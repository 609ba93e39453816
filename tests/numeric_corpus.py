"""Seeded inputs of the numeric tests: a grammar-aware fuzz of Atoi / ParseFloat strings and a rounding corpus of decimal
strings at and around the exact midpoints between adjacent doubles (the inputs that drive numeric.cu's rare path)."""
from __future__ import annotations

import random
import struct
from fractions import Fraction


def _digits(rng, lo, hi):
    return "".join(rng.choice("0123456789") for _ in range(rng.randint(lo, hi)))


def _hexdigits(rng, lo, hi):
    return "".join(rng.choice("0123456789abcdefABCDEF") for _ in range(rng.randint(lo, hi)))


def _sprinkle(rng, s, ch="_", p=0.15):
    """inserts ch at random places (valid and invalid underscore positions alike)"""
    out = []
    for c in s:
        if rng.random() < p:
            out.append(ch)
        out.append(c)
    if rng.random() < p:
        out.append(ch)
    return "".join(out)


JUNK = [b" ", b"\t", b"x", b"e", b"E", b".", b"+", b"-", b"_", b"\x00", b"\xff", b"\xc3\xa9", b"p", b"0x", b"i", b"n", b",", b'"']
WORDS = ["inf", "Inf", "INF", "infinity", "Infinity", "iNfInItY", "infin", "infinit", "infinityx", "nan", "NaN", "nAn", "nana",
         "na", "in", "i", "n"]


def fuzz_string(rng: random.Random) -> bytes:
    k = rng.random()
    sign = rng.choice(["", "", "", "+", "-"])
    if k < 0.22:  # integers, some near the int64 / uint64 bounds
        d = rng.choice([_digits(rng, 1, 4), _digits(rng, 1, 18), _digits(rng, 18, 21), str(rng.randrange(2 ** 63 - 50, 2 ** 63 + 50)),
                        str(rng.randrange(2 ** 64 - 50, 2 ** 64 + 50)), "0" * rng.randint(1, 30) + _digits(rng, 1, 19)])
        s = sign + d
    elif k < 0.55:  # decimal floats
        ip = _digits(rng, 0, rng.choice([3, 10, 25]))
        fp = _digits(rng, 0, rng.choice([3, 10, 30]))
        s = sign + ip + ("." + fp if rng.random() < 0.7 else "")
        if rng.random() < 0.5:
            s += rng.choice("eE") + rng.choice(["", "+", "-"]) + rng.choice([_digits(rng, 1, 3), _digits(rng, 1, 7), str(rng.randint(280, 360))])
    elif k < 0.65:  # underscores
        s = sign + _sprinkle(rng, _digits(rng, 1, 8) + ("." + _digits(rng, 0, 5) if rng.random() < 0.5 else "")
                             + ("e" + _digits(rng, 1, 3) if rng.random() < 0.3 else ""))
    elif k < 0.77:  # hex floats
        m = _hexdigits(rng, 0, rng.choice([4, 16, 20]))
        if rng.random() < 0.5:
            m += "." + _hexdigits(rng, 0, 14)
        s = sign + rng.choice(["0x", "0X"]) + (_sprinkle(rng, m, p=0.05) if rng.random() < 0.2 else m)
        if rng.random() < 0.9:
            s += rng.choice("pP") + rng.choice(["", "+", "-"]) + rng.choice([_digits(rng, 1, 2), str(rng.randint(1000, 1100))])
    elif k < 0.85:  # special words
        s = rng.choice(["", "", "+", "-"]) + rng.choice(WORDS)
    else:  # mutations of a valid string: a junk byte inserted, a byte dropped or the string cut
        b = fuzz_string(rng)
        if b:
            i = rng.randrange(len(b) + 1)
            op = rng.random()
            if op < 0.5:
                b = b[:i] + rng.choice(JUNK) + b[i:]
            elif op < 0.75:
                b = b[:i] + b[i + 1:]
            else:
                b = b[:i]
        return b
    return s.encode()


def fuzz(n: int, seed: int) -> list[bytes]:
    rng = random.Random(seed)
    return [fuzz_string(rng) for _ in range(n)]


def _bits(f: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", f))[0]


def _double(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def _decimal(fr: Fraction) -> str:
    """the exact decimal expansion of a dyadic rational > 0 (terminates)"""
    num, den = fr.numerator, fr.denominator
    k = den.bit_length() - 1  # den = 2^k
    assert den == 1 << k
    digits = str(num * 5 ** k)
    return f"0.{digits}e{len(digits) - k}" if k else str(num)


def _sci(digits: str, exp10: int) -> str:
    return f"{digits[0]}.{digits[1:]}e{exp10}" if len(digits) > 1 else f"{digits}e{exp10}"


def rounding_corpus(n: int, seed: int) -> list[bytes]:
    """for random doubles (normals, subnormals, the smallest subnormal, the largest finite): the exact decimal midpoint to
    the next double, the midpoint +- one unit in its last digit, the midpoint cut to 17-40 digits, and 19- / 20-digit
    mantissas around it"""
    rng = random.Random(seed)
    out = []
    fixed = [1, 0x7FEFFFFFFFFFFFFE, 0x000FFFFFFFFFFFFF, 0x0010000000000000, 0, 0x7FEFFFFFFFFFFFFF]
    while len(out) < n:
        r = rng.random()
        if fixed:
            b = fixed.pop()
        elif r < 0.6:
            b = rng.randrange(0x0010000000000000, 0x7FEFFFFFFFFFFFFF)
        elif r < 0.75:
            b = rng.randrange(1, 0x0010000000000000)
        else:  # doubles near powers of ten, where short mantissas sit close to midpoints
            b = _bits(float(f"1e{rng.randint(-320, 307)}")) + rng.randint(-3, 3)
            b = min(max(b, 1), 0x7FEFFFFFFFFFFFFE)
        lo = Fraction(_double(b)) if b else Fraction(0)
        hi = Fraction(_double(b + 1)) if b + 1 < 0x7FF0000000000000 else Fraction(2 ** 1024)
        mid = (lo + hi) / 2
        s = _decimal(mid)
        man, _, e = s.partition("e")
        if man.startswith("0."):
            digits, exp10 = man[2:].lstrip("0"), int(e or 0) - (len(man[2:]) - len(man[2:].lstrip("0"))) - 1
        else:
            digits, exp10 = man, len(man) - 1
        digits = digits.rstrip("0") or "0"
        sign = rng.choice(["", "-"])
        # the midpoint itself and +- one unit in its last digit
        out.append((sign + _sci(digits, exp10)).encode())
        up = str(int(digits) + 1)
        out.append((sign + _sci(up, exp10 + (len(up) - len(digits)))).encode())
        if int(digits) > 1:
            dn = str(int(digits) - 1)
            out.append((sign + _sci(dn, exp10 - (len(digits) - len(dn)))).encode())
        # cut to 17-40 digits, and the cut with a trailing 1 (just above)
        for _ in range(2):
            k = rng.randint(17, 40)
            if k < len(digits):
                out.append((sign + _sci(digits[:k], exp10)).encode())
                out.append((sign + _sci(digits[:k] + "0" * rng.randint(0, 5) + "1", exp10)).encode())
        # 19- and 20-digit mantissas at the midpoint's leading digits (Eisel-Lemire's refusals live here)
        for k in (19, 20):
            m = (digits + "0" * k)[:k]
            out.append((sign + _sci(m, exp10)).encode())
            out.append((sign + _sci(str(int(m) + 1), exp10 + (len(str(int(m) + 1)) - k))).encode())
        # the midpoint written with its digits padded by zeros past 800 significant digits, then a sticky 1
        if rng.random() < 0.02:
            out.append((sign + _sci(digits + "0" * (820 - len(digits)) + "1", exp10)).encode())
            out.append((sign + _sci(digits + "0" * (820 - len(digits)), exp10)).encode())
    return out[:n]
