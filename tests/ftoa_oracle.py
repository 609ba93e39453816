"""strconv.FormatInt(v, 10) and strconv.FormatFloat(x, fmt, prec, 64) restated from the rules of Go's strconv/ftoa.go.

Digits: a digit string d (no trailing zeros) and a decimal point dp with |x| ~ 0.d * 10^dp; zero has d = "", dp = 0.
  prec < 0   the shortest string that reads back as x, the closest to x among the shortest (ties to an even last digit).
             Two routes: shortest_digits_fraction restates the definition with exact fractions; shortest_digits takes
             Python's repr (also the shortest round-trip string, closest to x).  The CPU tests fuzz one against the other.
  prec >= 0  the exact value correctly rounded, ties to even, from Python's correctly rounded %.*e / %.*f:
             prec + 1 significant digits for 'e', max(prec, 1) for 'g', prec digits after the point for 'f'.
Layout: see format_digits.
"""
from __future__ import annotations

import math
import struct
from fractions import Fraction

VERBS = "eEfgG"


def format_int(v: int) -> str:
    return str(int(v))


def bits_of(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def float_of(u: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", u & (2**64 - 1)))[0]


def _trim(d: str, dp: int) -> tuple:
    d = d.rstrip("0")
    return (d, dp) if d else ("", 0)


def shortest_digits(x: float) -> tuple:
    """(digits, dp) of the shortest representation of |x| (finite), through repr"""
    x = abs(x)
    if x == 0:
        return "", 0
    r = repr(x)
    mant, _, exp = r.partition("e")
    ip, _, fp = mant.partition(".")
    d = (ip + fp).lstrip("0")
    lead = len(ip + fp) - len((ip + fp).lstrip("0"))
    dp = len(ip) - lead + (int(exp) if exp else 0)
    return _trim(d, dp)


def _parts(x: float) -> tuple:
    """(m, e, border) with |x| = m * 2^e; border: the gap below x is half the gap above"""
    u = bits_of(x) & (2**63 - 1)
    ex, fr = u >> 52, u & (2**52 - 1)
    m = fr | (1 << 52) if ex else fr
    e = ex - 1075 if ex else -1074
    return m, e, fr == 0 and ex > 1


def shortest_digits_fraction(x: float) -> tuple:
    """(digits, dp) of the shortest representation from the definition: the fewest digits n such that an n-digit
    decimal lies in the rounding interval of x (closed when the mantissa is even), and of those the closest to x"""
    x = abs(x)
    if x == 0:
        return "", 0
    m, e, border = _parts(x)
    X = Fraction(m) * Fraction(2) ** e
    h = Fraction(2) ** (e - 1)
    lo, hi = X - (h / 2 if border else h), X + h
    closed = m % 2 == 0

    def inside(c):
        return lo < c < hi or (closed and (c == lo or c == hi))

    dp = math.floor(math.log10(x)) + 1
    while X >= Fraction(10) ** dp:
        dp += 1
    while X < Fraction(10) ** (dp - 1):
        dp -= 1
    for n in range(1, 18):
        unit = Fraction(10) ** (dp - n)
        q = math.floor(X / unit)
        lower, upper = q * unit, (q + 1) * unit
        if lower == X:
            v = q
        else:
            lin, uin = inside(lower), inside(upper)
            if not lin and not uin:
                continue
            if lin and uin:
                dl, du = X - lower, upper - X
                up = du < dl or (du == dl and q % 2 == 1)
            else:
                up = uin
            v = q + (1 if up else 0)
        s = str(v)
        return _trim(s, dp + len(s) - n)
    raise AssertionError("no shortest representation within 17 digits")


def fixed_digits(x: float, n: int) -> tuple:
    """(digits, dp) of |x| correctly rounded to n >= 1 significant digits"""
    x = abs(x)
    if x == 0:
        return "", 0
    mant, _, exp = ("%.*e" % (n - 1, x)).partition("e")
    return _trim(mant.replace(".", ""), int(exp) + 1)


def f_digits(x: float, prec: int) -> tuple:
    """(digits, dp) of |x| correctly rounded to prec digits after the point"""
    s = "%.*f" % (prec, abs(x))
    ip, _, fp = s.partition(".")
    d = ip + fp
    dp = len(ip)
    stripped = d.lstrip("0")
    dp -= len(d) - len(stripped)
    return _trim(stripped, dp)


def format_digits(neg: bool, d: str, dp: int, fmt: str, prec: int) -> str:
    """formatDigits of strconv/ftoa.go over (digits, dp); prec < 0 means the digits are the shortest ones"""
    nd = len(d)
    lf = fmt.lower()
    if lf == "e":
        use_e, F = True, (nd - 1 if prec < 0 else prec)
    elif lf == "f":
        use_e, F = False, (max(nd - dp, 0) if prec < 0 else prec)
    else:
        eprec = 6 if prec < 0 else max(prec, 1)
        exp = dp - 1
        use_e = exp < -4 or exp >= eprec
        F = nd - 1 if use_e else max(nd - dp, 0)
    out = "-" if neg else ""
    if use_e:
        out += d[0] if nd else "0"
        if F > 0:
            out += "." + "".join(d[i] if i < nd else "0" for i in range(1, F + 1))
        x = dp - 1 if nd else 0
        out += ("E" if fmt in "EG" else "e") + ("-" if x < 0 else "+") + "%02d" % abs(x)
        return out
    out += "".join(d[i] if i < nd else "0" for i in range(dp)) if dp > 0 else "0"
    if F > 0:
        out += "." + "".join(d[j] if 0 <= j < nd else "0" for j in (dp + i - 1 for i in range(1, F + 1)))
    return out


def format_float(x: float, fmt: str = "g", prec: int = -1, shortest=shortest_digits) -> str:
    if fmt not in VERBS or not -1 <= prec <= 64:
        raise ValueError(f"unsupported FormatFloat({fmt!r}, {prec})")
    if math.isnan(x):
        return "NaN"
    neg = math.copysign(1.0, x) < 0
    if math.isinf(x):
        return "-Inf" if neg else "+Inf"
    lf = fmt.lower()
    if prec < 0:
        d, dp = shortest(x)
    elif lf == "e":
        d, dp = fixed_digits(x, prec + 1)
    elif lf == "g":
        d, dp = fixed_digits(x, max(prec, 1))
    else:
        d, dp = f_digits(x, prec)
    return format_digits(neg, d, dp, fmt, prec)


def format_bits(u: int, fmt: str = "g", prec: int = -1) -> str:
    return format_float(float_of(u), fmt, prec)
