"""Go 1.23 strconv.ParseFloat(s, 32) and FormatFloat(float64(x), fmt, prec, 32) restated for the float32 tests
(csrc/numeric.cu and csrc/format.cu with bitSize 32), on top of the float64 restatements in strconv_oracle.py (grammar,
specials) and ftoa_oracle.py (fixed digits, layout).

ParseFloat(s, 32): the exact decimal or hex value as a Fraction, rounded once to float32 (half to even).  Rounding a
  float64 to float32 would round twice and can differ (1.00000005960464477539062500000001 is 0x3f800001; through a double
  it is 0x3f800000).  Specials are Go's float32(special()): +-Inf, and NaN 0x7fc00000.
FormatFloat(float64(x), fmt, prec, 32): fixed precision is the exact value correctly rounded, as for 64 (a float32 is
  exactly a double), so ftoa_oracle's fixed digits apply unchanged.  Shortest digits use x's float32 rounding interval.
  Two routes: shortest_digits_fraction restates the definition with exact fractions; shortest_digits takes numpy's
  shortest float32 text.  The CPU tests fuzz one against the other."""
from __future__ import annotations

import math
import struct
from fractions import Fraction

from tests import ftoa_oracle as fo
from tests import strconv_oracle as so

INF, NAN = 0x7F800000, 0x7FC00000  # Go's float32(+Inf), float32(math.NaN())


def bits_of(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


def float_of(u: int) -> float:
    """the float32 of bits u, as the (exactly equal) Python float"""
    return struct.unpack("<f", struct.pack("<I", u & (2**32 - 1)))[0]


# ------------------------------------------------------------------ ParseFloat(s, 32)
def round_to_float32(v: Fraction) -> int:
    """the bits of v > 0 correctly rounded (half to even) to float32; INF when that reaches 2^128"""
    if v >= 2 ** 128:  # beyond every finite float32 and its rounding interval
        return INF
    e = max(v.numerator.bit_length() - v.denominator.bit_length() - 24, -149)
    while e > -149 and v < Fraction(2) ** (e + 23):  # the bit-length estimate can be one too high
        e -= 1
    while v >= Fraction(2) ** (e + 24):
        e += 1
    q = v / Fraction(2) ** e  # in [2^23, 2^24), or below 2^23 for a subnormal (e = -149)
    m = q.numerator // q.denominator
    rem = q - m
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and m & 1):
        m += 1
    if m == 1 << 24:
        m, e = m >> 1, e + 1
    if m < 1 << 23:  # subnormal (or zero)
        return m
    if e + 23 > 127:
        return INF
    return (e + 150) << 23 | (m - (1 << 23))


def parse_float(s: bytes) -> tuple[int, int]:
    """strconv.ParseFloat(s, 32) -> (float32 bits of the value, status)"""
    sp = so._special(s)
    if sp is not None:
        if sp[1] != len(s):
            return 0, so.SYNTAX
        b = sp[0]
        return ((b >> 63) << 31 | (NAN if b & (2 ** 52 - 1) else INF)), so.OK
    r = so.read_float(s)
    if r is None:
        return 0, so.SYNTAX
    neg, hexa, digits, dp = r
    sign = 1 << 31 if neg else 0
    if not digits.strip("0"):
        return sign, so.OK
    # 0.<digits> * base^dp; far outside the float32 range the result is known without the big powers
    if hexa:
        if dp > 132:
            return sign | INF, so.RANGE
        if dp < -160:
            return sign, so.OK
        v = Fraction(int(digits, 16)) * Fraction(2) ** (dp - 4 * len(digits))
    else:
        if dp > 40:
            return sign | INF, so.RANGE
        if dp < -50:
            return sign, so.OK
        v = Fraction(int(digits)) * Fraction(10) ** (dp - len(digits))
    b = round_to_float32(v)
    return sign | b, (so.RANGE if b == INF else so.OK)


# ------------------------------------------------------------------ FormatFloat(float64(x), fmt, prec, 32)
def _parts(x: float) -> tuple:
    """(m, e, border) with |x| = m * 2^e in float32 form (x must be a float32 value); border: the gap below x is half
    the gap above"""
    u = bits_of(x) & (2**31 - 1)
    assert float_of(u) == abs(x), x
    ex, fr = u >> 23, u & (2**23 - 1)
    m = fr | (1 << 23) if ex else fr
    e = ex - 150 if ex else -149
    return m, e, fr == 0 and ex > 1


def shortest_digits(x: float) -> tuple:
    """(digits, dp) of the shortest float32 representation of |x| (finite), through numpy"""
    import numpy as np
    x = abs(x)
    if x == 0:
        return "", 0
    mant, _, exp = np.format_float_scientific(np.float32(x), unique=True, trim="-").partition("e")
    ip, _, fp = mant.partition(".")
    d = (ip + fp).lstrip("0")
    lead = len(ip + fp) - len((ip + fp).lstrip("0"))
    return fo._trim(d, len(ip) - lead + (int(exp) if exp else 0))


def shortest_digits_fraction(x: float) -> tuple:
    """(digits, dp) from the definition: the fewest digits n such that an n-digit decimal lies in the float32 rounding
    interval of x (closed when the mantissa is even), and of those the closest to x, ties to an even last digit"""
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
    for n in range(1, 10):
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
        return fo._trim(s, dp + len(s) - n)
    raise AssertionError("no shortest float32 representation within 9 digits")


def format_float(x: float, fmt: str = "g", prec: int = -1, shortest=shortest_digits) -> str:
    """FormatFloat(float64(x), fmt, prec, 32) of a float32 value x: ftoa_oracle's rules with float32 shortest digits"""
    if not math.isnan(x) and not math.isinf(x):
        _parts(x)  # x must be a float32 value
    return fo.format_float(x, fmt, prec, shortest=shortest)


def format_bits(u: int, fmt: str = "g", prec: int = -1) -> str:
    return format_float(float_of(u), fmt, prec)
