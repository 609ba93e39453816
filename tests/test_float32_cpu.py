"""The float32 oracles (tests/float32_oracle.py: ParseFloat(s, 32), FormatFloat(float64(x), fmt, prec, 32)) against known answers derived
by exact arithmetic, their two shortest-digit routes against each other, and the float32 fixtures against their
generators."""
import importlib.util
import os
import random
from fractions import Fraction

import numpy as np
import pytest

from tests import float32_oracle as f32
from tests import ftoa_oracle as fo
from tests import strconv_oracle as so

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
HALF_MIN_SUB = Fraction(1, 2 ** 150)  # half the smallest subnormal


def _dec(fr: Fraction) -> bytes:
    """the exact decimal text of a dyadic rational > 0"""
    k = fr.denominator.bit_length() - 1
    assert fr.denominator == 1 << k
    d = str(fr.numerator * 5 ** k)
    return (d + "e-%d" % k).encode()


PARSE = [
    (b"1.000000059604644775390625", 0x3F800000, so.OK),  # 1 + 2^-24: halfway, to the even mantissa
    (_dec(1 + Fraction(3, 2 ** 24)), 0x3F800002, so.OK),  # halfway between odd 0x3f800001 and even 0x3f800002
    (b"1.00000005960464477539062500000001", 0x3F800001, so.OK),  # just above the tie
    (b"3.4028234663852886e38", 0x7F7FFFFF, so.OK),  # the largest finite value
    (str(2 ** 128 - 2 ** 103 - 1).encode(), 0x7F7FFFFF, so.OK),  # just below the overflow boundary
    (str(2 ** 128 - 2 ** 103).encode(), 0x7F800000, so.RANGE),  # the boundary: a tie that rounds to 2^128
    (b"-1e39", 0xFF800000, so.RANGE),
    (_dec(Fraction(1, 2 ** 149)), 0x00000001, so.OK),  # the smallest subnormal
    (_dec(HALF_MIN_SUB), 0x00000000, so.OK),  # half of it: a tie to zero
    (_dec(HALF_MIN_SUB) + b"1", 0x00000000, so.OK),  # the text with one more digit (a smaller value)
    (_dec(HALF_MIN_SUB * 3), 0x00000002, so.OK),  # 1.5 ulp: to even
    (b"-" + _dec(HALF_MIN_SUB + Fraction(1, 2 ** 170)), 0x80000001, so.OK),
    (b"16777216", 0x4B800000, so.OK), (b"16777217", 0x4B800000, so.OK), (b"16777219", 0x4B800002, so.OK),
    (b"0.1", 0x3DCCCCCD, so.OK), (b"-0", 0x80000000, so.OK), (b"nan", 0x7FC00000, so.OK), (b"-Inf", 0xFF800000, so.OK),
    (b"0x1p-149", 0x00000001, so.OK), (b"0x1p-150", 0x00000000, so.OK), (b"0x1.000001p0", 0x3F800000, so.OK),
    (b"0x1.000003p0", 0x3F800002, so.OK), (b"0x1.fffffep127", 0x7F7FFFFF, so.OK), (b"0x1.ffffffp127", 0x7F800000, so.RANGE),
    (b"1e", 0, so.SYNTAX), (b"infx", 0, so.SYNTAX),
]


@pytest.mark.parametrize("s,bits,st", PARSE)
def test_parse_known_answers(s, bits, st):
    assert f32.parse_float(s) == (bits, st)


def test_parse_is_one_rounding():
    s = b"1.00000005960464477539062500000001"
    two_step = int(np.float32(float(s)).view(np.uint32))
    assert two_step == 0x3F800000 and f32.parse_float(s)[0] == 0x3F800001


def test_parse_agrees_with_numpy_where_one_rounding_is_safe():
    """short decimal strings (<= 9 digits): the double is within far less than a float32 half-ulp of a tie unless the
    value is one, so float32(float(s)) is the correctly rounded float32 away from ties; every mismatch must be a tie"""
    rnd = random.Random(5)
    for _ in range(20000):
        s = ("%d.%de%d" % (rnd.randint(0, 99999), rnd.randint(0, 9999), rnd.randint(-46, 39))).encode()
        b, st = f32.parse_float(s)
        with np.errstate(over="ignore"):
            want = np.float32(float(s)).view(np.uint32)
        if st == so.RANGE:
            assert abs(float(s)) >= 3.4e38
        elif b != want:
            lo, hi = sorted((f32.float_of(b), f32.float_of(int(want))))
            assert Fraction(s.decode()) == (Fraction(lo) + Fraction(hi)) / 2, s


def _edge_f32():
    out = []
    for ex in range(0, 255):
        for fr in (0, 1, 2, 0x400000, 0x7FFFFE, 0x7FFFFF):
            out.append(ex << 23 | fr)
    return out


def test_shortest_routes_agree():
    rnd = random.Random(32)
    bits = _edge_f32() + [rnd.getrandbits(31) for _ in range(100_000)]
    for u in bits:
        if (u >> 23) & 0xFF == 0xFF:
            continue
        x = f32.float_of(u)
        d, dp = f32.shortest_digits(x)
        assert (d, dp) == f32.shortest_digits_fraction(x), hex(u)
        assert len(d) <= 9
        back = f32.parse_float(("0." + d + "e%d" % dp).encode() if d else b"0")[0]
        assert back == u, hex(u)


FORMAT = [
    (0x3DCCCCCD, "g", -1, "0.1"), (0x3DCCCCCD, "e", 10, "1.0000000149e-01"), (0x3DCCCCCD, "f", -1, "0.1"),
    (0x4B800000, "g", -1, "1.6777216e+07"), (0x4B800000, "f", -1, "16777216"), (0x7F7FFFFF, "g", -1, "3.4028235e+38"),
    (0x00000001, "g", -1, "1e-45"), (0x00000001, "e", 20, "1.40129846432481707092e-45"), (0x00800000, "g", -1, "1.1754944e-38"),
    (0x3F800001, "g", -1, "1.0000001"), (0x80000000, "g", -1, "-0"), (0x3EAAAAAB, "g", -1, "0.33333334"),
    (0x7FC00000, "g", -1, "NaN"), (0xFF800000, "e", 3, "-Inf"), (0x49742400, "G", -1, "1E+06"),
]


@pytest.mark.parametrize("bits,fmt,prec,want", FORMAT)
def test_format_known_answers(bits, fmt, prec, want):
    assert f32.format_bits(bits, fmt, prec) == want


def test_fixed_precision_does_not_depend_on_the_bit_size():
    rnd = random.Random(8)
    for _ in range(2000):
        u = rnd.getrandbits(32)
        if (u >> 23) & 0xFF == 0xFF:
            continue
        x = f32.float_of(u)
        for fmt, prec in (("e", 0), ("e", 12), ("f", 3), ("g", 5), ("g", 40)):
            assert f32.format_float(x, fmt, prec) == fo.format_float(x, fmt, prec)


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(GOLDEN, name + ".py"))
    g = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(g)
    return g


def test_numeric32_fixture_matches_its_generator():
    csv, expected = _load("make_numeric32_golden").rows()
    assert open(os.path.join(GOLDEN, "numeric32_kat.csv"), "rb").read() == csv
    assert open(os.path.join(GOLDEN, "numeric32_kat.expected")).read() == expected


def test_format32_fixture_matches_its_generator():
    want = ["%s,%s,%d,%s" % r for r in _load("make_format32_golden").rows()]
    assert open(os.path.join(GOLDEN, "format32_kat.csv")).read().splitlines() == want
