"""Known answers of the restated strconv (tests/strconv_oracle.py) for every grammar point numeric.cu implements, the
golden fixture against its generator, and the pow10 table build.py generates for Eisel-Lemire."""
import os

import pytest

from tests import strconv_oracle as so

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
INF, NINF = 0x7FF0000000000000, 0xFFF0000000000000


def f(s):
    return so.parse_float(s.encode() if isinstance(s, str) else s)


def bits(x):
    return so.bits_of(x)


def test_numerical_conversions_strings():  # csvplus_test.go:911-957
    assert so.atoi(b"12345") == (12345, so.OK)
    assert so.atoi(b"xyz") == (0, so.SYNTAX)
    b, st = f("3.1415926")
    assert st == so.OK and abs(so.float_of(b) - 3.1415926) < 1e-12
    assert f("xyz") == (0, so.SYNTAX)
    assert so.message("string", b"xyz", False, so.SYNTAX) == 'column "string": cannot convert "xyz" to integer: invalid syntax'
    assert so.message("string", b"xyz", True, so.SYNTAX) == 'column "string": cannot convert "xyz" to float: invalid syntax'
    assert so.message("q", b"1e999", True, so.RANGE) == 'column "q": cannot convert "1e999" to float: value out of range'


@pytest.mark.parametrize("s,want", [
    (b"", (0, so.SYNTAX)), (b"+", (0, so.SYNTAX)), (b"-", (0, so.SYNTAX)), (b" 1", (0, so.SYNTAX)), (b"1 ", (0, so.SYNTAX)),
    (b"+7", (7, so.OK)), (b"-7", (-7, so.OK)), (b"-0", (0, so.OK)), (b"007", (7, so.OK)), (b"1_0", (0, so.SYNTAX)),
    (b"0x10", (0, so.SYNTAX)), (b"1e3", (0, so.SYNTAX)),
    (b"9223372036854775807", (2 ** 63 - 1, so.OK)), (b"9223372036854775808", (2 ** 63 - 1, so.RANGE)),
    (b"-9223372036854775808", (-2 ** 63, so.OK)), (b"-9223372036854775809", (-2 ** 63, so.RANGE)),
    (b"18446744073709551616", (2 ** 63 - 1, so.RANGE)),
    # left to right: an overflow before a bad byte is ErrRange, a bad byte before the overflow ErrSyntax
    (b"99999999999999999999x", (2 ** 63 - 1, so.RANGE)), (b"-99999999999999999999x", (-2 ** 63, so.RANGE)),
    (b"1844674407370955161x", (0, so.SYNTAX)), (b"x99999999999999999999", (0, so.SYNTAX)),
])
def test_atoi(s, want):
    assert so.atoi(s) == want


@pytest.mark.parametrize("s,want", [
    ("1e400x", (0, so.SYNTAX)), ("1e400", (INF, so.RANGE)), ("-1e400", (NINF, so.RANGE)), ("1e-400", (0, so.OK)),
    ("-1e-400", (1 << 63, so.OK)), ("-0", (1 << 63, so.OK)), ("+0", (0, so.OK)), ("0e99999999999999999999", (0, so.OK)),
    ("1e", (0, so.SYNTAX)), ("1e+", (0, so.SYNTAX)), (".e1", (0, so.SYNTAX)), (".", (0, so.SYNTAX)), ("1.2.3", (0, so.SYNTAX)),
    ("", (0, so.SYNTAX)), ("+", (0, so.SYNTAX)), (" 1", (0, so.SYNTAX)), ("1 ", (0, so.SYNTAX)), (".5", (bits(0.5), so.OK)),
    ("1.", (bits(1.0), so.OK)), ("1e99999999999999999999", (INF, so.RANGE)), ("1e-99999999999999999999", (0, so.OK)),
    # underscores: only between digits, or after a base prefix
    ("1_000.5", (bits(1000.5), so.OK)), ("1__0", (0, so.SYNTAX)), ("_1", (0, so.SYNTAX)), ("1_", (0, so.SYNTAX)),
    ("1_.5", (0, so.SYNTAX)), ("1._5", (0, so.SYNTAX)), ("1_e5", (0, so.SYNTAX)), ("1e_5", (0, so.SYNTAX)),
    ("1e5_0", (bits(1e50), so.OK)), ("1e5_", (0, so.SYNTAX)), ("0x_1p0", (bits(1.0), so.OK)), ("0x1_p0", (0, so.SYNTAX)),
    ("0_1", (bits(1.0), so.OK)),
    # hex: mandatory p exponent, correct rounding, overflow
    ("0x1p-1074", (1, so.OK)), ("0x1p-1075", (0, so.OK)), ("0x1.8p-1074", (2, so.OK)), ("0x1.fffffffffffff8p1023", (INF, so.RANGE)),
    ("0x1.fffffffffffff7p1023", (0x7FEFFFFFFFFFFFFF, so.OK)), ("0x1p1024", (INF, so.RANGE)), ("0x1", (0, so.SYNTAX)),
    ("0x", (0, so.SYNTAX)), ("0xp1", (0, so.SYNTAX)), ("0X1P0", (bits(1.0), so.OK)), ("0x1.00000000000008p0", (bits(1.0), so.OK)),
    ("0x1.00000000000008000001p0", (bits(1.0) + 1, so.OK)), ("0x1.00000000000018p0", (bits(1.0) + 2, so.OK)),
    # special words
    ("inf", (INF, so.OK)), ("-Inf", (NINF, so.OK)), ("+INFINITY", (INF, so.OK)), ("infinity", (INF, so.OK)),
    ("infin", (0, so.SYNTAX)), ("infinityx", (0, so.SYNTAX)), ("nan", (so.NAN_BITS, so.OK)), ("NaN", (so.NAN_BITS, so.OK)),
    ("+nan", (0, so.SYNTAX)), ("-nan", (0, so.SYNTAX)), ("nanx", (0, so.SYNTAX)),
    # the extremes and halfway cases
    ("1.7976931348623157e308", (0x7FEFFFFFFFFFFFFF, so.OK)), ("1.7976931348623159e308", (INF, so.RANGE)),
    ("4.9406564584124654e-324", (1, so.OK)), ("2.4703282292062327e-324", (0, so.OK)), ("2.4703282292062328e-324", (1, so.OK)),
    ("9007199254740993", (bits(9007199254740992.0), so.OK)), ("9007199254740993.0000000000000000000000000001", (bits(9007199254740994.0), so.OK)),
])
def test_parse_float(s, want):
    assert f(s) == want


def test_very_long_inputs():
    # a halfway case padded with zeros past 800 significant digits: exact; a non-zero digit far beyond rounds it up
    half = "9007199254740993"
    assert f(half + "0" * 900) == (INF, so.RANGE)
    assert f("0." + half + "0" * 900 + "1e16")[0] == bits(9007199254740994.0)
    assert f("0." + half + "0" * 900 + "e16")[0] == bits(9007199254740992.0)
    assert f("0." + "0" * 400 + "1e401") == (bits(1.0), so.OK)


def test_golden_fixture_matches_its_generator():
    lines = open(os.path.join(GOLDEN, "numeric_kat.expected")).read().splitlines()
    csv = open(os.path.join(GOLDEN, "numeric_kat.csv"), "rb").read().split(b"\n")
    assert csv[0] == b"s"
    vals = [v[1:-1].replace(b'""', b'"') for v in csv[1:] if v]
    assert len(vals) == len(lines) > 100
    for v, line in zip(vals, lines):
        iv, ist, fb, fst = line.split()
        assert so.atoi(v) == (int(iv), int(ist)), v
        assert so.parse_float(v) == (int(fb, 16), int(fst)), v


def test_pow10_table():
    from csvplus_b200 import build
    t = build.pow10_table()
    assert len(t) == 696
    assert t[348] == (0, 1 << 63)                                    # 1e0
    assert t[347] == (0xCCCCCCCCCCCCCCCC, 0xCCCCCCCCCCCCCCCC)         # 1e-1, rounded down
    for e in (-348, -1, 0, 27, 28, 347):                               # 10^e = m * 2^k with m rounded down
        lo, hi = t[e + 348]
        m = hi << 64 | lo
        if e >= 0:
            v = 10 ** e
            assert m == (v << (128 - v.bit_length()) if v.bit_length() <= 128 else v >> (v.bit_length() - 128))
        else:
            assert m * 10 ** -e < 1 << (127 + (10 ** -e).bit_length()) <= (m + 1) * 10 ** -e
