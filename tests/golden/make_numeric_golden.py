"""Regenerates tests/golden/numeric_kat.{csv,expected} from the restated strconv (tests/strconv_oracle.py):

    python tests/golden/make_numeric_golden.py

numeric_kat.csv has one column `s`, every value quoted; numeric_kat.expected has one line per row:
`<Atoi value> <Atoi status> <ParseFloat bits, hex> <ParseFloat status>` (status 0 ok, 1 ErrSyntax, 2 ErrRange).
baseline/go/numeric/main.go writes the same .expected from the CSV with Go's own strconv, on a machine that has Go."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import strconv_oracle as so  # noqa: E402

KAT = [
    # TestNumericalConversions (csvplus_test.go:911-957)
    b"12345", b"3.1415926", b"xyz",
    # signs, empty, spaces
    b"", b"+", b"-", b"+0", b"-0", b"+1", b"-1", b" 1", b"1 ", b"1\t", b"--1", b"+-1", b"0", b"007", b"-007",
    # Atoi: left to right, int64 bounds and the first value past each
    b"9223372036854775807", b"9223372036854775808", b"-9223372036854775808", b"-9223372036854775809",
    b"18446744073709551615", b"18446744073709551616", b"99999999999999999999x", b"x99999999999999999999",
    b"1844674407370955161x", b"-99999999999999999999", b"000000000000000000000000000042", b"123456789012345678",
    b"1234567890123456789", b"1_000", b"0x10", b"1e3", b"\xff1",
    # ParseFloat: the whole string, exponents
    b"1e400x", b"1e400", b"-1e400", b"1e-400", b"-1e-400", b"1e", b"1e+", b"1e-", b".e1", b"e1", b".", b"1.", b".5", b"-.5",
    b"1.5e+3", b"1.5E-3", b"1.2.3", b"1e10000", b"1e99999999999999999999", b"0e99999999999999999999", b"1e-99999999999999999999",
    b"1" + b"0" * 400 + b"e-400", b"0." + b"0" * 400 + b"1e401",
    # underscores
    b"1_000.5", b"1__0", b"_1", b"1_", b"1_.5", b"1._5", b"1_e5", b"1e_5", b"1e5_0", b"1e5_", b"-1_0", b"+_1", b"0x_1p0", b"0x1_p0",
    b"0x1p1_0", b"0_1", b"0b1", b"0o7",
    # hex
    b"0x1p-1074", b"0x1p-1075", b"0x1.8p-1074", b"0x1.fffffffffffff8p1023", b"0x1.fffffffffffff7p1023", b"0x1p1024", b"0x1p1023",
    b"0x1", b"0x1.8", b"0x", b"0xp1", b"0x.p1", b"0x.8p1", b"0X1P0", b"-0x1p0", b"0x1.0000000000000000000001p0",
    b"0x1.00000000000008p0", b"0x1.00000000000008000001p0", b"0x1.00000000000018p0", b"0xABCDEFp-10", b"0xg1p0",
    # special words
    b"inf", b"+inf", b"-inf", b"Inf", b"INF", b"infinity", b"-Infinity", b"+INFINITY", b"infin", b"infinit", b"infinityx",
    b"infx", b"in", b"nan", b"NaN", b"NAN", b"+nan", b"-nan", b"nanx", b"na",
    # rounding: halfway cases, subnormals, the extremes
    b"2.2250738585072011e-308", b"2.2250738585072012e-308", b"4.9406564584124654e-324", b"2.4703282292062327e-324",
    b"2.4703282292062328e-324", b"1.7976931348623157e308", b"1.7976931348623158e308", b"1.7976931348623159e308",
    b"9007199254740993", b"9007199254740993.0000000000000000000000000001", b"9007199254740995", b"1.00000000000000011102230246251565404236316680908203125",
    b"1.00000000000000011102230246251565404236316680908203124", b"1.00000000000000011102230246251565404236316680908203126",
    b"123456789012345678901234567890", b"0.1", b"0.3", b"1e23", b"8.98846567431158e307", b"5e-324", b"1e-324",
]


def main():
    csv = b"s\n" + b"".join(b'"' + v.replace(b'"', b'""') + b'"\n' for v in KAT)
    lines = []
    for v in KAT:
        iv, ist = so.atoi(v)
        fb, fst = so.parse_float(v)
        lines.append(f"{iv} {ist} {fb:016x} {fst}")
    with open(os.path.join(HERE, "numeric_kat.csv"), "wb") as f:
        f.write(csv)
    with open(os.path.join(HERE, "numeric_kat.expected"), "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
