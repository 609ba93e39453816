"""Regenerates tests/golden/numeric32_kat.{csv,expected}: strconv.ParseFloat(s, 32) known answers from the restated
float32 strconv (tests/float32_oracle.py):

    python tests/golden/make_numeric32_golden.py

numeric32_kat.csv has one column `s`, every value quoted; numeric32_kat.expected has one line per row:
`<ParseFloat(s, 32) bits, 8 hex digits> <status>` (status 0 ok, 1 ErrSyntax, 2 ErrRange).  `go run ./numeric -32`
(baseline/go/numeric/main.go) writes the same .expected with Go's own strconv, on a machine that has Go."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import float32_oracle as f32  # noqa: E402

KAT = [
    # grammar and specials, as for 64
    b"", b"+", b"-", b"0", b"-0", b"+0", b"1", b"-1", b" 1", b"1 ", b"1e", b"1e+", b".", b".5", b"1.", b"1_000.5", b"1__0", b"_1",
    b"inf", b"-inf", b"+Infinity", b"infin", b"nan", b"NaN", b"-nan", b"nanx", b"1e400x", b"0x", b"0x1", b"0xp1",
    # the values of the float32 tests: 0.1, 2^24 and its neighbours, 1 + 2^-24 (a tie to even) and what double rounding breaks
    b"0.1", b"0.3", b"3.1415926", b"16777216", b"16777217", b"16777218", b"16777219", b"1.000000059604644775390625",
    b"1.00000005960464477539062500000001", b"1.000000178813934326171875", b"1.0000000596046448", b"1.00000006",
    # the largest finite value, the overflow boundary (2^128 - 2^103, a tie that rounds up to 2^128) and past it
    b"3.4028234663852886e38", b"3.4028235e38", b"340282356779733661637539395458142568447", b"340282356779733661637539395458142568448",
    b"3.4028236e38", b"1e39", b"-1e39", b"1e38", b"1e400",
    # the smallest normal and subnormal, half the smallest subnormal (a tie to zero) and just above it
    b"1.17549435e-38", b"1.1754942e-38", b"1.401298464324817e-45", b"1e-45", b"7.006492321624085e-46",
    b"7.00649232162408535461864791644958065640130970938257885878534141944895541342930300743319094181060791015625e-46",
    b"7.00649232162408535461864791644958065640130970938257885878534141944895541342930300743319094181060791015626e-46",
    b"-7.0064923216240854e-46", b"1e-46", b"1e-50", b"1e-400",
    # exact path bounds: mantissa < 2^24, |exponent| <= 10
    b"16777215e10", b"16777215e-10", b"16777217e10", b"1e10", b"1e11", b"1e-10", b"1e-11", b"123456789012345678901234567890",
    # hex with 23 mantissa bits
    b"0x1p-149", b"0x1p-150", b"0x1.8p-150", b"0x1.000001p0", b"0x1.000003p0", b"0x1.0000010000000000000001p0", b"0x1.fffffep127",
    b"0x1.ffffffp127", b"0x1p128", b"-0x1p128", b"0x1p-126", b"0x.8p-125", b"0xABCDEFp-10",
]


def rows():
    """(the CSV's bytes, the .expected text)"""
    csv = b"s\n" + b"".join(b'"' + v.replace(b'"', b'""') + b'"\n' for v in KAT)
    lines = []
    for v in KAT:
        b, st = f32.parse_float(v)
        lines.append(f"{b:08x} {st}")
    return csv, "\n".join(lines) + "\n"


def main():
    csv, expected = rows()
    with open(os.path.join(HERE, "numeric32_kat.csv"), "wb") as f:
        f.write(csv)
    with open(os.path.join(HERE, "numeric32_kat.expected"), "w") as f:
        f.write(expected)


if __name__ == "__main__":
    main()
