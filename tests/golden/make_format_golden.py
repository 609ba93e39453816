"""Writes tests/golden/format_kat.csv: strconv.FormatFloat / FormatInt known answers, one per line as
`kind,bits,fmt,prec,expected` (kind f: bits = the float64's bits in hex; kind i: bits = the int64 in decimal, fmt and
prec unused).  The expected texts come from tests/ftoa_oracle.py (oracle-pinned); baseline/go/format regenerates the
same file with Go's strconv to check them.

    python tests/golden/make_format_golden.py
"""
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from ftoa_oracle import bits_of, float_of, format_float, format_int  # noqa: E402

MODES = [("g", -1), ("e", -1), ("f", -1), ("f", 0), ("f", 2), ("f", 17), ("f", 40), ("e", 0), ("e", 5), ("e", 17), ("e", 25),
         ("g", 1), ("g", 6), ("g", 17), ("g", 30), ("E", 3), ("G", -1), ("e", 64), ("f", 64), ("g", 64)]
VALUES = [0.0, -0.0, 1.0, -1.0, 0.1, 0.125, 2.5, 0.5, 1.5, 1e23, 1e22, 1e21, 1e6, 100000.0, 123456.789, 5e-324, -5e-324,
          2.2250738585072014e-308, 2.225073858507201e-308, 1.7976931348623157e308, 9007199254740993.0, 2.0 ** 60, 2.0 ** -1022,
          0.3, 2.0 / 3, 1e-7, 123e-20, 999999.5, 9.5, 0.95, 0.005, 1e300, -1e-300, float("inf"), float("-inf"), float("nan")]
INTS = [0, 1, -1, 7, -7, 10, -10, 99, 100, 101, 2**31, -2**31, 2**53 + 1, 2**63 - 1, -2**63, 10**18, -10**18 - 1, 999999999999999999]


def rows():
    rnd = random.Random(20261015)
    vals = list(VALUES) + [float_of(rnd.getrandbits(64)) for _ in range(40)]
    out = []
    for x in vals:
        for fmt, prec in MODES:
            out.append(("f", "%016x" % bits_of(x), fmt, prec, format_float(x, fmt, prec)))
    for v in INTS:
        out.append(("i", str(v), "d", 0, format_int(v)))
    return out


def main():
    with open(os.path.join(HERE, "format_kat.csv"), "w") as f:
        for r in rows():
            f.write("%s,%s,%s,%d,%s\n" % r)


if __name__ == "__main__":
    main()
