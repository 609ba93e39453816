"""Writes tests/golden/format32_kat.csv: strconv.FormatFloat(float64(x), fmt, prec, 32) known answers of float32
values, one per line as `bits,fmt,prec,expected` (bits = the float32's bits in hex).  The expected texts come from
tests/float32_oracle.py (oracle-pinned); baseline/go/format checks them with Go's strconv.

    python tests/golden/make_format32_golden.py
"""
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.float32_oracle import bits_of, float_of, format_float  # noqa: E402

MODES = [("g", -1), ("e", -1), ("f", -1), ("f", 0), ("f", 2), ("f", 17), ("f", 40), ("e", 0), ("e", 5), ("e", 8), ("e", 17),
         ("g", 1), ("g", 6), ("g", 9), ("g", 30), ("E", 3), ("G", -1), ("e", 64), ("f", 64), ("g", 64)]
BITS = [0x00000000, 0x80000000, 0x3F800000, 0xBF800000, 0x3DCCCCCD, 0x3E99999A, 0x4B800000, 0x4B800001, 0x3F800001, 0x3F7FFFFF,
        0x7F7FFFFF, 0xFF7FFFFF, 0x00800000, 0x007FFFFF, 0x00000001, 0x80000001, 0x00000002, 0x7F000000, 0x01000000, 0x5E0AC723,
        0x49742400, 0x501502F9, 0x3A83126F, 0x358637BD, 0x40490FDB, 0x7F800000, 0xFF800000, 0x7FC00000]


def rows():
    rnd = random.Random(20261017)
    bits = list(BITS) + [rnd.getrandbits(32) for _ in range(40)]
    out = []
    for u in bits:
        x = float_of(u)
        assert u >> 23 & 0xFF == 0xFF or bits_of(x) == u
        for fmt, prec in MODES:
            out.append(("%08x" % u, fmt, prec, format_float(x, fmt, prec)))
    return out


def main():
    with open(os.path.join(HERE, "format32_kat.csv"), "w") as f:
        for r in rows():
            f.write("%s,%s,%d,%s\n" % r)


if __name__ == "__main__":
    main()
