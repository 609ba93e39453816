"""tests/ftoa_oracle.py against the known answers of strconv's documented behaviour, the golden fixture it wrote, and
its two shortest-digit routes (Python's repr, the exact-fraction restatement of the definition) against each other."""
import os
import random

import pytest

from tests import ftoa_oracle as fo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

KNOWN = [
    (1e23, "e", 17, "9.99999999999999916e+22"), (1e23, "g", -1, "1e+23"), (0.125, "f", 2, "0.12"), (2.5, "f", 0, "2"),
    (1e6, "g", -1, "1e+06"), (100000.0, "g", -1, "100000"), (5e-324, "e", -1, "5e-324"), (-0.0, "f", 2, "-0.00"),
    (0.0, "e", -1, "0e+00"), (0.0, "g", -1, "0"), (-0.0, "g", -1, "-0"), (1.5, "f", 0, "2"), (0.5, "f", 0, "0"),
    (0.006, "f", 2, "0.01"), (0.004, "f", 2, "0.00"), (1e21, "f", -1, "1000000000000000000000"), (1.0, "e", 0, "1e+00"),
    (1.0, "e", 3, "1.000e+00"), (123456789.0, "g", 3, "1.23e+08"), (0.0001, "g", -1, "0.0001"), (0.00001, "g", -1, "1e-05"),
    (1e100, "E", 3, "1.000E+100"), (float("nan"), "g", -1, "NaN"), (float("inf"), "f", 2, "+Inf"), (float("-inf"), "e", 3, "-Inf"),
    (1.7976931348623157e308, "g", -1, "1.7976931348623157e+308"), (2.0 ** -1074, "g", -1, "5e-324"), (100.0, "g", 1, "1e+02"),
    (3.0, "g", 0, "3"), (0.1, "e", 25, "1.0000000000000000555111512e-01"),
]


@pytest.mark.parametrize("x,fmt,prec,want", KNOWN)
def test_known_answers(x, fmt, prec, want):
    assert fo.format_float(x, fmt, prec) == want


def test_format_int():
    for v, s in ((0, "0"), (-7, "-7"), (-2**63, "-9223372036854775808"), (2**63 - 1, "9223372036854775807")):
        assert fo.format_int(v) == s


def test_refusals():
    for fmt, prec in (("b", -1), ("x", 2), ("g", 65), ("e", -2)):
        with pytest.raises(ValueError):
            fo.format_float(1.0, fmt, prec)


def test_shortest_routes_agree():
    rnd = random.Random(99)
    xs = [fo.float_of(rnd.getrandbits(64)) for _ in range(20000)]
    xs += [2.0 ** k for k in range(-1074, 1024)] + [fo.float_of(rnd.getrandbits(52)) for _ in range(2000)]
    xs += [float(k) for k in range(1, 2000)] + [k / 1000 for k in range(1, 2000)] + [10.0 ** k for k in range(-300, 300)]
    for x in xs:
        if x != x or abs(x) == float("inf"):
            continue
        assert fo.shortest_digits(x) == fo.shortest_digits_fraction(x), x
        assert float(("0." + fo.shortest_digits(x)[0] + "e%d" % fo.shortest_digits(x)[1]) if x else "0") == abs(x)


def test_golden_fixture_matches_the_oracle():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_format_golden", os.path.join(GOLDEN, "make_format_golden.py"))
    g = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(g)
    want = ["%s,%s,%s,%d,%s" % r for r in g.rows()]
    assert open(os.path.join(GOLDEN, "format_kat.csv")).read().splitlines() == want
