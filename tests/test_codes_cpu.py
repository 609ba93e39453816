"""The plain-Python categorical-codes reference (tests/codes_ref.py) against hand-derived answers and against an
independent numpy route; no device needed."""
import random

import numpy as np

from tests import codes_ref as cr


def test_first_appearance_order():
    codes, d = cr.factorize([b"b", b"a", b"b", b"c", b"a"])
    assert codes == [0, 1, 0, 2, 1] and d == [b"b", b"a", b"c"]


def test_empty_and_single():
    assert cr.factorize([]) == ([], [])
    assert cr.factorize([b""]) == ([0], [b""])
    assert cr.factorize([b"", b"x", b""]) == ([0, 1, 0], [b"", b"x"])


def test_bytes_not_text():
    vals = [b"a", b"a\0", b"aa", b"a", b"\xff\xfe", b"\xc3\xa9", b"e\xcc\x81", b"\xff\xfe"]
    codes, d = cr.factorize(vals)
    assert codes == [0, 1, 2, 0, 3, 4, 5, 3]  # no normalisation: the two spellings of e-acute differ
    assert d == [b"a", b"a\0", b"aa", b"\xff\xfe", b"\xc3\xa9", b"e\xcc\x81"]


def test_inverse_rebuilds_values():
    rng = random.Random(5)
    vals = [bytes(rng.choice(b"ab,\"\n") for _ in range(rng.randrange(4))) for _ in range(2000)]
    codes, d = cr.factorize(vals)
    assert [d[c] for c in codes] == vals
    assert len(set(d)) == len(d) and max(codes) + 1 == len(d)
    assert all(codes[vals.index(v)] == k for k, v in enumerate(d))


def test_ids_route_agrees():
    rng = np.random.default_rng(7)
    for k in (1, 3, 100, 5000):
        ids = rng.integers(0, k, 20000)
        codes, order = cr.factorize_ids(ids)
        want_codes, want_d = cr.factorize([b"%d" % i for i in ids])
        assert codes.tolist() == want_codes
        assert [b"%d" % i for i in order] == want_d
    assert [a.size for a in cr.factorize_ids(np.zeros(0, np.int64))] == [0, 0]


def test_column_of():
    d = [b"xy", b"", b"abc"]
    off, data = cr.column_of(d, np.array([2, 0, 1, 2]))
    assert off.tolist() == [0, 3, 5, 5, 8] and data.tobytes() == b"abcxyabc"
