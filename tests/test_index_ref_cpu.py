"""tests/index_ref.py (the plain-Python indexImpl) against the C++ oracle on sorted indexes: sort order, find, Join,
Except, the unique-key error and dedup.  The GPU index tests take index_ref as their expected answer where the oracle
cannot build the index (rows out of key order), so it is proved here first, where both apply."""
import random

import pytest

from oracle import oracle as orc
from tests import index_ref as ref

ALPHABET = [b"", b"a", b"b", b"\x00", b"\xff", b"a\x00", b"ab", b"b\xff", b"\x7f"]


def _rows(rng, n):
    return [{b"a": rng.choice(ALPHABET) + rng.choice(ALPHABET), b"b": b"%d" % rng.randrange(12), b"i": b"%05d" % i} for i in range(n)]


def _oracle_rows(o):
    return o.to_dicts()


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("keys", [(b"a",), (b"b", b"a"), (b"a", b"b", b"i")])
def test_sort_find_join_except(seed, keys):
    rng = random.Random(seed * 7 + len(keys))
    rows = _rows(rng, 600)
    cols = list(keys)
    srt = ref.index_on(rows, cols)
    oi = orc.take_rows(rows).index_on(*keys)
    assert srt == _oracle_rows(oi.rows())
    for _ in range(40):
        r = rng.choice(rows)
        nv = rng.randrange(1, len(cols) + 1)
        vals = [r[c] for c in cols[:nv]]
        if rng.random() < 0.3:
            vals[-1] = vals[-1] + rng.choice([b"\x00", b"z", b""])
        assert ref.find(srt, cols, vals) == _oracle_rows(oi.find(*vals)), vals
    # probes named differently from the index columns, on every prefix
    pnames = [b"p_" + c for c in cols]
    probe = [{**{pnames[j]: rng.choice(rows)[c] + (b"\x00" if rng.random() < 0.1 else b"") for j, c in enumerate(cols)}, b"q": b"%d" % k}
             for k in range(300)]
    op = orc.take_rows(probe)
    for nk in range(1, len(cols) + 1):
        assert ref.join(srt, cols, probe, pnames[:nk]) == _oracle_rows(op.join(oi, *pnames[:nk])), nk
        assert ref.except_(srt, cols, probe, pnames[:nk]) == _oracle_rows(op.except_(oi, *pnames[:nk])), nk
    # probes carrying the index's own column names: the probe value wins the collision
    same = [{c: p[pnames[j]] for j, c in enumerate(cols)} for p in probe]
    assert ref.join(srt, cols, same) == _oracle_rows(orc.take_rows(same).join(oi))


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("mode", ["first", "drop"])
def test_dedup(seed, mode):
    rng = random.Random(seed)
    n = rng.choice([2, 3, 50, 400])
    rows = [{b"k": b"%d" % rng.randrange(max(2, n // 3)), b"v": b"%d" % i} for i in range(n)]
    if seed == 3:  # the last sorted row a singleton after a group: lost (SURVEY §Q1)
        rows = [{b"k": b"a", b"v": b"0"}, {b"k": b"a", b"v": b"1"}, {b"k": b"b", b"v": b"2"}]
    srt = ref.index_on(rows, [b"k"])
    got, groups = ref.dedup(srt, [b"k"], (lambda g: g[0]) if mode == "first" else (lambda g: None))
    oi = orc.take_rows(rows).index_on("k")
    oi.dedup(mode)
    assert got == _oracle_rows(oi.rows())
    for lo, hi in groups:  # on sorted rows a group is a whole run of one key
        assert hi - lo >= 2 and len({r[b"k"] for r in srt[lo:hi]}) == 1
        assert (lo == 0 or srt[lo - 1][b"k"] != srt[lo][b"k"]) and (hi == len(srt) or srt[hi][b"k"] != srt[lo][b"k"])


def test_dedup_out_of_order_worked_example():
    """stored keys [b, b, a, c]: the group ends at the first row above b found by binary search from lower, so it takes
    in `a`, and the walk then runs off the end without copying `c`"""
    rows = [{b"k": k, b"v": b"%d" % i} for i, k in enumerate([b"b", b"b", b"a", b"c"])]
    seen = []
    got, groups = ref.dedup(rows, [b"k"], lambda g: seen.append(g) or {b"k": b"b'", b"v": b"x"})
    assert groups == [(0, 3)] and seen == [rows[:3]]
    assert got == [{b"k": b"b'", b"v": b"x"}]


def test_join_out_of_order_worked_example():
    """stored keys [a, d, c], probe pk = d: first() lands on d and the scan goes on through c (c <= d)"""
    rows = [{b"k": k, b"v": b"%d" % i} for i, k in enumerate([b"a", b"d", b"c"])]
    got = ref.join(rows, [b"k"], [{b"pk": b"d"}], [b"pk"])
    assert got == [{b"k": b"d", b"v": b"1", b"pk": b"d"}, {b"k": b"c", b"v": b"2", b"pk": b"d"}]


def test_sort_order_is_bytewise_and_stable():
    vals = [b"10", b"9", b"a", b"a\x00", b"", b"ab", b"a b", b"B", b"\xff", b"\x7f", b"aa", b"a", b"10", b"100", b"\xc3\xa9",
            b"z" * 300, b"z" * 299 + b"y"]
    rows = [{b"k": v, b"i": b"%d" % i} for i, v in enumerate(vals)]
    assert ref.index_on(rows, [b"k"]) == _oracle_rows(orc.take_rows(rows).index_on("k").rows())
    rows = [{b"p": b"ab", b"q": b"c"}, {b"p": b"a", b"q": b"bc"}, {b"p": b"a", b"q": b""}, {b"p": b"", b"q": b"abc"}, {b"p": b"a", b"q": b"b"}]
    for keys in ([b"p", b"q"], [b"q", b"p"]):
        assert ref.index_on(rows, keys) == _oracle_rows(orc.take_rows(rows).index_on(*keys).rows())


def test_unique_error_text():
    rows = [{b"x": b"2", b"y": b"b", b"z": b"0"}, {b"x": b"1", b"y": b"a", b"z": b"1"}, {b"x": b"2", b"y": b"b", b"z": b"2"}]
    with pytest.raises(ref.DuplicateKey) as e:
        ref.index_on(rows, [b"y", b"x"], unique=True)
    with pytest.raises(orc.OracleError) as oe:
        orc.take_rows(rows).unique_index_on("y", "x")
    assert str(e.value) == str(oe.value) == 'duplicate value while creating unique index: { "x" : "2", "y" : "b" }'
    assert ref.index_on(rows, [b"z"], unique=True) == _oracle_rows(orc.take_rows(rows).unique_index_on("z").rows())


def test_sub_index_keeps_stored_order():
    rows = [{b"a": b"1", b"b": b"z"}, {b"a": b"1", b"b": b"c"}, {b"a": b"2", b"b": b"a"}]
    sub, cols = ref.sub_index(rows, [b"a", b"b"], [b"1"])
    assert sub == rows[:2] and cols == [b"b"]
    with pytest.raises(ValueError):
        ref.sub_index(rows, [b"a", b"b"], [b"1", b"z"])
