"""GPU parity of what an index derives from its stored rows once those rows change (Join / Except after a dedup of a
unique index that was joined in source order), and of Index.Find on key images the other tests leave out: lookup
values longer than the key width, key columns of 255 bytes or more (two-byte length field), and a prefix Find that is
the first use of a lazily sorted unique index's order."""
import random

import pytest

from oracle import oracle as orc
from tests.helpers import assert_table_equals_oracle, gpu_ctx

pytestmark = pytest.mark.gpu


def _with_stats(fn):
    ctx = gpu_ctx()
    ctx.sync()
    ctx.stats(enable=True, reset=True)
    r = fn()
    ctx.sync()
    st = ctx.stats()
    ctx.stats(enable=False)
    return r, st


def _dicts(rows: "orc.Rows"):
    return [{k.decode(): v.decode() for k, v in r.items()} for r in rows.to_dicts()]


@pytest.mark.parametrize("n", [1000, 40_000])  # a probe table staged in shared memory / 16-byte slots
def test_join_after_dedup_of_a_source_order_index(n):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    rng = random.Random(n)
    keys = [str(i) for i in range(n)]  # at most 7 bytes: a one-word key image
    rng.shuffle(keys)
    rows = [{"k": k, "v": "v%019d" % i, "w": str(i % 7)} for i, k in enumerate(keys)]  # 20-byte payload column
    ix, st = _with_stats(lambda: cp.Table.from_rows(ctx, rows).index_on("k", unique=True))
    assert "rowhash_build" not in st, sorted(st)
    probe_rows = [{"k": k, "x": str(i)} for i, k in enumerate(keys + keys[::-1] + ["nope", str(n)])]
    tp, op = cp.Table.from_rows(ctx, probe_rows), orc.take_rows(probe_rows)
    oi = orc.take_rows(rows).unique_index_on("k")
    # every index key matches twice: the source-order row slots are laid out
    j, st = _with_stats(lambda: tp.join(ix, "k"))
    assert "slot_build" in st, sorted(st)
    assert_table_equals_oracle(j, op.join(oi, "k"))
    # a unique index has no duplicate group; with bug_compatible the last sorted row is dropped all the same
    ix.dedup_apply([0], bug_compatible=True)
    assert len(ix) == n - 1
    od = orc.take_rows(ix.table().rows()).unique_index_on("k")
    assert_table_equals_oracle(tp.join(ix, "k"), op.join(od, "k"))
    assert_table_equals_oracle(tp.join(ix, "k", anti=True), op.except_(od, "k"))


def test_find_value_longer_than_the_key_width():
    import csvplus_b200 as cp
    rows = [{"a": a, "b": b, "i": str(i)} for i, (a, b) in enumerate((a, b) for a in ("ab", "abc", "b", "") for b in ("1", "22", "333"))]
    random.Random(5).shuffle(rows)
    ix = cp.Table.from_rows(gpu_ctx(), rows).index_on("a", "b")
    oi = orc.take_rows(rows).index_on("a", "b")
    # "abcd" keeps the 3 bytes "abc" with an all-ones length: ordered after every "abc" key, never equal to one
    for probe in (("abcd",), ("abc", "3334"), ("abc", "333"), ("ab", "22"), ("abc",), ("b", "1111"), ("",)):
        assert ix.Find(*probe).ToRows() == _dicts(oi.find(*probe)), probe


def test_find_on_a_key_of_255_bytes_or_more():
    import csvplus_b200 as cp
    ks = ["z" * 300, "z" * 299 + "y", "z" * 255, "z" * 254, "z" * 256, "a", ""]
    rows = [{"k": k, "j": str(j), "i": "%d-%d" % (n, j)} for n, k in enumerate(ks) for j in range(3)]
    random.Random(7).shuffle(rows)
    ix = cp.Table.from_rows(gpu_ctx(), rows).index_on("k", "j")
    oi = orc.take_rows(rows).index_on("k", "j")
    for probe in (("z" * 300,), ("z" * 299 + "y", "2"), ("z" * 255,), ("z" * 254, "0"), ("z" * 256, "1"), ("z" * 299,),
                  ("z" * 301,), ("a",), ("", "1"), ("z" * 254, "00")):
        assert ix.Find(*probe).ToRows() == _dicts(oi.find(*probe)), (len(probe[0]), probe[1:])


@pytest.mark.parametrize("payload", [8, 20])  # the row-carrying table / the source-order key image
def test_prefix_find_first_on_a_lazily_sorted_unique_index(payload):
    import csvplus_b200 as cp
    rng = random.Random(payload)
    rows = [{"s": s, "id": str(i), "p": "p" * payload} for s in ("Ab", "Cd", "Ef") for i in range(500)]
    rng.shuffle(rows)
    ix, st = _with_stats(lambda: cp.Table.from_rows(gpu_ctx(), rows).index_on("s", "id", unique=True))
    assert ("rowhash_build" in st) == (payload <= 16), sorted(st)
    oi = orc.take_rows(rows).unique_index_on("s", "id")
    assert ix.Find("Cd").ToRows() == _dicts(oi.find("Cd"))
    assert ix.Find("Ef", "499").ToRows() == _dicts(oi.find("Ef", "499"))
    assert ix.Find("C").ToRows() == []
    assert_table_equals_oracle(ix.table(), oi.rows())
