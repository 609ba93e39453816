"""Known answers of tests/left_join_ref.py, the restatement LeftJoin's GPU results are compared against, on hand-written
rows: a natural-join miss keeps its key, a differently named key is empty on a miss, duplicate runs, a prefix join, an
empty index, stored rows out of key order and name collisions.  Also the argument errors of DataSource.LeftJoin and
Table.join(left=True), raised before anything runs."""
import pytest

from tests import index_ref as ref
from tests import left_join_ref as lj


def _r(**kv):
    return {k.encode(): v.encode() for k, v in kv.items()}


CUST = [_r(id="1", name="Ann"), _r(id="2", name="Bob"), _r(id="4", name="Dee")]  # sorted on id


def test_natural_join_miss_keeps_the_key():
    probe = [_r(id="2", qty="5"), _r(id="3", qty="7"), _r(id="1", qty="9")]
    got = lj.left_join(CUST, [b"id"], probe)
    assert got == [_r(id="2", name="Bob", qty="5"), _r(id="3", name="", qty="7"), _r(id="1", name="Ann", qty="9")]


def test_named_key_is_empty_on_a_miss():
    probe = [_r(cust_id="9", qty="1"), _r(cust_id="4", qty="2")]
    got = lj.left_join(CUST, [b"id"], probe, [b"cust_id"])
    assert got == [_r(id="", name="", cust_id="9", qty="1"), _r(id="4", name="Dee", cust_id="4", qty="2")]
    assert lj.schema([b"id", b"name"], [b"cust_id", b"qty"]) == [b"id", b"name", b"cust_id", b"qty"]


def test_duplicate_runs_give_every_row_in_index_order():
    rows = ref.index_on([_r(k="a", v="1"), _r(k="b", v="2"), _r(k="a", v="3"), _r(k="a", v="4")], [b"k"])
    probe = [_r(p="a"), _r(p="c"), _r(p="b")]
    got = lj.left_join(rows, [b"k"], probe, [b"p"])
    assert got == [_r(k="a", v="1", p="a"), _r(k="a", v="3", p="a"), _r(k="a", v="4", p="a"), _r(k="", v="", p="c"),
                   _r(k="b", v="2", p="b")]


def test_prefix_join_on_the_first_key_column():
    rows = ref.index_on([_r(a="x", b="1", v="p"), _r(a="x", b="2", v="q"), _r(a="y", b="1", v="r")], [b"a", b"b"])
    got = lj.left_join(rows, [b"a", b"b"], [_r(a="x"), _r(a="z")], [b"a"])
    assert got == [_r(a="x", b="1", v="p"), _r(a="x", b="2", v="q"), _r(a="z", b="", v="")]
    with pytest.raises(ValueError, match="too many source columns in LeftJoin"):
        lj.left_join(rows, [b"a"], [_r(a="x")], [b"a", b"b"])


def test_empty_index_keeps_every_probe_row():
    probe = [_r(cust_id="1"), _r(cust_id="")]
    got = lj.left_join([], [b"id"], probe, [b"cust_id"], index_columns=[b"id", b"name"])
    assert got == [_r(id="", name="", cust_id="1"), _r(id="", name="", cust_id="")]
    assert lj.left_join([], [b"id"], [], index_columns=[b"id"]) == []


def test_stored_rows_out_of_key_order_follow_joins_search():
    rows = [_r(k="b", v="1"), _r(k="a", v="2"), _r(k="c", v="3"), _r(k="a", v="4")]  # as LoadIndex stored them
    probe = [_r(k="a"), _r(k="b"), _r(k="c")]
    # first() lands on row 0 for "a" (above it: a miss) and on row 2 for "b" (a miss); for "c" on row 2, and the run
    # goes on through row 3, whose key "a" is not above "c"
    got = lj.left_join(rows, [b"k"], probe)
    assert got == [_r(k="a", v=""), _r(k="b", v=""), _r(k="c", v="3"), _r(k="c", v="4")]
    assert [g for g in got if g[b"v"]] == ref.join(rows, [b"k"], probe)


def test_probe_wins_name_collisions_on_matches_and_misses():
    probe = [_r(id="1", name="probe"), _r(id="7", name="other")]
    got = lj.left_join(CUST, [b"id"], probe)
    assert got == [_r(id="1", name="probe"), _r(id="7", name="other")]


def test_matched_rows_are_joins_result():
    rows = ref.index_on([_r(k=str(i % 5), v=str(i)) for i in range(20)], [b"k"])
    probe = [_r(p=str(i % 8), q=str(i)) for i in range(30)]
    got = lj.left_join(rows, [b"k"], probe, [b"p"])
    assert [g for g in got if g[b"k"]] == ref.join(rows, [b"k"], probe, [b"p"])
    assert sum(1 for g in got if not g[b"k"]) == sum(1 for p in probe if int(p[b"p"]) >= 5)


class _Ix:  # what DataSource.LeftJoin reads of an Index before anything runs
    columns = ["id"]


def test_left_join_argument_errors():
    import csvplus_b200 as cp
    src = cp.TakeRows([{"id": "1"}])
    with pytest.raises(ValueError, match=r"too many source columns in LeftJoin\(\)"):
        src.LeftJoin(_Ix(), "a", "b")
    ok = src.LeftJoin(_Ix(), "id")
    assert ok._ops[-1][0] == "leftjoin" and ok._ops[-1][2] == ("id",)
    with pytest.raises(ValueError, match="anti and left"):
        object.__new__(cp.Table).join(_Ix(), "id", anti=True, left=True)
