"""DataSource.OrderBy / Table.order_by on the GPU (csrc/order.cu, sort.cu's select_by_image; cpb_table_order_by, the C++
mirror) against the plain restatement of tests/order_ref.py, row for row and byte for byte: random tables of 0 to 5 M
rows, 1 to 4 keys of every kind and direction, string keys over 128 and over 255 bytes, floats dense in NaN, infinities,
signed zeros, subnormals and hex floats, few distinct values; every limit edge on both sides of the select / sort
crossover; IndexOn's order; streamed plans with their errors; streaming memory; host synchronisations per call."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest

from tests import order_ref as orf
from tests.helpers import gpu_ctx

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.abspath(__file__)).rsplit(os.sep, 1)[0]
SELECT_RATIO = 2  # order.cu: the select route when limit * 2 <= rows

FLOATS = [b"NaN", b"nan", b"+Inf", b"-Inf", b"inf", b"0", b"-0", b"+0", b"-0.0", b"5e-324", b"-5e-324", b"4.9e-324",
          b"2.2250738585072014e-308", b"2.225073858507201e-308", b"0x1p-1074", b"0x1.8p1", b"-0x1.fffffffffffffp1023", b"1e308",
          b"-1e308", b"1.5", b"-1.5", b"3", b"0x3p0"]
INTS = [b"0", b"-0", b"+7", b"7", b"9223372036854775807", b"-9223372036854775808", b"-1", b"1", b"-9223372036854775807"]
STRS = [b"", b"a", b"ab", b"a\x00", b"\xff", b"\x80", b"\x80a", b"b", b"A", b"\x7f"]


def _columns(seed: int, n: int, few: bool = False) -> dict:
    """column -> list of bytes: s (short strings, some over 128 bytes), w (some over 255 bytes), i (ints), f (floats),
    g (three values), id (the row); few: every column drawn from a handful of values, so ties dominate"""
    rng = np.random.default_rng(seed)
    k = 4 if few else 1000
    fl = FLOATS + [b"%.3g" % x for x in rng.normal(size=k) * 100]
    it = INTS + [b"%d" % x for x in rng.integers(-50, 50, k)]
    st = STRS + [bytes(rng.choice(list(b"ab\x00\xffz"), rng.integers(1, 6))) for _ in range(k)]
    st += [b"L" * 129 + b"x", b"L" * 129, b"L" * 130]
    wide = [b"W" * 256, b"W" * 300 + b"\x01", b"W" * 300, b""]
    pick = lambda pool, m: [pool[j] for j in rng.integers(0, min(len(pool), m), n)]  # noqa: E731
    m = 6 if few else 1 << 30
    return {"s": pick(st, m), "w": pick(wide + st, m), "i": pick(it, m), "f": pick(fl, m), "g": pick([b"x", b"y", b"z"], 3),
            "id": [b"%d" % r for r in range(n)]}


def _table(ctx, cols: dict):
    """cols as a device table, built from the bytes (cpb_table_from_host)"""
    from csvplus_b200 import _abi
    names = list(cols)
    n = len(cols[names[0]])
    offs, datas = [], []
    for c in names:
        off = np.zeros(n + 1, np.int64)
        np.cumsum(np.fromiter((len(v) for v in cols[c]), np.int64, n), out=off[1:])
        offs.append(off)
        datas.append(np.frombuffer(b"".join(cols[c]) + b"\0", np.uint8).copy())
    na = (_abi.Str * len(names))(*[_abi.Str(c.encode(), len(c)) for c in names])
    oa = (C.c_void_p * len(names))(*[o.ctypes.data for o in offs])
    da = (C.c_void_p * len(names))(*[d.ctypes.data for d in datas])
    return ctx._new_table("cpb_table_from_host", len(names), na, oa, da, n)


def _rows(cols: dict) -> list:
    names = list(cols)
    return [dict(zip(names, vals)) for vals in zip(*(cols[c] for c in names))]


def _check(t, want: list, columns=None):
    """table t holds the rows `want`, in order, byte for byte in every column"""
    assert len(t) == len(want)
    for c in columns or t.columns:
        off, data = t.column(c)
        exp = [r[c] for r in want]
        assert off.tolist() == [0] + np.cumsum([len(v) for v in exp], dtype=np.int64).tolist(), c
        assert data.tobytes() == b"".join(exp), c


def _norm(keys):
    return [(k, "str", "asc") if isinstance(k, str) else (tuple(k) + ("asc",))[:3] for k in keys]


KEYSETS = [
    [("f", "float64")],
    [("f", "float64", "desc")],
    [("i", "int", "desc")],
    ["s"],
    [("w", "str", "desc")],
    [("g", "str"), ("f", "float64", "desc")],
    [("g", "str", "desc"), ("i", "int"), ("s", "str", "desc")],
    [("f", "str"), ("i", "int", "desc"), "w", ("g", "str")],
    [("i", "int"), ("f", "float64"), ("g", "str", "desc"), ("s", "str")],
]


def _run_in_a_tie(want: list, keys) -> int:
    """a limit that cuts a run of rows equal in every key, or 1"""
    vals = [tuple(orf._value(kind, r[c])[0] for c, kind, _ in keys) for r in want]
    for j in range(1, len(vals) - 1):
        if vals[j] == vals[j + 1]:
            return j + 1
    return 1


@pytest.mark.parametrize("seed,n,few", [(1, 0, False), (2, 1, False), (3, 2, True), (4, 1000, False), (5, 50_000, False),
                                        (6, 300_000, True), (7, 300_000, False)])
def test_random_tables_every_kind_and_direction(seed, n, few):
    ctx = gpu_ctx()
    cols = _columns(seed, n, few)
    t = _table(ctx, cols)
    rows = _rows(cols)
    for keys in KEYSETS:
        nk = _norm(keys)
        want = orf.order(rows, nk)
        assert orf.error(rows, nk) is None
        _check(t.order_by(*keys), want)
        limits = {0, 1, _run_in_a_tie(want, nk), max(0, n - 1), n, n + 1, n // SELECT_RATIO, n // SELECT_RATIO + 1, n // 2}
        for lim in sorted(limits):
            _check(t.order_by(*keys, limit=lim), want[:lim], ["id", keys[0] if isinstance(keys[0], str) else keys[0][0]])


def test_every_row_equal_and_every_row_distinct():
    ctx = gpu_ctx()
    n = 200_000
    cols = {"k": [b"same"] * n, "f": [b"-0" if r % 2 else b"0" for r in range(n)], "id": [b"%d" % r for r in range(n)]}
    t = _table(ctx, cols)
    rows = _rows(cols)
    for keys in (["k"], [("f", "float64", "desc")], [("k", "str", "desc"), ("f", "float64")]):
        for lim in (None, 0, 1, 7, n // SELECT_RATIO, n // SELECT_RATIO + 1, n - 1, n, n + 1):
            _check(t.order_by(*keys, limit=lim), orf.order(rows, _norm(keys), lim), ["id"])
    rng = np.random.default_rng(9)
    perm = rng.permutation(n)
    cols = {"i": [b"%d" % (int(v) * 7919 - 10 ** 9) for v in perm], "id": [b"%d" % r for r in range(n)]}
    t = _table(ctx, cols)
    rows = _rows(cols)
    for d in ("asc", "desc"):
        want = orf.order(rows, [("i", "int", d)])
        for lim in (None, 1, 100, n // SELECT_RATIO, n // SELECT_RATIO + 1, n - 1):
            _check(t.order_by(("i", "int", d), limit=lim), want if lim is None else want[:lim], ["id", "i"])


def test_five_million_rows_with_few_distinct_values():
    ctx = gpu_ctx()
    n = 5_000_000
    rng = np.random.default_rng(11)
    fpool = [b"NaN", b"-0", b"0", b"1.5", b"-Inf", b"5e-324", b"0x1p-3", b"2"]
    ipool = [b"%d" % v for v in (-3, 0, 9223372036854775807, 5, -9223372036854775808)]
    cols = {"f": [fpool[j] for j in rng.integers(0, len(fpool), n)], "i": [ipool[j] for j in rng.integers(0, len(ipool), n)],
            "id": [b"%d" % r for r in range(n)]}
    t = _table(ctx, cols)
    rows = _rows(cols)
    keys = [("f", "float64", "desc"), ("i", "int")]
    want = orf.order(rows, _norm(keys))
    _check(t.order_by(*keys), want, ["id", "f", "i"])
    for lim in (100, n // SELECT_RATIO, n // SELECT_RATIO + 1):
        _check(t.order_by(*keys, limit=lim), want[:lim], ["id"])


def test_str_keys_give_index_on_order():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    cols = _columns(21, 40_000)
    cols = {"a": cols["s"], "b": cols["w"], "id": cols["id"]}
    t = _table(ctx, cols)
    got = cp.TakeTable(t).OrderBy("a", "b").ToRows()
    via_index = []
    cp.TakeTable(t).IndexOn("a", "b").Iterate(via_index.append)
    assert got == via_index
    assert [r["id"].encode() for r in got] == [r["id"] for r in orf.order(_rows(cols), _norm(["a", "b"]))]


def _orders_csv(n: int, bad_at=None, bad_value=b"12x") -> bytes:
    lines = [b"%d,c%03d,%s,%d" % (r, (r * 37) % 211, (b"%d.%02d" % ((r * 7919) % 1000, r % 100)) if r % 97 else b"NaN", r % 13)
             for r in range(n)]
    if bad_at is not None:
        f = lines[bad_at].split(b",")
        f[2] = bad_value
        lines[bad_at] = b",".join(f)
    return b"id,cust,price,q\n" + b"\n".join(lines) + b"\n"


def _csv_rows(csv: bytes) -> list:
    head, *body = csv.rstrip(b"\n").split(b"\n")
    names = head.decode().split(",")
    return [dict(zip(names, line.split(b","))) for line in body]


@pytest.mark.parametrize("k", [0, 1, 100, 2500, 20_000, 30_001])
def test_streamed_top_equals_materialised_order_and_reference(monkeypatch, k):
    import csvplus_b200 as cp
    from csvplus_b200 import api
    ctx = gpu_ctx()
    csv = _orders_csv(30_000)
    keys = [("price", "float64", "desc"), "cust", ("q", "int")]
    want = orf.order(_csv_rows(csv), _norm(keys), k)
    monkeypatch.setattr(api, "STREAM_BATCH_BYTES", 16 << 10)
    src = cp.Take(cp.FromBytes(csv, ctx))
    assert sum(1 for _ in src._batches()) > 5
    streamed = src.OrderBy(*keys).Top(k).ToRows()
    materialised = src.OrderBy(*keys).Drop(0).ToRows()[:k]
    assert streamed == materialised
    assert [r["id"].encode() for r in streamed] == [r["id"] for r in want]
    out = io.BytesIO()
    src.OrderBy(*keys).Top(k).ToCsv(out, "id", "price")
    assert out.getvalue() == b"id,price\n" + b"".join(r["id"] + b"," + r["price"] + b"\n" for r in want)


def test_conversion_error_in_a_late_batch_delivers_nothing(monkeypatch):
    import csvplus_b200 as cp
    from csvplus_b200 import api
    ctx = gpu_ctx()
    csv = _orders_csv(30_000, bad_at=27_001)
    monkeypatch.setattr(api, "STREAM_BATCH_BYTES", 16 << 10)
    src = cp.Take(cp.FromBytes(csv, ctx))
    with pytest.raises(cp.CsvPlusError) as want:
        src.ToTensors({"q": "int", "price": "float64"})
    assert want.value.row == 27_001
    for plan in (src.OrderBy(("q", "int"), ("price", "float64")).Top(10), src.OrderBy(("q", "int"), ("price", "float64")),
                 src.OrderBy("cust", ("price", "float64", "desc")).Top(10)):
        out = io.BytesIO()
        with pytest.raises(cp.CsvPlusError) as got:
            plan.ToCsv(out, "id")
        assert got.value.row == 27_001 and str(got.value) == str(want.value) and out.getvalue() == b""
        out = io.BytesIO()
        with pytest.raises(cp.CsvPlusError):
            plan.ToJSON(out)
        assert out.getvalue() == b""
    # the lowest row wins, ties to the earlier key
    rows = _csv_rows(csv)
    with pytest.raises(cp.CsvPlusError) as got:
        src.OrderBy(("q", "float64"), ("cust", "int")).Top(3).ToRows()
    assert (got.value.row, str(got.value)) == orf.error(rows, [("q", "float64", "asc"), ("cust", "int", "asc")])
    with pytest.raises(cp.CsvPlusError) as got:
        src.OrderBy(("zz", "int")).Top(3).ToRows()
    assert got.value.row == 0 and str(got.value) == 'missing column "zz"'


def test_source_error_delivers_nothing_and_a_conversion_error_before_it_wins(monkeypatch):
    import csvplus_b200 as cp
    from csvplus_b200 import api
    ctx = gpu_ctx()
    lines = _orders_csv(8000).split(b"\n")
    lines[6001] = b"1,2,3"  # a record of the wrong field count
    csv = b"\n".join(lines)
    monkeypatch.setattr(api, "STREAM_BATCH_BYTES", 8 << 10)
    src = cp.Take(cp.FromBytes(csv, ctx))
    with pytest.raises(cp.DataSourceError) as want:
        src.ToRows()
    for plan in (src.OrderBy(("price", "float64")).Top(5), src.OrderBy(("price", "float64"))):
        out = io.BytesIO()
        with pytest.raises(cp.DataSourceError) as got:
            plan.ToCsv(out, "id")
        assert str(got.value) == str(want.value) and out.getvalue() == b""
        out = io.BytesIO()
        with pytest.raises(cp.DataSourceError):
            plan.ToJSON(out)
        assert out.getvalue() == b""
        seen = []
        with pytest.raises(cp.DataSourceError):
            plan(seen.append)
        assert seen == []
    lines[3000] = b"3000,c1,zz,1"
    src = cp.Take(cp.FromBytes(b"\n".join(lines), ctx))
    with pytest.raises(cp.CsvPlusError) as got:
        src.OrderBy(("price", "float64")).Top(5).ToRows()
    assert got.value.row == 2999  # (line 3000 of the file holds row 2999)


def test_argument_errors_and_limits():
    import csvplus_b200 as cp
    from csvplus_b200 import _abi
    ctx = gpu_ctx()
    t = cp.Table.from_rows(ctx, [{"k": "x" * 5000, "v": "1"}, {"k": "y", "v": "2"}], ["k", "v"])
    with pytest.raises(cp.CsvPlusError) as e:
        t.order_by("k")
    assert e.value.status == _abi.CPB_ERR_UNSUPPORTED and "4 KiB" in str(e.value)
    assert [r["v"] for r in cp.TakeTable(t).OrderBy(("v", "int", "desc")).ToRows()] == ["2", "1"]
    # keys the C ABI refuses
    h = C.c_void_p()
    for keys in ([], [("v", 1), ("v", 2)], [("v", 7)]):
        arr = (_abi.OrderKey * max(1, len(keys)))(*[_abi.OrderKey(_abi.Str(c.encode(), len(c)), kd, 0) for c, kd in keys])
        e = _abi.Error()
        assert ctx.lib.cpb_table_order_by(ctx.h, t.h, arr, len(keys), 5, None, C.byref(h), C.byref(e)) == _abi.CPB_ERR_ARG
    arr = (_abi.OrderKey * 1)(_abi.OrderKey(_abi.Str(b"v", 1), 1, 0))
    other = cp.Table.from_rows(ctx, [{"v": "1"}], ["v"])
    assert ctx.lib.cpb_table_order_by(ctx.h, t.h, arr, 1, 5, other.h, C.byref(h), C.byref(_abi.Error())) == _abi.CPB_ERR_ARG
    assert ctx.lib.cpb_table_order_by(ctx.h, None, arr, 1, 5, None, C.byref(h), C.byref(_abi.Error())) == _abi.CPB_ERR_ARG
    # an empty plan keeps its columns; a missing key column of no rows is no error
    e = cp.Take(cp.FromBytes(b"a,b\n", ctx)).OrderBy(("zz", "int")).ToRows()
    assert e == []
    out = io.BytesIO()
    cp.Take(cp.FromBytes(b"a,b\n", ctx)).OrderBy("a").Top(3).ToCsv(out, "a", "b")
    assert out.getvalue() == b"a,b\n"


def test_operations_after_order_by_run_on_the_ordered_rows():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    csv = _orders_csv(5000)
    rows = _csv_rows(csv)
    want = orf.order(rows, [("price", "float64", "desc")])
    src = cp.Take(cp.FromBytes(csv, ctx))
    got = src.OrderBy(("price", "float64", "desc")).Drop(10).Filter(cp.Like({"cust": "c005"})).SelectColumns("id").Top(4).ToRows()
    assert [r["id"].encode() for r in got] == [r["id"] for r in want[10:] if r["cust"] == b"c005"][:4]
    got = src.Map(lambda r: dict(r)).OrderBy(("price", "float64", "desc")).Top(7).ToRows()
    assert [r["id"].encode() for r in got] == [r["id"] for r in want[:7]]


def test_streamed_top_memory_does_not_grow_with_the_input(monkeypatch):
    import csvplus_b200 as cp
    from csvplus_b200 import api
    ctx = gpu_ctx()
    buf = ctx.gen_csv("orders", (0, 4_000_000), n_cust=100_000, n_prod=50)
    data = buf.to_host().tobytes()
    buf.free()
    batch = 4 << 20
    monkeypatch.setattr(api, "STREAM_BATCH_BYTES", batch)
    keys = [("ts", "str", "desc"), ("qty", "int")]
    cut = data[: data.index(b"\n", 3 * batch) + 1]  # about three batches

    def high(d, top):
        ctx.sync()
        ctx.pool_used_high(reset=True)
        plan = cp.Take(cp.FromBytes(d, ctx)).OrderBy(*keys)
        rows = (plan.Top(100) if top else plan.Drop(0).Top(100)).ToRows()
        assert len(rows) == 100
        return ctx.pool_used_high(), rows
    (few, _), (many, streamed), (whole, materialised) = high(cut, True), high(data, True), high(data, False)
    assert len(data) > 20 * batch
    assert streamed == materialised
    assert many <= few * 1.25 + (1 << 20), (few, many)
    assert many * 4 < whole, (many, whole)


def test_host_syncs_per_call_on_each_route():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    n = 100_000
    t = cp.Table.from_rows(ctx, [{"s": "k%d" % (r % 777), "i": str(r % 1000), "f": "%d.5" % (r % 31)} for r in range(n)], ["s", "i", "f"])
    keys = ("s", ("i", "int", "desc"), ("f", "float64"))
    S, I = 1, 2

    def syncs(**kw):
        ctx.sync()
        s0 = ctx.host_syncs()
        r = t.order_by(*keys, **kw)
        return ctx.host_syncs() - s0, r
    assert syncs(limit=10)[0] == S + I + 3       # select route
    assert syncs(limit=n // SELECT_RATIO)[0] == S + I + 3
    assert syncs(limit=n // SELECT_RATIO + 1)[0] == S + I + 2  # sort route
    assert syncs()[0] == S + I + 2
    assert syncs(limit=0)[0] == S + I
    _, before = syncs(limit=10)
    # t's own 10 rows (select, gather), the concatenation, then the 20 rows of the union on the select route (2 * 10 <= 20)
    assert syncs(limit=10, before=before)[0] == (S + I + 2) + 1 + (S + I + 3)
    # every row of t, the concatenation, then the union on the sort route
    assert syncs(limit=n, before=before)[0] == (S + I) + 1 + (S + I + 2)


def test_cpp_order_example():
    exe = os.path.join(ROOT, "host", "order_example")
    if not os.path.exists(exe):
        import __graft_entry__ as g
        g.build()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "order example ok" in r.stdout
