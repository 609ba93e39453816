"""DataSource.GroupBy on the GPU (csrc/groupby.cu; cpb_groups_*, the C++ mirror) against the plain restatement of
tests/groupby_ref.py, bit for bit: random tables of 1 to 10^6 groups and 1 to 4 key columns (values over 128 bytes in
every warp position), every op x kind, plans streamed in many batches, the one-group and all-distinct extremes, the
reference's three per-customer folds, the errors, streaming memory, and the host synchronisations of a push."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from tests import groupby_ref as gr
from tests.helpers import gpu_ctx

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ALL_AGGS = {
    "n": ("count",),
    **{f"{op}_{kind}": (op, "i" if kind == "int" else "f", kind) for op in ("sum", "min", "max", "first", "last") for kind in ("int", "float64")},
}
SPECIAL_FLOATS = [b"-0", b"0", b"NaN", b"+Inf", b"-Inf", b"1e308", b"-1e308", b"5e-324", b"-0.0"]


def _key(g: int, j: int) -> bytes:
    """column j of group g's key: injective in column 0 (empty for group 1, over 128 bytes for every 7th group); the
    other columns repeat across groups, some of them long too"""
    if j == 0:
        return b"" if g == 1 else (b"L" * (129 + g % 300) + b"%d" % g if g % 7 == 3 else b"%d" % g)
    if j == 2 and g % 11 == 0:
        return b"M" * (200 + g % 5)
    return b"c%d" % (g % (3 + j))


def _data(seed: int, nrows: int, ngroups: int, nkeys: int):
    """(csv bytes, column names, columns) of nrows rows over ngroups groups (each appears at least once), in random order"""
    rng = np.random.default_rng(seed)
    gids = np.concatenate([rng.permutation(ngroups), rng.integers(0, ngroups, nrows - ngroups)])
    rng.shuffle(gids)
    small = rng.integers(-10 ** 6, 10 ** 6, nrows)
    big = rng.random(nrows) < 0.01
    ints = [b"%d" % (9_000_000_000_000_000_000 * (1 if v > 0 else -1) + int(v) if b else int(v)) for v, b in zip(small, big)]
    fv = rng.normal(size=nrows) * 1000
    sp = rng.integers(0, 2000, nrows)
    floats = [SPECIAL_FLOATS[s] if s < len(SPECIAL_FLOATS) else b"%.3f" % x for x, s in zip(fv, sp)]
    names = [f"k{j}" for j in range(nkeys)] + ["i", "f"]
    cols = [[_key(int(g), j) for g in gids] for j in range(nkeys)] + [ints, floats]
    csv = b",".join(n.encode() for n in names) + b"\n" + b"".join(b",".join(r) + b"\n" for r in zip(*cols))
    return csv, names, cols


def _rows(names, cols):
    return (dict(zip(names, vals)) for vals in zip(*cols))


def _check(g, keys, aggs, rows):
    """the Groups g equals the reference fold of rows, float values by their bits"""
    import torch
    order, acc, err = gr.fold(rows, keys, aggs)
    assert err is None
    assert g.table.columns == list(keys) and len(g.table) == len(order) == len(g)
    for j, k in enumerate(keys):
        assert g.table.values(k) == [o[j] for o in order], k
    for name, spec in aggs.items():
        v = g.values[name]
        assert v.device.type == "cuda" and v.numel() == len(order)
        if len(spec) == 3 and spec[0] != "count" and spec[2] == "float64":
            assert v.dtype == torch.float64
            got = [x & gr.MASK64 for x in v.view(torch.int64).cpu().tolist()]
        else:
            assert v.dtype == torch.int64
            got = v.cpu().tolist()
        assert got == acc[name], name


@pytest.mark.parametrize("ngroups,nkeys,nrows", [(1, 1, 5000), (7, 2, 20_000), (1000, 3, 60_000), (50_000, 4, 150_000), (1_000_000, 1, 1_200_000)])
def test_random_tables_every_op_and_kind(ngroups, nkeys, nrows):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    csv, names, cols = _data(ngroups + nkeys, nrows, ngroups, nkeys)
    keys = names[:nkeys]
    aggs = ALL_AGGS if ngroups < 1_000_000 else {k: ALL_AGGS[k] for k in ("n", "sum_int", "sum_float64", "min_float64", "last_int")}
    g = cp.Take(cp.FromBytes(csv, ctx)).GroupBy(keys, aggs)
    _check(g, keys, aggs, _rows(names, cols))


@pytest.mark.parametrize("batch", [97, 4096, 64 << 10])
def test_multi_batch_plans_equal_one_batch(monkeypatch, batch):
    import csvplus_b200 as cp
    from csvplus_b200 import api
    ctx = gpu_ctx()
    # group 0 in every batch, groups that first appear only in the last part of the input, and 3000 groups in all
    # (the slot table doubles from 64 to 8192 slots)
    rng = random.Random(batch)
    n = 3000 if batch == 97 else 40_000
    gids = [0 if r % 5 == 0 else (rng.randrange(1, 1500) if r < n // 2 else rng.randrange(1, 3000)) for r in range(n)]
    for x in range(1, 3000):  # the second half of the groups first appears here, group 0 still in between
        gids += [x, 0] if x % 4 == 0 else [x]
    names = ["k0", "k1", "i", "f"]
    cols = [[_key(g, 0) for g in gids], [_key(g, 2) for g in gids], [b"%d" % (g * 7 - r) for r, g in enumerate(gids)],
            [b"%.2f" % (g / 3 + r / 7) for r, g in enumerate(gids)]]
    csv = b"k0,k1,i,f\n" + b"".join(b",".join(r) + b"\n" for r in zip(*cols))
    keys = ["k0", "k1"]
    whole = cp.Take(cp.FromBytes(csv, ctx)).GroupBy(keys, ALL_AGGS)
    monkeypatch.setattr(api, "STREAM_BATCH_BYTES", batch)
    src = cp.Take(cp.FromBytes(csv, ctx))
    batches = sum(1 for _ in src._batches())
    assert batches > 5
    streamed = src.GroupBy(keys, ALL_AGGS)
    _check(streamed, keys, ALL_AGGS, _rows(names, cols))
    assert streamed.table.values("k0") == whole.table.values("k0") and len(streamed) == len(whole) == 3000
    for name in ALL_AGGS:
        assert streamed.values[name].view(-1).cpu().numpy().tobytes() == whole.values[name].cpu().numpy().tobytes(), name


def test_one_group_of_every_row_and_every_row_distinct():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    n = 400_000
    rng = np.random.default_rng(5)
    fv = [b"%.4f" % x for x in rng.normal(size=n) * 100]
    iv = [b"%d" % x for x in rng.integers(-10 ** 12, 10 ** 12, n)]
    csv = b"k,i,f\n" + b"".join(b"same," + a + b"," + b + b"\n" for a, b in zip(iv, fv))
    g = cp.Take(cp.FromBytes(csv, ctx)).GroupBy(["k"], ALL_AGGS)
    _check(g, ["k"], ALL_AGGS, ({"k": b"same", "i": a, "f": b} for a, b in zip(iv, fv)))
    m = 300_000
    csv = b"k,i,f\n" + b"".join(b"%d,%s,%s\n" % (r, iv[r], fv[r]) for r in range(m))
    g = cp.Take(cp.FromBytes(csv, ctx)).GroupBy(["k"], ALL_AGGS)
    _check(g, ["k"], ALL_AGGS, ({"k": b"%d" % r, "i": iv[r], "f": fv[r]} for r in range(m)))


def test_split_empty_and_nul_keys_on_table_sources():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    rows = [{"a": "ab", "b": "c", "v": "1"}, {"a": "a", "b": "bc", "v": "2"}, {"a": "", "b": "", "v": "3"},
            {"a": "\x00", "b": "", "v": "4"}, {"a": "ab", "b": "c", "v": "5"}, {"a": "", "b": "", "v": "6"}]
    t = cp.Table.from_rows(ctx, rows, ["a", "b", "v"])
    aggs = {"n": ("count",), "s": ("sum", "v", "int"), "f": ("first", "v", "int"), "l": ("last", "v", "float64")}
    g = cp.TakeTable(t).GroupBy(["a", "b"], aggs)
    _check(g, ["a", "b"], aggs, ({k: v.encode() for k, v in r.items()} for r in rows))
    assert len(g) == 4


def test_reference_patterns_on_generated_data():
    import torch
    import csvplus_b200 as cp
    from oracle import oracle as orc
    ctx = gpu_ctx()
    people = ctx.gen_csv("people", (0, 2000))
    orders = ctx.gen_csv("orders", (0, 50_000), n_cust=2000, n_prod=50)
    products = ctx.gen_csv("products", (0, 50), n_prod=50)
    ho, hp = orders.to_host(), products.to_host()
    oo = orc.reader_rows(ho, select=["cust_id", "prod_id", "qty"])
    ocust, oprod, oqty = oo.values("cust_id"), oo.values("prod_id"), oo.values("qty")
    po = orc.reader_rows(hp, select=["prod_id", "price"])
    prices = dict(zip(po.values("prod_id"), po.values("price")))

    # TestSimpleUniqueJoin: qty summed per customer after Join(custIdx, "cust_id")
    id_ix = cp.Take(cp.FromBytes(people, ctx).SelectColumns("id", "name", "surname")).UniqueIndexOn("id")
    g = cp.Take(cp.FromBytes(orders, ctx).SelectColumns("order_id", "cust_id", "qty")).Join(id_ix, "cust_id").GroupBy(
        ["id"], {"qty": ("sum", "qty", "int")})
    want: dict = {}
    for c, q in zip(ocust, oqty):  # the RowFunc: custQty[cid] += qty
        want[c] = want.get(c, 0) + int(q)
    assert g.table.values("id") == list(want) and g.values["qty"].cpu().tolist() == list(want.values())

    # TestTransformedSource: amount = FormatFloat(price * qty, 'f', 2), custAmounts[cid] += amount
    prod_ix = cp.Take(cp.FromBytes(products, ctx).SelectColumns("prod_id", "price")).UniqueIndexOn("prod_id")
    plan = cp.Take(cp.FromBytes(orders, ctx).SelectColumns("cust_id", "prod_id", "qty")).Join(prod_ix).MapTensors(
        {"qty": "int", "price": "float64"}, lambda v: {"amount": cp.FormatFloat(v["price"] * v["qty"].to(torch.float64), "f", 2)})
    g = plan.GroupBy(["cust_id"], {"amount": ("sum", "amount", "float64")})
    amounts = plan.ToTensors({"amount": "float64"})["amount"].cpu().tolist()
    custs = [int(x) for x in plan.ToTensors({"cust_id": "int"})["cust_id"].cpu().tolist()]
    want = {}
    for c, a in zip(custs, amounts):
        want[c] = want.get(c, 0.0) + a
    assert [int(x) for x in g.table.values("cust_id")] == list(want)
    assert g.values["amount"].view(torch.int64).cpu().tolist() == torch.tensor(list(want.values()), dtype=torch.float64).view(torch.int64).tolist()
    # the amounts are FormatFloat(price * qty, 'f', 2) of the oracle's rows, in the same order
    assert custs == [int(c) for c in ocust]
    assert amounts == [float("%.2f" % (float(prices[p]) * int(q))) for p, q in zip(oprod, oqty)]

    # TestSimpleTotals: price * qty of each customer's last order
    g = cp.Take(cp.FromBytes(orders, ctx).SelectColumns("cust_id", "prod_id", "qty")).Join(prod_ix).GroupBy(
        ["cust_id"], {"qty": ("last", "qty", "int"), "price": ("last", "price", "float64")})
    totals = g.values["price"] * g.values["qty"].to(torch.float64)
    want = {}
    for c, p, q in zip(ocust, oprod, oqty):
        want[c] = float(prices[p]) * int(q)
    assert g.table.values("cust_id") == list(want) and totals.cpu().tolist() == list(want.values())


def test_conversion_error_in_a_late_batch(monkeypatch):
    import csvplus_b200 as cp
    from csvplus_b200 import api
    ctx = gpu_ctx()
    lines = [b"%d,%d,%d.5" % (r % 13, r, r) for r in range(20_000)]
    lines[15_001] = b"3,12x,1.5"
    lines[15_001 + 7] = b"3,1,zz"
    csv = b"k,i,f\n" + b"\n".join(lines) + b"\n"
    monkeypatch.setattr(api, "STREAM_BATCH_BYTES", 4096)
    for aggs, kinds in (({"a": ("sum", "i", "int"), "b": ("max", "f", "float64")}, {"i": "int", "f": "float64"}),
                        ({"b": ("min", "f", "float64"), "a": ("first", "i", "int")}, {"f": "float64", "i": "int"})):
        with pytest.raises(cp.CsvPlusError) as want:
            cp.Take(cp.FromBytes(csv, ctx)).ToTensors(kinds)
        with pytest.raises(cp.CsvPlusError) as got:
            cp.Take(cp.FromBytes(csv, ctx)).GroupBy(["k"], aggs)
        assert got.value.row == want.value.row == 15_001 and str(got.value) == str(want.value)
    with pytest.raises(cp.CsvPlusError) as got:
        cp.Take(cp.FromBytes(csv, ctx)).Drop(15_002).GroupBy(["k"], {"x": ("sum", "f", "float64")})
    assert got.value.row == 6 and str(got.value) == 'column "f": cannot convert "zz" to float: invalid syntax'


def test_source_error_mid_stream_is_raised(monkeypatch):
    import csvplus_b200 as cp
    from csvplus_b200 import api
    ctx = gpu_ctx()
    lines = [b"%d,%d" % (r % 5, r) for r in range(5000)]
    lines[3000] = b"1,2,3"
    csv = b"k,v\n" + b"\n".join(lines) + b"\n"
    monkeypatch.setattr(api, "STREAM_BATCH_BYTES", 2048)
    with pytest.raises(cp.DataSourceError) as want:
        cp.Take(cp.FromBytes(csv, ctx)).ToRows()
    with pytest.raises(cp.DataSourceError) as got:
        cp.Take(cp.FromBytes(csv, ctx)).GroupBy(["k"], {"s": ("sum", "v", "int")})
    assert str(got.value) == str(want.value) and "wrong number of fields" in str(got.value)


def test_argument_and_missing_column_errors():
    import csvplus_b200 as cp
    from csvplus_b200 import _abi
    ctx = gpu_ctx()
    src = cp.Take(cp.FromBytes(b"k,v\na,1\nb,2\n", ctx))
    for keys, msg in (([], "empty column list in GroupBy()"), (["k", "k"], "duplicate column name(s) in GroupBy()")):
        with pytest.raises(ValueError) as e:
            src.GroupBy(keys, {"n": ("count",)})
        assert str(e.value) == msg
    for aggs in ({"x": ("avg", "v", "int")}, {"x": ("sum", "v", "float32")}, {"x": ("sum", "v")}, {"x": ("count", "v", "int")}):
        with pytest.raises(ValueError):
            src.GroupBy(["k"], aggs)
    for keys, aggs in ((["zz"], {"n": ("count",)}), (["k"], {"n": ("count",), "s": ("sum", "zz", "int")})):
        with pytest.raises(cp.CsvPlusError) as got:
            src.GroupBy(keys, aggs)
        assert str(got.value) == 'missing column "zz"' and got.value.row == 0 and got.value.kind == _abi.CPB_E_MISSING_COLUMN
    with pytest.raises(cp.CsvPlusError) as want:
        src.ToTensors({"zz": "int"})
    assert str(want.value) == 'missing column "zz"'
    # an empty plan: the key columns and no groups
    g = cp.Take(cp.FromBytes(b"k,v\n", ctx)).GroupBy(["v", "k"], {"n": ("count",), "f": ("sum", "v", "float64")})
    assert g.table.columns == ["v", "k"] and len(g) == 0 and g.values["n"].numel() == 0 and str(g.values["f"].dtype) == "torch.float64"
    # a null groups handle is refused
    e = _abi.Error()
    t = cp.Table.from_rows(ctx, [{"k": "a"}], ["k"])
    assert ctx.lib.cpb_groups_push(ctx.h, None, t.h, C.byref(e)) == _abi.CPB_ERR_ARG
    out, n = C.c_void_p(), C.c_uint64()
    assert ctx.lib.cpb_groups_result(ctx.h, None, C.byref(out), C.byref(n)) == _abi.CPB_ERR_ARG
    assert ctx.lib.cpb_groups_values(ctx.h, None, 0, None) == _abi.CPB_ERR_ARG


def test_opaque_map_before_groupby():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    csv, names, cols = _data(3, 20_000, 300, 2)
    keys = names[:2]
    direct = cp.Take(cp.FromBytes(csv, ctx)).GroupBy(keys, ALL_AGGS)
    mapped = cp.Take(cp.FromBytes(csv, ctx)).Map(lambda r: dict(r)).GroupBy(keys, ALL_AGGS)
    _check(mapped, keys, ALL_AGGS, _rows(names, cols))
    assert mapped.table.values("k0") == direct.table.values("k0")
    for name in ALL_AGGS:
        assert mapped.values[name].cpu().numpy().tobytes() == direct.values[name].cpu().numpy().tobytes()


def test_streaming_memory_stays_at_one_batch(monkeypatch):
    import csvplus_b200 as cp
    from csvplus_b200 import api
    ctx = gpu_ctx()
    buf = ctx.gen_csv("orders", (0, 8_000_000), n_cust=1000, n_prod=50)
    data = buf.to_host().tobytes()
    buf.free()
    batch = 4 << 20
    monkeypatch.setattr(api, "STREAM_BATCH_BYTES", batch)
    aggs = {"n": ("count",), "q": ("sum", "qty", "int"), "p": ("max", "prod_id", "float64")}
    cut = data[: data.index(b"\n", 3 * batch) + 1]  # about three batches

    def high(d):
        ctx.sync()
        ctx.pool_used_high(reset=True)
        g = cp.Take(cp.FromBytes(d, ctx)).GroupBy(["cust_id"], aggs)
        assert len(g) == 1000
        return ctx.pool_used_high()
    few, many = high(cut), high(data)
    assert len(data) > 80 * batch
    # 3 batches vs 80: the same high-water mark within 25 % (the groups are fixed, one batch is in flight at a time)
    assert many <= few * 1.25 + (1 << 20), (few, many)
    assert many < len(data), (many, len(data))


def test_host_syncs_and_launches_per_push():
    import csvplus_b200 as cp
    from csvplus_b200 import _abi
    ctx = gpu_ctx()
    aggs = [("n", 0, 0, b""), ("s", 1, 0, b"v"), ("m", 3, 1, b"w")]
    arr = (_abi.Agg * 3)(*[_abi.Agg(op, kind, _abi.Str(c, len(c))) for _, op, kind, c in aggs])
    ka = (_abi.Str * 1)(_abi.Str(b"k", 1))

    def table(n, offset):
        return cp.Table.from_rows(ctx, [{"k": str((r + offset) % 500), "v": str(r), "w": "%d.5" % r} for r in range(n)], ["k", "v", "w"])
    deltas = []
    for n in (1000, 20_000):
        h = C.c_void_p()
        ctx._call("cpb_groups_open", ka, 1, arr, 3, C.byref(h))
        try:
            for t in (table(n, 0), table(n, 7)):  # the first push creates every group, the second finds them all
                ctx.sync()
                s0, l0 = ctx.host_syncs(), ctx.kernel_launches()
                ctx._call("cpb_groups_push", h, t.h)
                deltas.append((ctx.host_syncs() - s0, ctx.kernel_launches() - l0))
        finally:
            ctx._call("cpb_groups_free", h)
    # two converted inputs + the miss count + the sort; + the new-group count and the key rows' gather on new groups
    assert [d[0] for d in deltas] == [6, 4, 6, 4], deltas
    assert deltas[0][1] == deltas[2][1] and deltas[1][1] == deltas[3][1], deltas


def test_cpp_groupby_example():
    exe = os.path.join(ROOT, "host", "groupby_example")
    if not os.path.exists(exe):
        import __graft_entry__ as g
        g.build()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "groupby example ok" in r.stdout
