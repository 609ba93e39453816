"""Row.ValueAsInt / ValueAsFloat64 on the GPU (csrc/numeric.cu, cpb_table_column_as_*) compared bit for bit with the
restated strconv of tests/strconv_oracle.py: the golden fixture, a grammar-aware fuzz, a rounding corpus that drives the
rare (exact) path, layouts (views, join results, empty tables and values), Table.values_as_* / DataSource.ToTensors in
both modes, the reference's TestSimpleTotals / TestSimpleUniqueJoin sums, and 100 M generated orders rows."""
import os

import numpy as np
import pytest

from tests import numeric_corpus as nc
from tests import strconv_oracle as so
from tests.helpers import gpu_ctx

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _table(values, name="v"):
    import csvplus_b200 as cp
    return cp.Table.from_rows(gpu_ctx(), [{name: v} for v in values], columns=[name])


def _check(t, name, values, is_float, check_msg=True):
    """converts column `name` of t (whose rows hold `values`) both ways and compares value bits, status and message"""
    import torch
    import csvplus_b200 as cp
    want = [so.parse_float(v) if is_float else so.atoi(v) for v in values]
    wv = np.array([w[0] for w in want], dtype=np.uint64 if is_float else np.int64)
    ws = np.array([w[1] for w in want], dtype=np.uint8)
    got, st = (t.values_as_float64 if is_float else t.values_as_int)(name, strict=False)
    assert got.dtype == (torch.float64 if is_float else torch.int64) and got.device.type == "cuda"
    gv = got.cpu().numpy().view(np.uint64 if is_float else np.int64)
    gs = st.cpu().numpy()
    bad = np.nonzero((gv != wv) | (gs != ws))[0]
    assert len(bad) == 0, [(values[i][:60], hex(int(gv[i])), int(gs[i]), hex(int(wv[i])), int(ws[i])) for i in bad[:10]]
    nbad = int((ws != 0).sum())
    if nbad:
        with pytest.raises(cp.CsvPlusError) as ei:
            (t.values_as_float64 if is_float else t.values_as_int)(name)
        first = int(np.nonzero(ws)[0][0])
        assert ei.value.row == first
        assert ei.value.kind == (16 if ws[first] == 1 else 17)
        if check_msg:
            assert str(ei.value) == so.message(name, values[first], is_float, int(ws[first]))
    else:
        assert bool(((t.values_as_float64 if is_float else t.values_as_int)(name).cpu().numpy().view(gv.dtype) == gv).all())
    return nbad


def _rare_rows(ctx):
    return ctx.stats().get("numeric_rare", {})


def test_golden_fixture():
    import csvplus_b200 as cp
    csv = open(os.path.join(GOLDEN, "numeric_kat.csv"), "rb").read()
    t, err = cp.parse_csv(gpu_ctx(), csv, spec=[("s", -1)])
    assert err is None
    want = [line.split() for line in open(os.path.join(GOLDEN, "numeric_kat.expected")).read().splitlines()]
    vals = t.values("s")
    assert len(vals) == len(want)
    iv, ist = t.values_as_int("s", strict=False)
    fv, fst = t.values_as_float64("s", strict=False)
    iv, ist = iv.cpu().numpy(), ist.cpu().numpy()
    fv, fst = fv.cpu().numpy().view(np.uint64), fst.cpu().numpy()
    for i, (ai, ais, fb, fs) in enumerate(want):
        assert (int(iv[i]), int(ist[i]), int(fv[i]), int(fst[i])) == (int(ai), int(ais), int(fb, 16), int(fs)), vals[i]


def test_fuzz_one_million():
    ctx = gpu_ctx()
    vals = nc.fuzz(1_000_000, 20261015)
    t = _table(vals)
    assert _check(t, "v", vals, False) > 0
    ctx.stats(enable=True, reset=True)
    assert _check(t, "v", vals, True) > 0
    ctx.stats(enable=False)


def test_rounding_corpus_drives_the_rare_path():
    ctx = gpu_ctx()
    vals = nc.rounding_corpus(200_000, 77)
    t = _table(vals)
    ctx.stats(enable=True, reset=True)
    s0 = ctx.host_syncs()
    got, st = t.values_as_float64("v", strict=False)
    assert ctx.host_syncs() - s0 == 1  # one synchronisation per call
    rare = _rare_rows(ctx)
    ctx.stats(enable=False)
    assert rare and rare["launches"] == 1 and rare["algo_bytes"] > 100_000 * 17  # the exact path converted rows
    _check(t, "v", vals, True)


def test_layouts():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    vals = nc.fuzz(5000, 3) + [b"1" * 3000, b"1." + b"7" * 2500 + b"e-2400", b"", b"-", b"12345678901234567890"] + nc.fuzz(2000, 4)
    t = _table(vals)
    for lo, hi in [(0, len(vals)), (1, 2), (7, 1000), (33, 5013), (5001, 5007), (4999, len(vals))]:
        s = t.slice(lo, hi)
        _check(s, "v", vals[lo:hi], False)
        _check(s, "v", vals[lo:hi], True)
    # a column of empty strings, and an empty table
    e = _table([b""] * 100)
    assert _check(e, "v", [b""] * 100, True) == 100
    z = t.slice(3, 3)
    v = z.values_as_int("v")
    assert v.numel() == 0
    assert z.values_as_float64("nope").numel() == 0  # no rows: nothing to convert, nothing missing
    # status=None through the C ABI
    import ctypes as C
    import torch
    from csvplus_b200 import _abi
    out = torch.empty(len(vals), dtype=torch.float64, device="cuda")
    nbad = C.c_uint64(); err = _abi.Error()
    st = ctx.lib.cpb_table_column_as_float64(ctx.h, t.h, _abi.Str(b"v", 1), C.c_void_p(out.data_ptr()), None, C.byref(nbad), C.byref(err))
    want = [so.parse_float(x) for x in vals]
    assert st == (1 if any(w[1] for w in want) else 0)
    assert nbad.value == sum(1 for w in want if w[1])
    assert out.cpu().numpy().view(np.uint64).tolist() == [w[0] for w in want]
    # the missing column
    with pytest.raises(cp.CsvPlusError) as ei:
        t.values_as_int("qty", strict=False)
    assert str(ei.value) == 'missing column "qty"' and ei.value.kind == 10


def test_join_columns_shared_and_gathered():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    people = ctx.gen_csv("people", (0, 20_000))
    orders = ctx.gen_csv("orders", (0, 300_000), n_cust=25_000, n_prod=100)
    cust, _ = cp.parse_csv(ctx, people, spec=[("id", -1), ("score", -1)])
    o, _ = cp.parse_csv(ctx, orders, spec=[("order_id", -1), ("cust_id", -1), ("qty", -1)])
    j = o.join(cust.index_on("id", unique=True), "cust_id")
    assert 0 < len(j) < len(o)
    for name, is_float in [("cust_id", False), ("id", False), ("qty", False), ("order_id", False), ("score", True), ("qty", True)]:
        assert _check(j, name, j.values(name), is_float) == 0
    js = j.slice(3, len(j) - 5)
    assert _check(js, "score", js.values("score"), True) == 0


def test_to_tensors_and_error_order():
    import torch
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    csv = b"a,b,c\n1,2.5,x\n2,3e1,y\n3,oops,z\n4,1,w\nx,1e999,q\n"
    src = cp.Take(cp.FromBytes(csv, ctx))
    with pytest.raises(cp.CsvPlusError) as ei:
        src.ToTensors({"a": "int", "b": "float64"})
    assert str(ei.value) == 'column "b": cannot convert "oops" to float: invalid syntax' and ei.value.row == 2
    with pytest.raises(cp.CsvPlusError) as ei:  # row 4 fails in both columns: the earlier column in dict order wins
        cp.Take(cp.FromBytes(csv, ctx)).Drop(3).ToTensors({"b": "float64", "a": "int"})
    assert ei.value.row == 1 and str(ei.value) == 'column "b": cannot convert "1e999" to float: value out of range'
    with pytest.raises(cp.CsvPlusError) as ei:
        cp.Take(cp.FromBytes(csv, ctx)).Drop(3).ToTensors({"a": "int", "b": "float64"})
    assert ei.value.row == 1 and str(ei.value) == 'column "a": cannot convert "x" to integer: invalid syntax'
    out = cp.Take(cp.FromBytes(csv, ctx)).Top(2).ToTensors({"a": "int", "b": "float64"})
    assert out["a"].tolist() == [1, 2] and out["b"].tolist() == [2.5, 30.0]
    with pytest.raises(cp.CsvPlusError) as ei:
        cp.Take(cp.FromBytes(csv, ctx)).Top(2).ToTensors({"a": "int", "zz": "int"})
    assert str(ei.value) == 'missing column "zz"'
    # a conversion error before a pending parse error is raised first; with none, the parse error
    bad = b"a,b\n1,2\nq,3\n4,5\n6,7,8\n"
    with pytest.raises(cp.CsvPlusError) as ei:
        cp.Take(cp.FromBytes(bad, ctx)).ToTensors({"a": "int"})
    assert ei.value.row == 1
    with pytest.raises(cp.DataSourceError) as ei:
        cp.Take(cp.FromBytes(bad, ctx)).ToTensors({"b": "int"})
    assert "wrong number of fields" in str(ei.value)
    # rows left on the host after an opaque closure are uploaded again
    out = cp.Take(cp.FromBytes(csv, ctx)).Top(2).Map(lambda r: {**r, "a": r["a"] + "0"}).ToTensors({"a": "int"})
    assert out["a"].tolist() == [10, 20]
    assert cp.Take(cp.FromBytes(b"a\n", ctx)).ToTensors({"a": "int"})["a"].numel() == 0
    # strict=False returns the values Go returns alongside the errors
    t = _table([b"7", b"99999999999999999999x", b"-99999999999999999999", b"x"])
    v, s = t.values_as_int("v", strict=False)
    assert v.tolist() == [7, 2 ** 63 - 1, -2 ** 63, 0] and s.tolist() == [0, 2, 2, 1]
    assert v.dtype == torch.int64


def _people_orders(ctx, n_people, n_orders, n_prod=50):
    import csvplus_b200 as cp
    people = ctx.gen_csv("people", (0, n_people))
    orders = ctx.gen_csv("orders", (0, n_orders), n_cust=n_people, n_prod=n_prod)
    products = ctx.gen_csv("products", (0, n_prod), n_prod=n_prod)
    return people, orders, products, cp


def test_simple_totals_and_unique_join_sums():
    import torch
    from oracle import oracle as orc
    ctx = gpu_ctx()
    people, orders, products, cp = _people_orders(ctx, 2000, 50_000)
    # TestSimpleTotals: totals[cust] = price * qty of the customer's last order
    prod_ix = cp.Take(cp.FromBytes(products, ctx).SelectColumns("prod_id", "price")).UniqueIndexOn("prod_id")
    got = cp.Take(cp.FromBytes(orders, ctx).SelectColumns("cust_id", "prod_id", "qty")).Join(prod_ix).ToTensors(
        {"cust_id": "int", "qty": "int", "price": "float64"})
    dev = got["qty"].device
    # rows come in probe order: each customer's last order is its highest row (scatter with duplicate indices has no
    # defined winner on the GPU, so take the row positions' maximum first)
    last = torch.full((2000,), -1, dtype=torch.int64, device=dev).scatter_reduce_(
        0, got["cust_id"], torch.arange(got["qty"].numel(), device=dev), reduce="amax")
    has = last >= 0
    totals = torch.zeros(2000, dtype=torch.float64, device=dev)
    totals[has] = got["price"][last[has]] * got["qty"][last[has]].to(torch.float64)
    ho, hp = orders.to_host(), products.to_host()
    po = orc.reader_rows(hp, select=["prod_id", "price"])
    prices = dict(zip(po.values("prod_id"), (float(x) for x in po.values("price"))))
    oo = orc.reader_rows(ho, select=["cust_id", "prod_id", "qty"])
    ocust, oprod, oqty = oo.values("cust_id"), oo.values("prod_id"), oo.values("qty")
    want = [0.0] * 2000
    for c, p, q in zip(ocust, oprod, oqty):
        want[int(c)] = prices[p] * int(q)
    assert totals.cpu().tolist() == want
    # TestSimpleUniqueJoin's per-customer qty sums
    id_ix = cp.Take(cp.FromBytes(people, ctx).SelectColumns("id", "name", "surname")).UniqueIndexOn("id")
    got = cp.Take(cp.FromBytes(orders, ctx).SelectColumns("order_id", "cust_id", "qty")).Join(id_ix, "cust_id").ToTensors(
        {"id": "int", "qty": "int"})
    sums = torch.zeros(2000, dtype=torch.int64, device=got["qty"].device).index_add_(0, got["id"], got["qty"])
    want = [0] * 2000
    for c, q in zip(ocust, oqty):
        want[int(c)] += int(q)
    assert sums.cpu().tolist() == want


def _gen_rnd(seed, kind, rows, col):
    """gen.cu's rnd(): splitmix64 of the seed, kind, row and column, vectorised"""
    M = np.uint64(0xFFFFFFFFFFFFFFFF)
    with np.errstate(over="ignore"):
        x = (np.uint64(seed) ^ np.uint64((kind + 1) << 56) ^ (rows * np.uint64(0xD1342543DE82EF95)) ^ np.uint64((col * 0xA24BAED4963EE407) & 0xFFFFFFFFFFFFFFFF)) & M
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def test_scale_orders_100m():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    n, chunk, ncust, nprod, seed = 100_000_000, 20_000_000, 10_000_000, 1000, 0xC5B200
    for lo in range(0, n, chunk):
        buf = ctx.gen_csv("orders", (lo, lo + chunk), n_cust=ncust, n_prod=nprod, header=lo == 0, seed=seed)
        spec = [("cust_id", 1), ("qty", 3)]
        t, err = cp.parse_csv(ctx, buf, spec=spec, header_from_first_row=lo == 0, num_fields=5)
        assert err is None and len(t) == chunk
        qty = t.values_as_int("qty").cpu().numpy()
        cust = t.values_as_int("cust_id").cpu().numpy()
        rows = np.arange(lo, lo + chunk, dtype=np.uint64)
        assert np.array_equal(cust, (_gen_rnd(seed, 1, rows, 1) % np.uint64(ncust)).astype(np.int64))
        assert np.array_equal(qty, (np.uint64(1) + _gen_rnd(seed, 1, rows, 3) % np.uint64(100)).astype(np.int64))
        del t, buf
    buf = ctx.gen_csv("products", (0, 1_000_000), n_prod=1_000_000, seed=seed)
    t, err = cp.parse_csv(ctx, buf, spec=[("price", -1)])
    price = t.values_as_float64("price").cpu().numpy()
    s = _gen_rnd(seed, 2, np.arange(0, 1_000_000, dtype=np.uint64), 2)
    whole, cents = (s % np.uint64(1000)).astype(np.int64), ((s >> np.uint64(32)) % np.uint64(100)).astype(np.int64)
    want = np.array([float(f"{a}.{b:02d}") for a, b in zip(whole.tolist(), cents.tolist())])
    assert np.array_equal(price.view(np.uint64), want.view(np.uint64))
