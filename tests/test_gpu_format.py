"""Computed columns on the GPU (csrc/format.cu, cpb_table_set_*, cpb_table_filter_flags, Table.with_column /
filter_mask, DataSource.MapTensors / FilterTensors) compared byte for byte with tests/ftoa_oracle.py: the golden
fixture, int and float fuzz under every format, the exact path, the ParseFloat round trip at 100 M rows, layouts,
limits, host synchronisations, streamed plan steps against the host closures, and the reference's pipelines."""
import io
import multiprocessing as mp
import os
import random
import subprocess
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

from tests import ftoa_oracle as fo
from tests.helpers import gpu_ctx

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
MODES = [("g", -1), ("e", -1), ("f", -1), ("f", 0), ("f", 2), ("f", 17), ("f", 40), ("e", 0), ("e", 5), ("e", 17), ("e", 25),
         ("g", 1), ("g", 6), ("g", 17), ("g", 30), ("E", 3), ("G", -1)]


def _base(n, ctx=None):
    """a device table of n rows with one column of empty strings"""
    import torch
    import csvplus_b200 as cp
    ctx = ctx or gpu_ctx()
    dev = torch.device("cuda", ctx.device)
    off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    data = torch.zeros(16, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    return cp.Table.from_device_columns(ctx, ["k"], [(off.data_ptr(), data.data_ptr())], n)


def _texts(t, name):
    off, data = t.column(name)
    d = data.tobytes()
    return [d[off[i]:off[i + 1]].decode() for i in range(len(off) - 1)]


def _tensor(vals, dtype):
    import torch
    return torch.tensor(np.asarray(vals).view(np.int64 if dtype == torch.int64 else np.float64), dtype=dtype, device="cuda")


def _fmt_chunk(args):
    xs, fmt, prec = args
    return [fo.format_float(x, fmt, prec) for x in xs]


def _oracle_many(xs, fmt, prec):
    """the oracle over many values, in worker processes (pure Python: nothing there touches the GPU)"""
    chunks = [(xs[i:i + 50_000], fmt, prec) for i in range(0, len(xs), 50_000)]
    with ProcessPoolExecutor(max_workers=min(16, os.cpu_count() or 1), mp_context=mp.get_context("fork")) as ex:
        return [s for part in ex.map(_fmt_chunk, chunks) for s in part]


def _diff(got, want, vals):
    bad = [i for i in range(len(want)) if got[i] != want[i]]
    return [(hex(int(np.asarray(vals[i]).view(np.uint64))) if isinstance(vals[i], float) else vals[i], got[i], want[i]) for i in bad[:10]]


def test_golden_fixture():
    import torch
    groups = {}
    for line in open(os.path.join(GOLDEN, "format_kat.csv")).read().splitlines():
        kind, v, fmt, prec, want = line.split(",", 4)
        groups.setdefault((kind, fmt, int(prec)), []).append((v, want))
    for (kind, fmt, prec), items in groups.items():
        t = _base(len(items))
        if kind == "i":
            out = t.with_column("v", _tensor([int(v) for v, _ in items], torch.int64))
        else:
            vals = np.array([int(v, 16) for v, _ in items], dtype=np.uint64).view(np.float64)
            out = t.with_column("v", _tensor(vals, torch.float64), fmt=fmt, prec=prec)
        got = _texts(out, "v")
        assert got == [w for _, w in items], (kind, fmt, prec, [(v, g, w) for (v, w), g in zip(items, got) if g != w][:10])


def test_int_fuzz():
    import torch
    rng = np.random.default_rng(7)
    edges = [0, 1, -1, 2**63 - 1, -2**63, -2**63 + 1]
    for k in range(19):
        for s in (1, -1):
            edges += [s * 10**k, s * (10**k - 1), s * (10**k + 1)]
    vals = np.concatenate([np.array(edges, dtype=np.int64), rng.integers(-2**63, 2**63 - 1, size=1_000_000, dtype=np.int64),
                           rng.integers(-10**6, 10**6, size=10_000, dtype=np.int64)])
    out = _base(len(vals)).with_column("n", torch.from_numpy(vals).cuda())
    got = _texts(out, "n")
    want = [str(v) for v in vals.tolist()]
    assert got == want, _diff(got, want, vals.tolist())


def _random_bits(n, seed):
    rng = np.random.default_rng(seed)
    u = rng.integers(0, 2**64, size=n, dtype=np.uint64)
    special = np.array([0, 1 << 63, 1, (1 << 63) | 1, 0x000FFFFFFFFFFFFF, 0x0010000000000000, 0x7FF0000000000000, 0xFFF0000000000000,
                        0x7FF8000000000001, 0x7FEFFFFFFFFFFFFF, 0x3FF0000000000000, 0x4415AF1D78B58C40], dtype=np.uint64)
    u[: len(special)] = special
    sub = rng.integers(0, 2**52, size=n // 50, dtype=np.uint64)  # subnormals
    u[len(special):len(special) + len(sub)] = sub
    return u


@pytest.mark.parametrize("fmt,prec", MODES)
def test_float_fuzz(fmt, prec):
    import torch
    u = _random_bits(1_000_000, 11 + MODES.index((fmt, prec)))
    xs = u.view(np.float64)
    out = _base(len(u)).with_column("x", torch.from_numpy(xs.copy()).cuda(), fmt=fmt, prec=prec)
    got = _texts(out, "x")
    want = _oracle_many(xs.tolist(), fmt, prec)
    assert got == want, _diff(got, want, xs.tolist())


def test_exact_path_runs():
    import torch
    ctx = gpu_ctx()
    for fmt, prec, vals in (("f", 40, [1e300, -1e300, 1.5e300]), ("e", 25, [0.1, 2.0 / 3, 1e-300, 5e-324])):
        ctx.stats(True, reset=True)
        ctx.stats(True)
        out = _base(len(vals)).with_column("x", torch.tensor(vals, dtype=torch.float64, device="cuda"), fmt=fmt, prec=prec)
        st = ctx.stats()
        ctx.stats(False)
        assert st.get("format_rare", {}).get("launches", 0) >= 1, st
        assert st["format_rare"]["algo_bytes"] == 8 * len(vals)  # the rows the exact path converted, 8 B each
        assert _texts(out, "x") == [fo.format_float(x, fmt, prec) for x in vals]


def test_round_trip_100m():
    import torch
    n = 100_000_000
    g = torch.Generator(device="cuda").manual_seed(5)
    bits = torch.randint(-2**63, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g)
    x = bits.view(torch.float64)
    finite = torch.isfinite(x)
    x = torch.where(finite, x, torch.zeros_like(x))
    t = _base(n).with_column("x", x)
    back = t.values_as_float64("x")
    assert torch.equal(back.view(torch.int64), x.view(torch.int64))
    idx = torch.randint(0, n, (1_000_000,), device="cuda", generator=g).sort().values
    sample = x[idx].cpu().numpy()
    part = t.select("x")
    ii = idx.cpu().numpy()
    off, data = part.column("x")
    d = data.tobytes()
    got = [d[off[i]:off[i + 1]].decode() for i in ii]
    want = _oracle_many(sample.tolist(), "g", -1)
    assert got == want, _diff(got, want, sample.tolist())


def test_layouts_slices_joins_replace_literal_empty():
    import torch
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    rows = [{"id": str(i), "name": "n%d" % (i % 7), "qty": str(i * 3 - 50)} for i in range(1000)]
    t = cp.Table.from_rows(ctx, rows, ["id", "name", "qty"])
    # a row-range view
    s = t.slice(100, 350)
    q = s.values_as_int("qty")
    out = s.with_column("qty2", q * 2)
    assert _texts(out, "qty2") == [str((i * 3 - 50) * 2) for i in range(100, 350)]
    assert _texts(out, "id") == [str(i) for i in range(100, 350)]
    # replacing a column keeps its place and every other column's buffers
    r = t.with_column("name", torch.arange(1000, dtype=torch.int64, device="cuda") - 500)
    assert r.columns == ["id", "name", "qty"]
    assert _texts(r, "name") == [str(i - 500) for i in range(1000)]
    for c in ("id", "qty"):
        assert r.device_column(c) == t.device_column(c)
    assert _texts(t, "name") == [row["name"] for row in rows]  # the input table is unchanged
    # a join result
    ix = cp.Table.from_rows(ctx, [{"id": str(i), "price": "%d.25" % i} for i in range(0, 1000, 3)], ["id", "price"]).index_on("id", unique=True)
    j = t.join(ix, "id")
    amt = j.values_as_float64("price") * j.values_as_int("qty").to(torch.float64)
    jr = j.with_column("amount", cp.FormatFloat(amt, "f", 2))
    want = [fo.format_float(float(p) * float(qq), "f", 2) for p, qq in zip(j.values("price"), j.values("qty"))]
    assert _texts(jr, "amount") == want
    # a literal, an empty literal and an empty table
    lit = t.with_column("name", "Julia")
    assert _texts(lit, "name") == ["Julia"] * 1000
    assert _texts(t.with_column("z", ""), "z") == [""] * 1000
    e = t.slice(5, 5)
    for v in ("x", torch.empty(0, dtype=torch.int64, device="cuda"), torch.empty(0, dtype=torch.float64, device="cuda")):
        ee = e.with_column("w", v)
        assert len(ee) == 0 and ee.columns == ["id", "name", "qty", "w"]
    assert len(e.filter_mask(torch.empty(0, dtype=torch.bool, device="cuda"))) == 0
    # filter_mask
    keep = torch.arange(1000, device="cuda") % 3 == 1
    f = t.filter_mask(keep)
    assert _texts(f, "id") == [str(i) for i in range(1000) if i % 3 == 1]


def test_side_stream_and_freed_tensor():
    import torch
    t = _base(1 << 20)
    dev = torch.device("cuda", gpu_ctx().device)
    side = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)  # the values are produced late on a side stream
        v = torch.arange(1 << 20, dtype=torch.int64, device=dev) * 7 - 12345
        out = t.with_column("v", v)
    want = [str(i * 7 - 12345) for i in range(1 << 20)]
    assert _texts(out, "v") == want
    # a tensor freed right after the call, its memory reused at once
    for _ in range(3):
        x = torch.full((1 << 20,), 0.1, dtype=torch.float64, device=dev)
        o2 = t.with_column("x", x, fmt="e", prec=25)
        del x
        torch.full((1 << 20,), 7.0, dtype=torch.float64, device=dev)
        assert set(_texts(o2, "x")) == {fo.format_float(0.1, "e", 25)}


def test_limits_and_refusals():
    import torch
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    n = 13_000_000  # "1" + 300 zeros + "." + 40 zeros: 342 bytes per row, 4.45 GB in all
    t = _base(n)
    with pytest.raises(cp.CsvPlusError) as ei:
        t.with_column("x", torch.full((n,), 1e300, dtype=torch.float64, device="cuda"), fmt="f", prec=40)
    assert ei.value.kind == 13 and ei.value.status == 1
    del t
    s = _base(10)
    x = torch.zeros(10, dtype=torch.float64, device="cuda")
    for fmt, prec in (("b", -1), ("x", 2), ("g", 65), ("e", -2), ("ff", 1)):
        with pytest.raises(ValueError):
            s.with_column("x", x, fmt=fmt, prec=prec)
        with pytest.raises(ValueError):
            cp.FormatFloat(x, fmt, prec)
    # the C ABI refuses them too
    import ctypes as C
    from csvplus_b200 import _abi
    h = C.c_void_p(); e = _abi.Error()
    for fmt, prec in ((b"b", -1), (b"g", 65), (b"e", -2)):
        st = ctx.lib.cpb_table_set_float64(ctx.h, s.h, _abi.Str(b"x", 1), C.c_void_p(x.data_ptr()), fmt, prec, C.byref(h), C.byref(e))
        assert st == 2
    with pytest.raises(TypeError):
        s.with_column("x", torch.zeros(10, dtype=torch.float32, device="cuda"))
    with pytest.raises(TypeError):
        s.with_column("x", torch.zeros(10, dtype=torch.int64, device="cuda"), fmt="f")
    with pytest.raises(TypeError):
        s.with_column("x", [1, 2, 3])
    with pytest.raises(ValueError):
        s.with_column("x", torch.zeros(11, dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError):
        s.with_column("x", torch.zeros(10, dtype=torch.int64))  # host memory
    with pytest.raises(TypeError):
        s.filter_mask(torch.zeros(10, dtype=torch.int64, device="cuda"))


def test_host_syncs_per_call():
    import torch
    ctx = gpu_ctx()
    t = _base(100_000)
    x = torch.linspace(-1e5, 1e5, 100_000, dtype=torch.float64, device="cuda")
    for fmt, prec in (("g", -1), ("f", 2), ("e", 25), ("f", 40)):
        before = ctx.host_syncs()
        t.with_column("x", x, fmt=fmt, prec=prec)
        assert ctx.host_syncs() - before <= 2
    before = ctx.host_syncs()
    t.with_column("i", torch.arange(100_000, device="cuda"))
    assert ctx.host_syncs() - before == 1
    before = ctx.host_syncs()
    t.slice(0, 0).with_column("i", torch.empty(0, dtype=torch.int64, device="cuda"))
    assert ctx.host_syncs() == before


# ------------------------------------------------------------------ plan steps
def _people_csv(n, seed=3):
    rnd = random.Random(seed)
    lines = ["id,name,surname,born,price,qty"]
    for i in range(n):
        lines.append("%d,%s,%s,%d,%s,%d" % (i, rnd.choice(["Amelia", "Jack", "Ava"]), rnd.choice(["Smith", "Jones"]), rnd.randint(1940, 2005),
                                            repr(rnd.uniform(0, 1000)) if i % 5 else str(rnd.randint(1, 99)), rnd.randint(-5, 50)))
    return ("\n".join(lines) + "\n").encode()


def _map_dev(v):
    import torch
    return {"amount": fo_marker(v["price"] * v["qty"].to(torch.float64)), "born2": v["born"] * 2 + 1, "tag": "x", "ratio": v["price"] * 0.3}


def fo_marker(t):
    import csvplus_b200 as cp
    return cp.FormatFloat(t, "f", 2)


def _map_host(row):
    p, q, b = float(row["price"]), int(row["qty"]), int(row["born"])
    row = dict(row)
    row["amount"] = fo.format_float(p * q, "f", 2)
    row["born2"] = str(b * 2 + 1)
    row["tag"] = "x"
    row["ratio"] = fo.format_float(p * 0.3, "g", -1)
    return row


INPUTS = {"price": "float64", "qty": "int", "born": "int"}


@pytest.mark.parametrize("batch", [64, 4096, 1 << 20])
def test_map_filter_tensors_streamed(monkeypatch, batch):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", batch)
    data = _people_csv(5000)
    cols = ["id", "name", "amount", "born2", "tag", "ratio"]

    def dev():
        return (cp.Take(cp.FromBytes(data, ctx)).MapTensors(INPUTS, _map_dev)
                .FilterTensors({"born": "int"}, lambda v: v["born"] > 1970))

    def host():
        return cp.Take(cp.FromBytes(data, ctx)).Map(_map_host).Filter(lambda r: int(r["born"]) > 1970)

    for sink in ("csv", "json"):
        a, b = io.BytesIO(), io.BytesIO()
        if sink == "csv":
            dev().ToCsv(a, *cols); host().ToCsv(b, *cols)
        else:
            dev().ToJSON(a); host().ToJSON(b)
        assert a.getvalue() == b.getvalue(), sink
    # Join and IndexOn after the steps
    ix = cp.Table.from_rows(ctx, [{"id": str(i), "w": "w%d" % i} for i in range(0, 5000, 7)], ["id", "w"]).index_on("id", unique=True)
    a, b = io.BytesIO(), io.BytesIO()
    dev().Join(ix, "id").ToCsv(a, "id", "w", "amount")
    host().Join(ix, "id").ToCsv(b, "id", "w", "amount")
    assert a.getvalue() == b.getvalue()
    ia, ib = dev().IndexOn("amount"), host().IndexOn("amount")
    assert ia.table().rows() == ib.table().rows()


def test_conversion_error_ordinals_and_prefix(monkeypatch):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 100)
    lines = ["a,b"] + ["%d,%d" % (i, i) for i in range(40)]
    lines[31] = "30,zz"  # row 30 (0-based) fails in column b
    lines[34] = "x33,33"
    data = ("\n".join(lines) + "\n").encode()
    seen = []

    def fn(v):
        seen.append(len(v["a"]))
        return {"c": v["a"] + v["b"]}

    out = io.BytesIO()
    with pytest.raises(cp.CsvPlusError) as ei:
        cp.Take(cp.FromBytes(data, ctx)).MapTensors({"a": "int", "b": "int"}, fn).ToCsv(out, "a", "c")
    assert ei.value.row == 30 and ei.value.kind == 16
    assert 'cannot convert "zz" to integer' in str(ei.value)
    assert out.getvalue() == ("a,c\n" + "".join("%d,%d\n" % (i, 2 * i) for i in range(30))).encode()
    assert sum(seen) == 30
    # the ordinal counts the rows that reached the step, after an upstream filter
    with pytest.raises(cp.CsvPlusError) as ei:
        (cp.Take(cp.FromBytes(data, ctx)).FilterTensors({"a": "int"}, lambda v: v["a"] % 2 == 0)
         .MapTensors({"b": "int"}, lambda v: {"d": v["b"]}).ToRows())
    assert ei.value.row == 15


def test_source_error_after_map_tensors(monkeypatch):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 64)
    data = b"a,b\n" + b"".join(b"%d,%d\n" % (i, i) for i in range(30)) + b"1,2,3\n" + b"5,5\n"
    a, b = io.BytesIO(), io.BytesIO()
    with pytest.raises(cp.DataSourceError) as ea:
        cp.Take(cp.FromBytes(data, ctx)).MapTensors({"a": "int"}, lambda v: {"c": v["a"] * 10}).ToCsv(a, "a", "c")
    with pytest.raises(cp.DataSourceError) as eb:
        cp.Take(cp.FromBytes(data, ctx)).Map(lambda r: dict(r, c=str(int(r["a"]) * 10))).ToCsv(b, "a", "c")
    assert str(ea.value) == str(eb.value)
    assert a.getvalue() == b.getvalue()


def test_reference_pipelines():
    import torch
    import csvplus_b200 as cp
    from oracle import oracle as orc
    ctx = gpu_ctx()
    people = ctx.gen_csv("people", (0, 2000))
    orders = ctx.gen_csv("orders", (0, 50_000), n_cust=2000, n_prod=50)
    products = ctx.gen_csv("products", (0, 50), n_prod=50)
    hp, ho, hpr = people.to_host().tobytes(), orders.to_host().tobytes(), products.to_host().tobytes()
    # createAmountsTable + TestSimpleTotals
    prod_ix = cp.Take(cp.FromBytes(hpr, ctx).SelectColumns("prod_id", "price")).UniqueIndexOn("prod_id")

    def amounts_dev():
        return (cp.Take(cp.FromBytes(ho, ctx).SelectColumns("cust_id", "prod_id", "qty")).Join(prod_ix)
                .MapTensors({"qty": "int", "price": "float64"},
                            lambda v: {"amount": cp.FormatFloat(v["price"] * v["qty"].to(torch.float64), "f", 2)})
                .DropColumns("price", "qty"))

    def amounts_host():
        def tr(row):
            row = dict(row)
            row["amount"] = fo.format_float(float(row["price"]) * int(row["qty"]), "f", 2)
            del row["price"], row["qty"]
            return row
        return cp.Take(cp.FromBytes(ho, ctx).SelectColumns("cust_id", "prod_id", "qty")).Join(prod_ix).Transform(tr)

    ra, rb = amounts_dev().ToRows(), amounts_host().ToRows()
    assert ra == rb and len(ra) == 50_000
    totals_dev, totals_host = {}, {}
    for r in ra:
        totals_dev[r["cust_id"]] = float(r["amount"])
    po = orc.reader_rows(hpr, select=["prod_id", "price"])
    prices = dict(zip(po.values("prod_id"), (float(x) for x in po.values("price"))))
    oo = orc.reader_rows(ho, select=["cust_id", "prod_id", "qty"])
    for c, p, q in zip(oo.values("cust_id"), oo.values("prod_id"), oo.values("qty")):
        totals_host[c.decode()] = float(fo.format_float(prices[p] * int(q), "f", 2))
    assert totals_dev == totals_host
    # the join test's born > 1970 filter
    a = cp.Take(cp.FromBytes(hp, ctx)).FilterTensors({"born": "int"}, lambda v: v["born"] > 1970).ToRows()
    b = cp.Take(cp.FromBytes(hp, ctx)).Filter(lambda r: int(r["born"]) > 1970).ToRows()
    assert a == b and 0 < len(a) < 2000
    # TestFilterMap
    a = (cp.Take(cp.FromBytes(hp, ctx).SelectColumns("name", "surname", "id")).Filter(cp.Like({"name": "Amelia"}))
         .MapTensors({}, lambda v: {"name": "Julia"}).ToRows())
    b = (cp.Take(cp.FromBytes(hp, ctx).SelectColumns("name", "surname", "id")).Filter(cp.Like({"name": "Amelia"}))
         .Map(lambda r: dict(r, name="Julia")).ToRows())
    assert a == b and len(a) > 0 and all(r["name"] == "Julia" for r in a)


def test_cpp_format_example():
    exe = os.path.join(ROOT, "host", "format_example")
    out = subprocess.run([exe], capture_output=True, check=True).stdout.decode()
    lines = out.splitlines()
    assert lines[0] == "cust_id,prod_id,amount"
    rows = [line.split(",") for line in lines[1:]]
    assert len(rows) == 1000
    for c, p, amt in rows:
        price = float(p) * 1.25 + 0.5
        assert amt == fo.format_float(price * (int(c) % 13 - 3), "f", 2), (c, p, amt)
