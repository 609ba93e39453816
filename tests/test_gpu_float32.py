"""Float32 columns on the GPU (ParseFloat(s, 32) in csrc/numeric.cu, FormatFloat(float64(x), fmt, prec, 32) in
csrc/format.cu; cpb_table_column_as_float32 / cpb_table_set_float32, Table.values_as_float32, FormatFloat(bit_size=32),
the "float32" kind of ToTensors / MapTensors / FilterTensors, the C++ mirror) compared bit for bit with the float32
oracles: the fixtures, a fuzz and a float32 midpoint corpus that reaches the rare parse kernel, shortest and fixed
formats of random bits, exponent borders and subnormals, streamed plan steps against host closures, host
synchronisations, and the round trip of every float32 bit pattern."""
import io
import multiprocessing as mp
import os
import random
import subprocess
from concurrent.futures import ProcessPoolExecutor
from fractions import Fraction

import numpy as np
import pytest

from tests import float32_oracle as f32
from tests import numeric_corpus as nc
from tests import strconv_oracle as so
from tests.helpers import gpu_ctx

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _pool_map(fn, items, chunk=20_000):
    """fn over chunks of items in worker processes (pure Python oracles: nothing there touches the GPU)"""
    parts = [items[i:i + chunk] for i in range(0, len(items), chunk)]
    with ProcessPoolExecutor(max_workers=min(16, os.cpu_count() or 1), mp_context=mp.get_context("fork")) as ex:
        return [y for part in ex.map(fn, parts) for y in part]


def _parse32_chunk(vals):
    return [f32.parse_float(v) for v in vals]


def _format32_chunk(args):
    us, fmt, prec = args
    return [f32.format_bits(int(u), fmt, prec) for u in us]


def _format32_many(bits, fmt, prec):
    parts = [(bits[i:i + 20_000], fmt, prec) for i in range(0, len(bits), 20_000)]
    with ProcessPoolExecutor(max_workers=min(16, os.cpu_count() or 1), mp_context=mp.get_context("fork")) as ex:
        return [s for part in ex.map(_format32_chunk, parts) for s in part]


def _table(values, name="v"):
    import csvplus_b200 as cp
    return cp.Table.from_rows(gpu_ctx(), [{name: v} for v in values], columns=[name])


def _base(n):
    """a device table of n rows with one column of empty strings"""
    import torch
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    dev = torch.device("cuda", ctx.device)
    off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    data = torch.zeros(16, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    return cp.Table.from_device_columns(ctx, ["k"], [(off.data_ptr(), data.data_ptr())], n)


def _texts(t, name):
    off, data = t.column(name)
    d = data.tobytes()
    return [d[off[i]:off[i + 1]].decode() for i in range(len(off) - 1)]


def _f32(bits):
    import torch
    return torch.from_numpy(np.asarray(bits, dtype=np.uint32).view(np.float32).copy()).cuda()


def _check_parse(t, name, values, want=None):
    """values_as_float32 of column `name` (rows holding `values`) against the oracle: bits, status, the strict error"""
    import torch
    import csvplus_b200 as cp
    want = want if want is not None else _parse32_chunk(values)
    wv = np.array([w[0] for w in want], dtype=np.uint32)
    ws = np.array([w[1] for w in want], dtype=np.uint8)
    got, st = t.values_as_float32(name, strict=False)
    assert got.dtype == torch.float32 and got.device.type == "cuda"
    gv, gs = got.cpu().numpy().view(np.uint32), st.cpu().numpy()
    bad = np.nonzero((gv != wv) | (gs != ws))[0]
    assert len(bad) == 0, [(values[i][:60], hex(int(gv[i])), int(gs[i]), hex(int(wv[i])), int(ws[i])) for i in bad[:10]]
    if ws.any():
        first = int(np.nonzero(ws)[0][0])
        with pytest.raises(cp.CsvPlusError) as ei:
            t.values_as_float32(name)
        assert ei.value.row == first and ei.value.kind == (16 if ws[first] == 1 else 17)
        assert str(ei.value) == so.message(name, values[first], True, int(ws[first]))
    return int((ws != 0).sum())


# ------------------------------------------------------------------ parse
def test_numeric32_fixture():
    import csvplus_b200 as cp
    csv = open(os.path.join(GOLDEN, "numeric32_kat.csv"), "rb").read()
    t, err = cp.parse_csv(gpu_ctx(), csv, spec=[("s", -1)])
    assert err is None
    want = [line.split() for line in open(os.path.join(GOLDEN, "numeric32_kat.expected")).read().splitlines()]
    v, st = t.values_as_float32("s", strict=False)
    v, st = v.cpu().numpy().view(np.uint32), st.cpu().numpy()
    vals = t.values("s")
    assert len(vals) == len(want)
    for i, (b, s) in enumerate(want):
        assert (int(v[i]), int(st[i])) == (int(b, 16), int(s)), vals[i]


def rounding_corpus32(n: int, seed: int) -> list:
    """for random float32 values (normals, subnormals, the extremes, values near powers of ten): the exact decimal
    midpoint to the next float32, +- one unit in its last digit, the midpoint cut to 9-40 digits (and the cut with a
    trailing 1), 19- / 20-digit mantissas around it, and now and then the midpoint padded past 800 digits"""
    rng = random.Random(seed)
    out = []
    fixed = [1, 0x7F7FFFFE, 0x007FFFFF, 0x00800000, 0, 0x7F7FFFFF, 0x3F800000, 0x4B7FFFFF]
    while len(out) < n:
        r = rng.random()
        if fixed:
            b = fixed.pop()
        elif r < 0.55:
            b = rng.randrange(0x00800000, 0x7F7FFFFF)
        elif r < 0.75:
            b = rng.randrange(1, 0x00800000)
        else:
            b = int(np.float32(float(f"1e{rng.randint(-45, 38)}")).view(np.uint32)) + rng.randint(-3, 3)
            b = min(max(b, 1), 0x7F7FFFFE)
        lo = Fraction(f32.float_of(b))
        hi = Fraction(f32.float_of(b + 1)) if b + 1 < 0x7F800000 else Fraction(2 ** 128)
        s = nc._decimal((lo + hi) / 2)
        man, _, e = s.partition("e")
        if man.startswith("0."):
            digits, exp10 = man[2:].lstrip("0"), int(e or 0) - (len(man[2:]) - len(man[2:].lstrip("0"))) - 1
        else:
            digits, exp10 = man, len(man) - 1
        digits = digits.rstrip("0") or "0"
        sign = rng.choice(["", "-"])
        out.append((sign + nc._sci(digits, exp10)).encode())
        up = str(int(digits) + 1)
        out.append((sign + nc._sci(up, exp10 + (len(up) - len(digits)))).encode())
        if int(digits) > 1:
            dn = str(int(digits) - 1)
            out.append((sign + nc._sci(dn, exp10 - (len(digits) - len(dn)))).encode())
        for _ in range(2):
            k = rng.randint(9, 40)
            if k < len(digits):
                out.append((sign + nc._sci(digits[:k], exp10)).encode())
                out.append((sign + nc._sci(digits[:k] + "0" * rng.randint(0, 5) + "1", exp10)).encode())
        for k in (19, 20):
            m = (digits + "0" * k)[:k]
            out.append((sign + nc._sci(m, exp10)).encode())
            out.append((sign + nc._sci(str(int(m) + 1), exp10 + (len(str(int(m) + 1)) - k))).encode())
        if rng.random() < 0.02:
            out.append((sign + nc._sci(digits + "0" * (820 - len(digits)) + "1", exp10)).encode())
            out.append((sign + nc._sci(digits + "0" * (820 - len(digits)), exp10)).encode())
    return out[:n]


def test_fuzz_and_midpoints_reach_the_rare_kernel():
    ctx = gpu_ctx()
    vals = nc.fuzz(1_000_000, 20261017) + rounding_corpus32(200_000, 32)
    want = _pool_map(_parse32_chunk, vals)
    t = _table(vals)
    ctx.stats(enable=True, reset=True)
    s0 = ctx.host_syncs()
    t.values_as_float32("v", strict=False)
    assert ctx.host_syncs() - s0 == 1  # one synchronisation per call, as for float64
    st = ctx.stats()
    ctx.stats(enable=False)
    assert st["numeric_float32"]["launches"] == 1 and "numeric_float" not in st and "numeric_rare" not in st
    rare = st.get("numeric_rare32", {})
    assert rare and rare["launches"] == 1 and rare["algo_bytes"] > 50_000 * 13  # the exact path converted rows
    assert _check_parse(t, "v", vals, want) > 0


def test_layouts_and_abi():
    import ctypes as C
    import torch
    import csvplus_b200 as cp
    from csvplus_b200 import _abi
    ctx = gpu_ctx()
    vals = nc.fuzz(3000, 5) + [b"1" * 3000, b"1." + b"7" * 2500 + b"e-30", b"", b"-", b"1e39"] + nc.fuzz(2000, 6)
    t = _table(vals)
    for lo, hi in [(0, len(vals)), (1, 2), (7, 1000), (2999, 3006), (4000, len(vals))]:
        _check_parse(t.slice(lo, hi), "v", vals[lo:hi])
    assert t.slice(3, 3).values_as_float32("nope").numel() == 0
    out = torch.empty(len(vals), dtype=torch.float32, device="cuda")
    nbad = C.c_uint64(); err = _abi.Error()
    st = ctx.lib.cpb_table_column_as_float32(ctx.h, t.h, _abi.Str(b"v", 1), C.c_void_p(out.data_ptr()), None, C.byref(nbad), C.byref(err))
    want = _parse32_chunk(vals)
    assert st == 1 and nbad.value == sum(1 for w in want if w[1])
    assert out.cpu().numpy().view(np.uint32).tolist() == [w[0] for w in want]
    with pytest.raises(cp.CsvPlusError) as ei:
        t.values_as_float32("qty", strict=False)
    assert str(ei.value) == 'missing column "qty"'
    with pytest.raises(cp.CsvPlusError) as ei:
        _table([b"1", b"1e39"]).values_as_float32("v")
    assert str(ei.value) == 'column "v": cannot convert "1e39" to float: value out of range' and ei.value.row == 1


# ------------------------------------------------------------------ format
def test_format32_fixture():
    import csvplus_b200 as cp
    groups = {}
    for line in open(os.path.join(GOLDEN, "format32_kat.csv")).read().splitlines():
        b, fmt, prec, want = line.split(",", 3)
        groups.setdefault((fmt, int(prec)), []).append((int(b, 16), want))
    for (fmt, prec), items in groups.items():
        out = _base(len(items)).with_column("v", cp.FormatFloat(_f32([b for b, _ in items]), fmt, prec, bit_size=32))
        got = _texts(out, "v")
        assert got == [w for _, w in items], (fmt, prec, [(hex(b), g, w) for (b, w), g in zip(items, got) if g != w][:10])


def _bits32(n, seed):
    """random bit patterns (NaN and Inf included), every exponent's border mantissas and a share of subnormals"""
    rng = np.random.default_rng(seed)
    u = rng.integers(0, 2**32, size=n, dtype=np.uint64).astype(np.uint32)
    edges = np.array([ex << 23 | fr for ex in range(256) for fr in (0, 1, 2, 0x400000, 0x7FFFFE, 0x7FFFFF)], dtype=np.uint32)
    edges = np.concatenate([edges, edges | np.uint32(0x80000000)])
    u[: len(edges)] = edges
    sub = rng.integers(1, 2**23, size=n // 20, dtype=np.uint64).astype(np.uint32)
    u[len(edges):len(edges) + len(sub)] = sub
    return u


MODES = [("g", -1, 1_000_000), ("e", -1, 300_000), ("f", -1, 300_000), ("G", -1, 100_000), ("f", 2, 1_000_000),
         ("e", 8, 300_000), ("g", 9, 300_000), ("e", 25, 100_000), ("f", 40, 300_000)]


@pytest.mark.parametrize("fmt,prec,n", MODES)
def test_format_fuzz(fmt, prec, n):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    u = _bits32(n, 100 + MODES.index((fmt, prec, n)))
    ctx.stats(enable=True, reset=True)
    out = _base(n).with_column("x", cp.FormatFloat(_f32(u), fmt, prec, bit_size=32))
    st = ctx.stats()
    ctx.stats(enable=False)
    assert st["format_float32"]["launches"] == 1 and "format_float" not in st and "format_rare" not in st
    if (fmt, prec) == ("f", 40):  # more than 18 significant digits: the exact path
        assert st["format_rare32"]["launches"] == 1 and st["format_rare32"]["algo_bytes"] > 4 * n // 10
    got = _texts(out, "x")
    want = _format32_many(u.tolist(), fmt, prec)
    assert got == want, [(hex(int(u[i])), got[i], want[i]) for i in range(n) if got[i] != want[i]][:10]


def test_format_refusals_and_syncs():
    import ctypes as C
    import torch
    import csvplus_b200 as cp
    from csvplus_b200 import _abi
    ctx = gpu_ctx()
    s = _base(10)
    x32 = torch.zeros(10, dtype=torch.float32, device="cuda")
    x64 = torch.zeros(10, dtype=torch.float64, device="cuda")
    with pytest.raises(TypeError):
        s.with_column("x", x32)  # a bare float32 tensor: the bit size is explicit
    for vals, bits in ((x64, 32), (x32, 64), (x32.to(torch.float16), 32), ([1.0], 32)):
        with pytest.raises(TypeError):
            cp.FormatFloat(vals, "g", -1, bit_size=bits)
    for bits in (16, 0, True):
        with pytest.raises(ValueError):
            cp.FormatFloat(x32, bit_size=bits)
    with pytest.raises(ValueError):
        cp.FormatFloat(x32, "b", -1, bit_size=32)
    h = C.c_void_p(); e = _abi.Error()
    for fmt, prec in ((b"b", -1), (b"g", 65), (b"e", -2)):
        assert ctx.lib.cpb_table_set_float32(ctx.h, s.h, _abi.Str(b"x", 1), C.c_void_p(x32.data_ptr()), fmt, prec, C.byref(h), C.byref(e)) == 2
    assert len(s.slice(2, 2).with_column("x", cp.FormatFloat(x32[:0], bit_size=32))) == 0
    t = _base(100_000)
    x = torch.linspace(-1e5, 1e5, 100_000, dtype=torch.float32, device="cuda")
    for fmt, prec in (("g", -1), ("f", 2), ("e", 25), ("f", 40)):
        before = ctx.host_syncs()
        t.with_column("x", cp.FormatFloat(x, fmt, prec, bit_size=32))
        assert ctx.host_syncs() - before <= 2
    before = ctx.host_syncs()
    t.slice(0, 0).with_column("x", cp.FormatFloat(x[:0], bit_size=32))
    assert ctx.host_syncs() == before


def test_round_trip_every_float32():
    """GPU 'g' -1 then GPU ParseFloat(s, 32) over all 2^32 bit patterns in chunks: every finite value comes back"""
    import torch
    import csvplus_b200 as cp
    chunk = 1 << 26
    t = _base(chunk)
    for lo in range(0, 1 << 32, chunk):
        bits = (torch.arange(lo, lo + chunk, dtype=torch.int64, device="cuda") - (1 << 31)).to(torch.int32)
        x = bits.view(torch.float32)
        x = torch.where(torch.isfinite(x), x, torch.zeros_like(x))
        back = t.with_column("x", cp.FormatFloat(x, bit_size=32)).values_as_float32("x")
        assert torch.equal(back.view(torch.int32), x.view(torch.int32)), lo


# ------------------------------------------------------------------ plan steps
def _csv(n, seed=3):
    rnd = random.Random(seed)
    lines = ["id,price,w,qty"]
    for i in range(n):
        lines.append("%d,%s,%s,%d" % (i, repr(rnd.uniform(0, 1000)) if i % 5 else "%.3f" % rnd.uniform(0, 1000),
                                      "%.9e" % rnd.uniform(-1e30, 1e30), rnd.randint(-5, 50)))
    return ("\n".join(lines) + "\n").encode()


def _map_dev(v):
    import torch
    import csvplus_b200 as cp
    return {"p2": cp.FormatFloat(v["price"] * 2.5, "g", -1, bit_size=32),
            "wq": cp.FormatFloat(v["w"] * v["qty"].to(torch.float32), "e", 4, bit_size=32)}


def _map_host(row):
    p = np.float32(f32.float_of(f32.parse_float(row["price"].encode())[0]))
    w = np.float32(f32.float_of(f32.parse_float(row["w"].encode())[0]))
    row = dict(row)
    row["p2"] = f32.format_float(float(p * np.float32(2.5)), "g", -1)
    row["wq"] = f32.format_float(float(w * np.float32(int(row["qty"]))), "e", 4)
    return row


def _keep_host(row):
    return np.float32(f32.float_of(f32.parse_float(row["price"].encode())[0])) > np.float32(400.5)


@pytest.mark.parametrize("batch", [64, 4096, 1 << 20])
def test_map_filter_tensors_streamed(monkeypatch, batch):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", batch)
    data = _csv(3000)
    dev = (cp.Take(cp.FromBytes(data, ctx)).MapTensors({"price": "float32", "w": "float32", "qty": "int"}, _map_dev)
           .FilterTensors({"price": "float32"}, lambda v: v["price"] > 400.5))
    host = cp.Take(cp.FromBytes(data, ctx)).Map(_map_host).Filter(_keep_host)
    a, b = io.BytesIO(), io.BytesIO()
    dev.ToCsv(a, "id", "price", "p2", "wq")
    host.ToCsv(b, "id", "price", "p2", "wq")
    assert a.getvalue() == b.getvalue() and a.getvalue().count(b"\n") > 1000
    import torch
    got = cp.Take(cp.FromBytes(data, ctx)).ToTensors({"price": "float32", "qty": "int"})
    assert got["price"].dtype == torch.float32 and got["qty"].dtype == torch.int64
    want = [f32.parse_float(r["price"].encode())[0] for r in cp.Take(cp.FromBytes(data, ctx)).ToRows()]
    assert got["price"].cpu().numpy().view(np.uint32).tolist() == want


def test_error_order_with_float32(monkeypatch):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    csv = b"a,b\n1,2.5\n2,1e39\nx,3\n4,oops\n"
    with pytest.raises(cp.CsvPlusError) as ei:
        cp.Take(cp.FromBytes(csv, ctx)).ToTensors({"a": "int", "b": "float32"})
    assert ei.value.row == 1 and str(ei.value) == 'column "b": cannot convert "1e39" to float: value out of range'
    with pytest.raises(cp.CsvPlusError) as ei:  # row 2 fails in a only, row 3 in b: the lower row first
        cp.Take(cp.FromBytes(csv, ctx)).Drop(2).ToTensors({"b": "float32", "a": "int"})
    assert ei.value.row == 0 and str(ei.value) == 'column "a": cannot convert "x" to integer: invalid syntax'
    both = b"a,b\n1,1\nq,zz\n"  # one row failing in both inputs: the earlier input wins
    with pytest.raises(cp.CsvPlusError) as ei:
        cp.Take(cp.FromBytes(both, ctx)).ToTensors({"b": "float32", "a": "int"})
    assert ei.value.row == 1 and 'cannot convert "zz" to float' in str(ei.value)
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 64)
    lines = ["a,b"] + ["%d,%d.5" % (i, i) for i in range(40)]
    lines[31] = "30,1e39"
    with pytest.raises(cp.CsvPlusError) as ei:
        cp.Take(cp.FromBytes(("\n".join(lines) + "\n").encode(), ctx)).MapTensors(
            {"b": "float32"}, lambda v: {"c": cp.FormatFloat(v["b"] * 2, bit_size=32)}).ToRows()
    assert ei.value.row == 30 and ei.value.kind == 17
    with pytest.raises(ValueError):
        cp.Take(cp.FromBytes(csv, ctx)).ToTensors({"a": "float16"})


def test_cpp_float32_example():
    exe = os.path.join(ROOT, "host", "float32_example")
    out = subprocess.run([exe], capture_output=True, check=True, timeout=300).stdout.decode()
    lines = out.splitlines()
    assert lines[0] == "s,g,f2"
    rows = [line.split(",") for line in lines[1:-1]]
    assert len(rows) == 1006
    for s, g, f2 in rows:
        b, st = f32.parse_float(s.encode())
        assert st == 0
        assert (g, f2) == (f32.format_bits(b, "g", -1), f32.format_bits(b, "f", 2)), s
    assert rows[1][1] == "1.0000001" and rows[0][1] == "0.1"
    assert lines[-1] == "error: " + so.message("s", b"1e39", True, so.RANGE)
