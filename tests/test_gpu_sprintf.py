"""fmt.Sprintf of string columns on the GPU (csrc/sprintf.cu; cpb_table_set_sprintf / cpb_table_sprintf_into,
Table.with_column(Sprintf), Table.sprintf_into, DataSource.Sprintf / ToText, the C++ mirror) against the plain-Python
restatement of tests/sprintf_ref.py, byte for byte: a fuzz corpus over edge values, every table route, the README's
Printf loop, the refusals, the errors and the 4 GiB limit on both sides."""
import ctypes as C
import io
import os
import random
import subprocess
import zlib

import numpy as np
import pytest

from tests import sprintf_ref as ref
from tests.helpers import gpu_ctx
from tests.test_sprintf_cpu import EDGE_VALUES, random_format

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
M = 1 << 20
README = "%s %s bought %s %ss for £%s each on %s\n"
README_COLS = ("name", "surname", "qty", "product", "price", "ts")


def _table(columns: dict):
    """a device table from host columns {name: [bytes per row]} (cpb_table_from_host)"""
    from csvplus_b200 import _abi
    ctx = gpu_ctx()
    names = list(columns)
    n = len(columns[names[0]]) if names else 0
    raw = [k.encode() for k in names]
    na = (_abi.Str * max(1, len(names)))(*[_abi.Str(b, len(b)) for b in raw])
    offs, datas = [], []
    for k in names:
        off = np.zeros(n + 1, np.int64)
        np.cumsum([len(v) for v in columns[k]], out=off[1:])
        offs.append(off)
        datas.append(np.frombuffer(b"".join(columns[k]) + b"\0", np.uint8))
    oa = (C.c_void_p * max(1, len(names)))(*[o.ctypes.data for o in offs])
    da = (C.c_void_p * max(1, len(names)))(*[d.ctypes.data for d in datas])
    return ctx._new_table("cpb_table_from_host", len(names), na, oa, da, n)


def _rows(t, cols) -> list:
    vals = [t.values(c) for c in cols]
    return [list(r) for r in zip(*vals)] if cols else [[] for _ in range(len(t))]


def _text(t, fmt, *cols) -> bytes:
    import csvplus_b200 as cp
    out = io.BytesIO()
    cp.TakeTable(t).ToText(out, fmt, *cols)
    return out.getvalue()


def _check(t, fmt: bytes, cols: tuple):
    """with_column, sprintf_into and ToText of t equal the restatement row by row"""
    import csvplus_b200 as cp
    want = [ref.sprintf(fmt, r) for r in _rows(t, cols)]
    got = t.with_column("out", cp.Sprintf(fmt, *cols))
    assert got.values("out") == want, fmt
    assert got.columns == t.columns + ["out"] if "out" not in t.columns else got.columns == t.columns
    assert _text(t, fmt, *cols) == b"".join(want), fmt
    assert t.sprintf_into(None, 0, fmt, *cols) == sum(len(w) for w in want)


def _corpus(rng: random.Random, n: int) -> list:
    tricky = EDGE_VALUES + [b"", b"\x00", b"\xe2\x82" * 3, b"\xf0\x9f\x98\x80" * 5, "日本語".encode() * 7]
    out = []
    for i in range(n):
        r = rng.random()
        if r < 0.5:
            out.append(b"".join(rng.choice(tricky) for _ in range(rng.randrange(5))))
        elif r < 0.9:
            out.append(bytes(rng.randrange(256) for _ in range(rng.randrange(20))))
        else:  # both sides of the warp's 4096-byte stage
            out.append(rng.choice([b"x", "é".encode(), b"\xff"]) * rng.choice([1360, 2047, 2048, 4080, 4095, 4096, 4097, 5000]))
    return out


# ---------------------------------------------------------------- the fuzz corpus
def test_fuzz_corpus():
    rng = random.Random(7)
    n = 3000
    t = _table({"a": _corpus(rng, n), "b": _corpus(rng, n), "c": _corpus(rng, n)})
    for k in range(60):
        nverbs = rng.randrange(4)
        fmt, _ = random_format(rng, nverbs)
        _check(t, fmt, tuple(rng.choice("abc") for _ in range(nverbs)))


def test_fixed_formats_over_edge_values():
    vals = EDGE_VALUES + [b"\xe2\x82a", b"ab\xe2", b"\x00\x00", b"\xf4\x90\x80\x80", "😀".encode() * 3, b"x" * 4095, b"y" * 4097]
    t = _table({"v": vals, "w": list(reversed(vals))})
    for fmt, cols in [(b"%5s", "v"), (b"%-5s|", "v"), (b"%.5s", "v"), (b"%.0s|%.1s|%.2s", "vvv"), (b"%4.2s", "v"),
                      (b"%.s", "v"), (b"%--5s|%v", "vw"), (b"%5.1s", "w"), (b"%%%s%%", "v"), (b"\xc2\xa3%s\x00\xff", "v"),
                      (b"%12v|%-12.3v|", "vw"), (b"%s%s%s", "vvv"), (b"%3s", "w")]:
        _check(t, fmt, tuple(cols))


def test_long_values_and_wide_fields():
    """values of 1 MiB, and widths of 10^6 runes on a few rows"""
    vals = [b"a" * M, "é".encode() * (M // 2), b"\xff" * M, b"", "日".encode() * 300_000, b"z"]
    t = _table({"v": vals})
    for fmt, cols in ((b"%s|", "v"), (b"%.100000s|", "v"), (b"%1000000s|", "v"), (b"%-1000000.7s|", "v"), (b"%999999v<%.s>", "vv")):
        _check(t, fmt, tuple(cols))


def test_column_twice_zero_verbs_and_empty_tables():
    import csvplus_b200 as cp
    t = _table({"v": [b"a", b"bc", b""], "w": [b"1", b"2", b"3"]})
    _check(t, b"%s=%s;%-3s", ("v", "v", "w"))
    assert t.with_column("k", cp.Sprintf("lit\n")).values("k") == [b"lit\n"] * 3
    assert _text(t, "lit\n") == b"lit\n" * 3
    assert t.with_column("k", cp.Sprintf("")).values("k") == [b""] * 3
    assert t.with_column("v", cp.Sprintf("<%s>", "v")).values("v") == [b"<a>", b"<bc>", b"<>"]  # replaced in place
    e = t.slice(0, 0)
    assert len(e.with_column("out", cp.Sprintf("%s", "v"))) == 0
    assert _text(e, "%s\n", "v") == b""
    none = cp.TakeTable(t).Filter(cp.Like({"w": "9"}))
    out = io.BytesIO()
    none.ToText(out, "%s\n", "v")
    assert out.getvalue() == b""
    assert none.Sprintf("s", "%s", "v").ToRows() == []


# ---------------------------------------------------------------- routes
def _csv(cols: dict) -> bytes:
    names = list(cols)
    lines = [",".join(names).encode()]
    for r in zip(*cols.values()):
        lines.append(b",".join(b'"' + v.replace(b'"', b'""') + b'"' for v in r))
    return b"\n".join(lines) + b"\n"


def test_routes(monkeypatch):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    rng = random.Random(11)
    n = 4000
    cols = {"a": [v.replace(b"\r", b"") for v in _corpus(rng, n)], "b": [b"%d" % i for i in range(n)], "c": _corpus(rng, n)}
    cols["c"] = [v.replace(b"\r", b"") for v in cols["c"]]
    data = _csv(cols)
    fmt, args = b"[%-6.3s|%5s|%v]\n", ("a", "b", "a")
    want_rows = [ref.sprintf(fmt, [cols[c][i] for c in args]) for i in range(n)]
    want = b"".join(want_rows)

    def text(ds):
        out = io.BytesIO()
        ds.ToText(out, fmt, *args)
        return out.getvalue()
    one = cp.Take(cp.FromBytes(data, ctx))
    assert text(one) == want
    assert [cp.api._enc(r["s"]) for r in one.Sprintf("s", fmt, *args).ToRows()] == want_rows
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 4096)  # many batches: the same text
    assert text(cp.Take(cp.FromBytes(data, ctx))) == want
    assert [cp.api._enc(r["s"]) for r in cp.Take(cp.FromBytes(data, ctx)).Sprintf("s", fmt, *args).ToRows()] == want_rows
    monkeypatch.undo()
    t = _table(cols)
    assert text(cp.TakeTable(t.slice(100, 2100))) == b"".join(want_rows[100:2100])
    assert text(cp.TakeTable(t).SelectColumns("b", "a")) == want
    assert text(cp.TakeTable(t).DropColumns("c")) == want
    sel = t.select("b", "a").slice(5, 50)
    _check(sel, fmt, args)
    cat = cp.Table.concat([t.slice(0, 1000), t.slice(1000, n)])
    assert text(cp.TakeTable(cat)) == want
    host = [{k: cp.api._dec(cols[k][i]) for k in cols} for i in range(300)]
    assert text(cp.TakeRows(host)) == b"".join(want_rows[:300])
    mapped = cp.TakeTable(t.slice(0, 300)).Map(lambda r: r)  # rows left on the host, uploaded with TakeRows semantics
    assert text(mapped) == b"".join(want_rows[:300])


def test_sprintf_step_then_filter_and_to_csv():
    import csvplus_b200 as cp
    t = _table({"name": [b"ann", b"bob", b"ann", b"cy"], "qty": [b"1", b"22", b"333", b"4"]})
    ds = cp.TakeTable(t).Sprintf("label", "%s:%3s", "name", "qty").Filter(cp.Like({"label": "ann:333"}))
    buf = io.BytesIO()
    ds.ToCsv(buf, "label", "qty")
    assert buf.getvalue() == b"label,qty\nann:333,333\n"


def test_map_tensors_reads_the_columns_before_the_step():
    import torch
    import csvplus_b200 as cp
    t = _table({"a": [b"x", b"yy", b"zzz"], "n": [b"1", b"2", b"3"]})
    ds = cp.TakeTable(t).MapTensors({"n": "int"}, lambda v: {"a": cp.Sprintf("%s-%s", "a", "n"), "n": v["n"] * 10,
                                                             "b": cp.Sprintf("%s/%s", "a", "n")})
    rows = ds.ToRows()
    assert [r["a"] for r in rows] == ["x-1", "yy-2", "zzz-3"]
    assert [r["b"] for r in rows] == ["x/1", "yy/2", "zzz/3"]  # the old a and n, though both were set before it
    assert [r["n"] for r in rows] == ["10", "20", "30"]
    assert list(rows[0]) == ["a", "n", "b"]
    del torch


# ---------------------------------------------------------------- the README's Printf loop
def test_readme_pipeline():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    people = ctx.gen_csv("people", (0, 20_000))
    orders = ctx.gen_csv("orders", (0, 200_000), n_cust=20_000, n_prod=500)
    products = ctx.gen_csv("products", (0, 500))
    cust = cp.Take(cp.FromBytes(people, ctx)).SelectColumns("id", "name", "surname").UniqueIndexOn("id")
    prod = cp.Take(cp.FromBytes(products, ctx)).UniqueIndexOn("prod_id")
    joined = cp.Take(cp.FromBytes(orders, ctx)).SelectColumns("cust_id", "prod_id", "qty", "ts").Join(cust, "cust_id").Join(prod)
    out = io.BytesIO()
    joined.ToText(out, README, *README_COLS)
    rows = joined.ToRows()
    assert len(rows) > 100_000
    enc = cp.api._enc
    want = b"".join(ref.sprintf(README.encode(), [enc(r[c]) for c in README_COLS]) for r in rows)
    assert out.getvalue() == want
    pct = "".join(README % tuple(r[c] for c in README_COLS) for r in rows).encode("utf-8", "surrogateescape")
    assert out.getvalue() == pct


def test_cpp_sprintf_example():
    import csvplus_b200 as cp
    exe = os.path.join(ROOT, "host", "sprintf_example")
    out = subprocess.run([exe, os.path.join(GOLDEN, "people.csv"), os.path.join(GOLDEN, "orders.csv")], capture_output=True, check=True,
                         timeout=300).stdout
    ctx = gpu_ctx()
    names = ["apple", "pear", "plum", "fig", "lime", "kiwi", "date", "quince"]
    products = "prod_id,product,price\n" + "".join("%d,%s,%d.%d\n" % (i, names[i], i * 3 + 1, 10 + i * 7) for i in range(8))
    cust = cp.Take(cp.FromFile(os.path.join(GOLDEN, "people.csv"), ctx).SelectColumns("id", "name", "surname")).UniqueIndexOn("id")
    prod = cp.Take(cp.FromBytes(products.encode(), ctx)).UniqueIndexOn("prod_id")
    joined = (cp.Take(cp.FromFile(os.path.join(GOLDEN, "orders.csv"), ctx).SelectColumns("cust_id", "prod_id", "qty", "ts"))
              .Join(cust, "cust_id").Join(prod))
    py = io.BytesIO()
    joined.ToText(py, README, *README_COLS)
    assert py.getvalue() and out.startswith(py.getvalue())
    tail = out[len(py.getvalue()):].split(b"\n")
    top = joined.Top(3).ToRows()
    for line, r in zip(tail[:3], top):
        assert line == b"label " + ref.sprintf(b"%-8s|%.3s|%5v", [cp.api._enc(r[c]) for c in ("name", "surname", "qty")])
    assert tail[3].startswith(b"error: Sprintf format: the verb 'd'") and b"at byte 1" in tail[3]


# ---------------------------------------------------------------- errors
def _launches(fn):
    ctx = gpu_ctx()
    ctx.sync()
    l0 = ctx.kernel_launches()
    try:
        r = fn()
    except Exception as e:  # noqa: BLE001 - returned to the caller, which checks its type
        r = e
    return r, ctx.kernel_launches() - l0


def test_missing_column_is_reported_as_to_csv_reports_it():
    import csvplus_b200 as cp
    t = _table({"a": [b"1", b"2"]})
    with pytest.raises(cp.DataSourceError) as csv_err:
        cp.TakeTable(t).ToCsv(io.BytesIO(), "a", "nope")
    out = io.BytesIO()
    with pytest.raises(cp.DataSourceError) as text_err:
        cp.TakeTable(t).ToText(out, "%s %s", "a", "nope")
    assert str(text_err.value) == str(csv_err.value) and out.getvalue() == b""
    r, n = _launches(lambda: t.with_column("x", cp.Sprintf("%s", "nope")))
    assert isinstance(r, cp.CsvPlusError) and r.kind == 10 and str(r) == 'missing column "nope"' and n == 0
    assert len(_table({"a": []}).with_column("x", cp.Sprintf("%s", "nope"))) == 0  # no row: no Sprintf call


@pytest.mark.parametrize("fmt,nargs", ref.REFUSED)
def test_refused_formats(fmt, nargs):
    import csvplus_b200 as cp
    t = _table({"a": [b"1", b"2"]})
    cols = ("a",) * nargs
    for call in (lambda: t.with_column("x", cp.Sprintf(fmt, *cols)), lambda: t.sprintf_into(None, 0, fmt, *cols),
                 lambda: cp.TakeTable(t).ToText(io.BytesIO(), fmt, *cols)):
        r, n = _launches(call)
        assert isinstance(r, ValueError) and "Sprintf format" in str(r) and "at byte" in str(r), r
        assert n == 0
    assert t.with_column("x", cp.Sprintf("<%s>", "a")).values("x") == [b"<1>", b"<2>"]  # the context still works


def test_argument_count():
    import csvplus_b200 as cp
    t = _table({"a": [b"1"], "b": [b"2"]})
    with pytest.raises(ValueError, match="2 columns for 1 verbs"):
        t.with_column("x", cp.Sprintf("%s", "a", "b"))
    with pytest.raises(ValueError, match="without a column"):
        cp.TakeTable(t).ToText(io.BytesIO(), "%s%s", "a")


# ---------------------------------------------------------------- the 4 GiB limit
class _Digest:
    n = crc = 0

    def write(self, b):
        self.n += len(b)
        self.crc = zlib.crc32(b, self.crc)


def test_limit_both_sides():
    """4400 rows of %1000000s are 4.4 GB: the column is refused before sprintf_write, ToText writes all of it in halved
    batches; 4294 rows (4 294 000 000 bytes, below 2^32) are one column"""
    import torch
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    vals = [b"%d" % i for i in range(4400)]
    t = _table({"v": vals})
    ctx.sync()
    ctx.stats(enable=True, reset=True)
    with pytest.raises(cp.CsvPlusError) as e:
        t.with_column("x", cp.Sprintf("%1000000s", "v"))
    st = ctx.stats()
    ctx.stats(enable=False)
    assert e.value.kind == 13 and "sprintf_len" in st and "sprintf_write" not in st
    d = _Digest()
    cp.TakeTable(t).ToText(d, "%1000000s", "v")
    crc = 0
    for v in vals:
        crc = zlib.crc32(b" " * (1_000_000 - len(v)) + v, crc)
    assert (d.n, d.crc) == (4_400_000_000, crc)
    below = t.slice(0, 4294).with_column("x", cp.Sprintf("%1000000s", "v"))
    assert len(below) == 4294 and below.values("x", 0, 1) == [b" " * 999_999 + b"0"]
    assert below.values("x", 4293, 4294) == [b" " * 999_996 + b"4293"]
    del below, t
    ctx.sync()
    torch.cuda.empty_cache()


def test_one_row_over_4_gib():
    """a 2 GiB value named three times is one row of 6 GiB: refused, nothing written"""
    import torch
    import csvplus_b200 as cp
    from csvplus_b200 import _abi
    ctx = gpu_ctx()
    big = np.zeros((1 << 31) + 1, np.uint8)
    off = np.array([0, 1 << 31], np.int64)
    name = b"v"
    na = (_abi.Str * 1)(_abi.Str(name, 1))
    t = ctx._new_table("cpb_table_from_host", 1, na, (C.c_void_p * 1)(off.ctypes.data), (C.c_void_p * 1)(big.ctypes.data), 1)
    del big
    out = io.BytesIO()
    with pytest.raises(cp.CsvPlusError) as e:
        cp.TakeTable(t).ToText(out, "%s%s%s", "v", "v", "v")
    assert e.value.kind == 13 and out.getvalue() == b""
    with pytest.raises(cp.CsvPlusError) as e:
        t.with_column("x", cp.Sprintf("%s%s%s", "v", "v", "v"))
    assert e.value.kind == 13
    assert t.sprintf_into(None, 0, "%.3s", "v") == 3
    del t
    ctx.sync()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- host synchronisations and kernel names
def test_host_synchronisations_and_kernels():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    t = _table({"v": [b"%d" % i for i in range(100_000)]})
    s0 = ctx.host_syncs()
    t.with_column("x", cp.Sprintf("%-8s|", "v"))
    assert ctx.host_syncs() - s0 == 1
    buf = ctx.host_alloc(2_000_000)
    s0 = ctx.host_syncs()
    n = t.sprintf_into(buf, 0, "%-8s|", "v")
    assert n == 900_000 and bytes(buf.array()[:18]) == b"0       |1       |"
    assert ctx.host_syncs() - s0 == 2  # the size, then the copy into buf (as to_csv_into)
    buf.free()
    ctx.stats(enable=True, reset=True)
    t.with_column("x", cp.Sprintf("%s", "v"))
    names = set(ctx.stats())
    ctx.stats(enable=False)
    assert {"sprintf_len", "sprintf_write"} <= names, names
