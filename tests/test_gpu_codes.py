"""Categorical codes on the GPU (csrc/codes.cu; cpb_table_column_codes / cpb_table_set_codes, Table.values_as_codes,
Categories in with_column and MapTensors, the "category" kind of ToTensors, the C++ mirror) against the plain-Python
reference of tests/codes_ref.py: edge values, values beyond any IndexOn key, 10 M-row columns, every table route,
determinism, the round trip and the errors."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest

from tests import codes_ref as cr
from tests.helpers import gpu_ctx

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _upload(columns: dict, n: int):
    """a device table from host columns {name: (offsets int64[n+1], data uint8[])} (cpb_table_from_host)"""
    import csvplus_b200 as cp
    from csvplus_b200 import _abi
    ctx = gpu_ctx()
    names = list(columns)
    raw = [n.encode() for n in names]
    na = (_abi.Str * len(names))(*[_abi.Str(b, len(b)) for b in raw])
    offs = [np.ascontiguousarray(columns[k][0], np.int64) for k in names]
    datas = [np.ascontiguousarray(np.concatenate([columns[k][1], np.zeros(1, np.uint8)]), np.uint8) for k in names]
    oa = (C.c_void_p * len(names))(*[o.ctypes.data for o in offs])
    da = (C.c_void_p * len(names))(*[d.ctypes.data for d in datas])
    return ctx._new_table("cpb_table_from_host", len(names), na, oa, da, n)


def _table(values: list, name="v"):
    off = np.zeros(len(values) + 1, np.int64)
    np.cumsum([len(v) for v in values], out=off[1:])
    return _upload({name: (off, np.frombuffer(b"".join(values), np.uint8))}, len(values))


def _col(t, name):
    off, data = t.column(name)
    return off - off[0], data


def _check(t, name, want_codes, want_dict):
    """values_as_codes(name) of t equals the reference, twice, and its round trip rebuilds the column byte for byte"""
    import csvplus_b200 as cp
    cat = t.values_as_codes(name)
    assert isinstance(cat, cp.Categories) and cat.codes.dtype.is_floating_point is False
    assert cat.codes.device.type == "cuda" and cat.codes.numel() == len(t)
    got = cat.codes.cpu().numpy()
    assert np.array_equal(got, np.asarray(want_codes, np.int64))
    assert cat.dictionary.columns == [name] and len(cat.dictionary) == len(want_dict)
    doff, ddata = _col(cat.dictionary, name)
    woff = np.zeros(len(want_dict) + 1, np.int64)
    np.cumsum([len(v) for v in want_dict], out=woff[1:])
    assert np.array_equal(doff, woff) and ddata.tobytes() == b"".join(want_dict)
    again = t.values_as_codes(name)
    assert np.array_equal(again.codes.cpu().numpy(), got)
    assert np.array_equal(_col(again.dictionary, name)[1], ddata)
    back = t.with_column(name, cat)
    assert back.columns == t.columns
    o1, d1 = _col(back, name)
    o0, d0 = _col(t, name)
    assert np.array_equal(o1, o0) and np.array_equal(d1, d0)
    return cat


EDGE_CASES = {
    "empty_table": [],
    "one_row": [b"x"],
    "all_equal": [b"same"] * 1000,
    "all_distinct": [b"%d" % i for i in range(5000)],
    "empty_strings": [b"", b"a", b"", b"", b"b", b"a", b""] * 300,
    "last_byte_and_length": [b"a", b"a\0", b"aa", b"a", b"ab", b"aa", b"a\0", b"", b"b"] * 50,
    "invalid_utf8": [b"\xff", b"\xc3\x28", b"\xff", b"e\xcc\x81", b"\xc3\xa9", b"\x80\x80", b"\xc3\x28"] * 40,
    "boundary_lengths": [b"q" * k for k in (0, 1, 7, 8, 9, 127, 128, 129, 255, 256, 257, 4095, 4096, 4097)] * 9,
    "long_values": [(b"L" * 5000) + bytes([k]) for k in range(40)] * 3 + [b"s%d" % k for k in range(70)] + [b"L" * 9000, b"L" * 9001],
    "long_last_byte": [b"z" * 8191 + b"1", b"z" * 8191 + b"2", b"z" * 8192, b"z" * 8191 + b"1", b"z" * 8191],
}


@pytest.mark.parametrize("case", sorted(EDGE_CASES))
def test_edge_values(case):
    vals = EDGE_CASES[case]
    codes, d = cr.factorize(vals)
    _check(_table(vals), "v", codes, d)


def test_long_and_short_in_every_warp_position():
    rng = np.random.default_rng(3)
    longs = [bytes(rng.integers(0, 256, int(rng.integers(129, 6000)), dtype=np.uint8)) for _ in range(50)]
    shorts = [bytes(rng.integers(97, 100, int(rng.integers(0, 5)), dtype=np.uint8)) for _ in range(50)]
    pool = longs + shorts
    vals = [pool[int(i)] for i in rng.integers(0, len(pool), 20000)]
    codes, d = cr.factorize(vals)
    _check(_table(vals), "v", codes, d)


def test_quoted_csv_values():
    import csvplus_b200 as cp
    data = b'id,name\n1,"a,b"\n2,"say ""hi"""\n3,"two\nlines"\n4,"a,b"\n5,\n6,plain\n7,"two\nlines"\n8,\xff\xfe\n9,\n'
    t, err = cp.parse_csv(gpu_ctx(), data)
    assert err is None
    vals = [b"a,b", b'say "hi"', b"two\nlines", b"a,b", b"", b"plain", b"two\nlines", b"\xff\xfe", b""]
    codes, d = cr.factorize(vals)
    _check(t, "name", codes, d)


def _big(dict_bytes, ids, name="v"):
    off, data = cr.column_of(dict_bytes, ids)
    return _upload({name: (off, data)}, len(ids))


def _check_big(t, dict_bytes, ids, name="v"):
    want, order = cr.factorize_ids(ids)
    cat = t.values_as_codes(name)
    got = cat.codes.cpu().numpy()
    assert np.array_equal(got, want)
    doff, ddata = _col(cat.dictionary, name)
    woff, wdata = cr.column_of(dict_bytes, order)
    assert np.array_equal(doff, woff) and np.array_equal(ddata, wdata)
    back = t.with_column(name, cat)
    o1, d1 = _col(back, name)
    o0, d0 = _col(t, name)
    assert np.array_equal(o1, o0) and np.array_equal(d1, d0)
    return cat


def _distinct_values(k, rng):
    """k distinct byte strings of 1..24 bytes: a decimal number, then filler"""
    fill = rng.integers(0, 16, k)
    return [b"%d" % i + b"#" * int(f) for i, f in enumerate(fill)]


@pytest.mark.parametrize("k", [10, 1000, 5_000_000])
def test_random_ten_million_rows(k):
    rng = np.random.default_rng(k)
    d = _distinct_values(k, rng)
    ids = rng.integers(0, k, 10_000_000)
    t = _big(d, ids)
    cat = _check_big(t, d, ids)
    fresh = _big(d, ids)  # the same bytes in a new allocation
    again = fresh.values_as_codes("v")
    assert np.array_equal(again.codes.cpu().numpy(), cat.codes.cpu().numpy())
    assert np.array_equal(_col(again.dictionary, "v")[1], _col(cat.dictionary, "v")[1])


def test_one_value_beside_a_million_singletons():
    rng = np.random.default_rng(11)
    n_rep, n_single = 10_000_000, 1_000_000
    d = [b"the-repeated-value"] + [b"u%d" % i for i in range(n_single)]
    ids = np.zeros(n_rep + n_single, np.int64)
    ids[rng.choice(ids.size, n_single, replace=False)] = np.arange(1, n_single + 1)
    _check_big(_big(d, ids), d, ids)


def test_views_and_routes(monkeypatch):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    rng = np.random.default_rng(19)
    names = [b"ann", b"bob", b"", b"c,d", b"eve" * 60, b"x" * 5000]
    lines = [b"id,name,grp"]
    rows = []
    for i in range(6000):
        nm = names[int(rng.integers(0, len(names)))]
        q = b'"' + nm + b'"' if b"," in nm else nm
        lines.append(b"%d,%s,%d" % (i, q, i % 7))
        rows.append(nm)
    data = b"\n".join(lines) + b"\n"
    t, err = cp.parse_csv(ctx, data)
    assert err is None
    _check(t, "name", *cr.factorize(rows))
    # row-range views: the codes of the rows of the view alone
    for lo, hi in ((0, 1), (1, 4097), (4000, 6000), (37, 38), (100, 100)):
        _check(t.slice(lo, hi), "name", *cr.factorize(rows[lo:hi]))
    # plan routes through ToTensors, against the host rows of the same plan
    def via_plan(src):
        got = src.ToTensors({"name": "category"})["name"]
        host = [cp.api._enc(r["name"]) for r in src.ToRows()]
        codes, d = cr.factorize(host)
        assert got.codes.cpu().tolist() == codes
        assert got.dictionary.values("name") == d
        return len(host)
    assert via_plan(cp.Take(cp.FromBytes(data, ctx)).SelectColumns("name", "id")) == 6000
    assert 0 < via_plan(cp.Take(cp.FromBytes(data, ctx)).Filter(cp.Like({"grp": "3"}))) < 6000
    grp = cp.TakeRows([{"grp": str(g), "label": "g%d" % (g % 3)} for g in range(7)]).UniqueIndexOn("grp")
    assert via_plan(cp.Take(cp.FromBytes(data, ctx)).Join(grp, "grp")) == 6000
    up = [{"name": cp.api._dec(nm), "k": str(i % 3)} for i, nm in enumerate(rows[:500])]
    assert via_plan(cp.TakeRows(up)) == 500
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 4096)  # many batches, concatenated before the codes are taken
    assert via_plan(cp.Take(cp.FromBytes(data, ctx))) == 6000
    sel = t.select("name", "id")
    _check(sel, "name", *cr.factorize(rows))


def test_remap_with_a_permuted_dictionary():
    import torch
    import csvplus_b200 as cp
    rng = np.random.default_rng(23)
    pool = [b"k%d" % i for i in range(300)] + [b"", b"K" * 5000]
    vals = [pool[int(i)] for i in rng.integers(0, len(pool), 50_000)]
    t = _table(vals)
    cat = t.values_as_codes("v")
    k = len(cat.dictionary)
    perm = torch.randperm(k, device=cat.codes.device)
    pdict = cat.dictionary.with_column("v", cp.Categories(perm, cat.dictionary))  # row j = old row perm[j]
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(k, device=perm.device)
    back = t.with_column("v", cp.Categories(inv[cat.codes], pdict))
    assert back.values("v") == vals
    # a remap to other values: the dictionary replaced, the codes kept
    codes, d = cr.factorize(vals)
    upper = cp.Table.from_rows(gpu_ctx(), [{"v": cp.api._dec(v.upper())} for v in d], ["v"])
    mapped = t.with_column("v", cp.Categories(cat.codes, upper))
    assert mapped.values("v") == [v.upper() for v in vals]
    # appended and replaced columns; the other columns are untouched
    two = _upload({"a": cr.column_of(pool, np.arange(len(pool))), "v": cr.column_of(pool[::-1], np.arange(len(pool)))}, len(pool))
    c2 = two.values_as_codes("a")
    app = two.with_column("copy", c2)
    assert app.columns == ["a", "v", "copy"] and app.values("copy") == pool and app.values("v") == pool[::-1]
    rep = two.with_column("v", c2)
    assert rep.columns == ["a", "v"] and rep.values("v") == pool and rep.values("a") == pool


def test_map_tensors_returning_categories(monkeypatch):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    labels = cp.Table.from_rows(ctx, [{"l": s} for s in ("low", "mid", "high")], ["l"])
    data = b"id,qty\n" + b"".join(b"%d,%d\n" % (i, (i * 37) % 101) for i in range(3000))
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 2048)
    dev = cp.Take(cp.FromBytes(data, ctx)).MapTensors({"qty": "int"}, lambda v: {"band": cp.Categories(v["qty"] // 34, labels)})
    host = cp.Take(cp.FromBytes(data, ctx)).Map(lambda r: {**r, "band": ("low", "mid", "high")[int(r["qty"]) // 34]})
    a, b = io.BytesIO(), io.BytesIO()
    dev.ToCsv(a, "id", "qty", "band")
    host.ToCsv(b, "id", "qty", "band")
    assert a.getvalue() == b.getvalue() and a.getvalue().count(b"\n") == 3001


def test_errors():
    import torch
    import csvplus_b200 as cp
    from csvplus_b200 import _abi
    t = _table([b"a", b"b", b"a", b"c", b"b"])
    with pytest.raises(cp.CsvPlusError) as want:
        t.values_as_int("nope")
    with pytest.raises(cp.CsvPlusError) as got:
        t.values_as_codes("nope")
    assert str(got.value) == str(want.value) == 'missing column "nope"'
    assert got.value.kind == want.value.kind == _abi.CPB_E_MISSING_COLUMN
    cat = t.values_as_codes("v")
    assert cat.codes.cpu().tolist() == [0, 1, 0, 2, 1]
    dev = cat.codes.device
    for bad, row in (([0, 1, -1, 2, 1], 2), ([0, 3, 0, 2, -5], 1), ([0, 1, 0, 2, 3], 4), ([2**40, 0, 0, 0, 0], 0)):
        with pytest.raises(cp.CsvPlusError) as ei:
            t.with_column("v", cp.Categories(torch.tensor(bad, dtype=torch.int64, device=dev), cat.dictionary))
        assert ei.value.row == row and ei.value.kind == _abi.CPB_E_BAD_CODE, (bad, str(ei.value))
        assert str(ei.value).startswith("row %d: code %d " % (row, bad[row]))
    two = _upload({"a": cr.column_of([b"x"], np.zeros(3, np.int64)), "b": cr.column_of([b"y"], np.zeros(3, np.int64))}, 3)
    with pytest.raises(cp.CsvPlusError, match="one"):
        t.with_column("v", cp.Categories(cat.codes, two))
    with pytest.raises(TypeError):
        t.with_column("v", cp.Categories(cat.codes.to(torch.int32), cat.dictionary))
    with pytest.raises(ValueError):
        t.with_column("v", cp.Categories(cat.codes[:4], cat.dictionary))
    with pytest.raises(ValueError):
        t.with_column("v", cp.Categories(cat.codes.cpu(), cat.dictionary))
    with pytest.raises(TypeError):
        cp.Categories(cat.codes, "not a table")
    src = cp.Take(cp.FromBytes(b"a,b\n1,x\n", gpu_ctx()))
    with pytest.raises(ValueError, match="batch"):
        src.MapTensors({"b": "category"}, lambda v: {})
    with pytest.raises(ValueError, match="batch"):
        src.FilterTensors({"b": "category"}, lambda v: v)
    with pytest.raises(ValueError):
        src.ToTensors({"b": "categories"})


def test_to_tensors_category_and_int():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    data = b"id,name\n" + b"".join(b"%d,%s\n" % (i, (b"n%d" % (i % 17)) if i % 5 else b"") for i in range(4000))
    out = cp.Take(cp.FromBytes(data, ctx)).ToTensors({"name": "category", "id": "int"})
    rows = cp.Take(cp.FromBytes(data, ctx)).ToRows()
    codes, d = cr.factorize([r["name"].encode() for r in rows])
    assert out["name"].codes.cpu().tolist() == codes and out["name"].dictionary.values("name") == d
    assert out["id"].cpu().tolist() == [int(r["id"]) for r in rows]
    empty = cp.Take(cp.FromBytes(b"id,name\n", ctx)).ToTensors({"name": "category", "id": "int"})
    assert empty["name"].codes.numel() == 0 and len(empty["name"].dictionary) == 0 and empty["name"].dictionary.columns == ["name"]
    # a source error: ToTensors raises it, as for the numeric kinds; the rows before it encode as the reference says
    bad = b"id,name\n1,a\n2,b\n3,a\n4,\"oops\n"
    with pytest.raises(cp.DataSourceError) as want:
        cp.Take(cp.FromBytes(bad, ctx)).ToRows()
    with pytest.raises(cp.DataSourceError) as got:
        cp.Take(cp.FromBytes(bad, ctx)).ToTensors({"name": "category", "id": "int"})
    assert str(got.value) == str(want.value)
    t, err = cp.parse_csv(ctx, bad)
    assert err is not None and str(err) == str(want.value)
    _check(t, "name", *cr.factorize([b"a", b"b", b"a"]))
    with pytest.raises(cp.CsvPlusError, match='missing column "nope"'):
        cp.Take(cp.FromBytes(data, ctx)).ToTensors({"id": "int", "nope": "category"})


def test_host_synchronisations_and_kernels():
    ctx = gpu_ctx()
    vals = [b"%d" % (i % 777) for i in range(100_000)] + [b"w" * 3000]
    t = _table(vals)
    s0 = ctx.host_syncs()
    cat = t.values_as_codes("v")
    assert ctx.host_syncs() - s0 == 2
    s0 = ctx.host_syncs()
    t.with_column("v", cat)
    assert ctx.host_syncs() - s0 == 2
    ctx.stats(enable=True, reset=True)
    t.with_column("v", t.values_as_codes("v"))
    names = set(ctx.stats())
    ctx.stats(enable=False)
    assert {"codes_hash", "codes_insert", "codes_flags", "codes_write", "codes_check", "gather_copy"} <= names, names


def test_cpp_codes_example():
    import csvplus_b200 as cp
    exe = os.path.join(ROOT, "host", "codes_example")
    out = subprocess.run([exe], capture_output=True, check=True, timeout=300).stdout
    vals = [b"red", b"", b'"a,b"', b"green", b"x" * 5000 + b"1", b"x" * 5000 + b"2", b"re"]
    csv = b"id,name\n" + b"".join(b"%d,%s\n" % (i, vals[(i * i + 3 * i) % 7 % (3 if i < 5 else 7)]) for i in range(3000))
    ref = _table([cp.api._enc(r["name"]) for r in cp.Take(cp.FromBytes(csv, gpu_ctx())).ToRows()])
    cat = ref.values_as_codes("v")
    lines = out.split(b"\n")
    assert lines[0] == b"rows 3000 distinct %d" % len(cat.dictionary)
    assert [int(x) for x in lines[1].split()] == cat.codes.cpu().tolist()
    dict_csv = cat.dictionary.to_csv("v").replace(b"v\n", b"name\n", 1)
    assert b"\n".join(lines[2:]).startswith(dict_csv)
    tail = b"\n".join(lines[2:])[len(dict_csv):].split(b"\n")
    assert tail[0] == b"round trip 3000 of 3000"
    assert tail[1] == b"error: row 2999: code %d outside a dictionary of %d values" % (len(cat.dictionary), len(cat.dictionary))
