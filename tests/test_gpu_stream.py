"""Streamed input (cpb_stream_*, csrc/stream.cu): the GPU cut against the restatement of tests/stream_cut_ref.py, and
plans over inputs parsed in batches of whole records against the single-shot parse and the oracle — rows, column bytes,
error text and line — for every source kind, batch sizes down to one byte, the reader option matrix, header specs, a
fused Like, multi-byte runes, the stateful operations with their boundary row on a batch edge, and every sink."""
import io
import itertools
import os

import numpy as np
import pytest

from oracle import oracle as orc
import tests.stream_cut_ref as ref
from tests.helpers import assert_table_equals_oracle, gpu_ctx, people_csv, random_csv
from tests.test_stream_cut_cpu import OPTION_MATRIX, soup

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cut(data, comma=",", comment="", lazy=False, trim=False):
    import csvplus_b200 as cp
    return cp.csv_stream_cut(gpu_ctx(), data, delimiter=comma, comment=comment, lazy_quotes=lazy, trim_leading_space=trim)


# ------------------------------------------------------------------ the cut
@pytest.mark.parametrize("comment,lazy,trim,nf", [m for m in OPTION_MATRIX if m[3] == 0])
def test_gpu_cut_equals_restatement(comment, lazy, trim, nf):
    for seed in range(6):
        data = soup(seed * 31 + lazy * 2 + trim)
        for k in range(len(data) + 1):
            assert _cut(data[:k], comment=comment, lazy=lazy, trim=trim) == ref.stream_cut(data[:k], comment=comment, lazy=lazy, trim=trim), (data[:k], k)


@pytest.mark.parametrize("comment,lazy", [("", False), ("#", False), ("", True)])
def test_gpu_cut_edges_and_scale(comment, lazy):
    kw = dict(comment=comment, lazy=lazy)
    assert _cut(b"", **kw) == 0
    assert _cut(b"no newline at all", **kw) == 0
    assert _cut(b'h\nx,"inside a quoted\nfield', **kw) == 2
    long_rec = b"h\n" + b'"' + b"y\n" * 150_000 + b'"\n'  # one record across several 64 KiB chunks and DFA blocks
    assert _cut(long_rec, **kw) == len(long_rec)
    assert _cut(long_rec[:-2], **kw) == 2
    # several MB of soup with long fields: chunk and block boundaries fall everywhere
    for seed in range(3):
        data = random_csv(seed, 4000, quoted_p=0.4, long_p=0.01, crlf_p=0.3, blank_p=0.1)
        data = data + b'tail,"open\n' + b"z" * (70_000 + seed * 4099)
        for k in (len(data), len(data) - 70_000, len(data) // 2 + seed, 65536 * 3 + 5):
            assert _cut(data[:k], **kw) == ref.stream_cut(data[:k], **kw), (seed, k)


def test_gpu_cut_multibyte_runes():
    nbsp, sect = "\u00a0".encode(), "\u00a7"
    cases = [(b'h\n' + nbsp + b'"a\nb\n', dict(lazy=True, trim=True)), (b'h\n' + nbsp + b'"a\nb\n', dict(lazy=True)),
             (b'h\nx' + sect.encode() + b'"a\nb\n', dict(comma=sect, lazy=True)),
             (b'h\n' + sect.encode() + b'"x\ny\n', dict(comment=sect)), (b'h\n' + sect.encode() + b'"x\ny\n', dict(comment="#"))]
    for data, kw in cases:
        for k in range(len(data) + 1):
            assert _cut(data[:k], **kw) == ref.stream_cut(data[:k], **kw), (data[:k], kw)


# ------------------------------------------------------------------ streamed parse
def _reader(kind, data, tmp_path):
    import csvplus_b200 as cp
    if kind == "bytes":
        return cp.FromBytes(data)
    if kind == "reader":
        return cp.FromReader(io.BytesIO(data))
    p = tmp_path / "in.csv"
    p.write_bytes(data)
    return cp.FromFile(str(p))


def _plan(kind, data, tmp_path, o, select=None, expect=None, assume=None, like=None):
    import csvplus_b200 as cp
    r = _reader(kind, data, tmp_path).Delimiter(o.comma).NumFields(o.fields_per_record)
    if o.comment:
        r.CommentChar(o.comment)
    if o.lazy_quotes:
        r.LazyQuotes()
    if o.trim_leading_space:
        r.TrimLeadingSpace()
    if select:
        r.SelectColumns(*select)
    elif expect:
        r.ExpectHeader(expect)
    elif assume:
        r.AssumeHeader(assume)
    ds = cp.Take(r)
    return ds.Filter(cp.Like(like)) if like else ds


def _same_tables(a, b):
    if a is None or b is None:
        assert (len(a) if a is not None else 0) == (len(b) if b is not None else 0)
        return
    assert a.columns == b.columns and len(a) == len(b)
    for c in a.columns:
        oa, da = a.column(c)
        ob, db = b.column(c)
        assert np.array_equal(oa, ob) and np.array_equal(da, db), c


def _parse_whole(data, o, select=None, expect=None, assume=None, like=None):
    """the input in one cpb_parse_csv call with the options, header spec and predicate of _plan"""
    import csvplus_b200 as cp
    spec = [(n, -1) for n in select] if select else list((expect or assume or {}).items())
    return cp.parse_csv(gpu_ctx(), data, delimiter=o.comma, comment=o.comment, num_fields=o.fields_per_record,
                        lazy_quotes=o.lazy_quotes, trim_leading_space=o.trim_leading_space, header_from_first_row=not assume,
                        spec=spec, pred=cp.Like(like) if like else None)


def check_stream(monkeypatch, tmp_path, data, o, batch, kind="bytes", **spec):
    """streamed == one piece == one cpb_parse_csv call == oracle: rows, column bytes, error text and line"""
    import csvplus_b200 as cp
    t0, e0 = _parse_whole(data, o, **spec)
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 1 << 40)
    t1, e1 = _plan(kind, data, tmp_path, o, **spec)._table()
    assert (str(e0), getattr(e0, "Line", None)) == (str(e1), getattr(e1, "Line", None)), data
    _same_tables(t0, t1)
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", batch)
    t2, e2 = _plan(kind, data, tmp_path, o, **spec)._table()
    assert (str(e1), getattr(e1, "Line", None)) == (str(e2), getattr(e2, "Line", None)), (data, batch)
    _same_tables(t1, t2)
    like = spec.pop("like", None)
    orows = orc.reader_rows(data, o, pred=orc.Like(like) if like else None, **spec)
    assert (str(e2) if e2 else None) == orows.error
    if t2 is not None and len(orows):
        assert_table_equals_oracle(t2, orows)
    return t2, e2


@pytest.mark.parametrize("batch", [1, 7, 64])
def test_streamed_soups_option_matrix(monkeypatch, tmp_path, batch):
    for i, (comment, lazy, trim, nf) in enumerate(OPTION_MATRIX):
        o = orc.Opts(comment=comment, lazy_quotes=lazy, trim_leading_space=trim, fields_per_record=nf)
        for seed in range(2 if batch == 1 else 4):
            data = soup(seed * 101 + i)
            check_stream(monkeypatch, tmp_path, data, o, batch, kind=("bytes", "reader", "file")[(seed + i) % 3])


@pytest.mark.parametrize("batch", [64, 4096, 1 << 20])
@pytest.mark.parametrize("kind", ["bytes", "reader", "file"])
def test_streamed_fixtures_and_specs(monkeypatch, tmp_path, batch, kind):
    people = open(os.path.join(GOLDEN, "people.csv"), "rb").read()
    nasty = open(os.path.join(GOLDEN, "nasty.csv"), "rb").read()
    big = random_csv(5, 30_000, quoted_p=0.3, crlf_p=0.3, blank_p=0.05)  # ~2 MB: several batches of 1 MiB
    check_stream(monkeypatch, tmp_path, people, orc.Opts(), batch, kind)
    check_stream(monkeypatch, tmp_path, people, orc.Opts(), batch, kind, select=["surname", "id"])
    check_stream(monkeypatch, tmp_path, people, orc.Opts(), batch, kind, expect={"id": 0, "born": 3})
    check_stream(monkeypatch, tmp_path, people, orc.Opts(), batch, kind, assume={"a": 0, "d": 3})
    check_stream(monkeypatch, tmp_path, people, orc.Opts(), batch, kind, select=["name", "id"], like={"name": "Jack"})
    check_stream(monkeypatch, tmp_path, nasty, orc.Opts(fields_per_record=-1), batch, kind)
    check_stream(monkeypatch, tmp_path, nasty, orc.Opts(comment="#", lazy_quotes=True), batch, kind)
    if batch >= 4096:
        check_stream(monkeypatch, tmp_path, big, orc.Opts(), batch, kind)
        check_stream(monkeypatch, tmp_path, big, orc.Opts(lazy_quotes=True, trim_leading_space=True), batch, kind, select=["c3", "c0"])


@pytest.mark.parametrize("batch", [1, 7, 64])
def test_streamed_multibyte_runes(monkeypatch, tmp_path, batch):
    sect, nbsp = "\u00a7", "\u00a0"
    rows = [f"h1{sect}h2{sect}h3", f"a{sect}\"b\nc\"{sect}d", f"{nbsp}\"q\"{sect}x{sect}y", f"\u00a7#{sect}2{sect}3", f"e{sect}f{sect}g"]
    data = ("\n".join(rows) + "\n").encode()
    for comment in ("", "#", "\u00b6"):
        for lazy, trim in itertools.product([False, True], [False, True]):
            o = orc.Opts(comma=sect, comment=comment, lazy_quotes=lazy, trim_leading_space=trim, fields_per_record=-1)
            check_stream(monkeypatch, tmp_path, data, o, batch)
            check_stream(monkeypatch, tmp_path, data.replace(b"#", "\u00b6".encode()), o, batch)


@pytest.mark.parametrize("batch", [64, 20_000])
def test_long_records_at_batch_starts(monkeypatch, tmp_path, batch):
    """data records above 16 KiB (a long quoted field) and above 1024 fields (NumFieldsAny) that start a batch parse like
    any other record: only a header row is limited to 16 KiB / 1024 fields"""
    blob = b'"' + b"text, with \"\"quotes\"\"\nand newlines " * 1500 + b'"'  # ~55 KB
    wide = b",".join(b"w%d" % i for i in range(1500))
    rows = [b"a,b,c", b"1,2,3", b"4," + blob + b",6", b"7,8,9", wide, b"x,y,z", blob + b",q,r", b"10,11,12"]
    data = b"\n".join(rows) + b"\n"
    for o in (orc.Opts(fields_per_record=-1), orc.Opts(fields_per_record=-1, comment="#", lazy_quotes=True),
              orc.Opts(fields_per_record=-1, trim_leading_space=True)):
        check_stream(monkeypatch, tmp_path, data, o, batch)
        check_stream(monkeypatch, tmp_path, data, o, batch, kind="reader", select=["c", "a"])
        check_stream(monkeypatch, tmp_path, data, o, batch, kind="file", assume={"a": 0, "c": 2})
    # a long first record without a header row is accepted by the single-shot parse too
    check_stream(monkeypatch, tmp_path, b"\n".join(rows[2:]) + b"\n", orc.Opts(fields_per_record=-1), batch,
                 assume={"a": 0, "c": 2})
    # the default field count: the wide record is the first failing one, in a later batch
    check_stream(monkeypatch, tmp_path, data, orc.Opts(), batch)


# ------------------------------------------------------------------ errors in a later batch
def _with_error(kind: str) -> tuple:
    body = people_csv(60).split(b"\n")
    if kind == "field_count":
        body[45] = body[45] + b",extra"
        return b"\n".join(body), {}
    if kind == "bare_quote":
        body[45] = body[45].replace(b",", b',x"y', 1)
        return b"\n".join(body), {}
    if kind == "quote":
        body[45] = body[45].replace(b",", b',"x"y', 1)
        return b"\n".join(body), {}
    if kind == "unclosed_start":
        return b'id,name\n"open,' + b"\n".join(body[1:]), {}
    if kind == "column_index":
        body[45] = b"1,2"
        return b"\n".join(body[1:]), {"assume": {"id": 0, "born": 3}}
    if kind == "long_header":
        return b",".join(b"col%04d" % i for i in range(300)) + b"\n" + b",".join(b"%d" % i for i in range(300)) + b"\n", {}
    if kind == "blank_start":
        return b"\n\r\n\n" * 40 + b"\n".join(body), {}
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["field_count", "bare_quote", "quote", "unclosed_start", "column_index", "long_header", "blank_start"])
@pytest.mark.parametrize("batch", [1, 64, 500])
def test_errors_in_later_batches(monkeypatch, tmp_path, kind, batch):
    data, spec = _with_error(kind)
    o = orc.Opts(fields_per_record=-1 if kind == "column_index" else 0)
    for comment in ("", "#"):
        o.comment = comment
        check_stream(monkeypatch, tmp_path, data, o, batch, kind=("bytes", "reader", "file")[batch % 3], **spec)


@pytest.mark.parametrize("kind", ["bare_quote", "quote_and_rows"])
def test_stuck_parity_stops_at_the_error(monkeypatch, tmp_path, kind):
    """a bare quote early in a large input flips the quote parity for the rest of it, so no batch can be cut; the carried
    tail is trial-parsed as it grows, and the stream ends at the error without reading the whole input"""
    import csvplus_b200 as cp
    body = people_csv(3000).split(b"\n")
    if kind == "bare_quote":
        body[5] = body[5].replace(b",", b',x"y', 1)
    else:  # a quoted field with trailing data, then more quote-free rows: ErrQuote in a record that others follow
        body[5] = body[5].replace(b",", b',"x"y', 1)
    data = b"\n".join(body)
    check_stream(monkeypatch, tmp_path, data, orc.Opts(), 64, kind="reader")
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 64)
    src = io.BytesIO(data)
    with pytest.raises(cp.DataSourceError) as e:
        cp.Take(cp.FromReader(src)).ToRows()
    assert e.value.Line == 6 and src.tell() < len(data) // 4, (e.value, src.tell(), len(data))


def test_top_hides_a_later_error(monkeypatch):
    import csvplus_b200 as cp
    data, _ = _with_error("bare_quote")
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 50)
    rows = cp.Take(cp.FromBytes(data)).Top(10).ToRows()
    assert [r["id"] for r in rows] == [str(i) for i in range(10)]
    with pytest.raises(cp.DataSourceError) as e:
        cp.Take(cp.FromBytes(data)).Top(44).ToRows()  # the 45th row is the failing record: Top pulls n + 1
    assert e.value.Line == 46


# ------------------------------------------------------------------ plans and sinks
def _sinks(ds_fn, tmp_path):
    """every sink's output for a fresh plan: bytes / rows / tensors"""
    import csvplus_b200 as cp
    out = {}
    for name, run in [("rows", lambda ds: ds.ToRows()), ("csv", lambda ds: _to(ds.ToCsv, "id", "name")),
                      ("json", lambda ds: _to(ds.ToJSON))]:
        try:
            out[name] = run(ds_fn())
        except (cp.DataSourceError, cp.CsvPlusError) as e:
            out[name] = ("error", str(e))
    f = str(tmp_path / "o.csv")
    try:
        ds_fn().ToCsvFile(f, "name", "id")
        out["csvfile"] = open(f, "rb").read()
    except cp.DataSourceError as e:
        out["csvfile"] = ("error", str(e), os.path.exists(f))
    f = str(tmp_path / "o.json")
    try:
        ds_fn().ToJSONFile(f)
        out["jsonfile"] = open(f, "rb").read()
    except cp.DataSourceError as e:
        out["jsonfile"] = ("error", str(e), os.path.exists(f))
    try:
        ix = ds_fn().IndexOn("name")
        out["index"] = ix.table().rows()
        uix = ds_fn().UniqueIndexOn("id")
        out["uindex"] = uix.table().rows()
        out["tensors"] = ds_fn().ToTensors({"id": "int"})["id"].cpu().tolist()
    except (cp.DataSourceError, cp.CsvPlusError) as e:
        out["index"] = ("error", str(e))
    return out


def _to(sink, *cols):
    b = io.BytesIO()
    sink(b, *cols)
    return b.getvalue()


def test_plans_and_sinks_batch_edges(monkeypatch, tmp_path):
    import csvplus_b200 as cp
    data = people_csv(40)
    per = len(b"12,Olivia,Jones,1955\n")  # ~ one row per batch at this size
    cust = cp.Take(cp.FromBytes(b"name,grp\nJack,1\nOlivia,2\nEmily,3\n")).UniqueIndexOn("name")
    plans = [lambda ds: ds, lambda ds: ds.Join(cust, "name"), lambda ds: ds.Except(cust, "name"),
             lambda ds: ds.Map(lambda r: {**r, "name": r["name"].upper()}), lambda ds: ds.Filter(lambda r: int(r["id"]) % 3 == 0),
             lambda ds: ds.Filter(cp.Like({"name": "Jack"}))]
    for k in (0, 1, 12, 13, 40):
        plans += [lambda ds, k=k: ds.Top(k), lambda ds, k=k: ds.Drop(k),
                  lambda ds, k=k: ds.TakeWhile(lambda r: int(r["id"]) < k), lambda ds, k=k: ds.DropWhile(lambda r: int(r["id"]) < k),
                  lambda ds, k=k: ds.TakeWhile(cp.Not(cp.Like({"id": str(k)}))), lambda ds, k=k: ds.DropWhile(cp.Not(cp.Like({"id": str(k)})))]
    for i, plan in enumerate(plans):
        monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 1 << 40)
        want = _sinks(lambda: plan(cp.Take(cp.FromBytes(data))), tmp_path)
        monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", per if i % 2 else 3 * per + 5)
        got = _sinks(lambda: plan(cp.Take(cp.FromBytes(data))), tmp_path)
        assert got == want, i


def test_streamed_json_on_error_keeps_the_prefix(monkeypatch):
    import csvplus_b200 as cp
    data, _ = _with_error("field_count")
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 64)
    out = io.BytesIO()
    with pytest.raises(cp.DataSourceError) as e:
        cp.Take(cp.FromBytes(data)).ToJSON(out)
    assert e.value.Line == 46
    t, _ = cp.Take(cp.FromBytes(data))._table()
    assert len(t) == 44 and out.getvalue() == t.to_json()[:-1]  # every delivered row, no closing ']'
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 1 << 40)
    out = io.BytesIO()
    with pytest.raises(cp.DataSourceError):
        cp.Take(cp.FromBytes(data)).ToJSON(out)
    assert out.getvalue() == b""  # one batch: nothing written, as before
    # the error inside the first batch of an input pushed in two pieces: the rows before it are still the written prefix
    body = people_csv(60).split(b"\n")
    body[10] = body[10] + b",extra"
    early = b"\n".join(body)
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", len(early) // 2 + 1)
    for kind in ("bytes", "reader"):
        src = (lambda: cp.FromBytes(early)) if kind == "bytes" else (lambda: cp.FromReader(io.BytesIO(early)))
        out = io.BytesIO()
        with pytest.raises(cp.DataSourceError) as e:
            cp.Take(src()).ToJSON(out)
        assert e.value.Line == 11
        t, _ = cp.Take(src())._table()
        assert len(t) == 9 and out.getvalue() == t.to_json()[:-1], kind


# ------------------------------------------------------------------ scale
def test_stream_scale_bounded_memory(monkeypatch):
    """a generated orders input of ~3.8 GB streamed from a reader that makes its bytes on the fly: the input is never held
    whole in host memory, the pool's peak device memory stays far below the input (two staging slots plus one batch's
    results), and the streamed ToCsv equals the single-shot results of the generator's row ranges"""
    import zlib

    import csvplus_b200 as cp
    ctx = gpu_ctx()
    rows, step = 80_000_000, 2_000_000
    batch = 32 << 20
    bound = 24 * batch  # 768 MiB
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", batch)

    def gen(lo):
        b = ctx.gen_csv("orders", (lo, lo + step), n_cust=50_000, n_prod=1000, header=True)
        h = b.to_host()
        b.free()
        return h if lo == 0 else h[int(np.argmax(h == 10)) + 1:]

    class Gen(io.RawIOBase):
        def __init__(self):
            self.lo, self.buf, self.off, self.max_held, self.total = 0, np.empty(0, np.uint8), 0, 0, 0

        def readable(self):
            return True

        def readinto(self, b):
            n = 0
            while n < len(b):
                if self.off == self.buf.size:
                    if self.lo >= rows:
                        break
                    self.buf, self.off = gen(self.lo), 0
                    self.lo += step
                    self.max_held = max(self.max_held, self.buf.size)
                k = min(len(b) - n, self.buf.size - self.off)
                b[n:n + k] = self.buf[self.off:self.off + k]
                n += k; self.off += k
            self.total += n
            return n

    class Crc:
        def __init__(self):
            self.crc, self.n = 0, 0

        def write(self, b):
            self.crc, self.n = zlib.crc32(b, self.crc), self.n + len(b)

    g, got = Gen(), Crc()
    ctx.pool_used_high(reset=True)
    cp.Take(cp.FromReader(g).SelectColumns("order_id", "qty")).ToCsv(got, "order_id", "qty")
    peak = ctx.pool_used_high()
    assert peak < bound, (peak / 2**20, g.total / 2**20)  # never the whole input on the device
    assert g.total > 4 * bound and g.max_held < g.total // 10, (g.total, g.max_held)  # nor in host memory
    want = Crc()
    for lo in range(0, rows, step):
        b = ctx.gen_csv("orders", (lo, lo + step), n_cust=50_000, n_prod=1000, header=True)
        t, err = cp.parse_csv(ctx, b, spec=[("order_id", -1), ("qty", -1)])
        assert err is None
        out = t.to_csv("order_id", "qty")
        want.write(out if lo == 0 else out[out.index(b"\n") + 1:])
        del t
        b.free()
    assert (got.n, got.crc) == (want.n, want.crc)


def test_column_above_4_gib(monkeypatch):
    """an input whose selected `ts` column totals more than 4 GiB: the single-shot parse fails with CPB_E_TOO_LARGE, the
    streamed ToCsv and ToTensors succeed and equal the results of the generator's row ranges parsed one by one"""
    import zlib

    import torch

    import csvplus_b200 as cp
    ctx = gpu_ctx()
    rows, step = 180_000_000, 20_000_000  # ts is 25 bytes: 4.5 GB in that column, ~8 GB of CSV
    pieces = []
    for lo in range(0, rows, step):
        b = ctx.gen_csv("orders", (lo, lo + step), header=lo == 0)
        pieces.append(b.to_host())
        b.free()
    host = np.concatenate(pieces)
    del pieces
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", host.size + 1)
    with pytest.raises(cp.CsvPlusError) as e:
        cp.Take(cp.FromBytes(host).SelectColumns("order_id", "ts")).ToCsv(io.BytesIO(), "order_id", "ts")
    assert e.value.kind == 13  # CPB_E_TOO_LARGE

    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 128 << 20)

    class Crc:
        def __init__(self):
            self.crc, self.n = 0, 0

        def write(self, b):
            self.crc, self.n = zlib.crc32(b, self.crc), self.n + len(b)

    got = Crc()
    cp.Take(cp.FromBytes(host).SelectColumns("order_id", "ts")).ToCsv(got, "order_id", "ts")
    want = Crc()
    for lo in range(0, rows, step):
        b = ctx.gen_csv("orders", (lo, lo + step), header=True)
        t, err = cp.parse_csv(ctx, b, spec=[("order_id", -1), ("ts", -1)])
        assert err is None
        out = t.to_csv("order_id", "ts")
        want.write(out if lo == 0 else out[out.index(b"\n") + 1:])
        del t
        b.free()
    assert (got.n, got.crc) == (want.n, want.crc) and got.n > 4 << 30
    ids = cp.Take(cp.FromBytes(host).SelectColumns("order_id", "ts")).DropColumns("ts").ToTensors({"order_id": "int"})["order_id"]
    assert ids.numel() == rows and bool((ids == torch.arange(rows, device=ids.device)).all())
