"""Results at the 4 GiB offset limit: every route that sizes a variable-length result from the length scan (ToCsv,
ToJSON, the column gathers of with_column(Categories) and Join, Table.concat) on both sides of 2^32 - 1 bytes, against
the exact sizes of tests/result_limits_ref.py.  The shapes put few long rows into one scan tile, so a 32-bit thread,
warp or tile sum would wrap.  A refused call launches no copy or write kernel and leaves the context usable.  Each case
builds its tables on the device and frees them before the next; none needs more than about 13 GB."""
import gc
import zlib

import numpy as np
import pytest

from oracle import oracle as orc
from tests import result_limits_ref as R
from tests.helpers import gpu_ctx

pytestmark = pytest.mark.gpu
M = R.MIB
TOO_LARGE = 13  # CPB_E_TOO_LARGE
WRITERS = ("gather_copy", "slot_copy", "csv_write", "json_write")


def _dev():
    import torch
    return torch.device("cuda", gpu_ctx().device)


def _column(runs):
    """(offsets int32[n + 1], bytes uint8) CUDA tensors of a column given as runs of (count, value)"""
    import torch
    dev = _dev()
    counts = torch.tensor([c for c, _ in runs], dtype=torch.int64, device=dev)
    lens = torch.tensor([len(v) for _, v in runs], dtype=torch.int64, device=dev)
    per_row = torch.repeat_interleave(lens, counts)
    off = torch.zeros(per_row.numel() + 1, dtype=torch.int64, device=dev)
    torch.cumsum(per_row, 0, out=off[1:])
    assert int(off[-1]) <= R.LIMIT
    off32 = (off & 0xFFFFFFFF).to(torch.int32)  # the low 32 bits: offsets above 2^31 - 1 read as uint32
    del off, per_row
    uniq = {}
    parts = []
    for c, v in runs:
        if c and v:
            if v not in uniq:
                uniq[v] = torch.frombuffer(bytearray(v), dtype=torch.uint8).to(dev)
            parts.append(uniq[v].repeat(c))
    parts.append(torch.zeros(16, dtype=torch.uint8, device=dev))
    data = torch.cat(parts)
    return off32, data


def _table(cols: dict):
    """a device table of columns name -> runs (every column the same number of rows)"""
    import torch
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    names, tensors = list(cols), [_column(r) for r in cols.values()]
    n = tensors[0][0].numel() - 1
    torch.cuda.synchronize()
    t = cp.Table.from_device_columns(ctx, names, [(o.data_ptr(), d.data_ptr()) for o, d in tensors], n)
    ctx.sync()
    del tensors
    torch.cuda.empty_cache()
    return t


def _flush():
    """returns the memory of the tables the caller has deleted (the next case starts from an empty pool)"""
    import torch
    gc.collect()
    gpu_ctx().sync()
    torch.cuda.empty_cache()


def _launches(fn):
    """fn() with kernel statistics on -> (result or the CsvPlusError raised, launches per kernel name)"""
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    ctx.sync()
    ctx.stats(enable=True, reset=True)
    try:
        r = fn()
    except cp.CsvPlusError as e:
        r = e
    ctx.sync()
    st = {k: v["launches"] for k, v in ctx.stats().items()}
    ctx.stats(enable=False)
    return r, st


def _refused(fn, kind=TOO_LARGE):
    """fn() raises CPB_E_TOO_LARGE without launching a copy or write kernel, and the context still computes right.
    (kind None: an entry without a cpb_error*, whose data error carries only its status and message)"""
    import csvplus_b200 as cp
    r, st = _launches(fn)
    assert isinstance(r, cp.CsvPlusError) and r.status == 1, r  # CPB_ERR_DATA
    assert r.kind == kind if kind is not None else "4 GiB" in str(r), (r.kind, str(r))
    assert not any(st.get(k) for k in WRITERS), st
    _still_right()


def _still_right():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    rows = [{"k": str(i % 7), "v": "v%d,\"%d" % (i, i)} for i in range(50)]
    idx_rows = [{"k": str(i), "w": "w" * i} for i in range(5)]
    t, ix = cp.Table.from_rows(ctx, rows, ["k", "v"]), cp.Table.from_rows(ctx, idx_rows, ["k", "w"])
    j = t.join(ix.index_on("k"), "k")
    oj = orc.take_rows(rows).join(orc.take_rows(idx_rows).index_on("k"), "k")
    assert len(j) == len(oj)
    for c in ("k", "v", "w"):
        assert j.values(c) == oj.values(c)
    assert j.to_csv("w", "v", "k") == oj.to_csv("w", "v", "k")[0]


def _crc_device(buf):
    """(bytes, CRC-32) of a DeviceBuffer, read back in pieces"""
    crc, step = 0, 1 << 30
    for lo in range(0, buf.nbytes, step):
        crc = zlib.crc32(buf.to_host(min(step, buf.nbytes - lo), lo), crc)
    return buf.nbytes, crc


# ---------------------------------------------------------------- the scan total at every level, through size-only ToCsv
@pytest.mark.parametrize("name", list(R.scan_shapes()))
def test_scan_total_at_every_level(name):
    runs, times, level = R.scan_shapes()[name]
    t = _table({"a": runs})
    cols = ["a"] * times
    want = R.csv_header_len(cols) + R.csv_body_size(R.repeated(runs, times))
    if R.csv_body_size(R.repeated(runs, times)) > R.LIMIT:
        _refused(lambda: t.to_csv_into(None, 0, *cols))
    else:
        assert t.to_csv_into(None, 0, *cols) == want
        assert t.to_csv_into(None, 0, *cols, header=False) == want - R.csv_header_len(cols)
    del t
    _flush()


# ---------------------------------------------------------------- ToCsv
def test_to_csv_one_row_of_quotes():
    """one row of 2^30 '"' written as "a","a" is 2^32 + 6 bytes: the row's length saturates instead of wrapping"""
    runs = [(1, b'"' * (1 << 30))]
    t = _table({"a": runs})
    assert R.csv_body_size(R.repeated(runs, 2)) == (1 << 32) + 6
    _refused(lambda: t.to_csv_device("a", "a"))
    del t
    _flush()


def test_to_csv_body_at_the_limit():
    """a body of exactly 2^32 - 1 bytes is written (the header is not counted against it); 2^32 bytes are refused"""
    runs = [(4095, R.x(M)), (1, R.x(1_044_479))]
    t = _table({"a": runs})
    body = R.csv_body_size(R.repeated(runs, 1))
    assert body == R.LIMIT
    assert t.to_csv_into(None, 0, "a") == body + 2
    b = t.to_csv_device("a")
    assert _crc_device(b) == R.crc_of([b"a\n"] + list(R.csv_body_chunks(R.repeated(runs, 1))))
    del b, t
    _flush()
    t = _table({"a": [(4095, R.x(M)), (1, R.x(1_044_480))]})
    _refused(lambda: t.to_csv_into(None, 0, "a", header=False))
    _refused(lambda: t.to_csv_device("a"))
    del t
    _flush()


# ---------------------------------------------------------------- ToJSON
def test_to_json_tile_wrap_and_batches():
    """700 rows of 2^20 bytes 0x01 escape to 4.4 GB in one scan tile: one call is refused, DataSource.ToJSON halves the
    batch and writes the whole document"""
    import csvplus_b200 as cp
    runs = [(700, b"\x01" * M)]
    t = _table({"a": runs})
    assert R.json_body_size([b"a"], R.repeated(runs, 1)) > R.LIMIT
    _refused(lambda: t.to_json_into(None))
    _refused(lambda: t.to_json_device())

    class Digest:
        n = crc = 0

        def write(self, b):
            self.n += len(b)
            self.crc = zlib.crc32(b, self.crc)
    d = Digest()
    cp.TakeTable(t).ToJSON(d)
    assert (d.n, d.crc) == R.crc_of(R.json_document_chunks([b"a"], R.repeated(runs, 1)))
    del t
    _flush()


def test_to_json_body_at_the_limit():
    """a body of 2^32 - 2 bytes is written (2^32 - 1 with the closing ']'); a body of 2^32 - 1 bytes is refused"""
    runs = [(4095, R.x(M)), (1, R.x(1_007_614))]
    t = _table({"a": runs})
    assert R.json_body_size([b"a"], R.repeated(runs, 1)) == R.LIMIT - 1
    assert t.to_json_into(None) == R.LIMIT
    b = t.to_json_device()
    assert _crc_device(b) == R.crc_of(R.json_document_chunks([b"a"], R.repeated(runs, 1)))
    del b, t
    _flush()
    t = _table({"a": [(4095, R.x(M)), (1, R.x(1_007_615))]})
    _refused(lambda: t.to_json_into(None))
    _refused(lambda: t.to_json_into(None, 0, False, False))
    del t
    _flush()


# ---------------------------------------------------------------- gathers
def _check_column(t, name, runs):
    """column `name` of t holds the values of runs (each value one repeated byte): its offsets and its bytes"""
    off, data = t.column(name)
    lens = np.repeat(np.array([len(v) for _, v in runs], np.int64), [c for c, _ in runs])
    assert off[0] == 0 and np.array_equal(np.diff(off), lens)
    pos, step = 0, 1 << 28
    for c, v in runs:
        assert len(set(v)) <= 1
        end = pos + c * len(v)
        for lo in range(pos, end, step):
            assert (data[lo:min(end, lo + step)] == v[0]).all()
        pos = end
    assert pos == int(off[-1]) == len(data)


def _codes(runs_of_codes):
    import torch
    return torch.cat([torch.full((c,), k, dtype=torch.int64, device=_dev()) for c, k in runs_of_codes])


@pytest.mark.parametrize("last", [None, 1_044_480, 1_044_481])
def test_set_codes_at_the_limit(last):
    """with_column(name, Categories): 4097 codes of one 2^20 + 1-byte value wrap one tile; 4095 of them and one value
    of `last` bytes make 2^32 - 1 bytes (written) or 2^32 bytes (refused)"""
    import csvplus_b200 as cp
    dvals = [b"a" * (M + 1)] + ([b"b" * last] if last else [])
    d = _table({"v": [(1, v) for v in dvals]})
    base = _table({"k": [(4097 if last is None else 4096, b"r")]})
    codes = _codes([(4097, 0)] if last is None else [(4095, 0), (1, 1)])
    size = R.gathered_size([len(v) for v in dvals], codes.tolist())
    if size > R.LIMIT:
        _refused(lambda: base.with_column("v", cp.Categories(codes, d)))
    else:
        r, st = _launches(lambda: base.with_column("v", cp.Categories(codes, d)))
        assert st.get("gather_copy") and len(r) == 4096
        _check_column(r, "v", [(4095, dvals[0]), (1, dvals[1])])
        del r
    _flush()
    del codes
    del base, d
    _flush()


def test_gather_group_holding_most_of_the_column():
    """one 32-row group of the gather holds 2^32 - 32 of a 2^32 - 1-byte column, behind 7 bytes that misalign it"""
    import csvplus_b200 as cp
    big = R.x((1 << 30) - 8)
    dvals = [big, b"s", b"", b"w" * 24]
    out = [(7, b"s"), (25, b""), (4, big), (28, b""), (1, b"w" * 24)]
    code_of = {v: k for k, v in enumerate(dvals)}
    d = _table({"v": [(1, v) for v in dvals]})
    base = _table({"k": [(65, b"r")]})
    codes = _codes([(c, code_of[v]) for c, v in out])
    assert R.gathered_size([len(v) for v in dvals], codes.tolist()) == R.LIMIT
    r = base.with_column("v", cp.Categories(codes, d))
    _check_column(r, "v", out)
    del codes
    del r, base, d
    _flush()


@pytest.mark.parametrize("last", [None, 1_044_480, 1_044_481])
def test_join_index_side_at_the_limit(last):
    """the index column of a join: one index row of 2^20 + 1 bytes matched by 4097 probe rows (refused), or by 4095
    probe rows beside one row of `last` bytes (2^32 - 1 bytes written, 2^32 refused).  Values over 255 bytes take the
    column gather, not row slots."""
    ivals = [b"a" * (M + 1)] + ([b"b" * last] if last else [])
    ix_t = _table({"k": [(1, b"1")] + ([(1, b"2")] if last else []), "v": [(1, v) for v in ivals]})
    probe = _table({"k": [(4097, b"1")] if last is None else [(4095, b"1"), (1, b"2")]})
    ix = ix_t.index_on("k")
    assert len(probe.slice(0, 1).join(ix, "k")) == 1  # the index's sorted rows are built here, not in the call below
    size = 4097 * (M + 1) if last is None else R.gathered_size([len(v) for v in ivals], [0] * 4095 + [1])
    if size > R.LIMIT:
        _refused(lambda: probe.join(ix, "k"))
    else:
        j, st = _launches(lambda: probe.join(ix, "k"))
        assert st.get("gather_copy") and not st.get("slot_copy"), st
        _check_column(j, "v", [(4095, ivals[0]), (1, ivals[1])])
        del j
    _flush()
    del ix, probe, ix_t
    _flush()


@pytest.mark.parametrize("last", [None, 1_044_480, 1_044_481])
def test_join_probe_side_at_the_limit(last):
    """the probe column of a join: one probe row of 2^20 + 1 bytes matching 4097 rows of a non-unique index (refused), or
    4095 rows beside a probe row of `last` bytes matching one (2^32 - 1 bytes written, 2^32 refused)"""
    pvals = [b"a" * (M + 1)] + ([b"b" * last] if last else [])
    probe = _table({"k": [(1, b"1")] + ([(1, b"2")] if last else []), "p": [(1, v) for v in pvals]})
    ix_t = _table({"k": [(4097, b"1")] if last is None else [(4095, b"1"), (1, b"2")]})
    ix = ix_t.index_on("k")
    size = 4097 * (M + 1) if last is None else R.gathered_size([len(v) for v in pvals], [0] * 4095 + [1])
    if size > R.LIMIT:
        _refused(lambda: probe.join(ix, "k"))
    else:
        j, st = _launches(lambda: probe.join(ix, "k"))
        assert st.get("gather_copy") and not st.get("slot_copy"), st
        _check_column(j, "p", [(4095, pvals[0]), (1, pvals[1])])
        del j
    _flush()
    del ix, ix_t, probe
    _flush()


# ---------------------------------------------------------------- concat
def test_concat_at_the_limit():
    """Table.concat sums the parts' bytes exactly: 2^32 - 1 bytes are accepted, 2^32 refused"""
    import csvplus_b200 as cp
    a = _table({"v": [(2047, R.x(M)), (1, b"t")]})
    b = _table({"v": [(2048, R.x(M)), (1, R.x(M - 2))]})
    assert (2047 * M + 1) + (2048 * M + M - 2) == R.LIMIT
    c = cp.Table.concat([a, b])
    _check_column(c, "v", [(2047, R.x(M)), (1, b"t"), (2048, R.x(M)), (1, R.x(M - 2))])
    del c
    _flush()
    e = _table({"v": [(1, b"u")]})
    _refused(lambda: cp.Table.concat([a, b, e]), kind=None)
    del a, b, e
    _flush()
