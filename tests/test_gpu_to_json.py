"""ToJSON on the GPU (csrc/json.cu, cpb_table_to_json*) byte for byte against the restated encoder of tests/json_oracle.py:
byte-soup tables, the escape fixture, views, empty and wide tables, escaped column names, a lazily sorted unique index,
a join at scale, streamed batches, and DataSource.ToJSON's batching, error and host-row paths."""
import io
import os
import random
import zlib

import pytest

from oracle import oracle as orc
from tests import json_oracle as jo
from tests.helpers import gpu_ctx, people_csv

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEED = 0xC5B200


def _doc(t, lo=0, hi=None, first=True, last=True):
    """the oracle's document of rows [lo, hi) of a device table (values fetched from the device)"""
    names = t.columns
    return jo.columns_document([n.encode("utf-8", "surrogateescape") for n in names], [t.values(n, lo, hi) for n in names],
                               first, last)


def _soup(rng, n):
    pool = list(range(0x20)) + [0x22, 0x5C, 0x7F] + list(range(0x80, 0x100, 7)) + [0xE2, 0x80, 0xA8, 0xA9, 0xF0, 0x9F, 0xC3]
    return bytes(rng.choice(pool) if rng.random() < 0.4 else rng.randrange(0x20, 0x7F) for _ in range(n))


def test_byte_soup_tables():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    rng = random.Random(11)
    rows = []
    for i in range(700):
        r = {"a": _soup(rng, rng.choice([0, 0, 1, 3, 8, 17, 40])), "bb": _soup(rng, rng.randrange(0, 90)), "c": b"plain %d" % i}
        if i in (5, 300, 301):
            r["a"] = _soup(rng, 9000)            # a value longer than a warp's stage
        if i == 450:
            r["bb"] = b"x" * 7000                 # a plain row longer than the stage
        rows.append(r)
    t = cp.Table.from_rows(ctx, rows, columns=["c", "bb", "a"])
    brows = [{k.encode(): v for k, v in r.items()} for r in rows]
    assert t.to_json() == jo.document(brows)
    # every row alone (groups of one row at every alignment)
    for lo in (0, 1, 5, 31, 32, 449, 699):
        assert t.slice(lo, lo + 1).to_json() == jo.document(brows[lo:lo + 1])
    # the device copy has the same bytes
    b = t.to_json_device()
    assert bytes(b.to_host()) == jo.document(brows)
    b.free()


def test_golden_fixture_parsed():
    import csvplus_b200 as cp
    csv = open(os.path.join(GOLDEN, "json_escapes.csv"), "rb").read()
    want = open(os.path.join(GOLDEN, "json_escapes.json"), "rb").read()
    names = ["a", "B", "\u00e9", 'k"\\<']
    t, err = cp.parse_csv(gpu_ctx(), csv, spec=[(n, -1) for n in names])
    assert err is None
    assert t.to_json() == want
    out = io.BytesIO()
    cp.Take(cp.FromBytes(csv).SelectColumns(*names)).ToJSON(out)
    assert out.getvalue() == want


def test_slice_empty_wide_and_escaped_names():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    rows = [{"id": str(i), "v": "\u00e9\x08%d\x0c" % i} for i in range(1000)]
    t = cp.Table.from_rows(ctx, rows)
    assert t.slice(123, 877).to_json() == _doc(t, 123, 877)
    assert t.slice(123, 877).to_json() == jo.document([{k.encode(): v.encode() for k, v in r.items()} for r in rows[123:877]])
    # 0 rows
    e = t.slice(10, 10)
    assert e.to_json() == b"[]" and e.to_json(True, False) == b"[" and e.to_json(False, True) == b"]" and e.to_json(False, False) == b""
    assert cp.Table.from_rows(ctx, [], columns=["a"]).to_json() == b"[]"
    # 80 columns
    rng = random.Random(80)
    wide = [{"col%02d" % k: _soup(rng, rng.randrange(0, 6)) for k in range(80)} for _ in range(300)]
    tw = cp.Table.from_rows(ctx, wide, columns=["col%02d" % k for k in reversed(range(80))])
    assert tw.to_json() == jo.document([{k.encode(): v for k, v in r.items()} for r in wide])
    # names that need escaping, in bytewise order ("B" < "a" < "\u00e9")
    named = [{'q"\\\n': "1", "\u00e9": "2", "\x01": "3", "B": "4", "a": "5", "\u2028": "6"}] * 3
    tn = cp.Table.from_rows(ctx, named, columns=list(named[0]))
    assert tn.to_json() == jo.document([{k.encode(): v.encode() for k, v in r.items()} for r in named])
    # a table whose key prefixes do not fit in shared memory
    long_names = [{"k%03d" % k + "n" * 300: "v" for k in range(60)}]
    tl = cp.Table.from_rows(ctx, long_names * 40, columns=list(long_names[0]))
    assert tl.to_json() == jo.document([{k.encode(): v.encode() for k, v in r.items()} for r in long_names * 40])


def test_lazily_sorted_unique_index():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    n = 60_000
    raw = ctx.gen_csv("customers", (0, n), n_cust=n, permute=True)
    t, _ = cp.parse_csv(ctx, raw, spec=[("id", -1), ("name", -1), ("surname", -1)])
    ix = t.index_on("id", unique=True)
    oi = orc.reader_rows(raw.to_host(), select=["id", "name", "surname"]).unique_index_on("id")
    out = io.BytesIO()
    cp.Take(ix).ToJSON(out)
    rows = oi.rows()
    assert out.getvalue() == jo.columns_document([b"id", b"name", b"surname"], [rows.values(c) for c in ("id", "name", "surname")])


def test_join_at_scale_and_streamed_batches():
    """a configs[3]-pattern join (orders x customers) at 2 M probe rows against the oracle's join; then the same
    document written in _into batches with first / last flags, and the too-small destination"""
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    n_orders, n_cust = 2_000_000, 200_000
    cust = ctx.gen_csv("customers", (0, n_cust), seed=SEED, n_cust=n_cust, permute=True)
    orders = ctx.gen_csv("orders", (0, n_orders), seed=SEED, n_cust=n_cust, n_prod=1000)
    tc, _ = cp.parse_csv(ctx, cust, spec=[("id", -1), ("name", -1), ("surname", -1)])
    to, _ = cp.parse_csv(ctx, orders, spec=[("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)])
    j = to.join(tc.index_on("id", unique=True), "cust_id")
    oj = orc.reader_rows(orders.to_host(), select=["cust_id", "prod_id", "qty", "ts"]).join(
        orc.reader_rows(cust.to_host(), select=["id", "name", "surname"]).unique_index_on("id"), "cust_id")
    names = sorted(j.columns)
    assert len(j) == len(oj) == n_orders and set(x.decode() for x in oj.header(0)) == set(names)
    whole = j.to_json()
    assert whole == jo.columns_document([n.encode() for n in names], [oj.values(n) for n in names])
    # streamed: uneven batches into one pinned buffer
    cuts = [0, 1, 33, 700_000, 700_001, 1_999_999, n_orders]
    hb = ctx.host_alloc(len(whole) + 64)
    w = 0
    for a, b in zip(cuts, cuts[1:]):
        w += j.slice(a, b).to_json_into(hb, w, first=(a == 0), last=(b == n_orders))
    assert w == len(whole) and bytes(hb.array()[:w]) == whole
    # too small: the size needed comes back and nothing is written
    small = ctx.host_alloc(1000)
    small.array()[:] = 0xAB
    part = j.slice(0, 100)
    need = part.to_json_into(small, 0)
    assert need == len(part.to_json()) > 1000 and (small.array() == 0xAB).all()
    assert j.to_json_into(None) == len(whole)
    hb.free(); small.free()


def test_datasource_batches_errors_and_host_rows(monkeypatch):
    import csvplus_b200 as cp
    import csvplus_b200.api as api
    data = people_csv(5000, seed=9)
    src = lambda d=data: cp.Take(cp.FromBytes(d).SelectColumns("id", "name", "surname"))
    o = orc.reader_rows(data, select=["id", "name", "surname"])
    want = jo.columns_document([b"id", b"name", b"surname"], [o.values(c) for c in ("id", "name", "surname")])
    out = io.BytesIO()
    src().ToJSON(out)
    assert out.getvalue() == want
    monkeypatch.setattr(api, "JSON_BATCH_ROWS", 7)  # 715 batches
    out = io.BytesIO()
    src().ToJSON(out)
    assert out.getvalue() == want
    monkeypatch.undo()
    # a parse error after the delivered rows: the same DataSourceError, nothing written
    bad = data + b"too,few\n"
    ob = orc.reader_rows(bad, select=["id", "name", "surname"])
    assert ob.error is not None
    out = io.BytesIO()
    with pytest.raises(cp.DataSourceError) as ei:
        src(bad).ToJSON(out)
    assert str(ei.value) == ob.error and out.getvalue() == b""
    # rows that stay on the host: different column sets, and after an opaque Map
    rows = [{"b": "x\x08y", "a": "1"}, {"c": "\x0c"}, {}]
    out = io.BytesIO()
    cp.TakeRows(rows).ToJSON(out)
    assert out.getvalue() == jo.document([{k.encode(): v.encode() for k, v in r.items()} for r in rows])
    out = io.BytesIO()
    src().Top(3).Map(lambda r: {**r, "tag": "\x08"}).ToJSON(out)
    top3 = [{b"id": o.values("id")[i], b"name": o.values("name")[i], b"surname": o.values("surname")[i], b"tag": b"\x08"} for i in range(3)]
    assert out.getvalue() == jo.document(top3)


class _Digest:
    def __init__(self):
        self.n, self.crc = 0, 0

    def write(self, b):
        self.n += len(b)
        self.crc = zlib.crc32(b, self.crc)


def test_output_above_4_gib():
    """one call produces < 4 GiB (CPB_E_TOO_LARGE); DataSource.ToJSON writes a larger document in row-range batches"""
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    n = 42_000_000
    raw = ctx.gen_csv("orders", (0, n), seed=SEED, n_cust=n // 10, n_prod=1000)
    t, err = cp.parse_csv(ctx, raw, spec=[("order_id", -1), ("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)])
    raw.free()
    assert err is None and len(t) == n
    with pytest.raises(cp.CsvPlusError) as ei:
        t.to_json()
    assert ei.value.kind == 13  # CPB_E_TOO_LARGE
    step = 5_000_000
    total, crc = 0, 0
    for lo in range(0, n, step):
        hi = min(n, lo + step)
        b = t.slice(lo, hi).to_json_device(first=(lo == 0), last=(hi == n))
        total += b.nbytes
        crc = zlib.crc32(b.to_host(), crc)
        b.free()
    assert total > 1 << 32
    d = _Digest()
    cp.TakeTable(t).ToJSON(d)
    assert (d.n, d.crc) == (total, crc)
    rng = random.Random(42)
    for lo in sorted(rng.sample(range(0, n - 1_000_000), 2)):
        assert t.slice(lo, lo + 1_000_000).to_json(first=False, last=False) == _doc(t, lo, lo + 1_000_000, False, False)
