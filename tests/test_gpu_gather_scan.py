"""GPU tests of the column gather and the look-back scans (gather.cu) that the route and parse tests leave out: each scan
source (scan_u32, scan_gather_len, slot_scan_lens, rowhash_scan_lens) at row counts around one, two and several tiles
(4096 rows per tile for the 32-bit scans, 2048 for the packed length scans) and past 8 tiles per SM, so that every CTA
takes several tickets; gather_copy groups longer than the 2048-byte stage, odd source alignments, empty values and
row-range views; and the kernel launches of the operations built on them.  Every result is compared byte for byte with
the oracle."""
import functools
import random

import numpy as np
import pytest

from oracle import oracle as orc
from tests.helpers import assert_table_equals_oracle, gpu_ctx

pytestmark = pytest.mark.gpu

SCAN_TILE, LENS_TILE = 4096, 2048
ALPHA = b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789 .-_"


def _sms():
    import torch
    return torch.cuda.get_device_properties(gpu_ctx().device).multi_processor_count


def _parse(data):
    import csvplus_b200 as cp
    t, err = cp.parse_csv(gpu_ctx(), data)
    assert err is None
    return t


def _word(rng, lo, hi):
    return bytes(rng.choice(ALPHA) for _ in range(rng.randint(lo, hi)))


def _table(n, seed, long_values=False):
    """k: a or b; v: 0-20 bytes (0-160 with long_values, a mean over 64); w: 0-3 bytes, so that the values of the other
    columns start at every alignment"""
    rng = random.Random(seed)
    vmax = 160 if long_values else 20
    rows = [b"%s,%s,%s" % (rng.choice(b"ab").to_bytes(1, "big"), _word(rng, 0, vmax), _word(rng, 0, 3)) for _ in range(n)]
    return b"k,v,w\n" + b"".join(r + b"\n" for r in rows)


def _oracle_values(o, col):
    off, data, _ = o.column(col)
    return [bytes(data[off[i]:off[i + 1]]) for i in range(len(off) - 1)]


def _customers(n, seed, long_payload):
    """a unique index source: id, name, surname; with long_payload every row's payload exceeds the 16 bytes the
    row-carrying table holds, so that a join takes the row slots"""
    rng = random.Random(seed)
    ids = list(range(n))
    rng.shuffle(ids)
    slo, shi = (17, 24) if long_payload else (0, 5)
    return b"id,name,surname\n" + b"".join(b"%d,%s,%s\n" % (i, _word(rng, 0, 6), _word(rng, slo, shi)) for i in ids)


def _orders(n, id_range, seed):
    rng = random.Random(seed)
    return b"cust_id,qty\n" + b"".join(b"%d,%d\n" % (rng.randrange(id_range), rng.randrange(1000)) for _ in range(n))


def _stats(fn):
    ctx = gpu_ctx()
    ctx.sync()
    ctx.stats(enable=True, reset=True)
    s0 = ctx.host_syncs()
    r = fn()
    ctx.sync()
    syncs = ctx.host_syncs() - s0
    st = ctx.stats()
    ctx.stats(enable=False)
    return r, {k: v["launches"] for k, v in st.items()}, syncs


AROUND_SCAN = [1, SCAN_TILE - 1, SCAN_TILE, SCAN_TILE + 1, 2 * SCAN_TILE, 2 * SCAN_TILE + 1, 5 * SCAN_TILE + 77]
AROUND_LENS = [1, LENS_TILE - 1, LENS_TILE, LENS_TILE + 1, 2 * LENS_TILE, 2 * LENS_TILE + 1, 5 * LENS_TILE + 77]


@pytest.mark.parametrize("n", AROUND_SCAN)
def test_scan_u32_and_gather_len(n):
    """ToCsv scans the row lengths (scan_u32); Filter scans the lengths of the kept rows (scan_gather_len)"""
    data = _table(n, seed=n)
    t, o = _parse(data), orc.reader_rows(data)
    _, st, _ = _stats(lambda: t.to_csv("k", "v", "w"))
    assert st.get("scan_u32") == 1
    assert t.to_csv("k", "v", "w") == o.to_csv("k", "v", "w")[0]
    import csvplus_b200 as cp
    f, st, _ = _stats(lambda: t.filter(cp.Like({"k": "a"})))
    assert st.get("scan_gather_len") == (3 if len(f) else None)
    assert_table_equals_oracle(f, o.filter(orc.Like({"k": "a"})))


@pytest.mark.parametrize("n", AROUND_LENS)
@pytest.mark.parametrize("route", ["rowhash", "slot"])
def test_length_scans(route, n):
    """a join against a unique index: rowhash_scan_lens over the probe's packed lengths, or slot_scan_lens over those of
    the row slots the probe rows pick (laid out on a first join with at least as many rows as the index)"""
    k = min(n, 1000) if route == "slot" else max(2, min(n, 1000))  # (a 1-row unique index has no row-carrying table)
    cdata, odata = _customers(k, seed=n, long_payload=route == "slot"), _orders(n, k, seed=n + 1)
    ix = _parse(cdata).index_on("id", unique=True)
    tp = _parse(odata)
    j, st, _ = _stats(lambda: tp.join(ix, "cust_id"))
    assert st.get(f"{route}_scan_lens") == 1, sorted(st)
    assert_table_equals_oracle(j, orc.reader_rows(odata).join(orc.reader_rows(cdata).unique_index_on("id"), "cust_id"))


def test_scans_with_several_tickets_per_cta():
    """more tiles than 8 CTAs per SM hold: every CTA of each scan takes several tickets"""
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    n = _sms() * 8 * SCAN_TILE * 3 // 2
    orders = ctx.gen_csv("orders", (0, n), n_cust=n // 4, n_prod=1000)
    host = orders.to_host()
    t, err = cp.parse_csv(ctx, orders, spec=[("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)])
    assert err is None
    o = orc.reader_rows(host, select=["cust_id", "prod_id", "qty", "ts"])
    assert t.to_csv("ts", "cust_id", "qty") == o.to_csv("ts", "cust_id", "qty")[0]
    assert_table_equals_oracle(t.filter(cp.Not(cp.Like({"qty": "1"}))), o.filter(orc.Not(orc.Like({"qty": "1"}))))
    # length scans: a join of more than 8 * 2048 probe rows per SM, rowhash and slot routes
    k = 50_000
    for long_payload, route in ((False, "rowhash"), (True, "slot")):
        cdata = _customers(k, seed=7, long_payload=long_payload)
        ix = _parse(cdata).index_on("id", unique=True)
        np_rows = _sms() * 8 * LENS_TILE * 3 // 2
        odata = _orders(np_rows, k, seed=8)
        tp = _parse(odata)
        j, st, _ = _stats(lambda: tp.join(ix, "cust_id"))
        assert st.get(f"{route}_scan_lens") == 1, sorted(st)
        assert_table_equals_oracle(j, orc.reader_rows(odata).join(orc.reader_rows(cdata).unique_index_on("id"), "cust_id"))


@pytest.mark.parametrize("lo,hi", [(0, 3000), (1, 3000), (37, 2900), (1000, 1001), (2999, 3000)])
@pytest.mark.parametrize("long_values", [False, True])
def test_gather_copy_views(lo, hi, long_values):
    """Filter over a row-range view (row0 = lo): kept rows come from every source alignment, some values are empty, and
    with long values most 32-row groups exceed the 2048-byte stage and are written directly"""
    import csvplus_b200 as cp
    data = _table(3000, seed=lo * 7 + hi, long_values=long_values)
    t, o = _parse(data), orc.reader_rows(data)
    want = {c: _oracle_values(o, c)[lo:hi] for c in ("k", "v", "w")}
    keep = [i for i, x in enumerate(want["k"]) if x == b"a"]
    f = t.slice(lo, hi).filter(cp.Like({"k": "a"}))
    assert len(f) == len(keep)
    for c in ("k", "v", "w"):
        assert f.values(c) == [want[c][i] for i in keep], c
    # every row of the view: the gather with consecutive ids
    g = t.slice(lo, hi).filter(cp.Not(cp.Like({"k": "no such value"})))
    for c in ("k", "v", "w"):
        assert g.values(c) == want[c], c
    if long_values and hi - lo >= 64:  # the views of many rows do take the direct path
        off, _ = g.column("v")
        groups = np.diff(np.asarray(off, dtype=np.int64)[::32])
        assert (groups > 2048).any()


# kernel launches and host synchronisations per operation, measured on an H100 80GB HBM3 before the scans shared one
# look-back chain; a change to the scans or the gather that alters them shows here
LAUNCHES = {'filter': {'host_syncs': 3,
            'kernels': {'compact_ids': 1, 'filter_like': 1, 'gather_copy': 2, 'scan_gather_len': 3, 'scan_u32': 1}},
 'format_float': {'host_syncs': 2, 'kernels': {'format_float': 1, 'format_write': 1, 'scan_u32': 1}},
 'index_on_table': {'host_syncs': 5,
                    'kernels': {'gather_copy': 3,
                                'image_gather': 1,
                                'key_pack': 1,
                                'key_width': 1,
                                'radix_pass': 21,
                                'scan_gather_len': 3,
                                'scan_u32': 7,
                                'sort_gather_word': 1,
                                'sort_hist': 1}},
 'join_plain': {'host_syncs': 3, 'kernels': {'gather_copy': 5, 'join_probe': 1, 'key_pack': 1, 'scan_gather_len': 5}},
 'join_rowhash': {'host_syncs': 2, 'kernels': {'rowhash_probe': 1, 'rowhash_scan_lens': 1, 'slot_copy': 1}},
 'join_slot': {'host_syncs': 3, 'kernels': {'join_probe': 1, 'key_pack': 1, 'slot_copy': 1, 'slot_scan_lens': 1}},
 'to_csv': {'host_syncs': 4, 'kernels': {'csv_row_len': 1, 'csv_write': 1, 'scan_u32': 1}},
 'to_json': {'host_syncs': 4, 'kernels': {'json_row_len': 1, 'json_write': 1, 'scan_u32': 1}},
 'write_to': {'host_syncs': 6, 'kernels': {'d2h_output': 0, 'gob_row_len': 2, 'gob_write': 1, 'scan_u32': 1}}}


@functools.lru_cache(maxsize=None)
def measure_launches():
    """{operation: {"kernels": {stat name: launches}, "host_syncs": n}}, each taken on the second call of the operation
    (the first builds what an index keeps)"""
    import os
    import tempfile

    import torch
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    people = _parse(_customers(5000, seed=3, long_payload=True))
    short = _parse(_customers(5000, seed=4, long_payload=False))
    orders = _parse(_orders(20000, 5000, seed=5))
    wide = _parse(b"id,a,b,c,d,e\n" + b"".join(b"%d,%d,x,yy,zzz,%d\n" % (i, i * 7, i % 13) for i in range(5000)))
    ix_slot, ix_rowhash, ix_plain = (x.index_on("id", unique=True) for x in (people, short, wide))
    vals = torch.arange(5000, dtype=torch.float64, device=f"cuda:{ctx.device}") / 7
    like = cp.Like({"surname": people.values("surname", 0, 1)[0].decode()})
    out = {}
    with tempfile.TemporaryDirectory() as d:
        ops = {
            "filter": lambda: people.filter(like),
            "index_on_table": lambda: people.index_on("name").table(),
            "join_slot": lambda: orders.join(ix_slot, "cust_id"),
            "join_rowhash": lambda: orders.join(ix_rowhash, "cust_id"),
            "join_plain": lambda: orders.join(ix_plain, "cust_id"),
            "to_csv": lambda: people.to_csv("id", "name", "surname"),
            "to_json": lambda: people.to_json(),
            "write_to": lambda: ix_slot.WriteTo(os.path.join(d, "ix.gob")),
            "format_float": lambda: people.with_column("x", vals, fmt="g", prec=-1),
        }
        for name, fn in ops.items():
            fn()
            _, st, syncs = _stats(fn)
            out[name] = {"kernels": st, "host_syncs": syncs}
    return out


@pytest.mark.parametrize("op", sorted(LAUNCHES))
def test_launches(op):
    assert measure_launches()[op] == LAUNCHES[op]


if __name__ == "__main__":
    import json
    print(json.dumps(measure_launches(), sort_keys=True))
