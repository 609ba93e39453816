"""GPU parity of the region-by-region build of the row-carrying hash table (UniqueIndexOn with a short key and a short
payload): region counts at and around the region size, keys whose probe sequence wraps inside its region, duplicates,
and a region that overflows and sends the index to the 16-byte probe table.  Keys aimed at given slots are chosen with a
restatement of the key image, the hash and the slot mapping of rowhash.cuh (tests/hash_ref.py)."""
import random

import numpy as np
import pytest

from oracle import oracle as orc
from tests.hash_ref import first_slots
from tests.helpers import assert_table_equals_oracle, gpu_ctx

pytestmark = pytest.mark.gpu

REGION = 1024  # RH_REGION (rowhash.cuh)


def _layout(n):
    """(slots per region, number of regions) of the table of an n-row index (join.cu: rowhash_build)"""
    want = 2 * n + 16
    rs = 1
    while rs < want and rs < REGION:
        rs *= 2
    return rs, -(-want // rs)


def _parse(data):
    import csvplus_b200 as cp
    t, err = cp.parse_csv(gpu_ctx(), data)
    assert err is None
    return t


def _with_stats(fn):
    ctx = gpu_ctx()
    ctx.sync()
    ctx.stats(enable=True, reset=True)
    s0 = ctx.host_syncs()
    r = fn()
    syncs = ctx.host_syncs() - s0
    ctx.sync()
    st = ctx.stats()
    ctx.stats(enable=False)
    return r, st, syncs


def _index_csv(keys, seed=1):
    rng = random.Random(seed)
    return b"k,name,city\n" + b"".join(b"%s,n%d,%s\n" % (k, rng.randrange(1000), rng.choice([b"", b"Oslo", b"Lima"])) for k in keys)


def _check(idata, pdata, key="k", pkey="k", path="rowhash"):
    """UniqueIndexOn(key) of idata built on `path` (rowhash: the row-carrying table, two host syncs; hash16: the build
    overflowed and the index took the 16-byte probe table); Join and Except of pdata checked against the oracle"""
    ti = _parse(idata)
    ix, st, syncs = _with_stats(lambda: ti.index_on(key, unique=True))
    assert {"rowhash_scatter", "rowhash_build"} <= set(st), sorted(st)
    if path == "rowhash":
        assert "hash_build" not in st and syncs == 2, (sorted(st), syncs)
    else:
        assert "hash_build" in st, sorted(st)
    oi = orc.reader_rows(idata).unique_index_on(key)
    tp, op = _parse(pdata), orc.reader_rows(pdata)
    j, st, _ = _with_stats(lambda: tp.join(ix, pkey))
    assert ("rowhash_probe" in st) == (path == "rowhash") and ("join_probe" in st) == (path != "rowhash"), sorted(st)
    assert_table_equals_oracle(j, op.join(oi, pkey))
    assert_table_equals_oracle(tp.join(ix, pkey, anti=True), op.except_(oi, pkey))


def _customers(n, seed=1):
    rng = random.Random(seed)
    ids = list(range(n))
    rng.shuffle(ids)
    return b"id,name,surname\n" + b"".join(b"%d,N%d,S%d\n" % (i, rng.randrange(50), rng.randrange(9)) for i in ids)


def _orders(n, id_range, seed=2):
    rng = random.Random(seed)
    return b"order_id,id,qty\n" + b"".join(b"%d,%d,%d\n" % (i, rng.randrange(id_range), rng.randrange(100)) for i in range(n))


@pytest.mark.parametrize("n", [2, 300, 504, 505, 1528, 2040, 1_050_000])
def test_region_counts(n):
    # one region (2, 300, 504: 2n + 16 <= 1024), exact multiples of the region (504, 1528, 2040: 2n + 16 = 1, 3, 4
    # regions), one past (505), and more than 1000 regions
    rs, nreg = _layout(n)
    assert (nreg == 1) == (n <= 504) and (n < 1_000_000 or nreg >= 1000)
    _check(_customers(n), _orders(min(4 * n, 400_000), n + n // 10 + 1), key="id", pkey="id")


def _ints(off, data):
    """the decimal values of a column of non-negative integers"""
    lens = np.diff(off)
    ends = np.repeat(off[1:], lens)
    place = ends - 1 - np.arange(off[0], off[-1])
    return np.add.reduceat((data.astype(np.int64) - 48) * 10 ** place, off[:-1] - off[0])


def _take(off, data, rows):
    """(offsets, bytes) of rows `rows` of a column"""
    lens = off[rows + 1] - off[rows]
    out = np.zeros(len(rows) + 1, np.int64)
    np.cumsum(lens, out=out[1:])
    return out, data[np.repeat(off[rows] - out[:-1], lens) + np.arange(out[-1])]


def test_10m_rows_against_numpy():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    ncust, nord = 10_000_000, 10_000_000
    cust = ctx.gen_csv("customers", (0, ncust), n_cust=ncust, permute=True)
    orders = ctx.gen_csv("orders", (0, nord), n_cust=ncust + ncust // 20, n_prod=1000)  # ids past ncust miss
    tc, _ = cp.parse_csv(ctx, cust, spec=[("id", -1), ("name", -1), ("surname", -1)])
    to, _ = cp.parse_csv(ctx, orders, spec=[("cust_id", -1), ("qty", -1)])
    ix, st, syncs = _with_stats(lambda: tc.index_on("id", unique=True))
    assert {"rowhash_scatter", "rowhash_build"} <= set(st) and "hash_build" not in st and syncs == 2
    row_of = np.full(ncust + ncust // 20, -1, np.int64)
    row_of[_ints(*tc.column("id"))] = np.arange(ncust)
    poff, pdata = to.column("cust_id")
    crow = row_of[_ints(poff, pdata)]
    hit = np.flatnonzero(crow >= 0)
    assert 0 < len(hit) < nord
    j = to.join(ix, "cust_id")
    assert len(j) == len(hit)
    for col, src, rows in (("cust_id", to, hit), ("qty", to, hit), ("name", tc, crow[hit]), ("surname", tc, crow[hit])):
        want = _take(*src.column(col), rows)
        got = j.column(col)
        assert np.array_equal(got[0] - got[0][0], want[0]) and np.array_equal(got[1], want[1]), col
    e = to.join(ix, "cust_id", anti=True)
    want = _take(poff, pdata, np.flatnonzero(crow < 0))
    got = e.column("cust_id")
    assert np.array_equal(got[0] - got[0][0], want[0]) and np.array_equal(got[1], want[1])


def test_probe_wraps_inside_the_region():
    n = 5000
    rs, nreg = _layout(n)
    cand = [b"%08d" % i for i in range(1_500_000)]
    slot = first_slots(cand, rs * nreg)
    by_slot = {}
    for i in np.flatnonzero((slot % rs == rs - 1) | (slot % rs == 0)):
        by_slot.setdefault(int(slot[i]), []).append(cand[i])
    aimed, misses = [], []
    for g in range(nreg):
        last, first = by_slot.get(g * rs + rs - 1, []), by_slot.get(g * rs, [])
        assert len(last) >= 7 and len(first) >= 2
        aimed += last[:4] + first[:2]  # three of the four wrap to the region's first slot, past its own two keys
        misses += last[4:7]            # walk the same slots to the first empty one
    used = set(aimed) | set(misses)
    keys = aimed + [k for k in cand[:3 * n] if k not in used][: n - len(aimed)]
    random.Random(3).shuffle(keys)
    probe = b"k\n" + b"".join(k + b"\n" for k in keys[::7] + aimed + misses)
    _check(_index_csv(keys), probe)


def test_duplicates():
    import csvplus_b200 as cp
    n = 6000
    rs, nreg = _layout(n)
    cand = [b"%07d" % i for i in range(3 * n)]
    slot = first_slots(cand, rs * nreg)
    region0 = [cand[i] for i in np.flatnonzero(slot[n:] // rs == 0) + n]  # keys not in base
    base = cand[:n]
    cases = [
        base + [region0[5], region0[9]] + [region0[9], region0[5]],  # two duplicated keys in one region
        base[:n // 2] + [base[77]] * 500 + base[n // 2:],             # one key 501 times
        base + [base[-1]],                                            # the duplicate is the last row
        base + [base[0]],
    ]
    for keys in cases:
        data = _index_csv(keys)
        with pytest.raises(cp.CsvPlusError) as e:
            _parse(data).index_on("k", unique=True)
        with pytest.raises(orc.OracleError) as oe:
            orc.reader_rows(data).unique_index_on("k")
        assert str(e.value) == str(oe.value)
        assert str(e.value).startswith("duplicate value while creating unique index: ")


def test_overflowing_region_takes_the_probe_table():
    n = 20000
    rs, nreg = _layout(n)
    cand = [b"%08d" % i for i in range(600_000)]
    region = first_slots(cand, rs * nreg) // rs
    crowd = [cand[i] for i in np.flatnonzero(region == 3)][: rs + 50]  # more keys than region 3 can hold
    assert len(crowd) == rs + 50
    others = [cand[i] for i in np.flatnonzero(region != 3)[: n - len(crowd)]]
    keys = crowd + others
    random.Random(5).shuffle(keys)
    outside = [cand[i] for i in np.flatnonzero(region == 3)[rs + 50: rs + 250]]
    probe = b"k\n" + b"".join(k + b"\n" for k in crowd[::3] + others[::11] + outside + [b"nope"])
    _check(_index_csv(keys), probe, path="hash16")
    # a duplicate inside the overflowing region is still found
    import csvplus_b200 as cp
    data = _index_csv(keys + [crowd[7]])
    with pytest.raises(cp.CsvPlusError) as e:
        _parse(data).index_on("k", unique=True)
    with pytest.raises(orc.OracleError) as oe:
        orc.reader_rows(data).unique_index_on("k")
    assert str(e.value) == str(oe.value)
