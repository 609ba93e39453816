"""GPU parity of Join / Except against a unique index held in the row-carrying hash table (a UniqueIndexOn whose full-key
image is at most 12 bytes and whose other columns, at most 4, take at most 16 bytes in every row), and of the indexes
just outside those limits, which keep the 16-byte probe table and the row slots."""
import random
import threading

import pytest

from oracle import oracle as orc
from tests.helpers import assert_table_equals_oracle, gpu_ctx

pytestmark = pytest.mark.gpu

NAMES = [b"Amelia", b"Olivia", b"Emily", b"Ava", b"Isla", b"Jack", b"Harry"]
SURNAMES = [b"Smith", b"Jones", b"Taylor", b"Williams", b"Brown", b"Davies", b""]


def _parse(data, ctx=None):
    import csvplus_b200 as cp
    t, err = cp.parse_csv(ctx or gpu_ctx(), data)
    assert err is None
    return t


def _customers(n, seed=1):
    rng = random.Random(seed)
    ids = list(range(n))
    rng.shuffle(ids)
    return b"id,name,surname\n" + b"".join(b"%d,%s,%s\n" % (i, rng.choice(NAMES), rng.choice(SURNAMES)) for i in ids)


def _orders(n, id_range, seed=2):
    rng = random.Random(seed)
    return b"order_id,cust_id,qty\n" + b"".join(b"%d,%d,%d\n" % (i, rng.randrange(id_range), rng.randrange(100)) for i in range(n))


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


def _check(idata, keys, pdata, *cols, rowhash=True):
    """Join and Except of pdata against UniqueIndexOn(keys) of idata, against the oracle; whether the row-carrying table
    was built must match `rowhash`"""
    ix, st, _ = _with_stats(lambda: _parse(idata).index_on(*keys, unique=True))
    assert ("rowhash_build" in st) == rowhash, sorted(st)
    oi = orc.reader_rows(idata).unique_index_on(*keys)
    tp, op = _parse(pdata), orc.reader_rows(pdata)
    assert_table_equals_oracle(tp.join(ix, *cols), op.join(oi, *cols))
    assert_table_equals_oracle(tp.join(ix, *cols, anti=True), op.except_(oi, *cols))
    return ix, oi, tp, op


@pytest.mark.parametrize("id_range,min_miss,max_miss", [(5000, 0, 0), (5100, 1, 1000), (10000, 5000, 15000)])
def test_join_all_match_and_misses(id_range, min_miss, max_miss):
    ix, oi, tp, op = _check(_customers(5000), ["id"], _orders(20000, id_range), "cust_id")
    miss = len(op.except_(oi, "cust_id"))
    assert min_miss <= miss <= max_miss
    _, st, syncs = _with_stats(lambda: len(tp.join(ix, "cust_id")))
    assert {"rowhash_probe", "rowhash_scan_lens", "slot_copy"} <= set(st)
    assert not {"hash_build", "join_probe", "slot_build", "slot_scan_lens"} & set(st), sorted(st)
    # one readback of the match count and the column totals; when rows miss, counting the hit rows and the column
    # totals of their gather add one each
    assert syncs == (1 if miss == 0 else 3)


def test_payload_of_16_and_17_bytes():
    rows = [(b"%d" % i, b"p" * (i % 9), b"q" * (8 - i % 9)) for i in range(300)]  # every row: 8 bytes of payload
    rows[17] = (b"17", b"p" * 8, b"q" * 8)
    data16 = b"k,p,q\n" + b"".join(b",".join(r) + b"\n" for r in rows)
    probe = b"k,x\n" + b"".join(b"%d,%d\n" % (i, i) for i in range(0, 320, 3))
    _check(data16, ["k"], probe, "k", rowhash=True)
    rows[17] = (b"17", b"p" * 8, b"q" * 9)
    data17 = b"k,p,q\n" + b"".join(b",".join(r) + b"\n" for r in rows)
    _check(data17, ["k"], probe, "k", rowhash=False)


def test_key_image_of_12_and_13_bytes():
    # one key column of width w: w value bytes + 1 length byte
    for w, rowhash in ((11, True), (12, False)):
        keys = [b"%0*d" % (w, i * 7919) for i in range(400)] + [b"x"]
        data = b"k,v\n" + b"".join(b"%s,v%d\n" % (k, i) for i, k in enumerate(keys))
        probe = b"k\n" + b"".join(k + b"\n" for k in keys[::3]) + b"nope\n" + b"0" * (w + 1) + b"\n"
        _check(data, ["k"], probe, "k", rowhash=rowhash)
    # two key columns: 5 + 1 and 5 + 1 bytes
    data = b"a,b,v\n" + b"".join(b"%d,%d,%d\n" % (i % 50, i // 50, i) for i in range(1000))
    probe = b"a,b\n" + b"".join(b"%d,%d\n" % (i % 60, i // 60) for i in range(0, 1200, 7))
    _check(data, ["a", "b"], probe, "a", "b")


def test_empty_values_and_empty_key():
    data = b"k,n,s\n,e0,\n1,,\n2,x,y\n3,,z\n"  # the empty key packs to an all-zero image
    probe = b"k,q\n,a\n3,b\n9,c\n,d\n1,e\n"
    ix, oi, tp, op = _check(data, ["k"], probe, "k")
    assert len(tp.join(ix, "k")) == 4


def test_probe_name_collisions():
    data = _customers(3000)
    oi = orc.reader_rows(data).unique_index_on("id")
    ix = _parse(data).index_on("id", unique=True)
    rng = random.Random(4)
    # the probe's `name` wins: the join needs `surname` only, a subset of the payload
    probe = b"cust_id,name\n" + b"".join(b"%d,P%d\n" % (rng.randrange(3100), i) for i in range(5000))
    assert_table_equals_oracle(_parse(probe).join(ix, "cust_id"), orc.reader_rows(probe).join(oi, "cust_id"))
    # ... and `surname`: no index column to fetch
    probe = b"id,surname,name\n" + b"".join(b"%d,S,N\n" % rng.randrange(3100) for _ in range(5000))
    assert_table_equals_oracle(_parse(probe).join(ix), orc.reader_rows(probe).join(oi))
    probe = b"id,surname,name\n" + b"".join(b"%d,S,N\n" % rng.randrange(3000) for _ in range(5000))
    assert_table_equals_oracle(_parse(probe).join(ix), orc.reader_rows(probe).join(oi))


def test_probe_views_and_empty_probe():
    data, pdata = _customers(4000), _orders(9000, 4100)
    oi = orc.reader_rows(data).unique_index_on("id")
    ix, tp = _parse(data).index_on("id", unique=True), _parse(pdata)
    allrows = orc.reader_rows(pdata)
    for lo, hi in ((0, 0), (1, 2), (37, 5000), (8999, 9000), (100, 9000)):
        view = tp.slice(lo, hi)
        sub = b"order_id,cust_id,qty\n" + b"".join(b"%s,%s,%s\n" % (r[b"order_id"], r[b"cust_id"], r[b"qty"])
                                                   for r in allrows.to_dicts()[lo:hi])
        assert_table_equals_oracle(view.join(ix, "cust_id"), orc.reader_rows(sub).join(oi, "cust_id"))
        assert_table_equals_oracle(view.join(ix, "cust_id", anti=True), orc.reader_rows(sub).except_(oi, "cust_id"))


def test_duplicate_key_error():
    import csvplus_b200 as cp
    data = _customers(2000) + b"1500,Dup,Row\n17,Two,Rows\n"
    with pytest.raises(cp.CsvPlusError) as e:
        _parse(data).index_on("id", unique=True)
    with pytest.raises(orc.OracleError) as oe:
        orc.reader_rows(data).unique_index_on("id")
    assert str(e.value) == str(oe.value)
    assert str(e.value).startswith("duplicate value while creating unique index: ")


def test_order_after_join():
    # the key image a qualifying index does not keep is packed on the first use of the order
    data = b"a,b,v\n" + b"".join(b"%d,%d,v%d\n" % ((i * 37) % 40, i, i) for i in range(800))
    ix, oi, tp, op = _check(data, ["a", "b"], b"a,b\n3,120\n39,799\n5,5\n", "a", "b")
    assert ix.Find("3").ToRows() == [{k.decode(): v.decode() for k, v in r.items()} for r in oi.find("3").to_dicts()]
    assert_table_equals_oracle(ix.table(), oi.rows())
    probe = b"a,q\n" + b"".join(b"%d,%d\n" % (i % 45, i) for i in range(100))
    assert_table_equals_oracle(_parse(probe).join(ix, "a"), orc.reader_rows(probe).join(oi, "a"))
    # and the full-key join still takes the row-carrying table
    _, st, _ = _with_stats(lambda: len(tp.join(ix, "a", "b")))
    assert "rowhash_probe" in st


def test_two_contexts_join_one_index():
    import csvplus_b200 as cp
    data, pdata = _customers(20000), _orders(60000, 20500)
    ix = _parse(data).index_on("id", unique=True)
    want = orc.reader_rows(pdata).join(orc.reader_rows(data).unique_index_on("id"), "cust_id")
    ctxs = [gpu_ctx(), cp.Context(gpu_ctx().device)]
    probes = [_parse(pdata, c) for c in ctxs]
    results, errors = [[], []], []

    def work(k):
        try:
            for _ in range(4):
                results[k].append(probes[k].join(ix, "cust_id"))
        except Exception as e:  # surfaced by the main thread
            errors.append(e)
    threads = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    try:
        assert not errors
        for k in range(2):
            for i in range(len(results[k])):
                assert_table_equals_oracle(results[k][i], want)
    finally:
        results.clear(); probes.clear()  # every table of the second context goes before it does
        ctxs[1].close()


def test_benchmark_shapes():
    """customers (id, name, surname) take the row-carrying table; products (prod_id, product, price: up to 17 bytes of
    payload) keep the 16-byte probe table and the row slots"""
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    ncust, nprod = 300_000, 100_000
    cust = ctx.gen_csv("customers", (0, ncust), n_cust=ncust, permute=True)
    prod = ctx.gen_csv("products", (0, nprod), n_prod=nprod, permute=True)
    orders = ctx.gen_csv("orders", (0, 400_000), n_cust=ncust, n_prod=nprod)
    tc, _ = cp.parse_csv(ctx, cust, spec=[("id", -1), ("name", -1), ("surname", -1)])
    tpr, _ = cp.parse_csv(ctx, prod, spec=[("prod_id", -1), ("product", -1), ("price", -1)])
    to, _ = cp.parse_csv(ctx, orders, spec=[("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)])
    cidx, st, _ = _with_stats(lambda: tc.index_on("id", unique=True))
    assert "rowhash_build" in st and "hash_build" not in st
    j, st, syncs = _with_stats(lambda: to.join(cidx, "cust_id"))
    assert {"rowhash_probe", "rowhash_scan_lens"} <= set(st) and not {"hash_build", "slot_build", "slot_scan_lens", "join_probe"} & set(st), sorted(st)
    assert syncs == 1
    pidx, st, _ = _with_stats(lambda: tpr.index_on("prod_id", unique=True))
    assert "rowhash_build" not in st and "hash_build" in st
    j2, st, _ = _with_stats(lambda: j.join(pidx))
    assert {"join_probe", "slot_build", "slot_scan_lens", "slot_copy"} <= set(st) and "rowhash_probe" not in st, sorted(st)
    oc = orc.reader_rows(cust.to_host(), select=["id", "name", "surname"])
    op = orc.reader_rows(prod.to_host(), select=["prod_id", "product", "price"])
    oo = orc.reader_rows(orders.to_host(), select=["cust_id", "prod_id", "qty", "ts"])
    assert_table_equals_oracle(j2, oo.join(oc.unique_index_on("id"), "cust_id").join(op.unique_index_on("prod_id")))
