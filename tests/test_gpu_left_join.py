"""LeftJoin on the GPU against tests/left_join_ref.py (the plain restatement over the index's stored rows), row for row and
byte for byte, with its columns in Join's order and its matched rows equal to Join's result:

1. every case of test_gpu_index_keys.CASES at every key prefix, on the probe route Join takes for it;
2. the row-carrying table: all, some, most and no probe rows matching; payloads of 16 and 17 bytes; an index key named
   unlike the probe's join column (empty on a miss); probe name collisions, row-range views and AssumeHeader aliases;
3. an empty index, an empty probe, a one-row index probed by b"a", b"a\\0" and b"";
4. indexes out of key order (LoadIndex of an unsorted file, ResolveDuplicates);
5. streamed plans: two LeftJoins in a multi-batch ToCsv, a source error in a later batch, a missing join column;
6. host synchronisations per route, and Join's kernels when every probe row matches once;
7. a result column at the 4 GiB limit on the index and the probe side, refused without writing;
8. host/left_join_example.cpp."""
import io
import os
import random
import subprocess

import pytest

from tests import index_ref as ref
from tests import left_join_ref as lj
from tests.helpers import gpu_ctx
from tests.hash_ref import image_bytes, probe_kind
from tests.test_gpu_index_keys import (CASES, _both, _case_data, _check_route, _columns, _device_table, _load, _resolve_both,
                                       _rowhash_fits, _trows, _with_stats)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check(pt, ix, pcols, probe=None, stored=None):
    """pt.join(ix, *pcols, left=True) against the restatement over ix's stored rows -> (LeftJoin table, Join table)"""
    stored = _trows(ix.table()) if stored is None else stored
    keys = [c.encode() for c in ix.columns]
    icols = [c.encode() for c in ix.table().columns]
    probe = _trows(pt) if probe is None else probe
    pc = [c.encode() for c in pcols]
    got = pt.join(ix, *pcols, left=True)
    assert [c.encode() for c in got.columns] == lj.schema(icols, [c.encode() for c in pt.columns])
    rows = _trows(got)
    assert rows == lj.left_join(stored, keys, probe, pc, index_columns=icols)
    j = pt.join(ix, *pcols)
    assert got.columns == j.columns
    # the matched rows, in order, are Join's result
    matched, at = [], 0
    for p in probe:
        k = len(ref.join(stored, keys, [p], pc))
        matched += rows[at:at + k]
        at += max(k, 1)
    assert at == len(rows) and matched == _trows(j)
    return got, j


# ------------------------------------------------------------------ 1. the route matrix
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_route_matrix(case):
    rows, knames, values, pay_lens, pnames, pvalues = _case_data(case)
    n, K = len(rows), len(knames)
    it, _ = _both(values)
    ix, st_build = _with_stats(lambda: it.index_on(*knames, unique=case.unique))
    rowhash = _rowhash_fits(case.unique, n, case.widths, pay_lens)
    stored = _trows(ix.table())
    full = _device_table(_columns(pvalues))
    part = _device_table(_columns({nm: v[:400] for nm, v in pvalues.items()}))
    for nk in [K] + list(range(1, K)):
        pt = full if nk == K else part
        nheads = len({r[:nk] for r in rows})
        pbytes = image_bytes(case.widths[:nk])
        if rowhash and nk == K:
            kind = "rowhash"
        else:
            if case.unique and nk == K:
                nheads = n
            kind = probe_kind(nheads, pbytes, n)
        # LeftJoin first: its stats hold the probe table's build, as Join's do in test_probe_routes
        _, st = _with_stats(lambda: pt.join(ix, *pnames[:nk], left=True))
        _check_route({**st_build, **st} if nk == K else st, kind, nheads, pbytes)
        _check(pt, ix, pnames[:nk], stored=stored)


# ------------------------------------------------------------------ 2. the row-carrying table
def _customers(n, name_len=6, seed=1):
    rnd = random.Random(seed)
    return [{"id": "c%07d" % i, "name": ("n%d" % rnd.randrange(10 ** 6)).ljust(name_len, "x")[:name_len],
             "city": "t%d" % (i % 10)} for i in range(n)]


def _orders(n, id_range, seed=2, key="cust_id"):
    rnd = random.Random(seed)
    return [{"order": "%d" % i, key: "c%07d" % rnd.randrange(id_range), "qty": "%d" % rnd.randrange(100)} for i in range(n)]


@pytest.mark.parametrize("id_range", [3000, 3030, 6000, 30000, 10 ** 7], ids=["all", "few", "half", "most", "none"])
@pytest.mark.parametrize("name_len", [14, 15], ids=["pay16", "pay17"])
def test_row_carrying_shapes(id_range, name_len):
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    cust = cp.Table.from_rows(ctx, _customers(3000, name_len), ["id", "name", "city"])
    ix, st = _with_stats(lambda: cust.index_on("id", unique=True))
    assert ("rowhash_build" in st) == (name_len == 14), sorted(st)  # payload name + city: 16 or 17 bytes
    ords = _orders(5000, id_range)
    pt = cp.Table.from_rows(ctx, ords, ["order", "cust_id", "qty"])
    got, j = _check(pt, ix, ["cust_id"])
    hits = sum(1 for o in ords if int(o["cust_id"][1:]) < 3000)
    assert len(j) == hits and len(got) == len(ords)
    ids = got.values("id")
    assert all((v == o["cust_id"].encode()) if int(o["cust_id"][1:]) < 3000 else v == b"" for v, o in zip(ids, ords))
    # a natural join keeps the probe's key on a miss
    pn = cp.Table.from_rows(ctx, [{"id": o["cust_id"], "qty": o["qty"]} for o in ords], ["id", "qty"])
    got, _ = _check(pn, ix, [])
    assert got.values("id") == [o["cust_id"].encode() for o in ords]


def test_row_carrying_collisions_views_and_aliases():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    cust = cp.Table.from_rows(ctx, _customers(2000), ["id", "name", "city"])
    ix = cust.index_on("id", unique=True)
    ords = [{**o, "name": "probe%d" % i} for i, o in enumerate(_orders(3000, 4000))]
    pt = cp.Table.from_rows(ctx, ords, ["order", "cust_id", "name", "qty"])
    got, _ = _check(pt, ix, ["cust_id"])  # the probe's name wins on matches and misses
    assert got.values("name") == [o["name"].encode() for o in ords]
    for lo, hi in ((0, 1), (17, 2900), (1500, 3000), (3000, 3000)):
        _check(pt.slice(lo, hi), ix, ["cust_id"])
    csv = "".join("%s,%s\n" % (o["cust_id"], o["qty"]) for o in ords).encode()
    at, err = cp.parse_csv(ctx, csv, header_from_first_row=False, spec=[("cust_id", 0), ("alias", 0), ("qty", 1)])
    assert err is None
    got, _ = _check(at, ix, ["alias"])
    _check(at.slice(5, 2000), ix, ["cust_id"])


# ------------------------------------------------------------------ 3. small cases
def test_empty_index_empty_probe_and_one_row_index():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    empty_ix = cp.Table.from_rows(ctx, [{"id": "1", "name": "a"}], ["id", "name"]).slice(0, 0).index_on("id")
    pt = cp.Table.from_rows(ctx, [{"cust_id": "1", "q": "x"}, {"cust_id": "", "q": "y"}], ["cust_id", "q"])
    (got, _), st = _with_stats(lambda: _check(pt, empty_ix, ["cust_id"], stored=[]))
    assert got.values("id") == [b"", b""] and got.values("name") == [b"", b""] and got.values("q") == [b"x", b"y"]
    assert "gather_copy" not in st and "slot_copy" not in st, sorted(st)
    ix = cp.Table.from_rows(ctx, [{"id": "1", "name": "a"}], ["id", "name"]).index_on("id")
    for t in (pt.slice(0, 0), pt.slice(1, 1)):
        got = t.join(ix, "cust_id", left=True)
        assert len(got) == 0 and got.columns == t.join(ix, "cust_id").columns == ["id", "name", "cust_id", "q"]
    for unique in (False, True):
        it, _ = _both({"k": [b"a\x00"], "v": [b"x"]})
        one = it.index_on("k", unique=unique)
        probe, _ = _both({"p": [b"a", b"a\x00", b"", b"a\x00\x00"], "q": [b"0", b"1", b"2", b"3"]})
        got, _ = _check(probe, one, ["p"])
        assert got.values("v") == [b"", b"x", b"", b""] and got.values("k") == [b"", b"a\x00", b"", b""]


# ------------------------------------------------------------------ 4. indexes out of key order
def test_load_index_of_an_unsorted_file(tmp_path):
    rng = random.Random(5)
    cols = [b"k", b"j"]
    stored = [{b"k": b"k%02d" % rng.randrange(30), b"j": b"%d" % rng.randrange(3), b"v": b"v%d" % i} for i in range(600)]
    ix = _load(stored, cols, tmp_path)
    probe = [{b"pk": r[b"k"], b"pj": r[b"j"] + (b"\x00" if rng.random() < 0.2 else b""), b"q": b"%d" % i}
             for i, r in enumerate(rng.choice(stored) for _ in range(400))]
    pt = _device_table(_columns({k.decode(): [p[k] for p in probe] for k in probe[0]}))
    for pn in (["pk"], ["pk", "pj"]):
        (_, _), st = _with_stats(lambda: _check(pt, ix, pn, probe=probe, stored=stored))
        assert "join_search" in st, sorted(st)


def test_after_resolve_duplicates():
    rng = random.Random(8)
    rows = [{b"k": b"key%03d" % rng.randrange(400), b"v": b"%d" % i} for i in range(5000)]
    it, _ = _both({"k": [r[b"k"] for r in rows], "v": [r[b"v"] for r in rows]})
    ix = it.index_on("k")
    stored = _resolve_both(ix, ref.index_on(rows, [b"k"]), [b"k"], lambda grp: {b"k": grp[0][b"k"][::-1], b"v": b"r"})
    probe = [{b"p": (b"key%03d" % rng.randrange(450))[::1 if rng.random() < 0.5 else -1], b"q": b"%d" % i} for i in range(2000)]
    pt = _device_table(_columns({k.decode(): [p[k] for p in probe] for k in probe[0]}))
    _check(pt, ix, ["p"], probe=probe, stored=stored)


# ------------------------------------------------------------------ 5. streamed plans
def _csv(rows, cols):
    return ("\n".join([",".join(cols)] + [",".join(r[c] for c in cols) for r in rows]) + "\n").encode()


def test_streamed_plan_of_two_left_joins(monkeypatch):
    import csvplus_b200 as cp
    from csvplus_b200 import api
    ctx = gpu_ctx()
    cust_rows = _customers(3000)
    prod_rows = [{"prod_id": "p%d" % i, "price": "%d.5" % i} for i in range(0, 400, 2)]
    cust = cp.Take(cp.FromBytes(_csv(cust_rows, ["id", "name", "city"]), ctx)).UniqueIndexOn("id")
    prod = cp.Take(cp.FromBytes(_csv(prod_rows, ["prod_id", "price"]), ctx)).UniqueIndexOn("prod_id")
    rnd = random.Random(3)
    ords = [{"order": "%d" % i, "cust_id": "c%07d" % rnd.randrange(3300), "prod_id": "p%d" % rnd.randrange(420)} for i in range(40000)]
    data = _csv(ords, ["order", "cust_id", "prod_id"])
    c_rows = ref.index_on([{k.encode(): v.encode() for k, v in r.items()} for r in cust_rows], [b"id"])
    p_rows = ref.index_on([{k.encode(): v.encode() for k, v in r.items()} for r in prod_rows], [b"prod_id"])
    want = lj.left_join(c_rows, [b"id"], [{k.encode(): v.encode() for k, v in o.items()} for o in ords], [b"cust_id"])
    want = lj.left_join(p_rows, [b"prod_id"], want)
    out_cols = ["order", "id", "name", "prod_id", "price"]
    monkeypatch.setattr(api, "STREAM_BATCH_BYTES", 64 << 10)  # about 15 batches
    buf = io.BytesIO()
    cp.Take(cp.FromBytes(data, ctx)).LeftJoin(cust, "cust_id").LeftJoin(prod).ToCsv(buf, *out_cols)
    assert buf.getvalue() == _csv([{c: w[c.encode()].decode() for c in out_cols} for w in want], out_cols)
    # a source error in a later batch: the rows before it are written, then the error, as after Join
    bad = data + b'1,"x\n'
    outs = []
    for step in ("Join", "LeftJoin"):
        b = io.BytesIO()
        with pytest.raises(cp.DataSourceError) as e:
            getattr(cp.Take(cp.FromBytes(bad, ctx)), step)(cust, "cust_id").ToCsv(b, "order", "cust_id")
        outs.append((b.getvalue(), str(e.value)))
    assert outs[0][1] == outs[1][1] and len(outs[1][0]) > len(outs[0][0]) > 0
    assert outs[1][0] == _csv([{"order": o["order"], "cust_id": o["cust_id"]} for o in ords], ["order", "cust_id"])
    # a missing join column: Join's text and row
    errs = []
    for step in ("Join", "LeftJoin"):
        with pytest.raises(cp.DataSourceError) as e:
            getattr(cp.Take(cp.FromBytes(data, ctx)), step)(cust, "nope").ToRows()
        errs.append((str(e.value), e.value.Line))
    assert errs[0] == errs[1]


# ------------------------------------------------------------------ 6. host synchronisations and kernels
def _syncs(fn):
    ctx = gpu_ctx()
    ctx.sync()
    s0 = ctx.host_syncs()
    r = fn()
    return ctx.host_syncs() - s0, r


def test_host_syncs_per_route_and_joins_kernels_on_all_match():
    import csvplus_b200 as cp
    ctx = gpu_ctx()
    cust = cp.Table.from_rows(ctx, _customers(3000, 14), ["id", "name", "city"])
    rix = cust.index_on("id", unique=True)  # row-carrying table
    sm_t = cp.Table.from_rows(ctx, [{"k": "k%d" % (i % 500), "v": "v%d" % i} for i in range(1000)], ["k", "v"])
    six = sm_t.index_on("k")  # runs of two, smem route
    all_match = cp.Table.from_rows(ctx, _orders(4000, 3000), ["order", "cust_id", "qty"])
    misses = cp.Table.from_rows(ctx, _orders(4000, 6000), ["order", "cust_id", "qty"])
    none = cp.Table.from_rows(ctx, _orders(4000, 10 ** 7, seed=9)[:0] + [{"order": "1", "cust_id": "zz", "qty": "1"}], ["order", "cust_id", "qty"])
    nat = cp.Table.from_rows(ctx, [{"id": o["cust_id"], "q": o["qty"]} for o in _orders(4000, 6000)], ["id", "q"])
    runs = cp.Table.from_rows(ctx, [{"k": "k%d" % (i % 700), "q": "%d" % i} for i in range(3000)], ["k", "q"])
    for t, ix, cols in ((all_match, rix, ["cust_id"]), (runs, six, ["k"])):
        t.join(ix, *cols), t.join(ix, *cols, left=True)  # probe tables, slots and sorted rows built once
    # row-carrying table: the miss rows' key column gathered again (named key) or nothing more (natural join)
    assert _syncs(lambda: misses.join(rix, "cust_id"))[0] == 3
    assert _syncs(lambda: misses.join(rix, "cust_id", left=True))[0] == 2
    assert _syncs(lambda: nat.join(rix, left=True))[0] == 1
    assert _syncs(lambda: none.join(rix, "cust_id", left=True))[0] == 1
    # run routes: one more than Join, the total of max(cnt, 1)
    sj, sl = _syncs(lambda: runs.join(six, "k"))[0], _syncs(lambda: runs.join(six, "k", left=True))[0]
    assert sl == sj + 1 and sj == 3, (sj, sl)
    # no match at all: the probe readback only; an empty index likewise
    none_k = cp.Table.from_rows(ctx, [{"k": "zz", "q": "1"}], ["k", "q"])
    assert _syncs(lambda: none_k.join(six, "k", left=True))[0] == 1
    # every probe row matching once: Join's result on Join's kernels, with the same synchronisations
    for t, ix, cols in ((all_match, rix, ["cust_id"]), (all_match.slice(0, 2500), rix, ["cust_id"])):
        (sj, j), st_j = _with_stats(lambda: _syncs(lambda: t.join(ix, *cols)))
        (sl, l), st_l = _with_stats(lambda: _syncs(lambda: t.join(ix, *cols, left=True)))
        assert sj == sl and {k: v["launches"] for k, v in st_j.items()} == {k: v["launches"] for k, v in st_l.items()}
        assert _trows(j) == _trows(l)
    one_t = cp.Table.from_rows(ctx, [{"k": "k%d" % i, "v": "v%d" % i} for i in range(500)], ["k", "v"])
    oix = one_t.index_on("k")
    probe1 = cp.Table.from_rows(ctx, [{"k": "k%d" % ((i * 7) % 500), "q": "%d" % i} for i in range(2000)], ["k", "q"])
    probe1.join(oix, "k")
    (sj, j), st_j = _with_stats(lambda: _syncs(lambda: probe1.join(oix, "k")))
    (sl, l), st_l = _with_stats(lambda: _syncs(lambda: probe1.join(oix, "k", left=True)))
    assert sj == sl and {k: v["launches"] for k, v in st_j.items()} == {k: v["launches"] for k, v in st_l.items()}
    assert _trows(j) == _trows(l)


# ------------------------------------------------------------------ 7. the 4 GiB column limit
def test_result_column_limit_on_both_sides():
    from tests import result_limits_ref as R
    from tests.test_gpu_result_limits import _flush, _refused, _table
    M = R.MIB
    # index side: one index row of 2^20 + 1 bytes matched by 4096 probe rows, beside a probe row that misses
    ix_t = _table({"k": [(1, b"1")], "v": [(1, b"a" * (M + 1))]})
    probe = _table({"k": [(4096, b"1"), (1, b"9")]})
    ix = ix_t.index_on("k")
    assert len(probe.slice(0, 1).join(ix, "k", left=True)) == 1
    assert 4096 * (M + 1) > R.LIMIT
    _refused(lambda: probe.join(ix, "k", left=True))
    del ix, ix_t, probe
    _flush()
    # probe side: one probe row of 2^20 + 1 bytes matching 4096 index rows, beside a probe row that misses
    probe = _table({"k": [(1, b"1"), (1, b"9")], "p": [(1, b"a" * (M + 1)), (1, b"b")]})
    ix_t = _table({"k": [(4096, b"1")]})
    ix = ix_t.index_on("k")
    _refused(lambda: probe.join(ix, "k", left=True))
    del ix, ix_t, probe
    _flush()


# ------------------------------------------------------------------ 8. the C++ example
def test_cpp_left_join_example():
    exe = os.path.join(ROOT, "host", "left_join_example")
    if not os.path.exists(exe):
        import __graft_entry__ as g
        g.build()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "left join example ok" in r.stdout
    assert "unknown customer" in r.stdout and "unknown product" in r.stdout
