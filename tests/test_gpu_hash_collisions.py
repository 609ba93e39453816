"""The GPU hash tables under keys built to collide, against their references bit for bit.

Both keyhash.cuh tables promise that a hash is never taken as equality, and every join table that its probe walks a
chain to the first empty slot, wrapping from the last slot to slot 0.  Random keys never test either: no two of them
share a 64-bit hash, and few chains cross the table's end.  tests/hash_ref.py inverts the value hash, so here
thousands of distinct values share one full hash (2^64 - 1 starts in the last slot of every power-of-two table; 0 is
the empty value's), GroupBy rows share the chained row hash while their columns do not, and join keys are aimed by
search at the last slot of the table their index builds:

1. the restatement against the device: tests/hash_harness.cu, built from the kernels' headers, hashes a crafted corpus
   and random values of every length 0..520 at every start misalignment; no mismatch is allowed;
2. codes (codes.cu) against tests/codes_ref.py: short, empty and long (warp-compared) values in one chain, repeated
   across warps, and the all-distinct route;
3. GroupBy (groupby.cu) against tests/groupby_ref.py, every op and kind: column-0 and row-level collisions in one push,
   in many pushes while the persistent table doubles, and through a streamed CSV;
4. Join, Except and LeftJoin on each probe table (smem, global, unique16, run32) against tests/index_ref.py and
   tests/left_join_ref.py, and a Filter on a large Like set against tests/pred_ref.py.

Every case asserts through hash_ref that its collisions or its wrap exist at the table size the kernel uses."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

from tests import hash_ref as hr
from tests import index_ref as ref
from tests.codes_ref import factorize
from tests.helpers import gpu_ctx
from tests.test_gpu_codes import _check as check_codes
from tests.test_gpu_codes import _table, _upload
from tests.test_gpu_groupby import ALL_AGGS, SPECIAL_FLOATS
from tests.test_gpu_groupby import _check as check_groups
from tests.test_gpu_index_keys import _both, _check_route, _trows, _with_stats
from tests.test_gpu_left_join import _check as check_left_join

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "csvplus_b200", "csrc")
M = hr.MASK
M1 = hr.row_target(M)  # the value hash of a one-column GroupBy key whose row hash is 2^64 - 1


# ------------------------------------------------------------------ 1. the restatement is the kernels' code
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    from csvplus_b200 import build
    d = tmp_path_factory.mktemp("hash_harness")
    exe = str(d / "hash_harness")
    r = subprocess.run([build.NVCC, *build.FLAGS, "-I", CSRC, os.path.join(HERE, "hash_harness.cu"), "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr

    def run(values, ks, mis, keys, widths, nslots):
        """device hashes: per value (thread, warp, row) and per key row (w0, w1, w2, hash3 x2, slot_of x2, hash_prefix)"""
        blob, recs = bytearray(), []
        for v, k, m in zip(values, ks, mis):
            pos = -(-len(blob) // 8) * 8 + m
            blob += b"\0" * (pos - len(blob)) + v
            recs.append((pos, len(v), k))
        out = [np.array([len(values), len(blob)], "<u8").tobytes(), np.array(recs, dtype=[("o", "<u8"), ("l", "<u4"), ("k", "<u4")]).tobytes(),
               bytes(blob)]
        pbytes = hr.image_bytes(widths)
        nwords = (pbytes + 7) // 8
        out.append(np.array([len(widths)], "<u4").tobytes() + np.array([len(keys), nslots], "<u8").tobytes()
                   + np.array([pbytes, nwords], "<u4").tobytes())
        for j, w in enumerate(widths):
            col = [key[j] for key in keys]
            off = np.zeros(len(col) + 1, "<u4")
            np.cumsum([len(v) for v in col], out=off[1:])
            out.append(np.array([w, hr.len_bytes(w)], "<u4").tobytes() + np.array([off[-1]], "<u8").tobytes() + off.tobytes() + b"".join(col))
        img = np.array([hr.image_words(hr.key_image(key, widths), nwords) for key in keys], "<u8").reshape(len(keys), nwords)
        out.append(np.ascontiguousarray(img.T).tobytes())
        with open(d / "in.bin", "wb") as f:
            f.write(b"".join(out))
        r = subprocess.run([exe, str(d / "in.bin"), str(d / "out.bin")], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stdout + r.stderr
        res = np.fromfile(d / "out.bin", "<u8")
        nv = 3 * len(values)
        return res[:nv].reshape(-1, 3), res[nv:].reshape(-1, 8)
    return run


def _mismatches(run, values, ks, mis, keys, widths, nslots):
    """the number of device hashes that differ from hash_ref's"""
    dv, dk = run(values, ks, mis, keys, widths, nslots)
    bad = 0
    for i, (v, k) in enumerate(zip(values, ks)):
        h = hr.value_hash(v)
        bad += (int(dv[i, 0]) != h) + (int(dv[i, 1]) != h) + (int(dv[i, 2]) != hr.row_hash(values[i - k:i + 1]))
    pbytes = hr.image_bytes(widths)
    for r, key in enumerate(keys):
        ws = hr.image_words(hr.key_image(key, widths), max(3, (pbytes + 7) // 8))
        h3, h2 = hr.hash3(ws[0], ws[1], ws[2]), hr.hash3(ws[0], ws[1], 0)
        want = ws[:3] + [h3, h2, hr.slot_of(h3, nslots), hr.slot_of(h2, nslots), hr.hash_prefix(ws, pbytes)]
        got = [int(x) for x in dk[r]]
        if pbytes > 24:  # pack3 keeps the first 3 words only for images of up to 24 bytes: hash_prefix alone
            want, got = want[-1:], got[-1:]
        bad += sum(a != b for a, b in zip(got, want))
    return bad


def _corpus():
    """crafted values: every LENGTHS at hashes 2^64 - 1, 0 and another, the empty value, and crafted 2- and 3-column
    rows; with each value's column in its row chain"""
    vals, ks = [b""], [0]
    for H in (M, 0, 0x0123456789ABCDEF):
        for n in (8, 9, 15, 16, 128, 129, 136, 4097):
            for s in range(1 if n == 8 else 3):
                vals.append(hr.collide(H, n, (H, n, s)))
                ks.append(0)
    for lengths in ([5, 16], [0, 12], [3, 200, 9], [130, 1, 136]):
        for s in range(4):
            row = hr.collide_row(M, lengths, (tuple(lengths), s))
            vals += list(row)
            ks += list(range(len(row)))
    return vals, ks


def _key_shapes():
    """(widths, nslots, keys): every probe kind's key shape, with short, empty, full-width and over-width values"""
    rng = random.Random(9)
    out = []
    for widths, nslots in (([7], 8192), ([11], 40016), ([23], 25516), ([24], 65536), ([5, 5], 40016), ([3, 3, 15], 25516), ([254, 3], 64)):
        keys = [tuple(rng.randbytes(rng.choice([0, 1, w // 2, w, w, w + 1])) for w in widths) for _ in range(300)]
        out.append((widths, nslots, keys))
    return out


def test_harness_matches_hash_ref(harness):
    vals, ks = _corpus()
    assert {hr.value_hash(v) for v in vals[1:4]} == {M} and hr.value_hash(vals[0]) == 0
    total = 0
    for widths, nslots, keys in _key_shapes():
        total += _mismatches(harness, vals, ks, [i % 8 for i in range(len(vals))], keys, widths, nslots)
    # random values of every length 0..520 at all 8 start misalignments, chained in rows of 1 to 3 columns
    rng = random.Random(4)
    rvals, rks, rmis = [], [], []
    for n in range(521):
        for m in range(8):
            rvals.append(rng.randbytes(n))
            rks.append(len(rks) % 3)
            rmis.append(m)
    total += _mismatches(harness, rvals, rks, rmis, [], [7], 64)
    assert total == 0


# ------------------------------------------------------------------ 2. codes
def _short(H, count, seed, lo=10, hi=hr.LONG_BYTES, reject=b""):
    """count distinct values of lo..hi bytes hashing to H"""
    rng = random.Random(str(seed))
    out = {hr.collide(H, rng.randrange(lo, hi + 1), (seed, i), reject) for i in range(count)}
    assert len(out) == count
    return sorted(out)


def _long(H, count, seed, reject=b""):
    return _short(H, count, seed, hr.LONG_BYTES + 1, 600, reject)


def _codes_case(vals):
    codes, d = factorize(vals)
    check_codes(_table(vals), "v", codes, d)


def _assert_chain(values, H, n):
    """non-vacuity: every value hashes to H, and in the table over n rows they start at its last slot (more than one of
    them: the chain wraps into slot 0)"""
    nslots = hr.codes_slots(n)
    assert {hr.value_hash(v) for v in values} == {H}
    assert H & (nslots - 1) == nslots - 1 and hr.chain_crosses_end([H & (nslots - 1)] * len(values), nslots)


def test_codes_short_values_share_one_hash_across_warps():
    crafted = _short(M, 2000, 1)
    rng = random.Random(2)
    vals = crafted * 3 + [rng.randbytes(rng.randrange(0, 40)) for _ in range(6000)]
    rng.shuffle(vals)
    assert len(set(crafted)) == 2000
    _assert_chain(crafted, M, len(vals))
    _codes_case(vals)


def test_codes_zero_hash_with_the_empty_value():
    crafted = _short(0, 1000, 3)
    vals = [b""] * 50 + crafted * 2 + [b""] * 50
    random.Random(4).shuffle(vals)
    assert hr.value_hash(b"") == 0 and 0 & (hr.codes_slots(len(vals)) - 1) == 0
    assert {hr.value_hash(v) for v in crafted} == {0}
    _codes_case(vals)


def test_codes_long_and_short_values_in_one_chain():
    short, long_ = _short(M, 600, 5), _long(M, 200, 6)
    rng = random.Random(7)
    vals = (short + long_) * 2 + [rng.randbytes(rng.randrange(0, 300)) for _ in range(2000)]
    rng.shuffle(vals)
    _assert_chain(short + long_, M, len(vals))
    assert min(map(len, long_)) > hr.LONG_BYTES >= max(map(len, short))
    _codes_case(vals)


def test_codes_all_distinct_every_value_colliding():
    vals = _short(M, 1500, 8) + _long(M, 100, 9)
    random.Random(10).shuffle(vals)
    _assert_chain(vals, M, len(vals))
    _codes_case(vals)


# ------------------------------------------------------------------ 3. GroupBy
def _agg_values(rng, n):
    ints = [b"%d" % rng.randrange(-10 ** 6, 10 ** 6) for _ in range(n)]
    floats = [rng.choice(SPECIAL_FLOATS) if rng.random() < 0.05 else b"%.3f" % rng.uniform(-1e3, 1e3) for _ in range(n)]
    return ints, floats


def _group_rows(groups, nrows, seed):
    """(column names, columns) of nrows rows over the key tuples `groups` (each at least once, first appearances spread
    over the rows), with int and float aggregate inputs"""
    rng = random.Random(str(seed))
    gids = list(range(len(groups))) + [rng.randrange(len(groups)) for _ in range(nrows - len(groups))]
    rng.shuffle(gids)
    nk = len(groups[0])
    ints, floats = _agg_values(rng, nrows)
    names = ["k%d" % j for j in range(nk)] + ["i", "f"]
    cols = [[groups[g][j] for g in gids] for j in range(nk)] + [ints, floats]
    return names, cols


def _device(names, cols):
    up = {}
    for nm, vals in zip(names, cols):
        off = np.zeros(len(vals) + 1, np.int64)
        np.cumsum([len(v) for v in vals], out=off[1:])
        up[nm] = (off, np.frombuffer(b"".join(vals), np.uint8))
    return _upload(up, len(cols[0]))


def _rows(names, cols):
    return [dict(zip(names, vals)) for vals in zip(*cols)]


def _pushed(t, keys, aggs, step):
    """GroupBy of t through cpb_groups_push of consecutive slices of `step` rows"""
    import csvplus_b200 as cp
    from csvplus_b200 import _abi
    ctx = gpu_ctx()
    specs = cp.api._group_aggs(aggs)
    ka, kkeep = cp.api._strs(keys)
    arr = (_abi.Agg * len(specs))()
    keep = []
    for i, (op, column, kind) in enumerate(specs.values()):
        b = column.encode()
        keep.append(b)
        arr[i] = _abi.Agg(_abi.CPB_AGG_OPS[op], _abi.CPB_AGG_KINDS[kind], _abi.Str(b, len(b)))
    h = C.c_void_p()
    ctx._call("cpb_groups_open", ka, len(keys), arr, len(specs), C.byref(h))
    try:
        for lo in range(0, len(t), step):
            part = t.slice(lo, min(lo + step, len(t)))  # (held: the handle must outlive the push)
            ctx._call("cpb_groups_push", h, part.h)
        return cp.api._groups_result(ctx, h, specs)
    finally:
        ctx._call("cpb_groups_free", h)


def _column0_groups(seed, reject=b""):
    """1500 short and 150 long one-column keys sharing the value hash M1 (so the row hash 2^64 - 1), and 800 random ones"""
    rng = random.Random(str(seed))
    crafted = _short(M1, 1500, (seed, 1), reject=reject) + _long(M1, 150, (seed, 2), reject=reject)
    other = {bytes(rng.choice(b"abcxyz019") for _ in range(rng.randrange(0, 12))) for _ in range(800)}
    return crafted, [(v,) for v in crafted + sorted(other)]


def _row_groups(ncols, seed):
    """1200 rows of ncols key columns sharing the row hash 2^64 - 1 (the last column 10..40 or 136 bytes), 600 random"""
    rng = random.Random(str(seed))
    crafted = set()
    while len(crafted) < 1200:
        lengths = [rng.randrange(0, 6) for _ in range(ncols - 1)] + [rng.choice([136] + list(range(10, 41)))]
        crafted.add(hr.collide_row(M, lengths, (seed, len(crafted), rng.random())))
    other = {tuple(b"r%d" % rng.randrange(10 ** 6) for _ in range(ncols)) for _ in range(600)}
    return sorted(crafted), sorted(crafted) + sorted(other)


def _assert_row_collisions(crafted, ngroups, nrows):
    """non-vacuity: the crafted rows share one row hash while their columns do not, at the sizes of both tables"""
    assert len(crafted) >= 1000 and {hr.row_hash(r) for r in crafted} == {M}
    assert len({hr.value_hash(r[0]) for r in crafted}) > 1 or len(crafted[0]) == 1
    for nslots in (hr.groupby_slots(ngroups), hr.groupby_first_slots(nrows)):
        assert M & (nslots - 1) == nslots - 1


@pytest.mark.parametrize("how", ["one_push", "pushes"])
def test_groupby_column0_collisions(how):
    import csvplus_b200 as cp
    crafted, groups = _column0_groups(11)
    names, cols = _group_rows(groups, 20_000, 12)
    _assert_row_collisions([(v,) for v in crafted], len(groups), len(cols[0]))
    assert {hr.value_hash(v) for v in crafted} == {M1}
    t = _device(names, cols)
    g = cp.TakeTable(t).GroupBy(["k0"], ALL_AGGS) if how == "one_push" else _pushed(t, ["k0"], ALL_AGGS, 700)
    check_groups(g, ["k0"], ALL_AGGS, _rows(names, cols))


@pytest.mark.parametrize("ncols", [2, 3])
@pytest.mark.parametrize("how", ["one_push", "pushes"])
def test_groupby_row_collisions(ncols, how):
    import csvplus_b200 as cp
    crafted, groups = _row_groups(ncols, 20 + ncols)
    names, cols = _group_rows(groups, 15_000, 30 + ncols)
    _assert_row_collisions(crafted, len(groups), len(cols[0]))
    keys = names[:ncols]
    t = _device(names, cols)
    g = cp.TakeTable(t).GroupBy(keys, ALL_AGGS) if how == "one_push" else _pushed(t, keys, ALL_AGGS, 500)
    check_groups(g, keys, ALL_AGGS, _rows(names, cols))


def test_groupby_pushes_while_the_table_doubles():
    """the colliding groups arrive a few per push: the persistent table grows from 64 slots to 8192, its chain always
    crossing the last slot, and every later push probes it"""
    crafted = _short(M1, 1500, 40)
    assert {hr.row_hash([v]) for v in crafted} == {M}
    rng = random.Random(41)
    gids = []
    for g in range(len(crafted)):
        gids += [g] + [rng.randrange(g + 1) for _ in range(3)]
    names = ["k0", "i", "f"]
    ints, floats = _agg_values(rng, len(gids))
    cols = [[crafted[g] for g in gids], ints, floats]
    sizes = [hr.groupby_slots(n) for n in (10, 100, 1500)]
    assert sizes == [64, 256, 4096] and all(M & (s - 1) == s - 1 for s in sizes)
    g = _pushed(_device(names, cols), ["k0"], ALL_AGGS, 40)  # 10 new groups a push
    check_groups(g, ["k0"], ALL_AGGS, _rows(names, cols))


def test_groupby_streamed_csv(monkeypatch):
    import csvplus_b200 as cp
    from csvplus_b200 import api
    crafted, groups = _column0_groups(50, reject=b"\r")  # (a quoted CRLF reads back as LF)
    names, cols = _group_rows(groups, 12_000, 51)
    _assert_row_collisions([(v,) for v in crafted], len(groups), len(cols[0]))

    def q(v):
        return b'"' + v.replace(b'"', b'""') + b'"'
    csv = b"k0,i,f\n" + b"".join(b",".join(q(v) for v in row) + b"\n" for row in zip(*cols))
    monkeypatch.setattr(api, "STREAM_BATCH_BYTES", 64 << 10)
    src = cp.Take(cp.FromBytes(csv, gpu_ctx()))
    assert sum(1 for _ in src._batches()) > 5
    check_groups(src.GroupBy(["k0"], ALL_AGGS), ["k0"], ALL_AGGS, _rows(names, cols))


# ------------------------------------------------------------------ 4. the join probe tables
# (kind, key width, distinct keys, rows): test_gpu_index_keys' shapes, one key column, no row-carrying table
JOIN_SHAPES = [("smem", 7, 3000, 5000), ("global", 24, 17000, 20000), ("unique16", 11, 20000, 20000), ("run32", 23, 17000, 20000)]
AIMED, MISSES = 5, 3


def _aimed_keys(kind, width, d):
    """(aimed, misses, fillers): AIMED keys and MISSES other keys that all start at the last slot of the table over d
    distinct keys, and d - AIMED keys that start at none of its first 64 slots nor its last (so the aimed chain holds
    the last slot and slots 0 .. AIMED - 2, and the misses walk it to slot AIMED - 1)"""
    nslots = hr.probe_slots(kind, d)
    aimed, fill, base = [], [], 0
    while len(aimed) < AIMED + MISSES or len(fill) < d - AIMED:
        cand = [b"%0*d" % (width, base + i) for i in range(200_000)]
        base += len(cand)
        s = hr.np_probe_start(kind, cand, width, nslots)
        aimed += [cand[i] for i in np.flatnonzero(s == nslots - 1)]
        fill += [cand[i] for i in np.flatnonzero((s >= 64) & (s != nslots - 1))[: d - AIMED - len(fill)]]
    return aimed[:AIMED], aimed[AIMED:AIMED + MISSES], fill, nslots


@pytest.mark.parametrize("kind,width,d,n", JOIN_SHAPES, ids=[s[0] for s in JOIN_SHAPES])
def test_join_chain_wraps(kind, width, d, n):
    aimed, misses, fill, nslots = _aimed_keys(kind, width, d)
    keys = aimed + fill
    rng = random.Random(d)
    rows = keys + [rng.choice(keys) for _ in range(n - d - 2 * AIMED)] + (aimed * 2 if n > d else [])
    rows = rows[:n]
    rng.shuffle(rows)
    nheads = len(set(rows))
    pbytes = hr.image_bytes([width])
    # non-vacuity: the kind and table size the kernel uses, and a chain across slot nslots - 1
    assert nheads == d and hr.probe_kind(nheads, pbytes, len(rows)) == kind and hr.probe_slots(kind, nheads) == nslots
    assert all(hr.probe_start(kind, [k], [width], nslots) == nslots - 1 for k in aimed + misses)
    assert all(hr.probe_start(kind, [k], [width], nslots) >= 64 for k in fill[:50])
    assert set(aimed) <= set(rows) and not set(misses) & set(rows)
    assert hr.chain_crosses_end([nslots - 1] * AIMED, nslots)
    it, _ = _both({"k": rows, "v": [b"%d" % i for i in range(len(rows))]})
    ix = it.index_on("k")
    probe = aimed + misses + rng.sample(fill, 300) + [b"x" * width, b"", b"0" * (width + 1)]
    probe += aimed[::-1] + misses
    pt, _ = _both({"p": probe, "q": [b"%d" % i for i in range(len(probe))]})
    j, st = _with_stats(lambda: pt.join(ix, "p"))
    _check_route(st, kind, nheads, pbytes)
    stored, prows = _trows(ix.table()), _trows(pt)
    assert _trows(j) == ref.join(stored, [b"k"], prows, [b"p"])
    assert _trows(pt.join(ix, "p", anti=True)) == ref.except_(stored, [b"k"], prows, [b"p"])
    got, _ = check_left_join(pt, ix, ["p"], probe=prows, stored=stored)
    assert sum(1 for r in _trows(got) if r[b"k"] in aimed) >= AIMED  # every aimed key was found


def test_filter_on_an_aimed_like_set():
    from tests.pred_ref import holds
    from tests.test_gpu_pred_sets import check_table_and_parse
    nlits = 2000
    aimed, misses, fill, nslots = _aimed_keys("smem", 7, nlits)
    lits = aimed + fill
    assert hr.probe_kind(nlits, 8, nlits) == "smem" and hr.ordinal_slots(nlits) == nslots
    assert all(hr.probe_start("smem", [k], [7], nslots) == nslots - 1 for k in aimed + misses)
    rng = random.Random(60)
    ids = aimed * 3 + misses * 3 + rng.sample(fill, 500) + [b"%07d" % rng.randrange(10 ** 7) for _ in range(500)]
    rng.shuffle(ids)
    data = b"id,x\n" + b"".join(b"%s,%d\n" % (v, i) for i, v in enumerate(ids))
    tree = ("any", [("like", {b"id": v}) for v in lits])
    rows, want, _ = check_table_and_parse(data, tree)
    assert sum(1 for r in want if r[b"id"] in aimed) == 3 * AIMED and not any(r[b"id"] in misses for r in want)
    for r in [r for r in rows if r[b"id"] in aimed or r[b"id"] in misses][:6]:  # the membership shortcut is holds
        assert holds(tree, r) == (r[b"id"] in aimed)
