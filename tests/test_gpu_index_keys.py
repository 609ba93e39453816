"""IndexOn / UniqueIndexOn / Find / SubIndex / Join / Except / ResolveDuplicates against the C++ oracle and against
tests/index_ref.py (the plain-Python indexImpl), on the shapes where the index code takes different routes:

a. every probe table of a join (join.cu: smem, global, unique16, run32, the row-carrying table), at key images of 8 to
   25 bytes in one column or split over several, long key columns (widths 0, 254, 255, 256), 16 384 / 16 385 distinct
   prefixes and awkward probe values; every case asserts the route it took from the kernel statistics;
b. the radix sort over several tiles per block (a partial last tile, constant words and digits skipped, heavy ties,
   0x00 / 0xff bytes), and UniqueIndexOn's duplicate error at that size;
c. indexes whose stored rows are out of key order (LoadIndex of an unsorted file, ResolveDuplicates storing rows whose
   keys sort elsewhere): Take, Find, SubIndex, Join, Except and ResolveDuplicates exactly as the reference's binary
   searches over those rows;
d. the limits: 16 key columns and a 4096-byte key image.

Key columns are built as numpy offsets and bytes, so values such as b"a" and b"a\\0" are exact, and reach the GPU from
torch tensors through Table.from_device_columns."""
import ctypes as C
import random
import zlib
from dataclasses import dataclass, field

import numpy as np
import pytest

from oracle import oracle as orc
from tests import gob_oracle as g
from tests import hash_ref as hr
from tests import index_ref as ref
from tests.helpers import assert_table_equals_oracle, gpu_ctx

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ fixtures
def _columns(values: dict) -> dict:
    """{name: list[bytes]} -> {name: (offsets int64[n+1], bytes uint8[])}"""
    out = {}
    for nm, vals in values.items():
        off = np.zeros(len(vals) + 1, np.int64)
        if vals:
            off[1:] = np.cumsum([len(v) for v in vals])
        out[nm] = (off, np.frombuffer(b"".join(vals), np.uint8))
    return out


def _device_table(cols: dict):
    """a device table of {name: (offsets, bytes)}, fed from torch tensors"""
    import torch

    import csvplus_b200 as cp
    ctx = gpu_ctx()
    dev = torch.device("cuda", ctx.device)
    names = list(cols)
    keep, ptrs = [], []
    for nm in names:
        off, data = cols[nm]
        to = torch.from_numpy(off.astype(np.int32)).to(dev)  # (uint32 offsets: every column here is far below 2 GiB)
        td = torch.from_numpy(np.concatenate([data, np.zeros(1, np.uint8)])).to(dev)
        keep += [to, td]
        ptrs.append((to.data_ptr(), td.data_ptr()))
    torch.cuda.synchronize(dev)
    t = cp.Table.from_device_columns(ctx, names, ptrs, len(cols[names[0]][0]) - 1)
    ctx.sync()
    return t


def _both(values: dict):
    """the same columns as a device table and as oracle rows"""
    cols = _columns(values)
    return _device_table(cols), orc.take_columns(cols)


def _trows(t) -> list:
    """a device table's rows as {bytes: bytes}"""
    vals = {c: t.values(c) for c in t.columns}
    return [{c.encode(): vals[c][i] for c in t.columns} for i in range(len(t))]


def _find(ix, vals):
    """Index.Find as a device table"""
    import csvplus_b200 as cp
    from csvplus_b200.api import _strs
    a, keep = _strs(vals)
    h = C.c_void_p()
    assert ix.ctx.lib.cpb_index_find(ix.ctx.h, ix.h, a, len(vals), C.byref(h)) == 0
    return cp.Table(ix.ctx, h)


def _with_stats(fn):
    ctx = gpu_ctx()
    ctx.sync()
    ctx.stats(enable=True, reset=True)
    r = fn()
    ctx.sync()
    st = ctx.stats()
    ctx.stats(enable=False)
    return r, st


def _s(rows):
    return [{k.decode("utf-8", "surrogateescape"): v.decode("utf-8", "surrogateescape") for k, v in r.items()} for r in rows]


def _b(rows):
    return [{k.encode("utf-8", "surrogateescape"): v.encode("utf-8", "surrogateescape") for k, v in r.items()} for r in rows]


# ------------------------------------------------------------------ the probe table a join takes (join.cu)
def _hash_build_bytes(kind, nheads, pbytes):  # join.cu: ensure_hash's hash_build record
    b = nheads * (pbytes + 8)
    if kind in ("unique16", "run32"):
        b += hr.probe_slots(kind, nheads) * (16 if kind == "unique16" else 32)
    return b


def _rowhash_fits(unique, n, widths, pay_lens):  # sort.cu: build_index, the row-carrying table's limits
    """pay_lens: per row, the lengths of its non-key columns"""
    return unique and n >= 2 and hr.image_bytes(widths) <= 12 and len(pay_lens[0]) <= 4 and max(map(sum, pay_lens)) <= 16


def _check_route(st, kind, nheads, pbytes):
    if kind == "rowhash":
        assert "rowhash_probe" in st or "rowhash_flags" in st, sorted(st)
        assert "hash_build" not in st and "join_search" not in st, sorted(st)
        return
    assert "rowhash_probe" not in st and "rowhash_flags" not in st and "join_search" not in st, sorted(st)
    hb = st.get("hash_build")
    assert hb is not None and hb["launches"] == 1, sorted(st)
    assert hb["algo_bytes"] == _hash_build_bytes(kind, nheads, pbytes), (kind, nheads, pbytes, hb)


BYTES = np.frombuffer(b"\x00\xff\x00\xffa\x01\x7f\x80", np.uint8)


def _value(rng, w, full=False):
    n = w if full else int(rng.integers(0, w + 1))
    if rng.random() < 0.5:
        return BYTES[rng.integers(0, len(BYTES), n)].tobytes()
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def _distinct_keys(rng, widths, d):
    keys = [tuple(_value(rng, w, full=True) for w in widths)]  # one key at the full width of every column
    seen = set(keys)
    while len(keys) < d:
        k = tuple(_value(rng, w) for w in widths)
        if k not in seen:
            seen.add(k)
            keys.append(k)
    return keys


@dataclass
class Case:
    name: str
    widths: list            # key column widths (longest value)
    d: int                  # distinct full keys
    n: int                  # rows (n > d: duplicates)
    route: str              # the route of the full-key join
    unique: bool = False    # UniqueIndexOn
    pay: list = field(default_factory=lambda: [4])  # payload columns: longest value of each
    lead_unique: bool = False  # the first key column alone is already unique (a prefix join on it sees runs of 1)


CASES = [
    Case("img8_smem", [7], 3000, 5000, "smem"),
    Case("img8_split_run32", [3, 3], 17000, 22000, "run32"),
    Case("img12_unique16", [11], 20000, 20000, "unique16"),
    Case("img12_split_unique16", [5, 5], 20000, 20000, "unique16"),
    Case("img13_run32", [12], 20000, 20000, "run32"),
    Case("img13_split_word_run32", [7, 4], 20000, 20000, "run32"),
    Case("img16_split_run32", [7, 7], 18000, 24000, "run32"),
    Case("img24_run32", [23], 17000, 20000, "run32"),
    Case("img24_split_word8_run32", [7, 15], 17000, 20000, "run32"),
    Case("img24_split3_run32", [3, 3, 15], 17000, 20000, "run32"),
    Case("img25_global", [24], 17000, 20000, "global"),
    Case("img25_split_word16_global", [7, 16], 17000, 20000, "global"),
    Case("img25_split_midword_global", [11, 12], 17000, 20000, "global"),
    Case("heads16384_smem", [7], 16384, 20000, "smem"),
    Case("heads16385_run32", [7], 16385, 20000, "run32"),
    Case("heads16384_long_smem", [24], 16384, 20000, "smem"),
    Case("heads16385_long_global", [24], 16385, 20000, "global"),
    Case("width0", [0], 1, 300, "smem"),
    Case("width0_then_key", [0, 6], 500, 900, "smem"),
    Case("width254", [254], 400, 700, "smem"),
    Case("width255", [255], 400, 700, "smem"),
    Case("width256", [256, 3], 400, 700, "smem"),
    Case("unique16_on_prefix", [7, 5], 20000, 20000, "run32", lead_unique=True),
    Case("unique_unique16", [11], 20000, 20000, "unique16", unique=True, pay=[2, 2, 2, 2, 2]),
    Case("unique_smem", [7], 3000, 3000, "smem", unique=True, pay=[6, 6, 6]),
    Case("unique_run32", [9, 4], 20000, 20000, "run32", unique=True),
    Case("rowhash_pay16", [11], 20000, 20000, "rowhash", unique=True, pay=[4, 4, 4, 4]),
    Case("rowhash_pay17", [11], 20000, 20000, "unique16", unique=True, pay=[5, 4, 4, 4]),
    Case("rowhash_small", [3, 3], 50, 50, "rowhash", unique=True, pay=[16]),
]


def test_matrix_covers_every_route():
    assert {c.route for c in CASES} == {"smem", "global", "unique16", "run32", "rowhash"}


def _case_data(case):
    rng = np.random.default_rng(zlib.crc32(case.name.encode()))
    keys = _distinct_keys(rng, case.widths, case.d)
    if case.lead_unique:  # the first column unique on its own
        firsts = {k[0] for k in keys}
        keys = list({k[0]: k for k in keys}.values())
        while len(keys) < case.d:
            k = tuple(_value(rng, w) for w in case.widths)
            if k[0] not in firsts:
                firsts.add(k[0])
                keys.append(k)
    rows = keys + [keys[int(i)] for i in rng.integers(0, len(keys), case.n - len(keys))]
    rows = [rows[i] for i in rng.permutation(len(rows))]
    knames = ["k%d" % j for j in range(len(case.widths))]
    values = {nm: [r[j] for r in rows] for j, nm in enumerate(knames)}
    full = int(rng.integers(0, len(rows)))  # the row whose payload columns are all at their longest
    for j, w in enumerate(case.pay):
        col = [_value(rng, w) for _ in rows]
        col[full] = b"p" * w
        values["v%d" % j] = col
    pay_lens = [tuple(len(values["v%d" % j][i]) for j in range(len(case.pay))) for i in range(len(rows))]
    # probe rows: stored keys, stored keys with a trailing \0 or cut short, values longer than the width, empty values
    probe = []
    for q in range(3000):
        k = list(rows[int(rng.integers(0, len(rows)))])
        u = rng.random()
        j = int(rng.integers(0, len(k)))
        if u < 0.15:
            k[j] = k[j] + b"\x00"
        elif u < 0.25:
            k[j] = k[j][:-1]
        elif u < 0.32:
            k[j] = k[j] + b"\xff" * (case.widths[j] + 1 - len(k[j]))  # one byte over the width
        elif u < 0.36:
            k = [b""] * len(k)
        elif u < 0.45:
            k = [_value(rng, w) for w in case.widths]
        probe.append(k)
    pnames = ["p%d" % j for j in range(len(case.widths))]
    pvalues = {nm: [p[j] for p in probe] for j, nm in enumerate(pnames)}
    pvalues["q"] = [b"%d" % i for i in range(len(probe))]
    return rows, knames, values, pay_lens, pnames, pvalues


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_probe_routes(case):
    rows, knames, values, pay_lens, pnames, pvalues = _case_data(case)
    n, K = len(rows), len(knames)
    it, ot = _both(values)
    ix, st_build = _with_stats(lambda: it.index_on(*knames, unique=case.unique))
    rowhash = _rowhash_fits(case.unique, n, case.widths, pay_lens)
    assert ("rowhash_build" in st_build) == rowhash, sorted(st_build)
    oi = ot.index_on(*knames, unique=case.unique)
    full = _both(pvalues)
    # (a prefix over a narrow column has long runs, the empty value's above all: fewer probe rows keep those joins small)
    part = _both({nm: v[:400] for nm, v in pvalues.items()})
    probe_keys = list(zip(*[pvalues[p] for p in pnames]))
    for nk in [K] + list(range(1, K)):
        pt, op = full if nk == K else part
        nheads = len({r[:nk] for r in rows})
        pbytes = hr.image_bytes(case.widths[:nk])
        if rowhash and nk == K:
            kind = "rowhash"
        else:
            if case.unique and nk == K:
                nheads = n  # a unique index probed on its full key: every row is its own run, in source order
            kind = hr.probe_kind(nheads, pbytes, n)
        if nk == K:
            assert kind == case.route, (case.name, kind, nheads, pbytes)  # the shape lands where the case says
        if case.lead_unique and nk == 1:
            assert kind == "unique16"
        j, st = _with_stats(lambda: pt.join(ix, *pnames[:nk]))
        # a unique index builds its full-key table when it checks the keys
        _check_route({**st_build, **st} if nk == K else st, kind, nheads, pbytes)
        assert_table_equals_oracle(j, op.join(oi, *pnames[:nk]))
        assert_table_equals_oracle(pt.join(ix, *pnames[:nk], anti=True), op.except_(oi, *pnames[:nk]))
        for k in probe_keys[:12]:
            assert_table_equals_oracle(_find(ix, list(k[:nk])), oi.find(*k[:nk]))
    assert_table_equals_oracle(ix.table(), oi.rows())


def test_one_row_index_and_empty_probe():
    for unique in (False, True):
        it, ot = _both({"k": [b"a\x00"], "v": [b"x"]})
        ix, oi = it.index_on("k", unique=unique), ot.index_on("k", unique=unique)
        pt, op = _both({"p": [b"a", b"a\x00", b"a\x00\x00", b"", b"b"], "q": [b"0", b"1", b"2", b"3", b"4"]})
        assert_table_equals_oracle(pt.join(ix, "p"), op.join(oi, "p"))
        assert_table_equals_oracle(pt.join(ix, "p", anti=True), op.except_(oi, "p"))
        e, _ = _both({"p": [], "q": []})
        assert len(e.join(ix, "p")) == 0 and len(e.join(ix, "p", anti=True)) == 0
        for v in (b"a", b"a\x00", b""):
            assert_table_equals_oracle(_find(ix, [v]), oi.find(v))


# ------------------------------------------------------------------ the sort over several tiles per block (sort.cu)
def test_sort_at_scale_and_unique_error():
    import torch
    sm = torch.cuda.get_device_properties(gpu_ctx().device).multi_processor_count
    n = 3 * 4 * sm * 2048 + 777  # tiles per block >= 3, the last tile partial
    rng = np.random.default_rng(11)
    pool0 = [_value(rng, 7) for _ in range(1500)] + [b"\x00" * 7, b"\xff" * 7, b"", b"\x00", b"\xff"]
    pool2 = [_value(rng, 9) for _ in range(40)] + [b"\x00" * 9, b"\xff" * 9]
    i0 = rng.integers(0, len(pool0), n)
    i2 = rng.integers(0, len(pool2), n)
    k0 = [pool0[i] for i in i0]
    k2 = [pool2[i] for i in i2]
    k1 = [b"CONSTANT-11"] * n  # bytes 8..19 of the image: the second word is constant and skipped whole
    rid = [b"%d" % i for i in range(n)]
    cols = _columns({"k0": k0, "k1": k1, "k2": k2, "i": rid})
    t = _device_table(cols)
    ix, st = _with_stats(lambda: t.index_on("k0", "k1", "k2"))
    words = (hr.image_bytes([7, 11, 9]) + 7) // 8
    assert words == 4 and st["sort_hist"]["launches"] == words
    assert st["sort_gather_word"]["launches"] == words - 1
    perm = sorted(range(n), key=lambda i: (k0[i], k1[i], k2[i]))  # index_ref.index_on: a stable sort on the key tuple
    got = ix.table()
    assert got.values("i") == [rid[i] for i in perm]
    assert got.values("k0") == [k0[i] for i in perm]
    assert got.values("k2") == [k2[i] for i in perm]
    del ix, got
    # UniqueIndexOn of that size with duplicates: it sorts to name the lowest duplicate key
    import csvplus_b200 as cp
    keys = [b"%08d" % i for i in rng.permutation(n)]
    a, b, c, d = (int(x) for x in rng.choice(n, 4, replace=False))
    keys[b] = keys[a]
    keys[d] = keys[c]
    low = min(keys[a], keys[c])
    tu = _device_table(_columns({"key": keys}))
    with pytest.raises(cp.CsvPlusError) as e:
        _with_stats(lambda: tu.index_on("key", unique=True))
    assert str(e.value) == "duplicate value while creating unique index: " + ref.row_string({b"key": low}).decode()


# ------------------------------------------------------------------ indexes whose rows are out of key order
def _load(rows, cols, tmp_path, name="ix.gob"):
    import csvplus_b200 as cp
    p = str(tmp_path / name)
    with open(p, "wb") as f:
        f.write(g.encode_index(cols, rows))
    return cp.LoadIndex(p)


def _probe_rows(rng, stored, cols, pnames, m):
    out = []
    for i in range(m):
        r = rng.choice(stored) if stored else {c: b"" for c in cols}
        vals = [r[c] for c in cols]
        if rng.random() < 0.2:
            vals[-1] += b"\x00"
        if rng.random() < 0.1:
            vals = [b"zz%d" % rng.randrange(9) for _ in cols]
        out.append({**{pn: v for pn, v in zip(pnames, vals)}, b"q": b"%d" % i})
    return out


def _check_out_of_order(ix, stored, cols, rng):
    """Take, Find, SubIndex (and Take / Find / Join on it), Join and Except of the index against index_ref over `stored`,
    with probe columns named unlike the index columns, on the full key and every prefix"""
    assert _trows(ix.table()) == stored
    K = len(cols)
    in_key_order = all([a[c] for c in cols] <= [b[c] for c in cols] for a, b in zip(stored, stored[1:]))
    pnames = [b"p_" + c for c in cols]
    probe = _probe_rows(rng, stored, cols, pnames, 400)
    pt = _device_table(_columns({k.decode(): [p[k] for p in probe] for k in probe[0]}))
    for nk in range(1, K + 1):
        pn = [p.decode() for p in pnames[:nk]]
        j, st = _with_stats(lambda: pt.join(ix, *pn))
        if not in_key_order:  # (rows that are in key order may take either route)
            assert "join_search" in st and "hash_build" not in st, sorted(st)
        assert _trows(j) == ref.join(stored, cols, probe, pnames[:nk]), nk
        assert _trows(pt.join(ix, *pn, anti=True)) == ref.except_(stored, cols, probe, pnames[:nk]), nk
        for r in rng.sample(stored, min(5, len(stored))) + [{c: b"zz" for c in cols}]:
            vals = [r[c] for c in cols[:nk]]
            assert _trows(_find(ix, vals)) == ref.find(stored, cols, vals), vals
    if K >= 2:
        for r in rng.sample(stored, min(4, len(stored))):
            v = [r[cols[0]]]
            sub = ix.SubIndex(*v)
            srows, scols = ref.sub_index(stored, cols, v)
            assert _trows(sub.table()) == srows
            if not srows:
                continue
            for s in rng.sample(srows, min(3, len(srows))):
                assert _trows(_find(sub, [s[scols[0]]])) == ref.find(srows, scols, [s[scols[0]]])
            sprobe = _probe_rows(rng, srows, scols, [b"s_" + c for c in scols], 50)
            spt = _device_table(_columns({k.decode(): [p[k] for p in sprobe] for k in sprobe[0]}))
            assert _trows(spt.join(sub, *["s_" + c.decode() for c in scols])) == ref.join(srows, scols, sprobe, [b"s_" + c for c in scols])


def _resolve_both(ix, stored, cols, resolver):
    """ResolveDuplicates on the GPU and in index_ref with the same resolver; the groups each was handed must agree"""
    seen_gpu, seen_ref = [], []

    def on_gpu(grp):
        seen_gpu.append(_b(grp))
        r = resolver(_b(grp))
        return None if r is None else _s([r])[0]

    def on_ref(grp):
        seen_ref.append(list(grp))
        return resolver(grp)

    ix.ResolveDuplicates(on_gpu)
    want, _ = ref.dedup(stored, cols, on_ref)
    assert seen_gpu == seen_ref
    assert _trows(ix.table()) == want
    return want


def test_worked_example_join_copies_index_keys(tmp_path):
    """stored keys [a, d, c], probe pk = d: the reference joins rows d and c, each with its own k"""
    import csvplus_b200 as cp
    rows = [{b"k": k, b"v": b"%d" % i} for i, k in enumerate([b"a", b"d", b"c"])]
    ix = _load(rows, [b"k"], tmp_path)
    got = cp.TakeRows([{"pk": "d"}]).Join(ix, "pk").ToRows()
    assert got == [{"k": "d", "v": "1", "pk": "d"}, {"k": "c", "v": "2", "pk": "d"}]


def test_worked_example_dedup_group_by_search(tmp_path):
    """stored keys [b, b, a, c]: the reference resolves [b, b, a] and keeps only the new row b'"""
    rows = [{b"k": k, b"v": b"%d" % i} for i, k in enumerate([b"b", b"b", b"a", b"c"])]
    ix = _load(rows, [b"k"], tmp_path)
    want = _resolve_both(ix, rows, [b"k"], lambda grp: {b"k": b"b'", b"v": b"x"})
    assert want == [{b"k": b"b'", b"v": b"x"}]


def test_sub_index_keeps_stored_order(tmp_path):
    import csvplus_b200 as cp
    rows = [{b"a": b"1", b"b": b"z", b"v": b"0"}, {b"a": b"1", b"b": b"c", b"v": b"1"}, {b"a": b"2", b"b": b"a", b"v": b"2"}]
    ix = _load(rows, [b"a", b"b"], tmp_path)
    sub = ix.SubIndex("1")
    assert _trows(sub.table()) == rows[:2]
    assert cp.Take(sub).ToRows() == _s(rows[:2])
    assert sub.Find("c").ToRows() == _s(ref.find(rows[:2], [b"b"], [b"c"]))


@pytest.mark.parametrize("shuffle", ["full", "partial"])
def test_loaded_out_of_order(tmp_path, shuffle):
    rng = random.Random(5 if shuffle == "full" else 6)
    cols = [b"k1", b"k2"]
    n = 20000
    rows = [{b"k1": b"%d" % rng.randrange(300), b"k2": rng.choice([b"", b"\x00", b"a", b"a\x00", b"\xff", b"b"]), b"v": b"%d" % i}
            for i in range(n)]
    if shuffle == "full":
        rng.shuffle(rows)
    else:  # sorted, then a few blocks moved
        rows.sort(key=lambda r: (r[b"k1"], r[b"k2"]))
        for _ in range(20):
            a = rng.randrange(n - 50)
            blk = rows[a:a + rng.randrange(1, 50)]
            del rows[a:a + len(blk)]
            b = rng.randrange(len(rows))
            rows[b:b] = blk
    ix = _load(rows, cols, tmp_path)
    _check_out_of_order(ix, rows, cols, rng)
    for resolver in (lambda grp: grp[0], lambda grp: None, lambda grp: {**grp[-1], b"k1": b"~" + grp[-1][b"k1"]}):
        ix = _load(rows, cols, tmp_path)
        after = _resolve_both(ix, rows, cols, resolver)
        _check_out_of_order(ix, after, cols, rng)


def _move(grp):
    """a third of the groups get a key that sorts before every other, a third the key of the next group (so that runs of
    equal keys form again, out of key order), the rest keep their second row"""
    k = grp[0][b"k"]
    h = int(k[3:]) % 3
    if h == 0:
        return {b"k": b"a" + k, b"v": b"%d" % len(grp)}
    if h == 1:
        return {b"k": b"key%03d" % (int(k[3:]) + 1), b"v": b"%d" % len(grp)}
    return grp[1]


def test_resolve_duplicates_out_of_order():
    """ResolveDuplicates storing rows whose keys sort elsewhere, every operation on the result, then a second
    ResolveDuplicates (first / drop / new-row resolvers) on those rows out of key order"""
    rng = random.Random(8)
    cols = [b"k"]
    rows = [{b"k": b"key%03d" % rng.randrange(400), b"v": b"%d" % i} for i in range(20000)]
    it, _ = _both({"k": [r[b"k"] for r in rows], "v": [r[b"v"] for r in rows]})
    stored = ref.index_on(rows, cols)

    def moved():
        ix = it.index_on("k")
        assert _trows(ix.table()) == stored
        return ix, _resolve_both(ix, stored, cols, _move)

    ix, once = moved()
    assert [r[b"k"] for r in once] != sorted(r[b"k"] for r in once)
    _check_out_of_order(ix, once, cols, rng)
    for resolver in (lambda grp: grp[0], lambda grp: None, lambda grp: {b"k": grp[0][b"k"] + b"!", b"v": b"n"}):
        ix, _ = moved()
        twice = _resolve_both(ix, once, cols, resolver)
        _check_out_of_order(ix, twice, cols, rng)


# ------------------------------------------------------------------ limits
def test_sixteen_key_columns():
    import csvplus_b200 as cp
    rng = random.Random(3)
    values = {"c%02d" % j: [rng.choice([b"", b"a", b"b", b"\x00"]) for _ in range(3000)] for j in range(17)}
    it, ot = _both(values)
    keys = sorted(values)
    ix = it.index_on(*keys[:16])
    oi = ot.index_on(*keys[:16])
    assert_table_equals_oracle(ix.table(), oi.rows())
    assert_table_equals_oracle(it.join(ix, *keys[:16]), ot.join(oi, *keys[:16]))
    with pytest.raises(cp.CsvPlusError) as e:
        it.index_on(*keys)
    assert e.value.status == 4  # CPB_ERR_UNSUPPORTED
    assert_table_equals_oracle(it.join(ix, *keys[:3], anti=True), ot.except_(oi, *keys[:3]))


def test_key_image_4096_bytes():
    import csvplus_b200 as cp
    w = 4096 - 2  # the value and its 2-byte length fill 512 image words exactly
    vals = [b"x" * w, b"x" * (w - 1) + b"\x00", b"x" * (w - 1), b"", b"x" * w]
    it, ot = _both({"k": vals, "v": [b"%d" % i for i in range(len(vals))]})
    ix, oi = it.index_on("k"), ot.index_on("k")
    assert_table_equals_oracle(ix.table(), oi.rows())
    pt, op = _both({"p": vals + [b"x" * (w + 1)], "q": [b"%d" % i for i in range(len(vals) + 1)]})
    assert_table_equals_oracle(pt.join(ix, "p"), op.join(oi, "p"))
    too = _device_table(_columns({"k": vals + [b"y" * (w + 1)]}))
    with pytest.raises(cp.CsvPlusError) as e:
        too.index_on("k")
    assert e.value.status == 4  # CPB_ERR_UNSUPPORTED
    # the context is still usable
    assert_table_equals_oracle(pt.join(ix, "p", anti=True), op.except_(oi, "p"))
    assert_table_equals_oracle(it.index_on("v", unique=True).table(), ot.unique_index_on("v").rows())
