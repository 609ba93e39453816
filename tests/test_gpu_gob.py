"""Index.WriteTo / LoadIndex (csvplus.go:655-705) on the GPU against the restatement of encoding/gob in
tests/gob_oracle.py: files the GPU writes decode to the index's key columns and rows in index order; files the oracle
writes (random pair order per row, other type ids and definition orders, adversarial values) load as the rows in file
order, and Find / Join / Except on the loaded index behave as the reference's binary searches over those rows
(indexImpl.find / first / has, csvplus.go:870-905), sorted or not."""
import os
import random
import subprocess
import zlib

import pytest

from tests import gob_oracle as g
from tests.index_ref import find as ref_find, join as ref_join
from tests.helpers import gpu_ctx, people_csv

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _rows(ix):
    """the index's rows in its stored order, as {bytes: bytes}"""
    t = ix.table()
    cols = t.columns
    vals = {c: t.values(c) for c in cols}
    return [{c.encode("utf-8", "surrogateescape"): vals[c][i] for c in cols} for i in range(len(t))]


def _written(ix, tmp_path, name="ix.gob"):
    p = str(tmp_path / name)
    ix.WriteTo(p)
    with open(p, "rb") as f:
        return f.read()


def _check_write(ix, tmp_path):
    data = _written(ix, tmp_path)
    keys, rows = g.decode_index(data)
    assert keys == [c.encode() for c in ix.columns]
    assert rows == _rows(ix)
    # the bytes are exactly the restatement's (pairs in bytewise name order)
    assert data == g.encode_index(keys, rows)
    return data


def _table(rows, columns=None):
    import csvplus_b200 as cp
    return cp.Table.from_rows(gpu_ctx(), rows, columns)


def test_write_unique_nonunique_multikey_sub(tmp_path):
    import csvplus_b200 as cp
    data = people_csv(3000, seed=5)
    src = lambda: cp.Take(cp.FromBytes(data).SelectColumns("id", "name", "surname", "born"))
    _check_write(src().UniqueIndexOn("id"), tmp_path)
    _check_write(src().IndexOn("surname"), tmp_path)
    ix3 = src().IndexOn("surname", "name", "born")
    _check_write(ix3, tmp_path)
    _check_write(ix3.SubIndex("Smith"), tmp_path)
    _check_write(ix3.SubIndex("Smith", "Amelia"), tmp_path)


def test_resolve_duplicates_with_replacement_out_of_key_order(tmp_path):
    """a replacement row that sorts elsewhere leaves the stored rows out of key order (csvplus.go:846 does not re-sort):
    WriteTo keeps that order, and Find / Join / Except search those rows as the reference's binary searches do"""
    import csvplus_b200 as cp
    rng = random.Random(4)
    rows = [{"k": "key%02d" % rng.randrange(30), "v": str(i)} for i in range(400)]
    ix = cp.TakeRows(rows).IndexOn("k")
    ix.ResolveDuplicates(lambda grp: {"k": "z" + grp[0]["k"] if grp[0]["k"] < "key10" else grp[0]["k"], "v": str(len(grp))})
    data = _check_write(ix, tmp_path)
    keys, frows = g.decode_index(data)
    assert [r[b"k"] for r in frows] != sorted(r[b"k"] for r in frows)
    stored, cols = _rows(ix), [b"k"]
    for v in ("key03", "key15", "zkey03", "key29", "a", "zz", ""):
        assert ix.Find(v).ToRows() == _s(ref_find(stored, cols, [v.encode()])), v
    probe = [{b"k": k, b"p": b"%d" % i} for i, k in enumerate(sorted({r[b"k"] for r in stored} | {b"key05", b"zkey99", b"0"}))]
    assert cp.TakeRows(_s(probe)).Join(ix).ToRows() == _s(ref_join(stored, cols, probe, cols))
    assert cp.TakeRows(_s(probe)).Except(ix).ToRows() == _s(ref_join(stored, cols, probe, cols, anti=True))


def test_write_empty_and_byte_values_and_sizes(tmp_path):
    import csvplus_b200 as cp
    _check_write(_table([], ["a", "b"]).index_on("a"), tmp_path)
    allb = bytes(range(256))
    rows = [{"k": (allb[i:] + allb[:i]).decode("utf-8", "surrogateescape"), "v": allb[::-1].decode("utf-8", "surrogateescape")} for i in range(256)]
    _check_write(cp.TakeRows(rows).IndexOn("k"), tmp_path)
    rng = random.Random(2)
    sizes = [0, 1, 127, 128, 255, 256, 65535, 65536, 70000]
    rows = [{"k": "%06d" % i, "v": "x" * sizes[i % len(sizes)]} for i in range(300)]
    _check_write(cp.TakeRows(rows).IndexOn("k"), tmp_path)
    for n in (127, 128, 255, 256, 65535, 65536, 70000):  # multi-byte row counts
        rows = [{"k": str(rng.randrange(1000)), "c": "v"} for _ in range(n)]
        _check_write(cp.TakeRows(rows).IndexOn("k"), tmp_path)


def test_write_in_batches(tmp_path, monkeypatch):
    import csvplus_b200 as cp
    from csvplus_b200 import api
    rows = [{"k": str(i % 97), "v": "val%d" % i} for i in range(5000)]
    ix = cp.TakeRows(rows).IndexOn("k")
    whole = _written(ix, tmp_path, "whole.gob")
    monkeypatch.setattr(api, "GOB_BATCH_ROWS", 333)
    assert _written(ix, tmp_path, "batched.gob") == whole


class _Digest:
    def __init__(self):
        self.n, self.crc = 0, 0

    def update(self, path):
        with open(path, "rb") as f:
            while True:
                b = f.read(1 << 26)
                if not b:
                    return self
                self.n += len(b)
                self.crc = zlib.crc32(b, self.crc)


def test_rows_message_above_4_gib(tmp_path, monkeypatch):
    """a rows message above 4 GiB: WriteTo halves a batch of 4 GiB or more (CPB_E_TOO_LARGE), the prefix declares the
    64-bit message length, and LoadIndex decodes the body in windows with 64-bit positions; the loaded index writes the
    same bytes again"""
    import csvplus_b200 as cp
    from csvplus_b200 import api
    ctx = gpu_ctx()
    n = 66_000_000
    raw = ctx.gen_csv("orders", (0, n), n_cust=n // 10, n_prod=1000)
    t, err = cp.parse_csv(ctx, raw, spec=[("order_id", -1), ("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)])
    raw.free()
    assert err is None and len(t) == n
    ix = t.index_on("cust_id")
    del t
    monkeypatch.setattr(api, "GOB_BATCH_ROWS", n)  # the first batch is above 4 GiB and gets halved
    p1 = str(tmp_path / "big1.gob")
    ix.WriteTo(p1)
    size = os.path.getsize(p1)
    with open(p1, "rb") as f:
        head = f.read(4096)
    i = 0
    for _ in range(4):  # []string def, columns, []Row def, Row def
        b = g._Buf(head[i:])
        i += b.uint() + b.i
    b = g._Buf(head[i:])
    body = b.uint()
    assert body > 1 << 32 and i + b.i + body == size
    assert b.int() == g.ID_ROWS and b.uint() == 0 and b.uint() == n
    assert g.decode_stream(head[:i]) == [[b"cust_id"]]
    d1 = _Digest().update(p1)
    ix2 = cp.LoadIndex(p1)
    os.remove(p1)
    assert len(ix2) == n and ix2.columns == ["cust_id"]
    assert ix2.Find("4242").ToRows() == ix.Find("4242").ToRows()
    del ix
    p2 = str(tmp_path / "big2.gob")
    ix2.WriteTo(p2)
    assert _Digest().update(p2).__dict__ == d1.__dict__
    os.remove(p2)


# ------------------------------------------------------------------ LoadIndex
def _s(rows):
    return [{k.decode(): v.decode() for k, v in r.items()} for r in rows]


def _load(data, tmp_path, name="in.gob"):
    import csvplus_b200 as cp
    p = str(tmp_path / name)
    with open(p, "wb") as f:
        f.write(data)
    return cp.LoadIndex(p)


@pytest.mark.parametrize("sort_rows", [True, False])
def test_load_random_pair_order(tmp_path, sort_rows):
    import csvplus_b200 as cp
    rng = random.Random(7 + sort_rows)
    cols = [b"k1", b"k2"]
    rows = [{b"k1": b"%d" % rng.randrange(20), b"k2": b"%d" % rng.randrange(5), b"v": b"row%d" % i, b"w": b"x" * rng.randrange(200)}
            for i in range(3000)]
    if sort_rows:
        rows.sort(key=lambda r: (r[b"k1"], r[b"k2"]))
    for ids, first in (((65, 66, 67), False), ((80, 70, 90), True)):
        data = g.encode_index(cols, rows, order=g.random_order(3), ids=ids, row_def_first=first)
        ix = _load(data, tmp_path)
        assert ix.columns == ["k1", "k2"] and len(ix) == len(rows)
        assert _rows(ix) == rows
        got = []
        ix.Iterate(got.append)
        assert got == _s(rows)
        for vals in ([], [b"3"], [b"3", b"1"], [b"19", b"4"], [b"nope"], [b""], [b"99"]):
            assert ix.Find(*[v.decode() for v in vals]).ToRows() == _s(ref_find(rows, cols, vals)), vals
        probe = [{b"k1": b"%d" % rng.randrange(25), b"k2": b"%d" % rng.randrange(6), b"p": b"%d" % i} for i in range(500)]
        sprobe = _s(probe)
        assert cp.TakeRows(sprobe).Join(ix).ToRows() == _s(ref_join(rows, cols, probe, cols))
        assert cp.TakeRows(sprobe).Join(ix, "k1").ToRows() == _s(ref_join(rows, cols, probe, cols[:1]))
        assert cp.TakeRows(sprobe).Except(ix).ToRows() == _s(ref_join(rows, cols, probe, cols, anti=True))
        # and written back as it was loaded (pairs now in bytewise order)
        assert _written(ix, tmp_path) == g.encode_index(cols, rows, ids=(65, 66, 67))


def test_index_store_round_trip(tmp_path):
    """TestIndexStore (csvplus_test.go:960-1014) on people.csv, and the pinned file of tests/golden/"""
    import csvplus_b200 as cp
    ix = cp.Take(cp.FromFile(os.path.join(GOLDEN, "people.csv")).SelectColumns("id", "name", "surname")).IndexOn("id")
    with open(os.path.join(GOLDEN, "people_index.gob"), "rb") as f:
        golden = f.read()
    assert _written(ix, tmp_path) == golden
    ix2 = cp.LoadIndex(str(tmp_path / "ix.gob"))
    assert ix2.columns == ix.columns
    assert cp.Take(ix2).ToRows() == cp.Take(ix).ToRows()
    assert ix2.Find("7").ToRows() == ix.Find("7").ToRows()


def test_adversarial_values(tmp_path):
    """values holding whole encoded rows (and the row header) put spurious candidates into the body that chain into true
    rows; the decode still follows the true rows only"""
    rng = random.Random(9)
    cols = [b"a"]
    rows = []
    for i in range(4000):
        fake = g.enc_row([(b"a", b"%d" % i), (b"b", b"fake")]) * rng.randrange(0, 4)
        fake += g.enc_row([(b"b", b"y"), (b"a", b"z")])[: rng.randrange(0, 9)]
        rows.append({b"a": b"%05d" % i, b"b": fake + bytes([2]) + g.enc_str(b"a")})
    data = g.encode_index(cols, rows, order=g.random_order(5))
    ix = _load(data, tmp_path)
    assert _rows(ix) == rows


def test_load_errors(tmp_path):
    import csvplus_b200 as cp
    with pytest.raises(FileNotFoundError):
        cp.LoadIndex(str(tmp_path / "missing.gob"))
    good = g.encode_index([b"id"], [{b"id": b"%d" % i, b"n": b"x%d" % i} for i in range(100)])
    with pytest.raises(cp.CsvPlusError, match="^EOF$"):
        _load(b"", tmp_path)
    first_two = len(g.message(g.slice_def(65, g.STRING))) + len(g.message(g.enc_int(65) + b"\0" + g.enc_uint(1) + g.enc_str(b"id")))
    with pytest.raises(cp.CsvPlusError, match="^EOF$"):  # ends between messages before the rows
        _load(good[:first_two], tmp_path)
    for cut in (1, 5, first_two + 3, len(good) - 1, len(good) - 40):
        with pytest.raises(cp.CsvPlusError, match="^unexpected EOF$"):
            _load(good[:cut], tmp_path)
    # wrong types: the columns as []int, the rows as []string
    bad1 = g.message(g.slice_def(65, 2)) + g.message(g.enc_int(65) + b"\0" + g.enc_uint(1) + g.enc_int(5))
    bad2 = g.message(g.slice_def(65, g.STRING)) + g.message(g.enc_int(65) + b"\0" + g.enc_uint(1) + g.enc_str(b"id"))
    bad2 += bad2[len(g.message(g.slice_def(65, g.STRING))):]
    for bad in (bad1, bad2):
        with pytest.raises(cp.CsvPlusError, match="type mismatch"):
            _load(bad, tmp_path)
    # rows with differing column sets, a row with a name twice, a key column the rows lack, a count that lies
    for rows in ([{b"id": b"1", b"n": b"a"}, {b"id": b"2", b"m": b"b"}], [{b"id": b"1", b"n": b"a"}, {b"id": b"2"}]):
        with pytest.raises(cp.CsvPlusError):
            _load(g.encode_index([b"id"], rows), tmp_path)
    twice = g.encode_index([b"id"], [{b"id": b"1", b"n": b"a"}, {b"id": b"2", b"n": b"b"}],
                           order=lambda r: [(b"id", r[b"id"]), (b"id", r[b"n"])] if r[b"id"] == b"2" else sorted(r.items()))
    with pytest.raises(cp.CsvPlusError):
        _load(twice, tmp_path)
    with pytest.raises(cp.CsvPlusError, match="key column"):
        _load(g.encode_index([b"zz"], [{b"id": b"1"}]), tmp_path)
    body = g.enc_int(67) + b"\0" + g.enc_uint(3) + g.enc_row([(b"id", b"1")]) + g.enc_row([(b"id", b"2")])
    lie = good[:good.index(g.message(g.slice_def(67, 66)))] + g.message(g.slice_def(67, 66)) + g.message(g.map_def(b"Row", 66, 6, 6)) + g.message(body)
    with pytest.raises(cp.CsvPlusError):
        _load(lie, tmp_path)
    # the context is still usable after every refusal
    assert len(_load(good, tmp_path)) == 100


def test_write_unwritable_path_leaves_no_file(tmp_path):
    import csvplus_b200 as cp
    ix = cp.TakeRows([{"k": "1"}]).IndexOn("k")
    bad = tmp_path / "no" / "such" / "dir" / "ix.gob"
    with pytest.raises(OSError):
        ix.WriteTo(str(bad))
    assert not bad.exists()


def test_cpp_gob_example():
    exe = os.path.join(ROOT, "host", "gob_example")
    if not os.path.exists(exe):
        import __graft_entry__ as ge
        ge.build()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "gob example ok" in r.stdout
