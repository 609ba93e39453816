"""The exact result sizes of tests/result_limits_ref.py against the full serialisers (the oracle's ToCsv, the restated
encoder of tests/json_oracle.py, a gather by row ids) on random small tables, so that they are a valid reference at GB
sizes; and the GPU shapes of tests/test_gpu_result_limits.py against the restated 32-bit sums, so that each shape
keeps wrapping where its test says it does."""
import random

import numpy as np
import pytest

from oracle import oracle as orc
from tests import json_oracle as jo
from tests import result_limits_ref as R

# values that exercise every quoting and escaping rule of both writers
_PIECES = [b"", b"a", b"plain", b",", b'"', b'""x', b"\r", b"\n", b" lead", b"\t", b"\\.", b"\\.x", b"\xc2\x85x", b"\xc2\xa0",
           b"\xe1\x9a\x80", b"\xe2\x80\x8a", b"\xe2\x80\xa8", b"\xe2\x80\xa9", b"\xe3\x80\x80", b"\xe2\x80\x8b", b"\x01", b"\x7f",
           b"\xff", b"\xc3", b"\xed\xa0\x80", b"\xf0\x9f\x98\x80", b"<&>", b"\\"]


def _value(rng):
    return b"".join(rng.choice(_PIECES) for _ in range(rng.choice([0, 1, 1, 2, 5])))


def _table(seed, nrows, ncols):
    rng = random.Random(seed)
    names = [("c%d" % k).encode() if rng.random() < 0.7 else _value(rng) + b"%d" % k for k in range(ncols)]
    return names, [tuple(_value(rng) for _ in range(ncols)) for _ in range(nrows)]


def _runs(rows):
    """rows -> runs of identical consecutive rows"""
    runs = []
    for r in rows:
        if runs and runs[-1][1] == r:
            runs[-1] = (runs[-1][0] + 1, r)
        else:
            runs.append((1, r))
    return runs


@pytest.mark.parametrize("seed", range(12))
def test_csv_sizes_match_the_oracle(seed):
    names, rows = _table(seed, nrows=random.Random(seed).choice([1, 2, 17, 300]), ncols=1 + seed % 4)
    rows = rows[:1] * 3 + rows  # a run of identical rows
    names = [n.decode("latin-1") for n in names]
    if len(set(names)) != len(names) or any(not n for n in names):
        names = ["c%d" % k for k in range(len(names))]
    t = orc.take_rows([{n: r[k] for k, n in enumerate(names)} for r in rows])
    # the columns in a different order, one of them twice
    cols = names[::-1] + names[:1]
    order = [names.index(c) for c in cols]
    want, err = t.to_csv(*cols)
    assert err is None
    crows = [tuple(r[k] for k in order) for r in rows]
    header = R.csv_header_len(cols)
    assert header + R.csv_body_size(_runs(crows)) == len(want)
    assert b"".join(R.csv_body_chunks(_runs(crows))) == want[header:]
    for r in crows:
        assert R.csv_row_len(r) == len(b",".join(R.csv_field(v) for v in r) + b"\n")


def test_csv_field_rules():
    assert [R.csv_field(v) for v in (b"", b"a", b"\\.", b"\\.x", b'a"b', b" a", b"\xc2\xa0a", b"\xc2\xa1a", b"\xe2\x80\x8ba",
                                     b"\xe2\x80\x8aa", b"\xc3", b"a,b")] == \
        [b"", b"a", b'"\\."', b"\\.x", b'"a""b"', b'" a"', b'"\xc2\xa0a"', b"\xc2\xa1a", b"\xe2\x80\x8ba", b'"\xe2\x80\x8aa"',
         b"\xc3", b'"a,b"']
    for v in (b'"' * 1000, b"x" * 1000 + b"\n"):
        assert R.csv_field_len(v) == len(R.csv_field(v))


@pytest.mark.parametrize("seed", range(12))
def test_json_sizes_match_the_encoder(seed):
    rng = random.Random(100 + seed)
    names, rows = _table(100 + seed, nrows=rng.choice([1, 2, 9, 250]), ncols=1 + seed % 5)
    if len(set(names)) != len(names):
        names = [b"c%d" % k for k in range(len(names))]
    rows = rows + rows[-1:] * 4
    runs = _runs(rows)
    for first, last in ((True, True), (True, False), (False, False), (False, True)):
        doc = jo.columns_document(names, [[r[k] for r in rows] for k in range(len(names))], first, last)
        assert R.json_body_size(names, runs, first) + (1 if last else 0) == len(doc)
    assert b"".join(R.json_document_chunks(names, runs)) == jo.document([dict(zip(names, r)) for r in rows])
    # the row layout of one call: '[' or ',', the object, '\n'
    assert R.json_row(names, rows[0], True) == jo.columns_document(names, [[v] for v in rows[0]], True, False)
    assert R.json_row(names, rows[0], False) == jo.columns_document(names, [[v] for v in rows[0]], False, False)
    assert b"".join(R.json_document_chunks(names, [])) == jo.document([])


@pytest.mark.parametrize("seed", range(6))
def test_gathered_size_matches_a_gather(seed):
    rng = random.Random(200 + seed)
    values = [_value(rng) * rng.randrange(1, 40) for _ in range(rng.randrange(1, 60))]
    ids = [rng.randrange(len(values)) for _ in range(rng.randrange(0, 500))]
    assert R.gathered_size([len(v) for v in values], ids) == len(b"".join(values[i] for i in ids))


def test_crc_of_chunks():
    import zlib
    parts = [b"abc", b"", b"\x00" * 1000, b"z"]
    assert R.crc_of(parts) == (1004, zlib.crc32(b"".join(parts)))


def test_scan_restatement_on_small_values():
    """without a wrap, the 32-bit sums equal the exact total; the total wraps by tile, not by the whole scan"""
    rng = np.random.default_rng(5)
    v = rng.integers(0, 1 << 20, size=3 * R.SCAN_TILE + 77, dtype=np.uint64)
    assert R.scan_total_u32(v) == int(v.sum()) and R.scan_wrap_level(v) is None
    w = np.zeros(2 * R.SCAN_TILE, np.uint64)
    w[0] = w[1] = 1 << 31  # one thread's two items: 2^32
    w[R.SCAN_TILE] = 5
    assert R.scan_wrap_level(w) == "thread" and R.scan_total_u32(w) == 5
    w[1] = 0; w[R.SCAN_ITEMS] = 1 << 31  # the next thread of the same warp
    assert R.scan_wrap_level(w) == "warp" and R.scan_total_u32(w) == 5
    w[R.SCAN_ITEMS] = 0; w[32 * R.SCAN_ITEMS] = 1 << 31  # the next warp of the same tile
    assert R.scan_wrap_level(w) == "tile" and R.scan_total_u32(w) == 5
    w[32 * R.SCAN_ITEMS] = 0; w[R.SCAN_TILE + 1] = 1 << 31  # the next tile: exact
    assert R.scan_wrap_level(w) is None and R.scan_total_u32(w) == int(w.sum()) == (1 << 32) + 5


@pytest.mark.parametrize("name", list(R.scan_shapes()))
def test_gpu_scan_shapes_wrap_where_stated(name):
    """every size-only ToCsv shape of the GPU tests wraps at its level under the old sums (so it would have reported a
    wrong size), and a shape without a wrap has the size its test expects"""
    runs, times, level = R.scan_shapes()[name]
    rows = R.repeated(runs, times)
    lens = R.run_lengths([(c, R.csv_row_len(r)) for c, r in rows])
    body = R.csv_body_size(rows)
    assert int(lens.sum()) == body
    assert R.scan_wrap_level(lens) == level
    if level is not None:
        assert body > R.LIMIT and R.scan_total_u32(lens) < R.LIMIT  # the old size passed the 4 GiB check
    else:
        assert R.scan_total_u32(lens) == body
    assert sum(c * len(v) for c, v in runs) < 1 << 32  # the source column itself fits


def test_gpu_limit_shapes():
    """the ToCsv, ToJSON and gather shapes of the GPU tests: their exact sizes on both sides of 2^32 - 1, and the sizes
    the 32-bit sums reported for the shapes that wrap"""
    M = R.MIB
    # ToCsv: 2049 rows of 2^20 + 1 bytes written as "a","a" wrap one tile (the parent's size-only answer 2 105 352)
    rows = R.repeated([(2049, R.x(M + 1))], 2)
    lens = R.run_lengths([(c, R.csv_row_len(r)) for c, r in rows])
    assert R.csv_header_len(["a", "a"]) + R.csv_body_size(rows) == 4_297_072_648
    assert R.csv_header_len(["a", "a"]) + R.scan_total_u32(lens) == 2_105_352
    # ToCsv: one row of 2^30 quotes written as "a","a": the row is 2^32 + 6 bytes, a uint32 sum says 6 (10 with the header)
    row = (b'"' * (1 << 30),) * 2
    assert R.csv_row_len(row) == (1 << 32) + 6 and R.csv_row_len_u32(row) + R.csv_header_len(["a", "a"]) == 10
    # ToCsv bodies of 2^32 - 1 and 2^32 bytes in 4096 rows (one tile; the second wraps to 0 under the old sums)
    for last, body in ((1_044_479, R.LIMIT), (1_044_480, R.LIMIT + 1)):
        runs = [(4095, (R.x(M),)), (1, (R.x(last),))]
        assert R.csv_body_size(runs) == body
        assert R.scan_total_u32(R.run_lengths([(c, R.csv_row_len(r)) for c, r in runs])) == body & R.LIMIT
    # ToJSON of one column "a": 10 bytes per row besides the value; bodies of 2^32 - 2 and 2^32 - 1 bytes
    assert R.json_row_len([b"a"], (b"v",), True) == R.json_row_len([b"a"], (b"v",), False) == 11
    for last, body in ((1_007_614, R.LIMIT - 1), (1_007_615, R.LIMIT)):
        assert R.json_body_size([b"a"], [(4095, (R.x(M),)), (1, (R.x(last),))]) == body
    # ToJSON: 700 rows of 2^20 bytes 0x01 (each escaped to \u0001) wrap one tile
    jruns = [(700, (b"\x01" * M,))]
    jlens = R.run_lengths([(699, R.json_row_len([b"a"], (b"\x01" * M,), False)), (1, 0)])
    assert R.json_body_size([b"a"], jruns) == 700 * (6 * M + 10) > R.LIMIT
    assert R.scan_wrap_level(jlens) == "tile"
    # gathers: 4097 copies of a 2^20 + 1-byte value wrap one tile; 4095 of them and one of 1 044 480 bytes are 2^32 - 1
    assert R.gathered_size([M + 1], [0] * 4097) == 4097 * (M + 1) > R.LIMIT
    assert R.scan_total_u32(R.run_lengths([(4097, M + 1)])) == 1_052_673
    assert R.gathered_size([M + 1, 1_044_480], [0] * 4095 + [1]) == R.LIMIT
    assert R.gathered_size([M + 1, 1_044_481], [0] * 4095 + [1]) == R.LIMIT + 1
