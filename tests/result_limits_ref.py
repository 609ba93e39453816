"""Exact result sizes in plain Python ints, for tables given as runs of identical rows, and a restatement of the 32-bit
sums the length scan kept before its total was exact.

A table is a list of runs (count, row): `count` copies of `row`, a tuple of bytes values, one per output column (a
column named twice in a ToCsv call appears twice).  Sizes are computed per run, so a multi-GiB table costs a few
lines of arithmetic; tests/test_result_limits_cpu.py checks every function against the full serialisers on small
tables.  Written from the rules of encoding/csv, encoding/json and the scan's tiling, not from the product code."""
from __future__ import annotations

import zlib

import numpy as np

from tests import json_oracle as jo

SCAN_THREADS, SCAN_ITEMS = 256, 16
SCAN_TILE = SCAN_THREADS * SCAN_ITEMS
LIMIT = (1 << 32) - 1  # the most bytes one result (a column, a ToCsv body) may hold: its offsets are 32-bit

# unicode.IsSpace of a rune that is not ASCII
_SPACE_RUNES = {0x85, 0xA0, 0x1680, 0x2028, 0x2029, 0x202F, 0x205F, 0x3000} | set(range(0x2000, 0x200B))


def _first_rune_is_space(v: bytes) -> bool:
    if v[0] < 0x80:
        return v[0] in b" \t\n\v\f\r"
    for k in (2, 3, 4):  # utf8.DecodeRune: the one valid sequence at the start, else RuneError (not a space)
        try:
            return ord(v[:k].decode("utf-8")) in _SPACE_RUNES
        except UnicodeDecodeError:
            continue
    return False


def csv_field(v: bytes) -> bytes:
    """encoding/csv.Writer's field: quoted when non-empty and `\\.`, or holding , " \\r \\n, or led by a space rune"""
    if v and (v == b"\\." or any(c in v for c in b',"\r\n') or _first_rune_is_space(v)):
        return b'"' + v.replace(b'"', b'""') + b'"'
    return v


def csv_field_len(v: bytes) -> int:
    """len(csv_field(v)) without building it"""
    if v and (v == b"\\." or any(v.find(bytes([c])) >= 0 for c in b',"\r\n') or _first_rune_is_space(v)):
        return len(v) + v.count(b'"') + 2
    return len(v)


def csv_row_len(row: tuple) -> int:
    """bytes of one ToCsv line: the fields, the commas between them and the newline"""
    return sum(csv_field_len(v) for v in row) + len(row)


def csv_header_len(names: list) -> int:
    return csv_row_len(tuple(n.encode() if isinstance(n, str) else n for n in names))


def csv_body_size(runs: list) -> int:
    """the ToCsv body (every line, no header) of a table given as runs"""
    return sum(count * csv_row_len(row) for count, row in runs)


def csv_body_chunks(runs: list):
    """the ToCsv body, one line at a time"""
    for count, row in runs:
        line = b",".join(csv_field(v) for v in row) + b"\n"
        for _ in range(count):
            yield line


def json_row_len(names: list, row: tuple, first: bool) -> int:
    """bytes of one ToJSON row of a table with columns `names`: ',' (or '[' for the first), the object, '\\n'"""
    return len(json_row(names, row, first))


def json_row(names: list, row: tuple, first: bool) -> bytes:
    order = sorted(range(len(names)), key=lambda k: names[k])
    return (b"[" if first else b",") + b"{" + b",".join(jo.enc(names[k]) + b":" + jo.enc(row[k]) for k in order) + b"}\n"


def json_body_size(names: list, runs: list, first: bool = True) -> int:
    """the ToJSON body of one call (every row with its leading '[' or ','; not the closing ']')"""
    total, lead = 0, first
    for count, row in runs:
        if count == 0:
            continue
        a, b = json_row_len(names, row, lead), json_row_len(names, row, False)
        total += a + (count - 1) * b
        lead = False
    return total


def json_document_chunks(names: list, runs: list):
    """the whole ToJSON document, one row at a time"""
    lead = True
    for count, row in runs:
        if count == 0:
            continue
        yield json_row(names, row, lead)
        rest = json_row(names, row, False) if count > 1 else b""
        for _ in range(count - 1):
            yield rest
        lead = False
    yield b"[]" if lead else b"]"


def gathered_size(lengths, ids) -> int:
    """bytes of a column gathered by row ids from a column whose values have these lengths"""
    lengths = np.asarray(lengths, dtype=np.int64)
    return int(lengths[np.asarray(ids, dtype=np.int64)].sum()) if len(ids) else 0


def crc_of(chunks) -> tuple:
    """(bytes, CRC-32) of a stream of chunks"""
    n, crc = 0, 0
    for c in chunks:
        n += len(c)
        crc = zlib.crc32(c, crc)
    return n, crc


# ---- the length scan's sums, as its 32-bit version kept them
def run_lengths(runs_of_lengths: list) -> np.ndarray:
    """the per-item values of a scan given as runs (count, value)"""
    return np.concatenate([np.full(c, v, dtype=np.uint64) for c, v in runs_of_lengths]) if runs_of_lengths \
        else np.zeros(0, np.uint64)


def scan_total_u32(values: np.ndarray) -> int:
    """the total the scan reported when each thread's 16 items, each warp's inclusive scan and each tile's sum of the 8
    warp totals were uint32 (only the chain across tiles 64-bit): the sum of every tile's total modulo 2^32"""
    v = np.asarray(values, dtype=np.uint64)
    pad = (-len(v)) % SCAN_TILE
    v = np.concatenate([v, np.zeros(pad, np.uint64)]).reshape(-1, SCAN_THREADS // 32, 32, SCAN_ITEMS)
    m = np.uint64(0xFFFFFFFF)
    thread = v.sum(axis=3) & m                      # a thread's 16 items
    warp = thread.sum(axis=2) & m                   # lane 31 of the warp's inclusive scan
    tile = warp.sum(axis=1) & m                     # the tile total handed to the look-back
    return int(tile.sum())


def scan_wrap_level(values: np.ndarray) -> str | None:
    """the first level at which an exact sum passes 2^32 - 1: 'thread', 'warp', 'tile', or None (no tile wraps; the
    total may still exceed it)"""
    v = np.asarray(values, dtype=np.uint64)
    pad = (-len(v)) % SCAN_TILE
    v = np.concatenate([v, np.zeros(pad, np.uint64)]).reshape(-1, SCAN_THREADS // 32, 32, SCAN_ITEMS)
    thread = v.sum(axis=3)
    if (thread > LIMIT).any():
        return "thread"
    if (thread.sum(axis=2) > LIMIT).any():
        return "warp"
    if (thread.sum(axis=(1, 2)) > LIMIT).any():
        return "tile"
    return None


def csv_row_len_u32(row: tuple) -> int:
    """a ToCsv line's length as a uint32 sum without saturation"""
    return csv_row_len(row) & 0xFFFFFFFF


# ---- the GPU shapes of tests/test_gpu_result_limits.py, as runs of one column's values (ToCsv names the column
# `times` times, so each row of the size functions holds the value that many times)
MIB = 1 << 20


def x(n: int) -> bytes:
    return b"x" * n


def scan_shapes() -> dict:
    """name -> (runs of (count, value), times, the level at which the old 32-bit sums wrap or None): size-only ToCsv
    calls that put the wrap of the row-length scan at each level"""
    tile_rows = lambda long: [r for w in range(8) for r in ([(1, x(1 << 28)), (511, b"")] if w < long else [(512, b"")])]
    return {
        "thread": ([(16, x(1 << 26))], 4, "thread"),            # 16 rows of 2^28 + 4 bytes in one thread's items
        "thread_fits": ([(15, x(1 << 26))], 4, None),
        "warp": ([(17, x((1 << 26) - 16))], 4, "warp"),         # no thread reaches 2^32, its first two lanes do
        "tile": (tile_rows(8), 2, "tile"),                      # one 2^29-byte row in each of the 8 warps
        "tile_fits": (tile_rows(7), 2, None),
        "tile_then_more": ([(2049, x(MIB + 1)), (10_000, b"yyyyyyy")], 2, "tile"),
        "no_tile_wraps": ([(3 * SCAN_TILE, x(1 << 17))], 4, None),  # 6.4 GB in tiles of 2 GiB each
    }


def repeated(runs: list, times: int) -> list:
    """runs of one column -> runs of rows that name it `times` times"""
    return [(c, (v,) * times) for c, v in runs]
