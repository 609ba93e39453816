"""A plain restatement of the fused parse's output sizing (csv_header_kernel's samples in parse_kernels.cuh and the
capacity estimate of run_scan in parse.cu), and builders of CSV inputs that land exactly on, or just past, the
capacities it predicts.

The header kernel samples three 64 KiB windows of the input: at byte 0, at n / 2 and at n - 64 KiB.  In each it counts
the '\\n' bytes of the 16-byte-aligned part, and 256 threads each split one line naively (quotes ignored): thread t
starts at lo + 256 t, skips to the byte after the next '\\n' within 4096 bytes, and splits the line that follows if it
ends within 4096 bytes; the bytes of every field that a delimiter or the '\\n' closes count, a line counts only when its
'\\n' is seen.  run_scan turns the samples into

    row_cap     = class_1MiB(min(body / avg * 1.1 + 4096, body / 2 + 2))
    data_cap[k] = min(body, 2^32 - 1, class_32MiB(row_cap * mean_k * 1.25 + 4 MiB))  (sampled fields < 64, >= 16 lines)

with the same double arithmetic in the same order: Python floats are IEEE doubles, so the caps agree bit for bit.
A first attempt whose rows or column bytes exceed these caps is rerun once at the exact size."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

TILE = 32768
WINDOW = 65536                # S of csv_header_kernel
SAMPLE_THREADS = 256          # the header kernel's block
LINE_LOOK = 4096              # how far a sampling thread looks for a line start, and then for its end
HDR_SAMPLE_FIELDS = 64
MIN_SAMPLED_LINES = 16
ROW_CLASS = 1 << 20
DATA_CLASS = 32 << 20
DATA_SLACK = 4 << 20
U32_MAX = 0xFFFFFFFF


@dataclass
class Sample:
    bytes: int                # aligned bytes the newline count covered (overlapping windows count again)
    newlines: int
    lines: int                # lines split to their '\n'
    field_bytes: list         # [HDR_SAMPLE_FIELDS] bytes of the fields closed in the split, per field index


@dataclass
class Caps:
    row_cap: int
    data_cap: list            # per selected field, in the order given


def windows(n: int) -> list:
    return [lo for lo in (0, n // 2, n - WINDOW if n > WINDOW else 0)]


def sample(data: bytes, delim: int = ord(",")) -> Sample:
    n = len(data)
    tot = nl = 0
    for lo in windows(n):
        hi = min(lo + WINDOW, n)
        lo16, hi16 = (lo + 15) & ~15, hi & ~15
        if lo16 < hi16:
            nl += data.count(b"\n", lo16, hi16)
            tot += hi16 - lo16
    lines, fb = 0, [0] * HDR_SAMPLE_FIELDS
    d = bytes([delim])
    for lo in windows(n):
        for t in range(SAMPLE_THREADS):
            p = lo + t * (WINDOW // SAMPLE_THREADS)
            lim = min(p + LINE_LOOK, n)
            j = data.find(b"\n", p, lim) if p < lim else -1
            if j < 0:
                continue        # no line start within reach
            p = j + 1
            if p >= n or p >= lim:
                continue
            lim = min(p + LINE_LOOK, n)
            e = data.find(b"\n", p, lim)
            seg = data[p:lim] if e < 0 else data[p:e]
            fields = seg.split(d)
            closed = fields if e >= 0 else fields[:-1]  # an unterminated line keeps the fields its delimiters closed
            for f, v in enumerate(closed[:HDR_SAMPLE_FIELDS]):
                fb[f] += len(v)
            lines += e >= 0
    return Sample(tot, nl, lines, fb)


def size_class(v: int, gran: int) -> int:
    return (v + gran - 1) // gran * gran


def estimate(s: Sample, n: int, data_start: int, sel_fields: list) -> Caps:
    """run_scan's capacities for an input of n bytes whose records start at data_start"""
    avg = float(s.bytes) / float(s.newlines) if s.newlines else float(n)
    if avg < 2:
        avg = 2.0
    body = n - data_start
    row_cap = int(float(body) / avg * 1.10) + 4096
    if row_cap > body // 2 + 2:
        row_cap = body // 2 + 2
    row_cap = size_class(row_cap, ROW_CLASS)
    data_cap = []
    for f in sel_fields:
        cap = min(body, U32_MAX)
        if s.lines >= MIN_SAMPLED_LINES and f < HDR_SAMPLE_FIELDS:
            mean = float(s.field_bytes[f]) / float(s.lines)
            est = int(float(row_cap) * mean * 1.25) + DATA_SLACK
            cap = min(cap, size_class(est, DATA_CLASS))
        data_cap.append(cap)
    return Caps(row_cap, data_cap)


def caps(data: bytes, data_start: int, sel_fields: list, delim: int = ord(",")) -> Caps:
    return estimate(sample(data, delim), len(data), data_start, sel_fields)


# ------------------------------------------------------------------ builders
# Every builder lays its input out as
#     header | A | first half of the filler | M | second half of the filler | E
# where A, M and E are zones of "window" lines that hold the three sampling windows (M is centred on n / 2 because
# the two filler halves have equal sizes), and the filler is what the samples do not see.  Window lines are long, so
# that the row estimate is small (row_cap = 1 MiB rows), and their fields are short except one pad field, so that the
# data estimate is small (data_cap = 32 MiB); the filler then holds the rows or the column bytes that meet the caps.
ZONE_AE = 72 << 10            # a window plus a line look-ahead
ZONE_M = 256 << 10            # the middle window, with room for n / 2 to move


@dataclass
class Built:
    data: bytes
    data_start: int
    sel_fields: list
    caps: Caps
    rows: int                 # data records (every one a row without a predicate)
    col_bytes: list           # bytes of each selected field over all rows
    error_row: int | None = None  # data-record ordinal (0-based) of the one malformed record


def _zone(size: int, line) -> list:
    out, n, i = [], 0, 0
    while n < size:
        ln = line(i)
        out.append(ln); n += len(ln); i += 1
    return out


def _assemble(header: bytes, win_line, filler: list) -> tuple:
    """filler: lines, split in two halves of (about) equal bytes around the middle zone -> (input, zones A, M, E, the
    index of the filler's second half)"""
    sizes = np.cumsum([len(x) for x in filler]) if filler else np.zeros(1, np.int64)
    half = int(np.searchsorted(sizes, sizes[-1] / 2)) if filler else 0
    a, m, e = _zone(ZONE_AE, win_line), _zone(ZONE_M, win_line), _zone(ZONE_AE, win_line)
    return b"".join([header] + a + filler[:half] + m + filler[half:] + e), (a, m, e), half


def _fields(line: bytes, delim: bytes = b",") -> list:
    return line.rstrip(b"\n").split(delim)


def rows_input(extra: int, *, trim: bool = False, comment: bool = False, error_at: int | None = None) -> Built:
    """a 2-column file of row_cap + extra data records.  trim: fields written with leading spaces (for
    TrimLeadingSpace); comment: '#' lines among the filler (for CommentChar '#'); error_at: the filler record of that
    index (negative: from the end) has three fields, and error_row is its data-record ordinal"""
    sp = b" " if trim else b""
    # 10-byte records make every filler tile a dense one (more than TILE / 16 terminators); the checked scan sends a
    # comment line in a dense tile to the general path, so next to comments the records are 21 bytes long
    tail = b"c" * 10 + b"\n" if comment else b"\n"
    header = b"a," + sp + b"b\n"
    win_line = lambda i: sp + b"W%06d" % i + b"w" * 56 + b"," + sp + b"p" * 64 + b"\n"
    nwin = sum(len(_zone(z, win_line)) for z in (ZONE_AE, ZONE_M, ZONE_AE))
    row_cap = ROW_CLASS
    for _ in range(3):
        nfill = row_cap + extra - nwin
        filler, rec_at = [], []
        for i in range(nfill):
            rec_at.append(len(filler))
            filler.append(sp + b"%07d," % i + sp + b"%d" % (i % 7) + tail)
            if comment and i % 64 == 5:
                filler.append(b"#note %d\n" % i)
        if error_at is not None:
            filler[rec_at[error_at]] = b"%07d,x,y\n" % (error_at % nfill)
        data, (a, m, e), half = _assemble(header, win_line, filler)
        c = caps(data, len(header), [0, 1])
        if c.row_cap == row_cap:
            break
        row_cap = c.row_cap
    assert c.row_cap == row_cap
    b = Built(data, len(header), [0, 1], c, row_cap + extra, [])
    if error_at is not None:
        at = rec_at[error_at]
        b.error_row = len(a) + sum(1 for x in rec_at if x < at) + (len(m) if at >= half else 0)
    return b


def column_input(ncols: int, k: int, extra: int, *, line_len: int = 128) -> Built:
    """an ncols-column file whose field k totals data_cap[k] + extra bytes over its rows; every other field stays
    short (one pad field of the window lines aside).  The filler's field k values run from 1.5 KB to 40 KB (records
    past the 2 KiB look-ahead, fields longer than a tile)."""
    pad = (k + 1) % ncols
    header = b",".join(b"c%d" % i for i in range(ncols)) + b"\n"
    pad_len = max(1, line_len - 2 * ncols)

    def win_line(i):
        f = [b"%d" % (i % 10)] * ncols
        f[pad] = b"p" * pad_len
        return b",".join(f) + b"\n"

    def fill_line(v: bytes, i: int):
        f = [b""] * ncols
        f[k] = v
        f[pad] = b"%d" % (i % 10)
        return b",".join(f) + b"\n"

    nwin = sum(len(_zone(z, win_line)) for z in (ZONE_AE, ZONE_M, ZONE_AE))
    target = DATA_CLASS + extra
    for _ in range(3):
        left, filler, cyc = target - nwin, [], [1500, 2500, 5000, 1900, 40000, 3000]
        while left > 50000:
            ln = cyc[len(filler) % len(cyc)]
            filler.append(fill_line(b"%c" % (65 + len(filler) % 26) * ln, len(filler))); left -= ln
        while left > 0:
            ln = min(left, 3000)
            filler.append(fill_line(b"z" * ln, len(filler))); left -= ln
        data, _, _ = _assemble(header, win_line, filler)
        c = caps(data, len(header), list(range(ncols)))
        if c.data_cap[k] + extra == target:
            break
        target = c.data_cap[k] + extra
    assert c.data_cap[k] + extra == target
    col = [nwin * (pad_len if f == pad else 1) + sum(len(_fields(ln)[f]) for ln in filler) for f in range(ncols)]
    return Built(data, len(header), list(range(ncols)), c, nwin + len(filler), col)


def flood_input(rows: int = 6 << 20) -> Built:
    """a 2-column file of `rows` filler records of 6-byte field 0 values: rows far over row_cap and field 0 over its
    data_cap (36 MiB against 32 MiB for the default count), so that many tiles straddle both caps"""
    header = b"k,p\n"
    win_line = lambda i: b"%d," % (i % 10) + b"p" * 126 + b"\n"
    i = np.arange(rows, dtype=np.int64)
    arr = np.empty((rows, 8), np.uint8)
    for d in range(6):
        arr[:, d] = 48 + (i // 10 ** (5 - d)) % 10
    arr[:, 6], arr[:, 7] = ord(","), ord("\n")
    half = rows // 2
    a, m, e = _zone(ZONE_AE, win_line), _zone(ZONE_M, win_line), _zone(ZONE_AE, win_line)
    data = b"".join([header] + a + [arr[:half].tobytes()] + m + [arr[half:].tobytes()] + e)
    nwin = len(a) + len(m) + len(e)
    c = caps(data, len(header), [0, 1])
    return Built(data, len(header), [0, 1], c, rows + nwin, [nwin + 6 * rows, 126 * nwin])
