"""A plain-Python restatement of the reference's indexImpl (csvplus.go:784-920) and of the DataSource operations built on
it: Join with mergeRows (:545-583), Except (:588-608), SubIndex (:632-641), createIndex / createUniqueIndex (:707-756)
and dedup (:810-867).

Rows are dict[bytes, bytes] held in STORED order: nothing here assumes that the rows are sorted, so the restatement is
also the expected answer for an index whose rows are out of key order (a LoadIndex of an unsorted file, or a
ResolveDuplicates that stored a row whose key sorts elsewhere).  Values compare as Go's strings.Compare does: bytewise.
The sort is stable (the CUDA sort and the C++ oracle with stable=True both keep input order inside a run of equal keys;
the reference's pdqsort does not promise it, SURVEY §Q2)."""
from __future__ import annotations

Row = dict  # dict[bytes, bytes]


def cmp(row: Row, cols: list, values: list, eq: bool) -> bool:
    """indexImpl.cmp (:907-920): True when the row's key prefix is above `values`; `eq` when it is equal"""
    for j, v in enumerate(values):
        a = row[cols[j]]
        if a > v:
            return True
        if a < v:
            return False
    return eq


def search(n: int, f) -> int:
    """sort.Search: the smallest i in [0, n) with f(i), or n; f is only assumed monotone, never checked"""
    i, j = 0, n
    while i < j:
        h = (i + j) // 2
        if not f(h):
            i = h + 1
        else:
            j = h
    return i


def find(rows: list, cols: list, values: list) -> list:
    """indexImpl.find (:870-891): upper bound first, then the lower bound below it"""
    if not values:
        return rows
    if len(values) > len(cols):
        raise ValueError("too many columns in indexImpl.find()")
    upper = search(len(rows), lambda i: cmp(rows[i], cols, values, False))
    lower = search(upper, lambda i: cmp(rows[i], cols, values, True))
    return rows[lower:upper]


def first(rows: list, cols: list, values: list) -> int:
    """indexImpl.first (:893-897)"""
    return search(len(rows), lambda i: cmp(rows[i], cols, values, True))


def has(rows: list, cols: list, values: list) -> bool:
    """indexImpl.has (:899-905)"""
    i = first(rows, cols, values)
    return i < len(rows) and not cmp(rows[i], cols, values, False)


def join(rows: list, cols: list, probe: list, pcols: list | None = None, anti: bool = False) -> list:
    """DataSource.Join (:545-569) / Except (:588-608) of the probe rows against the index rows, matched on the probe's
    columns `pcols` (default: the index's key columns).  Join takes every index row from first() on while the row is not
    above the probe's values, and merges it with the probe row, the probe winning name collisions (mergeRows, :571-583)"""
    pcols = list(cols) if not pcols else list(pcols)
    if len(pcols) > len(cols):
        raise ValueError("too many source columns in Join()")
    out = []
    for p in probe:
        values = [p[c] for c in pcols]
        if anti:
            if not has(rows, cols, values):
                out.append(p)
            continue
        i = first(rows, cols, values)
        while i < len(rows) and not cmp(rows[i], cols, values, False):
            out.append({**rows[i], **p})
            i += 1
    return out


def except_(rows: list, cols: list, probe: list, pcols: list | None = None) -> list:
    return join(rows, cols, probe, pcols, anti=True)


def sub_index(rows: list, cols: list, values: list) -> tuple:
    """Index.SubIndex (:632-641): the find() slice in stored order (no sort) and the remaining key columns"""
    if len(values) >= len(cols):
        raise ValueError("too many values in SubIndex()")
    return find(rows, cols, values), list(cols[len(values):])


def row_string(row: Row) -> bytes:
    """Row.String (:90-104): pairs in name order"""
    if not row:
        return b"{}"
    return b"{ " + b", ".join(b'"' + k + b'" : "' + row[k] + b'"' for k in sorted(row)) + b" }"


class DuplicateKey(Exception):
    pass


def index_on(rows: list, cols: list, unique: bool = False) -> list:
    """createIndex (:707-738) with a stable sort, and createUniqueIndex's adjacent duplicate check (:740-756)"""
    out = sorted(rows, key=lambda r: tuple(r[c] for c in cols))
    if unique:
        for i in range(1, len(out)):
            if all(out[i - 1][c] == out[i][c] for c in cols):
                raise DuplicateKey("duplicate value while creating unique index: "
                                   + row_string({c: out[i][c] for c in cols}).decode("utf-8", "surrogateescape"))
    return out


def _equal(cols: list, a: Row, b: Row) -> bool:  # equalRows (:759-767)
    return all(a[c] == b[c] for c in cols)


def dedup(rows: list, cols: list, resolve) -> tuple:
    """indexImpl.dedup (:810-867) step for step: -> (the rows after it, the groups handed to `resolve` as [lo, hi)).

    A group starts at an adjacent equal pair and ends at sort.Search from `lower` for the first row above the key (:831),
    so on rows out of key order it can take in rows with other keys.  The walk copies the row before `lower` while no
    pair is found; when it runs off the end that way the last row is never copied (SURVEY §Q1).  `resolve` returns a row,
    or None / a row with fewer entries than key columns to drop the group (:845)."""
    rows = list(rows)
    groups = []
    n = len(rows)
    lower = 1
    while lower < n and not _equal(cols, rows[lower - 1], rows[lower]):
        lower += 1
    if lower >= n:
        return rows, groups
    dest = lower - 1
    while lower < n:
        values = [rows[lower][c] for c in cols]
        lo = lower
        upper = lo + search(n - lo, lambda i: cmp(rows[lo + i], cols, values, False))
        groups.append((lower - 1, upper))
        row = resolve(rows[lower - 1:upper])
        lower = upper + 1
        if row is not None and len(row) >= len(cols):
            rows[dest] = row
            dest += 1
        while lower < n:
            if _equal(cols, rows[lower - 1], rows[lower]):
                break
            rows[dest] = rows[lower - 1]
            lower += 1
            dest += 1
    return rows[:dest], groups
