"""A plain-Python restatement of DataSource.LeftJoin, built on index_ref's first / cmp (indexImpl.first and indexImpl.cmp).

Per probe row, in order: the rows Join gives (every index row from first() on while the row is not above the probe's
values, merged with the probe row, the probe winning name collisions); when there is none, the probe row alone with ""
in every index column whose name the probe lacks (Row.SafeGetValue(col, "") read from the probe row).  Rows are
dict[bytes, bytes] in stored order, so indexes out of key order are covered as index_ref covers them."""
from __future__ import annotations

from tests.index_ref import cmp, first


def left_join(rows: list, cols: list, probe: list, pcols: list | None = None, index_columns: list | None = None) -> list:
    """LeftJoin of the probe rows against the index rows (stored order) keyed on cols, matched on the probe's columns
    pcols (default: cols).  index_columns: the index's column names (needed when the index has no rows; default: the
    first stored row's)"""
    pcols = list(cols) if not pcols else list(pcols)
    if len(pcols) > len(cols):
        raise ValueError("too many source columns in LeftJoin()")
    if index_columns is None:
        index_columns = list(rows[0]) if rows else list(cols)
    out = []
    for p in probe:
        values = [p[c] for c in pcols]
        i = first(rows, cols, values)
        matched = False
        while i < len(rows) and not cmp(rows[i], cols, values, False):
            out.append({**rows[i], **p})
            matched = True
            i += 1
        if not matched:
            out.append({**{c: b"" for c in index_columns if c not in p}, **p})
    return out


def schema(index_columns: list, probe_columns: list) -> list:
    """Join's (and LeftJoin's) column order: the index columns the probe lacks in index order, then the probe's"""
    return [c for c in index_columns if c not in probe_columns] + list(probe_columns)
