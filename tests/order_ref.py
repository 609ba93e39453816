"""DataSource.OrderBy restated in plain Python: Go's slices.SortStableFunc with the comparator cmp.Or(cmp.Compare(key 0),
cmp.Compare(key 1), ...), written as stable sorts from the last key to the first.  Values are tests/strconv_oracle.py's
conversions; floats compare as cmp.Compare on float64 (every NaN below every number and all NaNs equal, -0 == +0).

    keys: (column, kind, direction), kind "str" | "int" | "float64", direction "asc" | "desc"
    rows: dicts column -> bytes"""
from __future__ import annotations

import functools

from tests import strconv_oracle as so


@functools.lru_cache(maxsize=1 << 16)
def _value(kind: str, raw: bytes):
    """(sort key as cmp.Compare orders it, status)"""
    if kind == "str":
        return raw, so.OK  # Python compares bytes as strings.Compare does: unsigned, a prefix first
    if kind == "int":
        return so.atoi(raw)
    bits, st = so.parse_float(raw)
    f = so.float_of(bits)
    return ((0, 0.0) if f != f else (1, f)), st  # NaN first and all NaNs equal; -0.0 == 0.0 in Python too


def error(rows: list, keys: list):
    """(row, message) of the conversion error OrderBy raises, or None: per key the first failing row (a key column the
    rows lack fails at row 0), the lowest row over the keys, ties to the earlier key"""
    best = None
    if not rows:
        return None
    for ki, (column, kind, _) in enumerate(keys):
        found = None
        if column not in rows[0]:
            found = (0, "missing column " + so.go_quote(column.encode()).decode())
        elif kind != "str":
            for r, row in enumerate(rows):
                _, st = _value(kind, row[column])
                if st:
                    found = (r, so.message(column, row[column], kind == "float64", st))
                    break
        if found is not None and (best is None or found[0] < best[0]):
            best = found
    return best


def order(rows: list, keys: list, limit: int | None = None) -> list:
    """the rows in OrderBy's order (the first `limit` of them); the rows convert without error"""
    out = list(rows)
    for column, kind, direction in reversed(keys):
        out.sort(key=lambda row: _value(kind, row[column])[0], reverse=direction == "desc")  # reverse keeps ties in order
    return out if limit is None else out[:limit]
