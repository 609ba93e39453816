"""DataSource.GroupBy restated as the Go RowFunc it stands for: the rows folded one by one, in plan order, into a map
from the key values to one accumulator per aggregate.  Values are Python ints: int64 for count and "int" inputs, the
IEEE bits for "float64" inputs, so results compare bit for bit.  Conversions are tests/strconv_oracle.py's.

    groups := map[key][]acc{}; order := []key{}
    for each row:  k := (row[keys[0]], ...); if new: order = append(order, k), acc = init
                   for each aggregate in order: v, err := row.ValueAsInt / ValueAsFloat64(column); if err: stop
                   count: acc++   sum: acc += v   min / max: math.Min / math.Max (floats), < / > (ints)
                   first: v of the group's first row   last: v of its last row"""
from __future__ import annotations

from tests import strconv_oracle as so

MASK64 = (1 << 64) - 1
POS_INF, NEG_INF = 0x7FF0000000000000, 0xFFF0000000000000
X86_NAN = 0xFFF8000000000000  # the default NaN an x86 addition (Go's ADDSD) returns for Inf + -Inf
INT64_MAX, INT64_MIN = so.INT64_MAX, so.INT64_MIN


def is_nan(b: int) -> bool:
    return (b & POS_INF) == POS_INF and (b & ((1 << 52) - 1)) != 0


def go_min(x: int, y: int) -> int:
    """math.Min on IEEE bits: -Inf wins, then NaN (math.NaN()), Min(-0, +0) = -0"""
    if x == NEG_INF or y == NEG_INF:
        return NEG_INF
    if is_nan(x) or is_nan(y):
        return so.NAN_BITS
    fx, fy = so.float_of(x), so.float_of(y)
    if fx == 0 and fx == fy:
        return x if x >> 63 else y
    return x if fx < fy else y


def go_max(x: int, y: int) -> int:
    """math.Max on IEEE bits: +Inf wins, then NaN (math.NaN()), Max(-0, +0) = +0"""
    if x == POS_INF or y == POS_INF:
        return POS_INF
    if is_nan(x) or is_nan(y):
        return so.NAN_BITS
    fx, fy = so.float_of(x), so.float_of(y)
    if fx == 0 and fx == fy:
        return y if x >> 63 else x
    return x if fx > fy else y


def go_add(a: int, b: int) -> int:
    """acc += v on float64 bits, as Go on amd64 computes it: rounded to nearest; a NaN result is the NaN operand (acc
    first), or the x86 default NaN when both operands are numbers (Inf + -Inf)"""
    r = so.bits_of(so.float_of(a) + so.float_of(b))
    if not is_nan(r):
        return r
    return a if is_nan(a) else b if is_nan(b) else X86_NAN


def _to_int64(v: int) -> int:
    v &= MASK64
    return v - (1 << 64) if v >> 63 else v


INIT = {("count", "int"): 0, ("sum", "int"): 0, ("sum", "float64"): 0, ("min", "int"): INT64_MAX, ("min", "float64"): POS_INF,
        ("max", "int"): INT64_MIN, ("max", "float64"): NEG_INF}


def step(op: str, kind: str, acc: int, v: int, new: bool) -> int:
    """one row's value v folded into acc; new: the row is its group's first"""
    if op == "count":
        return acc + 1
    if op == "first":
        return v if new else acc
    if op == "last":
        return v
    if kind == "int":
        if op == "sum":
            return _to_int64(acc + v)
        return min(acc, v) if op == "min" else max(acc, v)
    if op == "sum":
        return go_add(acc, v)
    return go_min(acc, v) if op == "min" else go_max(acc, v)


def fold(rows: list, keys: list, aggs: dict) -> tuple:
    """rows: dicts column -> bytes; aggs: {name: (op, column, kind) or ("count",)} -> (key tuples in group order,
    {name: [value per group]}, error or None).  The error is (row, message) of the first row whose key column is missing
    or whose conversion fails (the aggregates in order); the rows before it are folded, that row is not."""
    specs = {name: (("count", "", "int") if tuple(s) == ("count",) else tuple(s)) for name, s in aggs.items()}
    index: dict = {}
    order: list = []
    acc: dict = {name: [] for name in specs}
    for r, row in enumerate(rows):
        missing = [k for k in keys if k not in row]
        if missing:
            return order, acc, (r, "missing column " + so.go_quote(missing[0].encode()).decode())
        vals, conv = {}, {}
        for name, (op, column, kind) in specs.items():
            if op == "count":
                continue
            if column not in row:
                return order, acc, (r, "missing column " + so.go_quote(column.encode()).decode())
            if (column, kind) not in conv:
                conv[column, kind] = so.atoi(row[column]) if kind == "int" else so.parse_float(row[column])
            v, st = conv[column, kind]
            if st:
                return order, acc, (r, so.message(column, row[column], kind == "float64", st))
            vals[name] = v
        key = tuple(row[k] for k in keys)
        g = index.get(key)
        new = g is None
        if new:
            g = index[key] = len(order)
            order.append(key)
            for name, (op, _, kind) in specs.items():
                acc[name].append(INIT.get((op, kind), 0))
        for name, (op, _, kind) in specs.items():
            acc[name][g] = step(op, kind, acc[name][g], vals.get(name, 0), new)
    return order, acc, None
