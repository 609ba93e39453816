"""ctypes binding of the CPU oracle (oracle/oracle.cpp).

TEST INFRASTRUCTURE ONLY — imported by tests/, __graft_entry__.smoke() and the
cpu_baseline / --impl reference legs of bench.py.  The product package
(csvplus_b200) never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "oracle.cpp")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _LIB_PATH


class _Opts(C.Structure):
    _fields_ = [("comma", C.c_uint32), ("comment", C.c_uint32), ("fields_per_record", C.c_int32),
                ("lazy_quotes", C.c_uint8), ("trim_leading_space", C.c_uint8),
                ("header_from_first_row", C.c_uint8), ("_pad", C.c_uint8)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, i64, u64, cp = C.c_void_p, C.c_int64, C.c_uint64, C.c_char_p
        P = C.POINTER
        L.orc_csv_records.restype = i64
        L.orc_csv_records.argtypes = [vp, u64, P(_Opts), vp, u64, P(u64), P(C.c_int)]
        L.orc_reader_rows.restype = vp
        L.orc_reader_rows.argtypes = [vp, u64, P(_Opts), cp, P(i64), P(C.c_int32), C.c_int]
        L.orc_reader_filter_rows.restype = vp
        L.orc_reader_filter_rows.argtypes = [vp, u64, P(_Opts), cp, P(i64), P(C.c_int32), C.c_int, vp]
        L.orc_result_free.argtypes = [vp]
        L.orc_result_nrows.restype = i64; L.orc_result_nrows.argtypes = [vp]
        L.orc_result_failed.restype = C.c_int; L.orc_result_failed.argtypes = [vp]
        L.orc_result_line.restype = u64; L.orc_result_line.argtypes = [vp]
        L.orc_result_kind.restype = C.c_int; L.orc_result_kind.argtypes = [vp]
        L.orc_result_error.restype = i64; L.orc_result_error.argtypes = [vp, vp, u64]
        L.orc_result_row_header.restype = i64; L.orc_result_row_header.argtypes = [vp, i64, vp, u64]
        L.orc_result_column.restype = i64; L.orc_result_column.argtypes = [vp, cp, i64, vp, vp, vp]
        L.orc_row_string.restype = i64; L.orc_row_string.argtypes = [vp, i64, vp, u64]
        L.orc_result_from_columns.restype = vp
        L.orc_result_from_columns.argtypes = [C.c_int, cp, P(i64), P(vp), P(vp), i64]
        L.orc_pred_like.restype = vp; L.orc_pred_like.argtypes = [C.c_int, cp, P(i64), cp, P(i64)]
        L.orc_pred_combine.restype = vp; L.orc_pred_combine.argtypes = [C.c_int, C.c_int, P(vp)]
        L.orc_pred_free.argtypes = [vp]
        L.orc_filter.restype = vp; L.orc_filter.argtypes = [vp, vp]
        L.orc_select.restype = vp; L.orc_select.argtypes = [vp, C.c_int, cp, P(i64), u64]
        L.orc_cut.restype = vp; L.orc_cut.argtypes = [vp, C.c_int, u64, vp]
        L.orc_drop_columns.restype = vp; L.orc_drop_columns.argtypes = [vp, C.c_int, cp, P(i64)]
        L.orc_index_create.restype = vp
        L.orc_index_create.argtypes = [vp, C.c_int, cp, P(i64), C.c_int, C.c_int, vp, u64]
        L.orc_index_free.argtypes = [vp]
        L.orc_index_nrows.restype = i64; L.orc_index_nrows.argtypes = [vp]
        L.orc_index_rows.restype = vp; L.orc_index_rows.argtypes = [vp]
        L.orc_index_find.restype = vp; L.orc_index_find.argtypes = [vp, C.c_int, cp, P(i64)]
        L.orc_join.restype = vp; L.orc_join.argtypes = [vp, vp, C.c_int, cp, P(i64), u64]
        L.orc_except.restype = vp; L.orc_except.argtypes = [vp, vp, C.c_int, cp, P(i64)]
        L.orc_index_dedup.argtypes = [vp, C.c_int, cp, i64]
        L.orc_to_csv.restype = i64; L.orc_to_csv.argtypes = [vp, C.c_int, cp, P(i64), vp, u64, vp, u64]
        _lib = L
    return _lib


ERR_NAMES = {0: None, 1: "bare_quote", 2: "quote", 3: "field_count", 4: "invalid_delim", 5: "eof", 6: "other"}


def _b(s) -> bytes:
    return s if isinstance(s, (bytes, bytearray)) else str(s).encode()


def _pack(strs):
    bs = [_b(s) for s in strs]
    lens = (C.c_int64 * max(1, len(bs)))(*[len(x) for x in bs])
    return b"".join(bs), lens, len(bs)


def _buf(data):
    """bytes-like / numpy uint8 -> (pointer, length, keepalive)."""
    if isinstance(data, np.ndarray):
        a = np.ascontiguousarray(data, dtype=np.uint8)
        return a.ctypes.data, a.size, a
    b = bytes(data)
    return C.cast(C.c_char_p(b), C.c_void_p).value, len(b), b


@dataclass
class Opts:
    comma: str = ","
    comment: str = ""
    fields_per_record: int = 0
    lazy_quotes: bool = False
    trim_leading_space: bool = False
    header_from_first_row: bool = True

    def c(self) -> _Opts:
        return _Opts(ord(self.comma), ord(self.comment) if self.comment else 0, self.fields_per_record,
                     int(self.lazy_quotes), int(self.trim_leading_space), int(self.header_from_first_row), 0)


def csv_records(data, opts: Opts | None = None):
    """encoding/csv.Reader.ReadAll restated: -> (list of records (list[bytes]), error-name or None)."""
    o = (opts or Opts()).c()
    p, n, keep = _buf(data)
    cap = max(1024, 2 * n + 16)
    out = C.create_string_buffer(cap)
    out_len = C.c_uint64(); err = C.c_int()
    cnt = lib().orc_csv_records(p, n, C.byref(o), out, cap, C.byref(out_len), C.byref(err))
    raw = out.raw[: out_len.value]
    recs = [r.split(b"\x1f") for r in raw.split(b"\x1e")[:-1]] if cnt else []
    assert len(recs) == cnt
    return recs, ERR_NAMES[err.value]


class Pred:
    def __init__(self, h):
        self.h = h

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_pred_free(self.h); self.h = None


def Like(match: dict) -> Pred:
    if not match:
        raise ValueError("empty match row in Like() predicate")  # csvplus.go:1280-1282 (panic)
    kb, kl, n = _pack(match.keys()); vb, vl, _ = _pack(match.values())
    return Pred(lib().orc_pred_like(n, kb, kl, vb, vl))


def _combine(op, preds):
    arr = (C.c_void_p * len(preds))(*[p.h for p in preds])
    return Pred(lib().orc_pred_combine(op, len(preds), arr))


def All(*preds): return _combine(1, preds)
def Any(*preds): return _combine(2, preds)
def Not(pred): return _combine(3, [pred])


class Rows:
    """A pulled DataSource: rows delivered + optional DataSourceError."""

    def __init__(self, h):
        self.h = h

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_result_free(self.h); self.h = None

    def __len__(self):
        return lib().orc_result_nrows(self.h)

    @property
    def error(self):
        if not lib().orc_result_failed(self.h):
            return None
        b = C.create_string_buffer(4096); lib().orc_result_error(self.h, b, 4096)
        return b.value.decode("utf-8", "replace")

    @property
    def error_line(self): return lib().orc_result_line(self.h)

    @property
    def error_kind(self): return ERR_NAMES[lib().orc_result_kind(self.h)] if lib().orc_result_failed(self.h) else None

    def header(self, i=0):
        b = C.create_string_buffer(1 << 16); n = lib().orc_result_row_header(self.h, i, b, 1 << 16)
        return b.raw[:n].split(b"\x1f") if n else []

    def column(self, name):
        """-> (offsets int64[n+1], data uint8[], present uint8[n])"""
        nb = _b(name); n = len(self)
        total = lib().orc_result_column(self.h, nb, len(nb), None, None, None)
        off = np.empty(n + 1, np.int64); data = np.empty(max(1, total), np.uint8); pres = np.empty(max(1, n), np.uint8)
        lib().orc_result_column(self.h, nb, len(nb), off.ctypes.data, data.ctypes.data, pres.ctypes.data)
        return off, data[:total], pres[:n]

    def values(self, name):
        off, data, pres = self.column(name)
        d = data.tobytes()
        return [d[off[i]:off[i + 1]] if pres[i] else None for i in range(len(self))]

    def row_string(self, i):
        b = C.create_string_buffer(1 << 16); lib().orc_row_string(self.h, i, b, 1 << 16); return b.value.decode()

    def to_dicts(self):
        if len(self) == 0:
            return []
        names = set()
        for i in range(len(self)):
            names.update(self.header(i))
        cols = {nm: self.values(nm) for nm in names}
        return [{nm: cols[nm][i] for nm in names if cols[nm][i] is not None} for i in range(len(self))]

    # ---- DataSource combinators
    def filter(self, pred: Pred): return Rows(lib().orc_filter(self.h, pred.h))

    def select(self, *cols, line_base=0):
        b, l, n = _pack(cols); return Rows(lib().orc_select(self.h, n, b, l, line_base))

    def top(self, n): return Rows(lib().orc_cut(self.h, 0, n, None))
    def drop(self, n): return Rows(lib().orc_cut(self.h, 1, n, None))
    def take_while(self, pred: Pred): return Rows(lib().orc_cut(self.h, 2, 0, pred.h))
    def drop_while(self, pred: Pred): return Rows(lib().orc_cut(self.h, 3, 0, pred.h))

    def drop_columns(self, *cols):
        b, l, n = _pack(cols); return Rows(lib().orc_drop_columns(self.h, n, b, l))

    def index_on(self, *cols, unique=False, stable=True):
        b, l, n = _pack(cols); eb = C.create_string_buffer(8192)
        h = lib().orc_index_create(self.h, n, b, l, int(unique), int(stable), eb, 8192)
        if not h:
            raise OracleError(eb.value.decode("utf-8", "replace"))
        return Index(h)

    def unique_index_on(self, *cols, stable=True): return self.index_on(*cols, unique=True, stable=stable)

    def join(self, index, *cols, line_base=0):
        b, l, n = _pack(cols); return Rows(lib().orc_join(self.h, index.h, n, b, l, line_base))

    def except_(self, index, *cols):
        b, l, n = _pack(cols); return Rows(lib().orc_except(self.h, index.h, n, b, l))

    def to_csv(self, *cols):
        b, l, n = _pack(cols); eb = C.create_string_buffer(8192)
        size = lib().orc_to_csv(self.h, n, b, l, None, 0, eb, 8192)
        out = C.create_string_buffer(max(1, size))
        lib().orc_to_csv(self.h, n, b, l, out, size, eb, 8192)
        err = eb.value.decode() or None
        return out.raw[:size], err


class OracleError(Exception):
    pass


class Index:
    def __init__(self, h): self.h = h

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_index_free(self.h); self.h = None

    def __len__(self): return lib().orc_index_nrows(self.h)
    def rows(self): return Rows(lib().orc_index_rows(self.h))

    def find(self, *vals):
        b, l, n = _pack(vals); return Rows(lib().orc_index_find(self.h, n, b, l))

    def dedup(self, mode="min", col=""):
        m = {"min": 0, "drop": 1, "first": 2}[mode]; cb = _b(col)
        lib().orc_index_dedup(self.h, m, cb, len(cb))


def reader_rows(data, opts: Opts | None = None, select=None, expect=None, assume=None, pred: Pred | None = None):
    """Take(FromFile(..)[.SelectColumns(select) | .ExpectHeader(expect) | .AssumeHeader(assume)])[.Filter(pred)] pulled."""
    o = opts or Opts()
    names, idx = [], []
    if select is not None:
        names, idx = list(select), [-1] * len(select)
    elif expect is not None:
        names, idx = list(expect.keys()), list(expect.values())
    elif assume is not None:
        names, idx = list(assume.keys()), list(assume.values())
        o = Opts(**{**o.__dict__, "header_from_first_row": False})
    co = o.c()
    b, l, n = _pack(names)
    ia = (C.c_int32 * max(1, n))(*idx)
    p, ln, keep = _buf(data)
    if pred is None:
        return Rows(lib().orc_reader_rows(p, ln, C.byref(co), b, l, ia, n))
    return Rows(lib().orc_reader_filter_rows(p, ln, C.byref(co), b, l, ia, n, pred.h))


def take_rows(rows: list[dict]) -> Rows:
    """TakeRows of literal rows that all share the same columns (csvplus.go:218)."""
    names = sorted({k for r in rows for k in r})
    offs, datas = [], []
    for nm in names:
        vals = [_b(r[nm]) for r in rows]
        off = np.zeros(len(rows) + 1, np.int64); off[1:] = np.cumsum([len(v) for v in vals])
        datas.append(np.frombuffer(b"".join(vals) or b"\0", np.uint8).copy()); offs.append(off)
    b, l, n = _pack(names)
    oa = (C.c_void_p * n)(*[o.ctypes.data for o in offs]); da = (C.c_void_p * n)(*[d.ctypes.data for d in datas])
    return Rows(lib().orc_result_from_columns(n, b, l, oa, da, len(rows)))


def take_columns(columns: dict) -> Rows:
    """take_rows from columns: {name: (offsets int[n+1], bytes uint8[])}, every column of the same n rows."""
    names = list(columns)
    offs = [np.ascontiguousarray(columns[nm][0], dtype=np.int64) for nm in names]
    datas = [np.ascontiguousarray(columns[nm][1], dtype=np.uint8) for nm in names]
    datas = [d if d.size else np.zeros(1, np.uint8) for d in datas]
    nrows = len(offs[0]) - 1 if offs else 0
    b, l, n = _pack(names)
    oa = (C.c_void_p * max(1, n))(*[o.ctypes.data for o in offs]); da = (C.c_void_p * max(1, n))(*[d.ctypes.data for d in datas])
    return Rows(lib().orc_result_from_columns(n, b, l, oa, da, nrows))
