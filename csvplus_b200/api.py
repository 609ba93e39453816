"""Host-side mirror of the csvplus Go API (csvplus.go) over the C ABI (include/csvplus_b200.h).

The reference's toolchain (Go) is absent from this image, so this module — together with
host/csvplus.hpp (C++) — plays the role of the thin Go package described in INTEGRATION.md:
same names, argument meaning and error text as the reference, so that tests read like
csvplus_test.go.  Nothing here parses, filters, sorts or joins on the CPU: a `DataSource` is a
*plan*; a sink (ToRows / ToCsv / IndexOn / UniqueIndexOn / calling the source with a RowFunc)
lowers the recognisable prefix (parse -> SelectColumns -> Filter(Like/All/Any/Not) -> Join ...) to
C-ABI calls running CUDA kernels.  Opaque Python callables (Map, Filter(func), Transform, ...)
run on the host at a materialisation boundary, exactly like opaque Go closures would (SURVEY §8b),
and whatever follows them is uploaded again with TakeRows semantics (cpb_table_from_host).
"""
from __future__ import annotations

import contextlib
import ctypes as C
import io
import os
import stat
from typing import Callable, Iterable

import numpy as np

from . import _abi

Row = dict  # map[string]string, csvplus.go:59 (values are str; bytes survive via surrogateescape)

# rows per cpb_table_to_json_into call when DataSource.ToJSON writes a device table: one call produces < 4 GiB, and
# about 2.4 GB for joined rows of ~150 B.  A batch that is still too large is split in halves.
JSON_BATCH_ROWS = 1 << 24
# rows per cpb_index_gob_into call of Index.WriteTo (one call produces < 4 GiB; a batch that is still too large is halved)
GOB_BATCH_ROWS = 1 << 24
# bytes per host push of an input (FromFile / FromReader / host FromBytes, cpb_stream_*): one batch is parsed per push, so
# every column of a batch stays far below the 4 GiB a column of one table may hold.  An input of at most this size is one
# push.  128 MiB: on an H100 the streamed orders join of DESIGN §3.7 ran as fast as at 64 MiB with half the host
# synchronisations, and slower with larger batches (less copy / compute overlap).
STREAM_BATCH_BYTES = 128 << 20


def _enc(s) -> bytes:
    return s if isinstance(s, (bytes, bytearray)) else str(s).encode("utf-8", "surrogateescape")


def _dec(b: bytes) -> str:
    return b.decode("utf-8", "surrogateescape")


def _go_json_string(s) -> bytes:
    """encoding/json's string encoding with HTML escaping off: `"` `\\` and control characters escaped (\\n \\r \\t \\b \\f,
    else \\u00xx), U+2028 / U+2029 escaped, every invalid UTF-8 byte replaced by \\ufffd, everything else verbatim"""
    b = _enc(s)
    out = bytearray(b'"')
    i, n = 0, len(b)
    while i < n:
        c = b[i]
        if c < 0x80:
            if c == 0x22: out += b'\\"'
            elif c == 0x5C: out += b"\\\\"
            elif c == 0x0A: out += b"\\n"
            elif c == 0x0D: out += b"\\r"
            elif c == 0x09: out += b"\\t"
            elif c == 0x08: out += b"\\b"
            elif c == 0x0C: out += b"\\f"
            elif c < 0x20: out += b"\\u00" + b"%02x" % c
            else: out.append(c)
            i += 1
            continue
        width = 2 if 0xC2 <= c <= 0xDF else 3 if 0xE0 <= c <= 0xEF else 4 if 0xF0 <= c <= 0xF4 else 0
        chunk = b[i:i + width]
        try:
            ch = chunk.decode("utf-8") if width and len(chunk) == width else None
        except UnicodeDecodeError:
            ch = None
        if ch is None:
            out += b"\\ufffd"; i += 1
        elif ch in ("\u2028", "\u2029"):
            out += b"\\u2028" if ch == "\u2028" else b"\\u2029"; i += width
        else:
            out += chunk; i += width
    out += b'"'
    return bytes(out)


class DataSourceError(Exception):
    """csvplus.go:1230-1238: `row %d: %s`"""

    def __init__(self, line: int, err: str, kind: int = 0):
        self.Line, self.Err, self.kind = line, err, kind
        super().__init__(f"row {line}: {err}")


class CsvPlusError(Exception):
    """errors the reference returns without a row number (e.g. duplicate key) or panics with"""

    def __init__(self, msg, status=0, kind=0):
        super().__init__(msg)
        self.status, self.kind = status, kind


class StopIterationEOF(Exception):
    """a RowFunc raises this to stop the iteration cleanly (io.EOF, csvplus.go:238-239)"""


def _strs(items: Iterable) -> tuple:
    bs = [_enc(x) for x in items]
    arr = (_abi.Str * max(1, len(bs)))()
    for i, b in enumerate(bs):
        arr[i].ptr = b
        arr[i].len = len(b)
    return arr, bs  # keep bs alive


def _raise(st: int, err: _abi.Error, ctx=None):
    msg = err.msg.decode("utf-8", "replace") if err is not None else ""
    if st == _abi.CPB_ERR_DATA:
        if err.has_line:
            raise _data_error(err)
        raise CsvPlusError(msg, st, err.kind)
    if not msg and ctx is not None:
        msg = _abi.load().cpb_last_error(ctx.h).decode("utf-8", "replace")
    raise CsvPlusError(msg or f"csvplus_b200 call failed with status {st}", st, err.kind if err is not None else 0)


def _data_error(e: _abi.Error) -> DataSourceError:
    return DataSourceError(e.line, e.msg.decode("utf-8", "replace"), e.kind)


class Context:
    """cpb_ctx: one device, one stream.  `default()` gives a process-wide context on cuda:LOCAL_RANK."""

    _default = None

    def __init__(self, device: int = 0):
        self.lib = _abi.load()
        h = C.c_void_p()
        st = self.lib.cpb_init(device, C.byref(h))
        if st != 0:
            raise CsvPlusError(f"cpb_init(device={device}) failed with status {st}: no usable CUDA device "
                               "(csvplus_b200 has no CPU fallback)", st)
        self.h, self.device = h, device

    @classmethod
    def default(cls) -> "Context":
        if cls._default is None:
            cls._default = cls(int(os.environ.get("LOCAL_RANK", "0")))
        return cls._default

    def close(self):
        if self.h:
            self.lib.cpb_shutdown(self.h)
            self.h = None

    def sync(self):
        self.lib.cpb_sync(self.h)

    def reserve(self, nbytes: int) -> bool:
        """cpb_pool_reserve: map `nbytes` of device memory into this context's pool ahead of time (False: not available)"""
        return self.lib.cpb_pool_reserve(self.h, int(nbytes)) == 0

    def _call(self, name: str, *args, err: "_abi.Error | None" = None, accept: tuple = (), h=None) -> int:
        """lib.<name>(h, *args[, err]) -> its status.  h is the handle passed first, this context's by default; an entry
        whose last parameter is a cpb_error* is given err (a fresh one by default).  A non-zero status that is not in
        accept raises (_raise)."""
        fn = getattr(self.lib, name)
        if fn.argtypes[-1] is C.POINTER(_abi.Error):
            err = _abi.Error() if err is None else err
            args += (C.byref(err),)
        st = fn(self.h if h is None else h, *args)
        if st and st not in accept:
            _raise(st, err, self)
        return st

    def _new_table(self, name: str, *args) -> "Table":
        """an entry whose out-parameter, after args, is a new table handle"""
        h = C.c_void_p()
        self._call(name, *args, C.byref(h))
        return Table(self, h)

    def _new_index(self, name: str, *args, columns: list) -> "Index":
        """an entry whose out-parameter, after args, is a new index handle; columns: the index's key columns"""
        h = C.c_void_p()
        self._call(name, *args, C.byref(h))
        return Index(self, h, columns)

    def pool_used_high(self, reset: bool = False) -> int:
        """cpb_pool_used_high: the most device memory this context's pool has had allocated at once since the last reset
        (reset=True starts a new window at the current use)"""
        out = C.c_uint64()
        self._call("cpb_pool_used_high", int(reset), C.byref(out))
        return out.value

    @property
    def stream(self) -> int:
        return self.lib.cpb_ctx_stream(self.h) or 0

    # ---- measurement
    def stats(self, enable: bool | None = None, reset: bool = False):
        if enable is not None:
            self.lib.cpb_stats_enable(self.h, int(enable))
        if reset:
            self.lib.cpb_stats_reset(self.h)
            return {}
        arr = (_abi.KStat * 64)()
        n = C.c_int()
        self.lib.cpb_stats_get(self.h, arr, 64, C.byref(n))
        return {arr[i].name.decode(): {"launches": arr[i].launches, "ms": arr[i].ms, "algo_bytes": arr[i].algo_bytes}
                for i in range(min(n.value, 64))}

    def kernel_launches(self) -> int:
        return self.lib.cpb_kernel_launches(self.h)

    def host_syncs(self) -> int:
        return self.lib.cpb_host_syncs(self.h)

    # ---- staging memory
    def host_alloc(self, n: int) -> "HostBuffer":
        return HostBuffer(self, n)

    def device_alloc(self, n: int) -> "DeviceBuffer":
        return DeviceBuffer(self, n)

    def gen_csv(self, kind: str, rows: tuple, seed=0xC5B200, n_cust=1, n_prod=1, header=True, permute=False,
                chunk_rows=20_000_000) -> "DeviceBuffer":
        """synthetic CSV of SURVEY §8(d) generated on the GPU (bench / tests only)"""
        k = {"people": 0, "customers": 0, "orders": 1, "products": 2}[kind]
        lo, hi = rows

        def gen(r0, r1, dst, cap) -> int:
            nb = C.c_uint64()
            self._call("cpb_gen_csv", k, seed, r0, r1, n_cust, n_prod, int(header and r0 == lo), int(permute), dst, cap, C.byref(nb))
            return nb.value
        sizes, r = [], lo
        while True:
            e = min(hi, r + chunk_rows)
            sizes.append((r, e, gen(r, e, None, 0)))
            r = e
            if r >= hi:
                break
        total = sum(nb for _, _, nb in sizes)
        buf = self.device_alloc(total)
        off = 0
        for (r0, r1, nb) in sizes:
            off += gen(r0, r1, C.c_void_p(buf.ptr + off), nb)
        buf.nbytes = total
        return buf


class HostBuffer:
    def __init__(self, ctx: Context, n: int):
        self.ctx, self.nbytes = ctx, n
        p = C.c_void_p()
        ctx._call("cpb_host_alloc", n, C.byref(p))
        self.ptr = p.value

    def array(self) -> np.ndarray:
        return np.ctypeslib.as_array((C.c_uint8 * self.nbytes).from_address(self.ptr))

    def free(self):
        if self.ptr:
            self.ctx.lib.cpb_host_free(self.ctx.h, C.c_void_p(self.ptr)); self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class DeviceBuffer:
    def __init__(self, ctx: Context, n: int, ptr: int | None = None):
        """n bytes of new device memory (cpb_device_alloc), or the n bytes at ptr that the library allocated"""
        self.ctx, self.nbytes = ctx, n
        if ptr is None:
            p = C.c_void_p()
            ctx._call("cpb_device_alloc", n, C.byref(p))
            ptr = p.value
        self.ptr = ptr

    @classmethod
    def adopt(cls, ctx: Context, ptr: int, nbytes: int) -> "DeviceBuffer":
        """device memory a call returned (cpb_table_to_csv_device, ...): released with the buffer, like its own"""
        return cls(ctx, nbytes, ptr)

    def to_host(self, n: int | None = None, offset: int = 0) -> np.ndarray:
        n = self.nbytes - offset if n is None else n
        out = np.empty(n, np.uint8)
        self.ctx._call("cpb_memcpy_d2h", out.ctypes.data, C.c_void_p(self.ptr + offset), n)
        return out

    def free(self):
        if self.ptr:
            self.ctx.lib.cpb_device_free(self.ctx.h, C.c_void_p(self.ptr)); self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


# ------------------------------------------------------------------ predicates (csvplus.go:1240-1293)
# what an index key can hold (a set term is an index over its literals): key columns, key image bytes (csvplus_b200.h)
_MAX_INDEX_KEYS, _MAX_KEY_IMAGE = 16, 4096
# cpb_str and cpb_pred as numpy records (set terms are lowered in bulk)
_STR_DTYPE = np.dtype([("ptr", "<u8"), ("len", "<u8")])
_PRED_DTYPE = np.dtype([("op", "<i4"), ("n", "<i4"), ("keys", "<u8"), ("values", "<u8"), ("children", "<u8")])
assert _STR_DTYPE.itemsize == C.sizeof(_abi.Str) and _PRED_DTYPE.itemsize == C.sizeof(_abi.Pred)


class Predicate:
    """A recognisable predicate: callable on a Row (host) and lowerable to cpb_pred (device)."""

    def __init__(self, op: int, match: dict | None = None, kids: list | None = None):
        self.op, self.match, self.kids = op, match or {}, kids or []
        # computed once per node: a plan that filters batch by batch asks for them on every batch
        self._sets = self._lowerable = self._lowered = None

    def __call__(self, row: Row) -> bool:
        if self.op == 0:
            return all(k in row and row[k] == v for k, v in self.match.items())
        if self.op == 1:
            return all(k(row) for k in self.kids)
        if self.op == 2:
            return any(k(row) for k in self.kids)
        return not self.kids[0](row)

    def lowerable(self) -> bool:
        """True when the device compiles the tree: every node is a Predicate and the tree stays within the header's
        CPB_PRED_MAX_* limits, a set term (_set_groups) counting as one term.  Terms are counted as if every Like key named
        a column (a missing one compiles to a constant false), so a tree over missing columns may be declined where the
        device would have taken it.  A declined tree is evaluated on host rows, as an opaque function is."""
        if self._lowerable is not None:
            return self._lowerable
        terms = ops = 0

        def walk(p, depth) -> bool:
            nonlocal terms, ops
            if not isinstance(p, Predicate) or depth > _abi.PRED_MAX_DEPTH:
                return False
            if p.op == 0:  # one term per pair, ANDed together
                terms += len(p.match); ops += 2 * len(p.match) - 1
                return True
            if not p.kids:  # All() / Any(): a constant
                ops += 1
                return True
            sets = p._set_groups()
            grouped = {i for _, members in sets for i in members}
            terms += len(sets); ops += len(sets)  # one term each; its Likes add no depth
            ops += 1 if p.op == 3 else len(p.kids) - len(grouped) + len(sets) - 1
            return all(walk(k, depth + 1) for i, k in enumerate(p.kids) if i not in grouped)

        self._lowerable = walk(self, 0) and terms <= _abi.PRED_MAX_TERMS and ops <= _abi.PRED_MAX_OPS
        return self._lowerable

    def _set_groups(self) -> list:
        """The set terms of an Any node (CPB_PRED_SET_MIN, csvplus_b200.h), as the device forms them: the direct Like children
        grouped by the set of column names they compare; a group of at least PRED_SET_MIN children whose literals fit an
        index key image is one term.  -> [(keys in the order of the group's first Like, child positions)], by first child."""
        if self._sets is None:
            self._sets = []
            if self.op == 2 and len(self.kids) >= _abi.PRED_SET_MIN:
                groups: dict = {}
                for i, k in enumerate(self.kids):
                    if isinstance(k, Predicate) and k.op == 0 and 0 < len(k.match) <= _MAX_INDEX_KEYS:
                        m = k.match  # (a one-column Like is grouped by its name: a str never equals a frozenset)
                        groups.setdefault(next(iter(m)) if len(m) == 1 else frozenset(m), []).append(i)
                for members in groups.values():
                    if len(members) < _abi.PRED_SET_MIN:
                        continue
                    keys = list(self.kids[members[0]].match)
                    widths = [max(len(_enc(self.kids[i].match[key])) for i in members) for key in keys]
                    if sum(w + (1 if w < 255 else 2 if w < 65535 else 4) for w in widths) <= _MAX_KEY_IMAGE:
                        self._sets.append((keys, members))
                self._sets.sort(key=lambda s: s[1][0])
        return self._sets

    def columns(self) -> set:
        """the distinct column names the tree's Like terms compare"""
        return set(self.match).union(*(k.columns() for k in self.kids))

    def _c(self, keep: list) -> _abi.Pred:
        """the cpb_pred tree, lowered once per node; keep receives what must stay alive while the tree is in use"""
        if self._lowered is None:
            own: list = []
            self._lowered = (self._lower(own), own)
        keep.append(self._lowered)
        return self._lowered[0]

    def _lower(self, keep: list) -> _abi.Pred:
        p = _abi.Pred()
        p.op = self.op
        if self.op == 0:
            ka, kb = _strs(self.match.keys()); va, vb = _strs(self.match.values())
            keep += [ka, kb, va, vb]
            p.n, p.keys, p.values = len(self.match), ka, va
            return p
        ptrs = np.zeros(max(1, len(self.kids)), np.uint64)
        bulk = np.zeros(len(ptrs), bool)
        for keys, members in self._set_groups():
            ptrs[members] = self._lower_group(keys, members, keep)
            bulk[members] = True
        for i, k in enumerate(self.kids):
            if not bulk[i]:
                ptrs[i] = C.addressof(k._c(keep))
        arr = (C.POINTER(_abi.Pred) * len(ptrs)).from_buffer(ptrs)
        keep += [ptrs, arr]
        p.n, p.children = len(self.kids), arr
        return p

    def _lower_group(self, keys: list, members: list, keep: list) -> np.ndarray:
        """the Likes of one set term in bulk: every child's pairs in the order of keys, all children on one keys array, the
        values in one cpb_str array over one byte string, the nodes in one array.  -> the nodes' addresses"""
        nk, m = len(keys), len(members)
        ka, kb = _strs(keys)
        vals = [_enc(self.kids[i].match[k]) for i in members for k in keys]
        blob = b"".join(vals)
        lens = np.fromiter(map(len, vals), np.uint64, len(vals))
        offs = np.zeros(len(vals), np.uint64)
        np.cumsum(lens[:-1], out=offs[1:])
        base = np.frombuffer(blob, np.uint8) if blob else np.zeros(1, np.uint8)
        strs = np.empty(len(vals), _STR_DTYPE)
        strs["ptr"] = np.uint64(base.ctypes.data) + offs
        strs["len"] = lens
        nodes = np.zeros(m, _PRED_DTYPE)
        nodes["n"] = nk
        nodes["keys"] = C.addressof(ka)
        nodes["values"] = np.uint64(strs.ctypes.data) + np.arange(m, dtype=np.uint64) * np.uint64(_STR_DTYPE.itemsize * nk)
        keep += [ka, kb, blob, base, strs, nodes]
        return np.uint64(nodes.ctypes.data) + np.arange(m, dtype=np.uint64) * np.uint64(_PRED_DTYPE.itemsize)


def Like(match: Row) -> Predicate:
    if len(match) == 0:
        raise ValueError("empty match row in Like() predicate")  # panic, csvplus.go:1280-1282
    return Predicate(0, {str(k): (v if isinstance(v, str) else _dec(_enc(v))) for k, v in match.items()})


def All(*funcs) -> Callable[[Row], bool]:
    return Predicate(1, kids=list(funcs)) if all(isinstance(f, Predicate) for f in funcs) else (lambda row: all(f(row) for f in funcs))


def Any(*funcs) -> Callable[[Row], bool]:
    return Predicate(2, kids=list(funcs)) if all(isinstance(f, Predicate) for f in funcs) else (lambda row: any(f(row) for f in funcs))


def Not(pred) -> Callable[[Row], bool]:
    return Predicate(3, kids=[pred]) if isinstance(pred, Predicate) else (lambda row: not pred(row))


# ------------------------------------------------------------------ device tables
class Table:
    """cpb_table handle: a columnar batch of rows in HBM."""

    def __init__(self, ctx: Context, h):
        self.ctx, self.h = ctx, h

    def __del__(self):
        try:
            if self.h:
                self.ctx.lib.cpb_table_free(self.h); self.h = None
        except Exception:
            pass

    def __len__(self):
        return self.ctx.lib.cpb_table_num_rows(self.h)

    @property
    def columns(self) -> list[str]:
        out = []
        for i in range(self.ctx.lib.cpb_table_num_cols(self.h)):
            s = _abi.Str()
            self.ctx.lib.cpb_table_col_name(self.h, i, C.byref(s))
            out.append(_dec(C.string_at(s.ptr, s.len)))
        return out

    def column(self, name: str, lo: int = 0, hi: int | None = None):
        """-> (offsets int64[n+1], data uint8[]) of rows [lo,hi) copied to the host"""
        hi = len(self) if hi is None else hi
        idx = self.columns.index(name)
        nb = C.c_uint64()
        self.ctx._call("cpb_table_col_bytes", self.h, idx, lo, hi, C.byref(nb))
        off = np.empty(hi - lo + 1, np.int64)
        data = np.empty(max(1, nb.value), np.uint8)
        self.ctx._call("cpb_table_fetch_column", self.h, idx, lo, hi, off.ctypes.data, data.ctypes.data, data.size)
        return off, data[: nb.value]

    def values(self, name: str, lo: int = 0, hi: int | None = None) -> list[bytes]:
        off, data = self.column(name, lo, hi)
        d = data.tobytes()
        return [d[off[i]:off[i + 1]] for i in range(len(off) - 1)]

    def rows(self, lo: int = 0, hi: int | None = None) -> list[Row]:
        cols = self.columns
        vals = {c: self.values(c, lo, hi) for c in cols}
        n = (len(self) if hi is None else hi) - lo
        return [{c: _dec(vals[c][i]) for c in cols} for i in range(n)]

    def parsed_from(self) -> tuple:
        """(name -> field index of every column, field count of the file's first record) of a parsed table: the resolved
        header that the shards of a file after the first are given (cpb_table_col_field / cpb_table_record_fields)"""
        cols = self.columns
        return ({c: self.ctx.lib.cpb_table_col_field(self.h, i) for i, c in enumerate(cols)}, self.ctx.lib.cpb_table_record_fields(self.h))

    def device_column(self, name: str):
        """raw device pointers (offsets uint32[n+1], data) for zero-copy interop (torch / NCCL)"""
        po, pd = C.c_void_p(), C.c_void_p()
        self.ctx.lib.cpb_table_column_device(self.h, self.columns.index(name), C.byref(po), C.byref(pd))
        return po.value, pd.value

    @staticmethod
    def from_rows(ctx: Context, rows: list[Row], columns: list[str] | None = None) -> "Table":
        """TakeRows (csvplus.go:218): rows must share one column set on the device path"""
        cols = columns if columns is not None else (sorted(rows[0].keys()) if rows else [])
        for r in rows:
            if set(r.keys()) != set(cols):
                raise CsvPlusError("TakeRows on the device requires rows with identical column sets")
        na, nb = _strs(cols)
        offs, datas = [], []
        for cname in cols:
            vals = [_enc(r[cname]) for r in rows]
            off = np.zeros(len(rows) + 1, np.int64)
            if vals:
                off[1:] = np.cumsum([len(v) for v in vals])
            datas.append(np.frombuffer(b"".join(vals) + b"\0", np.uint8).copy()); offs.append(off)
        oa = (C.c_void_p * max(1, len(cols)))(*[o.ctypes.data for o in offs])
        da = (C.c_void_p * max(1, len(cols)))(*[d.ctypes.data for d in datas])
        return ctx._new_table("cpb_table_from_host", len(cols), na, oa, da, len(rows))

    @staticmethod
    def from_device_columns(ctx: Context, names: list[str], columns: list[tuple], nrows: int) -> "Table":
        """cpb_table_from_device: columns[k] = (device pointer of uint32 offsets[nrows+1], device pointer of the bytes);
        the buffers are copied, so the caller may release them once the ctx has been synchronised"""
        na, keep = _strs(names)
        oa = (C.c_void_p * max(1, len(names)))(*[c[0] for c in columns])
        da = (C.c_void_p * max(1, len(names)))(*[c[1] or 0 for c in columns])
        return ctx._new_table("cpb_table_from_device", len(names), na, oa, da, nrows)

    # thin wrappers of the table-level ABI
    def select(self, *cols) -> "Table":
        a, keep = _strs(cols)
        return self.ctx._new_table("cpb_table_select", self.h, a, len(cols))

    def drop(self, *cols) -> "Table":
        a, keep = _strs(cols)
        return self.ctx._new_table("cpb_table_drop", self.h, a, len(cols))

    def filter(self, pred: Predicate) -> "Table":
        keep = []; p = pred._c(keep)
        return self.ctx._new_table("cpb_table_filter", self.h, C.byref(p))

    def first_false(self, pred: Predicate) -> int:
        """index of the first row for which the recognisable predicate is false (len(self) if none): cpb_table_first_false"""
        keep = []; p = pred._c(keep); out = C.c_int64()
        self.ctx._call("cpb_table_first_false", self.h, C.byref(p), C.byref(out))
        return out.value

    def slice(self, lo: int, hi: int) -> "Table":
        return self.ctx._new_table("cpb_table_slice", self.h, lo, hi)

    def index_on(self, *cols, unique=False) -> "Index":
        a, keep = _strs(cols)
        return self.ctx._new_index("cpb_index_build", self.h, a, len(cols), int(unique), columns=list(cols))

    def join(self, index: "Index", *cols, anti=False) -> "Table":
        a, keep = _strs(cols)
        return self.ctx._new_table("cpb_except" if anti else "cpb_join", self.h, index.h, a, len(cols))

    def _pinned_bytes(self, name: str, *args) -> bytes:
        """an entry that returns its bytes in new pinned host memory"""
        p = C.c_void_p(); n = C.c_uint64()
        self.ctx._call(name, self.h, *args, C.byref(p), C.byref(n))
        out = C.string_at(p.value, n.value)
        self.ctx.lib.cpb_host_free(self.ctx.h, p)
        return out

    def _device_bytes(self, name: str, *args) -> "DeviceBuffer":
        """an entry that leaves its bytes in new device memory"""
        p = C.c_void_p(); n = C.c_uint64()
        self.ctx._call(name, self.h, *args, C.byref(p), C.byref(n))
        return DeviceBuffer.adopt(self.ctx, p.value, n.value)

    def to_csv(self, *cols) -> bytes:
        a, keep = _strs(cols)
        return self._pinned_bytes("cpb_table_to_csv", a, len(cols))

    def to_csv_into(self, dst: "HostBuffer | None", offset: int, *cols, header: bool = True) -> int:
        """one batch of ToCsv into pinned host memory (cpb_table_to_csv_into).  Returns the batch's size in bytes; when
        that exceeds the room left in dst (or dst is None), nothing is written."""
        a, keep = _strs(cols)
        return _into(self.ctx, "cpb_table_to_csv_into", self.h, a, len(cols), int(header), dst=dst, offset=offset)

    def to_csv_device(self, *cols) -> "DeviceBuffer":
        """ToCsv with the serialised bytes left in HBM (cpb_table_to_csv_device)"""
        a, keep = _strs(cols)
        return self._device_bytes("cpb_table_to_csv_device", a, len(cols))

    def to_json(self, first: bool = True, last: bool = True) -> bytes:
        """DataSource.ToJSON of every column (cpb_table_to_json); first / last: the batch opens / closes the array"""
        return self._pinned_bytes("cpb_table_to_json", int(first), int(last))

    def to_json_into(self, dst: "HostBuffer | None", offset: int = 0, first: bool = True, last: bool = True) -> int:
        """one batch of a streamed ToJSON into pinned host memory (cpb_table_to_json_into).  Returns the batch's size in
        bytes; when that exceeds the room left in dst (or dst is None), nothing is written."""
        return _into(self.ctx, "cpb_table_to_json_into", self.h, int(first), int(last), dst=dst, offset=offset)

    def to_json_device(self, first: bool = True, last: bool = True) -> "DeviceBuffer":
        """ToJSON with the serialised bytes left in HBM (cpb_table_to_json_device)"""
        return self._device_bytes("cpb_table_to_json_device", int(first), int(last))

    def values_as_int(self, name: str, strict: bool = True):
        """Row.ValueAsInt (strconv.Atoi, csvplus.go:165-183) of every row of a column, as an int64 CUDA tensor on the
        ctx's device.  strict: the first failing row raises CsvPlusError with the reference's text (.row = its index), as
        a RowFunc returning the helper's error does; else -> (values, status uint8: 0 ok, 1 ErrSyntax, 2 ErrRange), the
        values being what Go returns alongside each error."""
        return self._values_as(name, False, strict)

    def values_as_float64(self, name: str, strict: bool = True):
        """Row.ValueAsFloat64 (strconv.ParseFloat(s, 64), csvplus.go:187-205): as values_as_int, float64 values"""
        return self._values_as(name, True, strict)

    def _values_as(self, name: str, is_float: bool, strict: bool):
        values, status, err = self._convert(name, is_float)
        if err is not None and (strict or err.kind == _abi.CPB_E_MISSING_COLUMN):  # fails in both modes
            raise err
        return values if strict else (values, status)

    def _convert(self, name: str, is_float: bool):
        """-> (values, status, CsvPlusError of the first failing row or None); one host synchronisation"""
        import torch
        dev = torch.device("cuda", self.ctx.device)
        n = len(self)
        values = torch.empty(n, dtype=torch.float64 if is_float else torch.int64, device=dev)
        status = torch.empty(n, dtype=torch.uint8, device=dev)
        # the ctx stream writes into memory torch's current stream allocated: it waits for that stream first; the
        # synchronisation inside the call orders the way back
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dev))
        torch.cuda.ExternalStream(self.ctx.stream, device=dev).wait_event(ev)
        b = _enc(name); nbad = C.c_uint64(); e = _abi.Error()
        st = self.ctx._call("cpb_table_column_as_float64" if is_float else "cpb_table_column_as_int64", self.h, _abi.Str(b, len(b)),
                            C.c_void_p(values.data_ptr()), C.c_void_p(status.data_ptr()), C.byref(nbad), err=e, accept=(_abi.CPB_ERR_DATA,))
        if st:
            err = CsvPlusError(e.msg.decode("utf-8", "replace"), st, e.kind)
            err.row = e.line
            return values, status, err
        return values, status, None

    def with_column(self, name: str, value, fmt: str | None = None, prec: int = -1) -> "Table":
        """the reference's Map(func(row) Row { row[name] = value; return row }) on the GPU: a new table with column `name`
        set, replaced in place when it exists, else appended; every other column shares this table's buffers.  value is a
        str (the same bytes in every row), an int64 CUDA tensor (strconv.FormatInt(v, 10)), a float64 CUDA tensor
        (strconv.FormatFloat(x, fmt, prec, 64); fmt defaults to 'g', prec -1 gives the shortest digits that read back as x)
        or a FormatFloat marker.  A tensor holds one value per row; it may be freed as soon as the call returns."""
        if isinstance(value, FormatFloat):
            if fmt is not None:
                raise TypeError("with_column: the format of a FormatFloat value is given in FormatFloat")
            value, fmt, prec = value.values, value.fmt, value.prec
        b = _enc(name); column = _abi.Str(b, len(b))
        if isinstance(value, (str, bytes)):
            if fmt is not None:
                raise TypeError("with_column: fmt applies to float64 tensors only")
            v = _enc(value)
            return self.ctx._new_table("cpb_table_set_literal", self.h, column, _abi.Str(v, len(v)))
        import torch
        values = _device_tensor(self, value, (torch.int64, torch.float64), "with_column")
        if values.dtype == torch.float64:
            fmt = "g" if fmt is None else fmt
            _check_format(fmt, prec)
            return self.ctx._new_table("cpb_table_set_float64", self.h, column, C.c_void_p(values.data_ptr()), fmt.encode(), prec)
        if fmt is not None:
            raise TypeError("with_column: fmt applies to float64 tensors only")
        return self.ctx._new_table("cpb_table_set_int64", self.h, column, C.c_void_p(values.data_ptr()))

    def filter_mask(self, mask) -> "Table":
        """the rows where the bool CUDA tensor mask (one value per row) is true, in order: the reference's
        Filter(func(row) bool) with the predicate computed on the GPU"""
        import torch
        keep = _device_tensor(self, mask, (torch.bool,), "filter_mask")
        return self.ctx._new_table("cpb_table_filter_flags", self.h, C.c_void_p(keep.data_ptr()))

    @staticmethod
    def concat(parts: list["Table"]) -> "Table":
        ctx = parts[0].ctx
        arr = (C.c_void_p * len(parts))(*[p.h for p in parts])
        return ctx._new_table("cpb_table_concat", arr, len(parts))


FORMAT_VERBS = "eEfgG"


def _check_format(fmt, prec):
    if not isinstance(fmt, str) or len(fmt) != 1 or fmt not in FORMAT_VERBS:
        raise ValueError(f"FormatFloat: unsupported format {fmt!r} (want one of e E f g G)")
    if isinstance(prec, bool) or not isinstance(prec, int) or not -1 <= prec <= 64:
        raise ValueError(f"FormatFloat: precision {prec!r} outside -1..64")


class FormatFloat:
    """strconv.FormatFloat(x, fmt, prec, 64) of every value of a float64 CUDA tensor: a value for Table.with_column and
    MapTensors.  fmt is one of e E f g G; prec runs from -1 (the shortest digits that read back as x) to 64."""

    def __init__(self, values, fmt: str = "g", prec: int = -1):
        _check_format(fmt, prec)
        self.values, self.fmt, self.prec = values, fmt, prec


def _device_tensor(t: Table, x, dtypes: tuple, what: str):
    """x as a contiguous 1-D CUDA tensor of one of dtypes with one value per row of t, on t's device, ready to be read on
    the ctx stream: the ctx stream waits for torch's current stream (where x was produced), and x's memory is not reused
    before the ctx stream's work is done, so the caller may free x at once"""
    import torch
    if not isinstance(x, torch.Tensor) or x.dtype not in dtypes:
        got = x.dtype if isinstance(x, torch.Tensor) else type(x).__name__
        raise TypeError(f"{what}: want a CUDA tensor of {' or '.join(str(d) for d in dtypes)}, got {got}")
    dev = torch.device("cuda", t.ctx.device)
    if x.device != dev:
        raise ValueError(f"{what}: the tensor is on {x.device}, the table on {dev}")
    if x.dim() != 1 or x.numel() != len(t):
        raise ValueError(f"{what}: want one value per row ({len(t)}), got shape {tuple(x.shape)}")
    x = x.contiguous()
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(dev))
    s = torch.cuda.ExternalStream(t.ctx.stream, device=dev)
    s.wait_event(ev)
    x.record_stream(s)
    return x


def _tensor_kinds(inputs: dict, what: str) -> dict:
    kinds = {}
    for name, kind in inputs.items():
        if kind not in ("int", "float64"):
            raise ValueError(f"{what}: unknown type {kind!r} for column {name!r} (want 'int' or 'float64')")
        kinds[name] = kind == "float64"
    return kinds


def parse_csv(ctx: Context, data, *, on_device=False, nbytes=None, delimiter=",", comment="", num_fields=0, lazy_quotes=False,
              trim_leading_space=False, header_from_first_row=True, spec: list | None = None, pred: Predicate | None = None):
    """cpb_parse_csv.  data: bytes / numpy uint8 / HostBuffer (host) or DeviceBuffer / int pointer (device).
    Returns (Table, DataSourceError | None): the table holds the rows delivered before the error."""
    opts = _reader_opts(delimiter, comment, num_fields, lazy_quotes, trim_leading_space, header_from_first_row)
    keep = []
    ptr, n, dev = _input_ptr(data, nbytes, on_device, keep)
    sa, nspec, pp = _spec_and_pred(spec, pred, keep)
    h = C.c_void_p(); e = _abi.Error()
    st = ctx._call("cpb_parse_csv", C.c_void_p(ptr), n, int(dev), C.byref(opts), sa, nspec, pp, C.byref(h), err=e, accept=(_abi.CPB_ERR_DATA,))
    return _rows_before_error(ctx, Table(ctx, h), st, e)


def _rows_before_error(ctx: Context, t: "Table | None", st: int, e: _abi.Error) -> tuple:
    """the outcome of a parse whose status may be CPB_ERR_DATA -> (table of the rows before the error, that error or None);
    a data error that comes without a table is raised"""
    if st and (t is None or not t.h.value):
        _raise(st, e, ctx)
    return t, _data_error(e) if st else None


def _reader_opts(delimiter=",", comment="", num_fields=0, lazy_quotes=False, trim_leading_space=False,
                 header_from_first_row=True) -> _abi.ReaderOpts:
    return _abi.ReaderOpts(ord(delimiter), ord(comment) if comment else 0, num_fields, int(lazy_quotes), int(trim_leading_space),
                           int(header_from_first_row), 0)


def _spec_and_pred(spec: list | None, pred: Predicate | None, keep: list) -> tuple:
    """-> (HeaderCol array of spec's (name, index) pairs, their count, pointer to pred's cpb_pred tree or None); keep
    holds what they point to"""
    spec = spec or []
    sa = (_abi.HeaderCol * max(1, len(spec)))()
    for i, (name, idx) in enumerate(spec):
        nb = _enc(name); keep.append(nb)
        sa[i].name.ptr, sa[i].name.len, sa[i].index = nb, len(nb), idx
    pp = None
    if pred is not None:
        pc = pred._c(keep); keep.append(pc); pp = C.byref(pc)
    keep.append(sa)
    return sa, len(spec), pp


def _input_ptr(data, nbytes, on_device, keep):
    if isinstance(data, DeviceBuffer):
        return data.ptr, data.nbytes if nbytes is None else nbytes, True
    if isinstance(data, HostBuffer):
        return data.ptr, data.nbytes if nbytes is None else nbytes, on_device
    if isinstance(data, np.ndarray):
        a = np.ascontiguousarray(data, np.uint8); keep.append(a)
        return a.ctypes.data, a.size if nbytes is None else nbytes, on_device
    if isinstance(data, int):
        return data, nbytes, on_device
    b = bytes(data); keep.append(b)
    return C.cast(C.c_char_p(b), C.c_void_p).value, len(b) if nbytes is None else nbytes, on_device


def csv_quote_parity(ctx: Context, data, *, nbytes=None, on_device=False) -> int:
    """cpb_csv_quote_parity: parity of the quote bytes of a shard's own byte range"""
    keep = []
    ptr, n, dev = _input_ptr(data, nbytes, on_device, keep)
    out = C.c_uint32()
    ctx._call("cpb_csv_quote_parity", C.c_void_p(ptr), n, int(dev), C.byref(out))
    return out.value


def csv_stream_cut(ctx: Context, data, *, nbytes=None, on_device=False, delimiter=",", comment="", lazy_quotes=False,
                   trim_leading_space=False) -> int:
    """cpb_csv_stream_cut: the end of the last complete record of data (0: none), the cut of one stream batch"""
    opts = _reader_opts(delimiter, comment, 0, lazy_quotes, trim_leading_space)
    keep = []
    ptr, n, dev = _input_ptr(data, nbytes, on_device, keep)
    out = C.c_uint64()
    ctx._call("cpb_csv_stream_cut", C.c_void_p(ptr), n, int(dev), C.byref(opts), C.byref(out))
    return out.value


def parse_csv_shard(ctx: Context, data, *, own_bytes: int, shard_index: int, is_last: bool, initial_parity: int, nbytes=None, on_device=False,
                    delimiter=",", num_fields=0, header_from_first_row=True, spec: list | None = None, pred: Predicate | None = None):
    """cpb_parse_csv_shard.  Returns (Table, records owned by the shard, DataSourceError | None) — the error's Line is the
    LOCAL 0-based ordinal of the failing record among the shard's records."""
    opts = _reader_opts(delimiter, num_fields=num_fields, header_from_first_row=header_from_first_row)
    keep = []
    ptr, n, dev = _input_ptr(data, nbytes, on_device, keep)
    sa, nspec, pp = _spec_and_pred(spec, pred, keep)
    h = C.c_void_p(); e = _abi.Error(); recs = C.c_uint64()
    st = ctx._call("cpb_parse_csv_shard", C.c_void_p(ptr), n, int(dev), own_bytes, shard_index, int(is_last), initial_parity, C.byref(opts), sa,
                   nspec, pp, C.byref(h), C.byref(recs), err=e, accept=(_abi.CPB_ERR_DATA,))
    t, err = _rows_before_error(ctx, Table(ctx, h), st, e)
    return t, recs.value, err


# ------------------------------------------------------------------ Index (csvplus.go:610-705)
class Index:
    def __init__(self, ctx: Context, h, columns: list[str]):
        self.ctx, self.h, self.columns = ctx, h, columns

    def __del__(self):
        try:
            if self.h:
                self.ctx.lib.cpb_index_free(self.h); self.h = None
        except Exception:
            pass

    def __len__(self):
        return self.ctx.lib.cpb_index_num_rows(self.h)

    def table(self) -> Table:
        return self.ctx._new_table("cpb_index_table", self.h)

    def Iterate(self, fn):  # csvplus.go:618-620
        return TakeTable(self.table(), line_base=0)(fn)

    def Find(self, *values) -> "DataSource":  # csvplus.go:625-627
        a, keep = _strs(values)
        try:
            return TakeTable(self.ctx._new_table("cpb_index_find", self.h, a, len(values)), line_base=0)
        except CsvPlusError as e:
            if e.status != _abi.CPB_ERR_ARG:
                raise
            raise ValueError("too many columns in indexImpl.find()") from None

    def SubIndex(self, *values) -> "Index":  # csvplus.go:632-641
        if len(values) >= len(self.columns):
            raise ValueError("too many values in SubIndex()")
        a, keep = _strs(values)
        return self.ctx._new_index("cpb_index_sub", self.h, a, len(values), columns=self.columns[len(values):])

    def dup_groups(self):
        """[lo, hi) sorted-row ranges of every run of >= 2 rows with equal keys (cpb_index_dup_groups) as two int64 arrays"""
        ng = C.c_int64(); lo = C.POINTER(C.c_int64)(); hi = C.POINTER(C.c_int64)()
        self.ctx._call("cpb_index_dup_groups", self.h, C.byref(ng), C.byref(lo), C.byref(hi))
        n = ng.value
        try:
            a = np.ctypeslib.as_array(lo, shape=(max(n, 1),))[:n].copy()
            b = np.ctypeslib.as_array(hi, shape=(max(n, 1),))[:n].copy()
        finally:
            self.ctx.lib.cpb_free(lo); self.ctx.lib.cpb_free(hi)
        return a, b

    def dedup_apply(self, keep, bug_compatible: bool = True):
        """keep[g] = sorted position of the row kept for group g, or -1 to drop the group (cpb_index_dedup_apply)"""
        k = np.ascontiguousarray(keep, dtype=np.int64)
        self.ctx._call("cpb_index_dedup_apply", self.h, len(k), k.ctypes.data_as(C.POINTER(C.c_int64)), int(bug_compatible))

    def ResolveDuplicates(self, resolve: Callable[[list[Row]], Row | None], bug_compatible: bool = True):
        """csvplus.go:651-653 / dedup :810-867.  `resolve` gets each group of rows with equal keys and returns the row to
        keep — one of the group's rows or any other row with the index's columns (:846 stores whatever comes back,
        without re-sorting) — or an empty row / None to drop the group, or raises (the index is left unchanged)."""
        lo, hi = self.dup_groups()
        n = len(lo)
        keep = np.full(max(1, n), -1, np.int64)
        replacements: list[Row] = []
        t = self.table()
        for g in range(n):
            rows = t.rows(int(lo[g]), int(hi[g]))
            chosen = resolve(rows)
            if not chosen or len(chosen) < len(self.columns):  # csvplus.go:845
                keep[g] = -1
                continue
            pick = next((i for i, r in enumerate(rows) if r is chosen), None)
            if pick is None:
                pick = next((i for i, r in enumerate(rows) if r == chosen), None)
            if pick is None:
                keep[g] = -2 - len(replacements)
                replacements.append(chosen)
            else:
                keep[g] = lo[g] + pick
        rt = Table.from_rows(self.ctx, replacements, columns=t.columns) if replacements else None
        self.ctx._call("cpb_index_dedup_apply2", self.h, n, keep.ctypes.data_as(C.POINTER(C.c_int64)), rt.h if rt is not None else None,
                       int(bug_compatible))

    def WriteTo(self, fileName: str):  # csvplus.go:655-680: the file is removed on error
        """the index as the reference's encoding/gob file (its key columns, then its rows in stored order), encoded on the
        GPU and written in row-range batches through one pinned buffer.  A path that cannot be created raises the OS
        error and leaves no file; any later error removes the file."""
        with _new_file(fileName) as f:
            self._write_gob(f)

    def _write_gob(self, out: io.IOBase):
        # one pinned buffer, sized up front so that the prefix and every batch are serialised in one call each: the prefix
        # holds the key column names and about 100 bytes more, a batch at most the rows' total (and less than 4 GiB)
        bound = 256 + sum(len(_enc(c)) + 10 for c in self.columns)
        hold: list = [HostBuffer(self.ctx, bound)]
        try:
            plen, total = C.c_uint64(), C.c_uint64()
            _write_into(out, hold, self.ctx, lambda buf: self._gob_begin(buf, plen, total))
            rows_bytes = total.value - plen.value
            if rows_bytes > hold[0].nbytes:
                hold[0].free()
                hold[:] = [HostBuffer(self.ctx, min(rows_bytes, 1 << 32) + 64)]
            _row_batches(len(self), GOB_BATCH_ROWS, lambda lo, hi: _write_into(out, hold, self.ctx, lambda buf: self._gob_into(buf, lo, hi)))
        finally:
            for b in hold:
                b.free()

    def _gob_begin(self, buf: "HostBuffer | None", plen, total) -> int:
        return _into(self.ctx, "cpb_index_gob_begin", self.h, dst=buf, size=plen, more=(C.byref(total),))

    def _gob_into(self, buf: "HostBuffer | None", lo: int, hi: int) -> int:
        return _into(self.ctx, "cpb_index_gob_into", self.h, lo, hi, dst=buf)


def LoadIndex(fileName: str, ctx: Context | None = None) -> Index:  # csvplus.go:683-705
    """an index from a file Index.WriteTo (or the reference) wrote, decoded on the GPU: its rows in file order, its key
    columns from the file.  A missing file raises the OS error; an empty file raises CsvPlusError("EOF"), a cut one
    CsvPlusError("unexpected EOF"), any other file that is not an index CsvPlusError with a description."""
    ctx = ctx or Context.default()
    with open(fileName, "rb") as f:
        size = os.fstat(f.fileno()).st_size
        buf = HostBuffer(ctx, max(size, 1))  # pinned: the rows are copied to the device from here
        try:
            got = f.readinto(memoryview(buf.array())[:size]) if size else 0
            if got != size:
                raise OSError(f"read {fileName}: short read")
            ix = ctx._new_index("cpb_index_load_gob", C.c_void_p(buf.ptr), size, columns=[])
        finally:
            buf.free()
    for k in range(ctx.lib.cpb_index_num_keys(ix.h)):
        s = _abi.Str()
        ctx.lib.cpb_index_key_col(ix.h, k, C.byref(s))
        ix.columns.append(_dec(C.string_at(s.ptr, s.len)))
    return ix


# ------------------------------------------------------------------ Reader (csvplus.go:922-1146)
class Reader:
    def __init__(self, pieces: Callable[[], Iterable], ctx: Context | None = None):
        """pieces: -> an iterator of (piece, is the last piece), each host piece (numpy uint8) left untouched until the
        next one is asked for; a DeviceBuffer is the whole input as one piece"""
        self._pieces, self._ctx = pieces, ctx
        self.delimiter, self.comment = ",", ""
        self.numFields, self.lazyQuotes, self.trimLeadingSpace = 0, False, False
        self.header: dict | None = None
        self.headerFromFirstRow = True
        self._pred: Predicate | None = None

    @property
    def ctx(self) -> Context:
        return self._ctx or Context.default()

    def Delimiter(self, c): self.delimiter = c; return self
    def CommentChar(self, c): self.comment = c; return self
    def LazyQuotes(self): self.lazyQuotes = True; return self
    def TrimLeadingSpace(self): self.trimLeadingSpace = True; return self

    def AssumeHeader(self, spec: dict):  # csvplus.go:998-1012
        if len(spec) == 0:
            raise ValueError("Empty header spec")
        for name, col in spec.items():
            if col < 0:
                raise ValueError("header spec: negative index for column " + name)
        self.header, self.headerFromFirstRow = dict(spec), False
        return self

    def ExpectHeader(self, spec: dict):  # csvplus.go:1020-1033
        if len(spec) == 0:
            raise ValueError("empty header spec")
        self.header, self.headerFromFirstRow = dict(spec), True
        return self

    def SelectColumns(self, *names):  # csvplus.go:1039-1056
        if len(names) == 0:
            raise ValueError("empty header spec")
        h = {}
        for n in names:
            if n in h:
                raise ValueError("header spec: duplicate column name: " + n)
            h[n] = -1
        self.header, self.headerFromFirstRow = h, True
        return self

    def NumFields(self, n): self.numFields = n; return self
    def NumFieldsAuto(self): return self.NumFields(0)
    def NumFieldsAny(self): return self.NumFields(-1)

    def _options(self) -> dict:
        """the reader's options and header spec as keyword arguments of parse_csv"""
        return dict(delimiter=self.delimiter, comment=self.comment, num_fields=self.numFields, lazy_quotes=self.lazyQuotes,
                    trim_leading_space=self.trimLeadingSpace, header_from_first_row=self.headerFromFirstRow,
                    spec=list(self.header.items()) if self.header else [])

    def _batches(self, pred: Predicate | None = None):
        """-> (Table, DataSourceError | None, several) per batch, several: the input was pushed in more than one piece;
        the error comes with the last batch.  Host pieces go through cpb_stream_*: one piece is one push, parsed as one
        batch.  Closing the generator early stops reading the input."""
        pieces = iter(self._pieces())
        st = None
        try:
            piece, last = next(pieces, (None, True))
            if isinstance(piece, DeviceBuffer):  # device memory cannot be pushed: one cpb_parse_csv call
                t, err = parse_csv(self.ctx, piece, pred=pred, **self._options())
                yield t, err, False
                return
            st = _Stream(self.ctx, pred, **self._options())
            # one cpb_stream_next per push parses every complete record pushed so far.  A batch is delivered after the
            # next piece has been pushed: that piece's host-to-device copy (the stream's copy stream) overlaps what the
            # consumer does with the batch on the context's stream, and it is parsed only after the batch was delivered.
            # An iterator that ends without a last piece is closed by an empty last push.
            several = not last  # known from the first piece, so every batch, the first one included, reports it
            pending = None
            while True:
                st.push(piece, last)
                if pending is not None:
                    yield (*pending, several)
                    pending = None
                t, err, done = st.next()
                if t is not None or err is not None:
                    pending = (t, err)
                if last or done or err is not None:
                    break
                piece, last = next(pieces, (None, True))
            if pending is not None:
                yield (*pending, several)
        finally:
            if st is not None:
                st.free()
            close = getattr(pieces, "close", None)
            if close is not None:
                close()

    def Iterate(self, fn):  # csvplus.go:1080
        return Take(self)(fn)


class _Stream:
    """cpb_stream: one input parsed in batches of whole records"""

    def __init__(self, ctx: Context, pred: Predicate | None, spec: list | None = None, **opts):
        """opts: the reader options of parse_csv"""
        self.ctx, self._keep, self._pushed = ctx, [], None
        o = _reader_opts(**opts)
        sa, nspec, pp = _spec_and_pred(spec, pred, self._keep)  # the predicate is borrowed by the stream until it is freed
        self.h = C.c_void_p()
        ctx._call("cpb_stream_open", C.byref(o), sa, nspec, pp, C.byref(self.h))

    def push(self, piece, last: bool):
        if piece is None:
            ptr, n = None, 0
        else:
            a = piece if isinstance(piece, np.ndarray) else np.frombuffer(piece, np.uint8)
            ptr, n = a.ctypes.data, a.size
        self._pushed = piece  # untouched until the next cpb_stream_next returns
        self.ctx._call("cpb_stream_push", C.c_void_p(ptr), n, int(last), h=self.h)

    def next(self):
        h = C.c_void_p(); done = C.c_int(); e = _abi.Error()
        st = self.ctx._call("cpb_stream_next", C.byref(h), C.byref(done), err=e, accept=(_abi.CPB_ERR_DATA,), h=self.h)
        t, err = _rows_before_error(self.ctx, Table(self.ctx, h) if h.value else None, st, e)
        return t, err, bool(st or done.value)

    def free(self):
        if self.h:
            self.ctx.lib.cpb_stream_free(self.h)
            self.h = None


def _pinned_pieces(f, ctx: Context):
    """the pieces of the open file f, read by a helper thread into two pinned host buffers: piece k+1 is read while piece
    k is being parsed.  Closes f."""
    from concurrent.futures import ThreadPoolExecutor
    step = STREAM_BATCH_BYTES
    bufs = [HostBuffer(ctx, step), HostBuffer(ctx, step)]
    views = [b.array() for b in bufs]
    ex = ThreadPoolExecutor(1)
    try:
        with f:
            def fill(k):
                n, v = 0, memoryview(views[k])
                while n < step:
                    got = f.readinto(v[n:])
                    if not got:
                        break
                    n += got
                return n
            k = 0
            fut = ex.submit(fill, 0)
            while True:
                n = fut.result()
                if n == 0:
                    return
                # the other buffer held the piece before this one: its parse has returned by now
                fut = ex.submit(fill, k ^ 1) if n == step else None
                yield views[k][:n], fut is None
                if fut is None:
                    return
                k ^= 1
    finally:
        ex.shutdown(wait=True)
        for b in bufs:
            b.free()


def _reader_pieces(inp):
    """the pieces of an io reader, read with readinto (or read(n)); a piece is known to be the last one when it is short
    or the next one is empty"""
    step = STREAM_BATCH_BYTES

    def read_piece():
        a = np.empty(step, np.uint8)
        n = 0
        if hasattr(inp, "readinto"):
            v = memoryview(a)
            while n < step:
                got = inp.readinto(v[n:])
                if not got:
                    break
                n += got
        else:
            while n < step:
                b = inp.read(step - n)
                if not b:
                    break
                a[n:n + len(b)] = np.frombuffer(b, np.uint8); n += len(b)
        return a[:n]

    p = read_piece()
    while True:
        q = read_piece() if p.size == step else None
        last = q is None or q.size == 0
        yield p, last
        if last:
            return
        p = q


def FromFile(name: str, ctx: Context | None = None) -> Reader:  # csvplus.go:950
    """a regular file that fits one piece is read whole into pageable memory; a larger one is read by a helper thread
    into two pinned buffers; any other file (a FIFO, a character device) is read as FromReader reads it"""
    def pieces():
        try:
            f = open(name, "rb", buffering=0)
        except OSError as e:  # mapError's *os.PathError branch, csvplus.go:1216-1220
            raise DataSourceError(1, f"open: {e.strerror.lower() if e.strerror else e}") from None
        st = os.fstat(f.fileno())
        if not stat.S_ISREG(st.st_mode):
            return _closing(f, _reader_pieces(f))
        if st.st_size > STREAM_BATCH_BYTES:
            return _pinned_pieces(f, r.ctx)
        with f:
            return [(np.fromfile(f, dtype=np.uint8), True)]
    r = Reader(pieces, ctx)
    return r


def _closing(f, pieces):
    with f:
        yield from pieces


def FromReader(inp: io.IOBase, ctx: Context | None = None) -> Reader:  # csvplus.go:936
    return Reader(lambda: _reader_pieces(inp), ctx)


FromReadCloser = FromReader


def FromBytes(data, ctx: Context | None = None) -> Reader:
    """bytes / numpy / HostBuffer / DeviceBuffer already in memory.  Host memory is pushed in pieces of STREAM_BATCH_BYTES
    (one piece when it fits); a DeviceBuffer is parsed in one call."""
    def pieces():
        if isinstance(data, DeviceBuffer):
            return [(data, True)]
        if isinstance(data, HostBuffer):
            a = data.array()
        elif isinstance(data, np.ndarray):
            a = np.ascontiguousarray(data, np.uint8).reshape(-1)
        else:
            a = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.frombuffer(bytes(data), np.uint8)
        step = STREAM_BATCH_BYTES
        return ((a[i:i + step], i + step >= a.size) for i in range(0, max(a.size, 1), step))
    return Reader(pieces, ctx)


# ------------------------------------------------------------------ DataSource (csvplus.go:207-608)
class DataSource:
    """A lazily evaluated plan: source + operations.  Calling it with a RowFunc pulls the rows."""

    def __init__(self, source, ops: tuple = ()):
        self._src, self._ops = source, ops  # source: Reader | ("table", Table, line_base) | ("rows", list[Row])

    def _with(self, op) -> "DataSource":
        return DataSource(self._src, self._ops + (op,))

    # ---- combinators
    def Transform(self, trans): return self._with(("transform", trans))
    def Filter(self, pred): return self._with(("filter", pred))
    def Map(self, mf): return self._with(("map", mf))
    def Validate(self, vf): return self._with(("validate", vf))
    def Top(self, n: int): return self._with(("top", n))
    def Drop(self, n: int): return self._with(("drop", n))
    def TakeWhile(self, pred): return self._with(("takewhile", pred))
    def DropWhile(self, pred): return self._with(("dropwhile", pred))

    def MapTensors(self, inputs: dict, fn):
        """a device Map (an extension beyond the reference API, like ToTensors): inputs = {column: "int" | "float64"} are
        converted per batch as ToTensors converts them, fn(dict of CUDA tensors) returns {name: value} and each name is set
        as Table.with_column sets it (an int64 / float64 tensor with one value per row, a FormatFloat, a str).  fn is called
        once per non-empty batch and must be row-wise.  A conversion error (the lowest failing row, ties to the earlier
        input) ends the plan there like a source error: the rows before it flow on and the sink raises CsvPlusError with
        .row = the row's ordinal among the rows that reached the step."""
        return self._with(("maptensors", _tensor_kinds(inputs, "MapTensors"), fn))

    def FilterTensors(self, inputs: dict, fn):
        """a device Filter: as MapTensors, fn returns a bool CUDA tensor with one value per row; the rows where it is true
        are kept"""
        return self._with(("filtertensors", _tensor_kinds(inputs, "FilterTensors"), fn))

    def DropColumns(self, *columns):
        if len(columns) == 0:
            raise ValueError("no columns specified in DropColumns()")
        return self._with(("dropcols", columns))

    def SelectColumns(self, *columns):
        if len(columns) == 0:
            raise ValueError("no columns specified in SelectColumns()")
        return self._with(("select", columns))

    def Join(self, index: Index, *columns):
        if len(columns) > len(index.columns):
            raise ValueError("too many source columns in Join()")
        return self._with(("join", index, columns))

    def Except(self, index: Index, *columns):
        if len(columns) > len(index.columns):
            raise ValueError("too many source columns in Except()")
        return self._with(("except", index, columns))

    # ---- evaluation
    def _ctx(self) -> Context:
        s = self._src
        if isinstance(s, Reader):
            return s.ctx
        if s[0] == "table":
            return s[1].ctx
        return Context.default()

    def _batches(self):
        """-> (state, pending error, several) per batch of the source; state: ("table", Table | None) or ("rows", list[Row]).
        A Reader yields one batch per parsed batch (several: its input was pushed in more than one piece), every other
        source one.
        Top / Drop / TakeWhile / DropWhile carry their counters across batches; when one of them has pulled all it will
        ever deliver, the input is no longer read."""
        ops = list(self._ops)
        s = self._src
        carry: dict = {}
        if isinstance(s, Reader):
            pred = None
            # fused into the parse kernel, which extracts the predicate's columns beside every group of output columns
            # (CPB_MAX_PARSE_COLS at a time); a predicate over more columns filters the parsed table instead
            if (ops and ops[0][0] == "filter" and isinstance(ops[0][1], Predicate) and ops[0][1].lowerable()
                    and len(ops[0][1].columns()) < _abi.MAX_PARSE_COLS):
                pred = ops.pop(0)[1]
            src = s._batches(pred)
            try:
                for t, err, several in src:
                    state, err, stop = self._apply(("table", t), err, ops, carry)
                    yield state, err, several
                    if stop or err is not None:
                        return
            finally:
                src.close()
            return
        if s[0] == "table":
            state = ("table", s[1])
        else:
            state = ("rows", [dict(r) for r in s[1]])  # iterate() clones, csvplus.go:230
        state, err, _ = self._apply(state, None, ops, carry)
        yield state, err, False

    def _apply(self, state, err, ops, carry: dict):
        """the operations over one batch -> (state, err, stop); carry: per-operation state across batches"""
        ctx = self._ctx()
        stop = False
        for i, op in enumerate(ops):
            kind = op[0]
            device_ok = (kind in ("select", "dropcols", "join", "except", "top", "drop", "maptensors", "filtertensors")
                         or (kind in ("filter", "takewhile", "dropwhile") and isinstance(op[1], Predicate) and op[1].lowerable()))
            if device_ok:
                if state[0] == "rows":
                    state = ("table", Table.from_rows(ctx, state[1]) if state[1] else None)
                t = state[1]
                if t is None:
                    continue
                try:
                    if kind == "select": t = t.select(*op[1])
                    elif kind == "dropcols": t = t.drop(*op[1])
                    elif kind == "filter": t = t.filter(op[1])
                    elif kind == "join": t = t.join(op[1], *op[2])
                    elif kind == "except": t = t.join(op[1], *op[2], anti=True)
                    elif kind == "top":  # note: the reference pulls one extra row (SURVEY §Q8)
                        seen = carry.get(i, 0)
                        t = t.slice(0, min(len(t), max(0, op[1] - seen)))
                    elif kind == "drop":
                        seen = carry.get(i, 0)
                        t = t.slice(min(len(t), max(0, op[1] - seen)), len(t))
                        carry[i] = seen + len(state[1])
                    elif kind == "takewhile":  # csvplus.go:346-358: io.EOF at the first failing row — a later error is never met
                        cut = t.first_false(op[1])
                        if cut < len(t):
                            err = None; stop = True
                        t = t.slice(0, cut)
                    elif kind in ("maptensors", "filtertensors"):
                        seen = carry.get(i, 0)
                        carry[i] = seen + len(t)
                        t, step_err = _tensor_step(t, op, seen)
                        if step_err is not None:  # the rows before it flow on; the sink raises it as a source error
                            err = step_err; stop = True
                    elif kind == "dropwhile":  # :361-374
                        if carry.get(i, True):
                            k = t.first_false(op[1])
                            if k < len(t):
                                carry[i] = False
                            t = t.slice(k, len(t))
                except DataSourceError as e:
                    if err is None or kind in ("select", "join", "except"):
                        return ("rows", []), e, True
                    raise
                if kind == "top":
                    carry[i] = carry.get(i, 0) + len(state[1])
                    if carry[i] > op[1]:  # Top(n) pulls n+1 rows then stops (io.EOF): the failing record is never reached
                        err = None; stop = True
                state = ("table", t)
            else:
                rows = state[1].rows() if state[0] == "table" and state[1] is not None else (state[1] or [])
                out = []
                fn = op[1]
                dropping = carry.get(i, True)
                for r in rows:
                    if kind == "filter":
                        if fn(r): out.append(r)
                    elif kind == "map":
                        out.append(fn(r))
                    elif kind == "transform":
                        r2 = fn(r)
                        if r2: out.append(r2)
                    elif kind == "validate":
                        fn(r); out.append(r)
                    elif kind == "takewhile":
                        if not fn(r):
                            stop = True; err = None
                            break
                        out.append(r)
                    elif kind == "dropwhile":
                        dropping = dropping and fn(r)
                        if not dropping: out.append(r)
                carry[i] = dropping
                state = ("rows", out)
        return state, err, stop

    def _evaluate(self):
        """-> (state, pending error) of the whole plan: the batches' tables concatenated"""
        parts, err = [], None
        for state, err, _ in self._batches():
            parts.append(state)
        if len(parts) == 1:
            return parts[0], err
        t = _concat([self._as_table(st) for st in parts])
        return ("table", t), err

    def _as_table(self, state):
        if state[0] == "rows":
            return Table.from_rows(self._ctx(), state[1]) if state[1] else None
        return state[1]

    def _table(self) -> tuple:
        state, err = self._evaluate()
        return self._as_table(state), err

    def __call__(self, fn: Callable[[Row], None]):
        for state, err, _ in self._batches():  # each batch is delivered before the next one is parsed
            rows = state[1].rows() if state[0] == "table" and state[1] is not None else (state[1] or [])
            for r in rows:
                try:
                    fn(r)
                except StopIterationEOF:
                    return
            if err is not None:
                raise err

    # ---- sinks
    def ToRows(self) -> list[Row]:  # csvplus.go:483-490
        out = []
        self(out.append)
        return out

    def ToCsv(self, out: io.IOBase, *columns):  # csvplus.go:379-406
        if len(columns) == 0:
            raise ValueError("empty column list in ToCsv() function")
        wrote_header = False
        hold: list = []  # the pinned buffer every batch is serialised into
        try:
            for state, err, _ in self._batches():
                t = self._as_table(state)
                if t is not None:  # the csv.Writer writes the header once, before the first batch (csvplus.go:387)
                    _write_into(out, hold, t.ctx, lambda buf: t.to_csv_into(buf, 0, *columns, header=not wrote_header))
                elif not wrote_header:
                    out.write((",".join(columns) + "\n").encode())
                wrote_header = True
                if err is not None:
                    raise err
        finally:
            for b in hold:
                b.free()

    def ToCsvFile(self, name: str, *columns):  # csvplus.go:411-443: the file is removed on error
        with _new_file(name) as f:
            self.ToCsv(f, *columns)

    def ToJSON(self, out: io.IOBase):  # csvplus.go:446-474
        """all rows as a JSON array, formatted the way the reference's json.Encoder (SetEscapeHTML(false), no indent) writes
        it: `[`, then per row the object with its keys sorted and a newline, a `,` before every row but the first, `]`.
        A device table is serialised by the GPU in row-range batches; rows left on the host (after an opaque Map or
        Filter(func), or TakeRows of rows with different columns) are encoded here.  On a source error nothing is written
        when the input was pushed in one piece; an input pushed in several keeps what its batches wrote (a prefix of the
        array, without `]`), as the reference's encoder has flushed them."""
        hold: list = []  # the pinned buffer every batch is serialised into
        opened = False
        try:
            for state, err, several in self._batches():
                if err is not None and not several:
                    raise err
                if state[0] == "table":
                    if state[1] is not None and len(state[1]):
                        _json_batches(state[1], out, not opened, hold)
                        opened = True
                elif state[1]:
                    out.write(_json_rows(state[1], not opened, False))
                    opened = True
                if err is not None:
                    raise err
            out.write(b"]" if opened else b"[]")
        finally:
            for b in hold:
                b.free()

    def ToJSONFile(self, name: str):  # csvplus.go:477-479
        with _new_file(name) as f:
            self.ToJSON(f)

    def ToTensors(self, columns: dict) -> dict:
        """{name: "int" | "float64"} -> {name: CUDA tensor}: Row.ValueAsInt / ValueAsFloat64 of every row of each column,
        converted on the GPU (an extension beyond the reference API, like TakeTable).  The plan is evaluated once.  The
        error raised is the one a RowFunc converting the columns in dict order would meet first: the lowest failing row,
        ties to the earlier column (CsvPlusError, .row = the row).  When no row fails, a pending source error is raised:
        the table only holds the rows delivered before it."""
        kinds = _tensor_kinds(columns, "ToTensors")
        t, err = self._table()
        if t is None:
            import torch
            dev = torch.device("cuda", self._ctx().device)
            out = {name: torch.empty(0, dtype=torch.float64 if f else torch.int64, device=dev) for name, f in kinds.items()}
        else:
            out, first = _convert_all(t, kinds)
            if first is not None:
                raise first
        if err is not None:
            raise err
        return out

    def IndexOn(self, *columns) -> Index:  # csvplus.go:529-531
        return self._index(columns, False)

    def UniqueIndexOn(self, *columns) -> Index:  # csvplus.go:535-537
        return self._index(columns, True)

    def _index(self, columns, unique) -> Index:
        if len(columns) == 0:
            raise ValueError("empty column list in CreateIndex()")
        if len(set(columns)) != len(columns):
            raise ValueError("duplicate column name(s) in CreateIndex()")
        t, err = self._table()
        if err is not None:
            raise err
        if t is None:
            t = Table.from_rows(self._ctx(), [], list(columns))
        return t.index_on(*columns, unique=unique)


def _convert_all(t: Table, kinds: dict) -> tuple:
    """Table._convert of every input -> ({name: values}, CsvPlusError of the lowest failing row, ties to the earlier
    input, or None)"""
    vals, first = {}, None
    for name, is_float in kinds.items():
        values, _, e = t._convert(name, is_float)
        vals[name] = values
        if e is not None and (first is None or e.row < first.row):
            first = e
    return vals, first


def _tensor_step(t: Table, op, seen: int):
    """MapTensors / FilterTensors over one batch -> (table, CsvPlusError of the first failing conversion or None)"""
    kind, kinds, fn = op
    vals, first = _convert_all(t, kinds)
    err = None
    if first is not None:
        err = CsvPlusError(str(first), first.status, first.kind)
        err.row = seen + first.row
        t = t.slice(0, first.row)
        vals = {name: v[: first.row] for name, v in vals.items()}
    if len(t):
        res = fn(vals)
        if kind == "maptensors":
            if not isinstance(res, dict):
                raise TypeError(f"MapTensors: fn must return a dict of column values, got {type(res).__name__}")
            for name, value in res.items():
                t = t.with_column(name, value)
        else:
            t = t.filter_mask(res)
    return t, err


def _concat(tables: list) -> "Table | None":
    """the batches' tables as one (cpb_table_concat); None when no batch has a table"""
    parts = [t for t in tables if t is not None]
    if not parts:
        return None
    return parts[0] if len(parts) == 1 else Table.concat(parts)


def _json_rows(rows: list, first: bool, last: bool) -> bytes:
    """host rows as (a piece of) the JSON array: `[` when first, `,` before every other row, `]` when last"""
    parts = [b"["] if first else []
    for i, row in enumerate(rows):
        if i or not first:
            parts.append(b",")
        parts.append(b"{" + b",".join(_go_json_string(k) + b":" + _go_json_string(row[k]) for k in sorted(row, key=_enc)) + b"}\n")
    if last:
        parts.append(b"]")
    return b"".join(parts)


@contextlib.contextmanager
def _new_file(name: str):
    """name opened for writing; any error while it is written removes it.  A path that cannot be created raises the OS
    error and leaves nothing behind."""
    f = open(name, "wb")
    try:
        with f:
            yield f
    except BaseException:
        os.remove(name)
        raise


def _into(ctx: Context, name: str, *args, dst: "HostBuffer | None", offset: int = 0, size=None, more: tuple = ()) -> int:
    """an entry that writes into caller-owned host memory: args are followed by the room of dst from offset on (none when
    dst is None), the size out-parameter and more.  Returns the size the entry reports; when that exceeds the room the
    entry answered CPB_ERR_ARG and wrote nothing."""
    size = C.c_uint64() if size is None else size
    e = _abi.Error()
    ptr, cap = (dst.ptr + offset, dst.nbytes - offset) if dst is not None else (None, 0)
    st = ctx._call(name, *args, C.c_void_p(ptr), cap, C.byref(size), *more, err=e, accept=(_abi.CPB_ERR_ARG,))
    if st and size.value <= cap:
        _raise(st, e, ctx)
    return size.value


def _row_batches(n: int, step: int, write: Callable[[int, int], None]):
    """write(lo, hi) for row ranges of at most step rows that cover [0, n); a range that fails with CPB_E_TOO_LARGE is
    halved"""
    lo = 0
    while lo < n:
        hi = min(n, lo + step)
        try:
            write(lo, hi)
        except CsvPlusError as e:
            if e.kind != _abi.CPB_E_TOO_LARGE or hi - lo < 2:
                raise
            step = (hi - lo) // 2
            continue
        lo = hi


def _write_into(out: io.IOBase, hold: list, ctx: Context, serialise: Callable[["HostBuffer | None"], int]):
    """serialise(buf) writes one batch into the pinned buffer buf and returns its size, or writes nothing when the size
    exceeds buf (or buf is None).  The buffer hold[0] is grown to the size reported and the batch serialised again, then
    the batch is written to out; hold keeps the buffer for the next batch (the caller frees it)."""
    while True:
        buf = hold[0] if hold else None
        n = serialise(buf)
        if n <= (buf.nbytes if buf is not None else 0):
            if n:
                out.write(memoryview(buf.array()[:n]))
            return
        if buf is not None:
            buf.free()
        hold[:] = [HostBuffer(ctx, n + n // 4 + 64)]


def _json_batches(t: Table, out: io.IOBase, first: bool, hold: list):
    """ToJSON of a device table with rows, without the closing `]`: row-range slices of at most JSON_BATCH_ROWS rows, each
    written through the pinned buffer of hold (_write_into).  first: the table opens the array."""
    n = len(t)

    def write(lo, hi):
        part = t if (lo, hi) == (0, n) else t.slice(lo, hi)
        _write_into(out, hold, t.ctx, lambda buf: part.to_json_into(buf, 0, first and lo == 0, False))
    _row_batches(n, JSON_BATCH_ROWS, write)


def Take(src) -> DataSource:  # csvplus.go:252-256
    if isinstance(src, Reader):
        return DataSource(src)
    if isinstance(src, Index):
        return TakeTable(src.table(), line_base=0)
    raise TypeError("Take() needs a Reader or an Index")


def TakeRows(rows: list[Row]) -> DataSource:  # csvplus.go:218-222
    return DataSource(("rows", rows))


def TakeTable(t: Table, line_base: int = 0) -> DataSource:
    return DataSource(("table", t, line_base))
