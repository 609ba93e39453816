"""ctypes prototypes for include/csvplus_b200.h.  Loading fails loudly when the CUDA library is
missing: there is no CPU fallback anywhere in this package."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("CPB_LIB", os.path.join(HERE, "libcsvplus_b200.so"))  # CPB_LIB: A/B builds of the same ABI

# the header's limits (tests check that these equal its #defines)
MAX_PARSE_COLS = 16  # CPB_MAX_PARSE_COLS
PRED_MAX_TERMS = 32  # CPB_PRED_MAX_TERMS
PRED_MAX_OPS = 64    # CPB_PRED_MAX_OPS
PRED_MAX_DEPTH = 48  # CPB_PRED_MAX_DEPTH
PRED_SET_MIN = 33    # CPB_PRED_SET_MIN
# the cpb_status and cpb_err_kind values the host layer tells apart (tests check them against the header's enums)
CPB_ERR_DATA = 1
CPB_ERR_ARG = 2
CPB_ERR_UNSUPPORTED = 4
CPB_E_MISSING_COLUMN = 10
CPB_E_TOO_LARGE = 13
CPB_E_BAD_CODE = 19
# GroupBy aggregates (cpb_agg): ops and input kinds
CPB_AGG_OPS = {"count": 0, "sum": 1, "min": 2, "max": 3, "first": 4, "last": 5}
CPB_AGG_KINDS = {"int": 0, "float64": 1}
# OrderBy key kinds (cpb_order_key)
CPB_ORDER_KINDS = {"str": 0, "int": 1, "float64": 2}
MAX_ORDER_KEYS = 16  # the most keys of one cpb_table_order_by


class Str(C.Structure):
    _fields_ = [("ptr", C.c_char_p), ("len", C.c_uint64)]


class Error(C.Structure):
    _fields_ = [("kind", C.c_int32), ("column_index", C.c_int32), ("line", C.c_uint64), ("has_line", C.c_int32),
                ("_pad", C.c_int32), ("msg", C.c_char * 488)]


class ReaderOpts(C.Structure):
    _fields_ = [("delimiter", C.c_uint32), ("comment", C.c_uint32), ("num_fields", C.c_int32),
                ("lazy_quotes", C.c_uint8), ("trim_leading_space", C.c_uint8), ("header_from_first_row", C.c_uint8),
                ("_pad", C.c_uint8)]


class HeaderCol(C.Structure):
    _fields_ = [("name", Str), ("index", C.c_int32), ("_pad", C.c_int32)]


class Pred(C.Structure):
    pass


Pred._fields_ = [("op", C.c_int32), ("n", C.c_int32), ("keys", C.POINTER(Str)), ("values", C.POINTER(Str)),
                 ("children", C.POINTER(C.POINTER(Pred)))]


class Agg(C.Structure):
    _fields_ = [("op", C.c_int32), ("kind", C.c_int32), ("column", Str)]


class OrderKey(C.Structure):
    _fields_ = [("column", Str), ("kind", C.c_int32), ("descending", C.c_int32)]


class KStat(C.Structure):
    _fields_ = [("name", C.c_char * 48), ("launches", C.c_uint64), ("ms", C.c_double), ("algo_bytes", C.c_uint64)]


# every symbol include/csvplus_b200.h declares (tests check the library exports all of them)
SYMBOLS = [
    "cpb_abi_version", "cpb_init", "cpb_shutdown", "cpb_ctx_stream", "cpb_sync", "cpb_pool_reserve", "cpb_pool_used_high", "cpb_last_error",
    "cpb_host_alloc", "cpb_host_free", "cpb_device_alloc", "cpb_device_free", "cpb_memcpy_h2d", "cpb_memcpy_d2h",
    "cpb_parse_csv", "cpb_stream_open", "cpb_stream_push", "cpb_stream_next", "cpb_stream_free", "cpb_csv_stream_cut",
    "cpb_csv_quote_parity", "cpb_parse_csv_shard", "cpb_table_col_field", "cpb_table_record_fields",
    "cpb_table_num_rows", "cpb_table_num_cols", "cpb_table_col_name", "cpb_table_find_col", "cpb_table_col_bytes",
    "cpb_table_fetch_column", "cpb_table_column_device", "cpb_table_from_host", "cpb_table_from_device",
    "cpb_table_concat", "cpb_table_select", "cpb_table_drop", "cpb_table_filter", "cpb_table_first_false", "cpb_table_slice",
    "cpb_table_free",
    "cpb_index_build", "cpb_index_num_rows", "cpb_index_num_keys", "cpb_index_table", "cpb_index_find", "cpb_index_sub",
    "cpb_index_dup_groups", "cpb_index_dedup_apply", "cpb_index_dedup_apply2", "cpb_free", "cpb_index_free",
    "cpb_index_key_col", "cpb_index_gob_begin", "cpb_index_gob_into", "cpb_index_load_gob",
    "cpb_join", "cpb_except", "cpb_left_join", "cpb_table_to_csv", "cpb_table_to_csv_device", "cpb_table_to_csv_into",
    "cpb_table_to_json", "cpb_table_to_json_device", "cpb_table_to_json_into",
    "cpb_table_column_as_int64", "cpb_table_column_as_float64", "cpb_table_column_as_float32",
    "cpb_table_set_int64", "cpb_table_set_float64", "cpb_table_set_float32", "cpb_table_set_literal", "cpb_table_filter_flags",
    "cpb_table_column_codes", "cpb_table_set_codes", "cpb_table_set_sprintf", "cpb_table_sprintf_into",
    "cpb_groups_open", "cpb_groups_push", "cpb_groups_result", "cpb_groups_values", "cpb_groups_free",
    "cpb_table_order_by",
    "cpb_comm_unique_id", "cpb_comm_init_rank", "cpb_init_multi", "cpb_comm_size", "cpb_comm_rank", "cpb_allgather_table",
    "cpb_allgather_tables", "cpb_allgather_u64", "cpb_allgather_layout",
    "cpb_stats_enable", "cpb_stats_reset", "cpb_stats_get", "cpb_kernel_launches", "cpb_host_syncs", "cpb_gen_csv",
]

_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: build it with `python -m csvplus_b200.build` "
                           "(csvplus_b200 has no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, i64, u64, i32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_int
    P = C.POINTER
    sig = {
        "cpb_abi_version": (i32, []),
        "cpb_init": (i32, [i32, P(vp)]),
        "cpb_shutdown": (None, [vp]),
        "cpb_ctx_stream": (vp, [vp]),
        "cpb_sync": (i32, [vp]),
        "cpb_pool_reserve": (i32, [vp, u64]),
        "cpb_last_error": (C.c_char_p, [vp]),
        "cpb_pool_used_high": (i32, [vp, i32, P(u64)]),
        "cpb_host_alloc": (i32, [vp, u64, P(vp)]),
        "cpb_host_free": (i32, [vp, vp]),
        "cpb_device_alloc": (i32, [vp, u64, P(vp)]),
        "cpb_device_free": (i32, [vp, vp]),
        "cpb_memcpy_h2d": (i32, [vp, vp, vp, u64]),
        "cpb_memcpy_d2h": (i32, [vp, vp, vp, u64]),
        "cpb_parse_csv": (i32, [vp, vp, u64, i32, P(ReaderOpts), P(HeaderCol), i32, P(Pred), P(vp), P(Error)]),
        "cpb_stream_open": (i32, [vp, P(ReaderOpts), P(HeaderCol), i32, P(Pred), P(vp), P(Error)]),
        "cpb_stream_push": (i32, [vp, vp, u64, i32]),
        "cpb_stream_next": (i32, [vp, P(vp), P(i32), P(Error)]),
        "cpb_stream_free": (None, [vp]),
        "cpb_csv_stream_cut": (i32, [vp, vp, u64, i32, P(ReaderOpts), P(u64)]),
        "cpb_table_col_field": (i32, [vp, i32]),
        "cpb_table_record_fields": (i32, [vp]),
        "cpb_csv_quote_parity": (i32, [vp, vp, u64, i32, P(C.c_uint32)]),
        "cpb_parse_csv_shard": (i32, [vp, vp, u64, i32, u64, i32, i32, C.c_uint32, P(ReaderOpts), P(HeaderCol), i32, P(Pred), P(vp),
                                      P(u64), P(Error)]),
        "cpb_table_num_rows": (i64, [vp]),
        "cpb_table_num_cols": (i32, [vp]),
        "cpb_table_col_name": (i32, [vp, i32, P(Str)]),
        "cpb_table_find_col": (i32, [vp, Str]),
        "cpb_table_col_bytes": (i32, [vp, vp, i32, i64, i64, P(u64)]),
        "cpb_table_fetch_column": (i32, [vp, vp, i32, i64, i64, vp, vp, u64]),
        "cpb_table_column_device": (i32, [vp, i32, P(vp), P(vp)]),
        "cpb_table_from_host": (i32, [vp, i32, P(Str), P(vp), P(vp), i64, P(vp)]),
        "cpb_table_from_device": (i32, [vp, i32, P(Str), P(vp), P(vp), i64, P(vp)]),
        "cpb_table_concat": (i32, [vp, P(vp), i32, P(vp)]),
        "cpb_table_select": (i32, [vp, vp, P(Str), i32, P(vp), P(Error)]),
        "cpb_table_drop": (i32, [vp, vp, P(Str), i32, P(vp)]),
        "cpb_table_filter": (i32, [vp, vp, P(Pred), P(vp)]),
        "cpb_table_first_false": (i32, [vp, vp, P(Pred), P(i64)]),
        "cpb_table_slice": (i32, [vp, vp, i64, i64, P(vp)]),
        "cpb_table_free": (None, [vp]),
        "cpb_index_build": (i32, [vp, vp, P(Str), i32, i32, P(vp), P(Error)]),
        "cpb_index_num_rows": (i64, [vp]),
        "cpb_index_num_keys": (i32, [vp]),
        "cpb_index_table": (i32, [vp, vp, P(vp)]),
        "cpb_index_find": (i32, [vp, vp, P(Str), i32, P(vp)]),
        "cpb_index_sub": (i32, [vp, vp, P(Str), i32, P(vp)]),
        "cpb_index_dup_groups": (i32, [vp, vp, P(i64), P(P(i64)), P(P(i64))]),
        "cpb_index_dedup_apply": (i32, [vp, vp, i64, P(i64), i32]),
        "cpb_index_dedup_apply2": (i32, [vp, vp, i64, P(i64), vp, i32, P(Error)]),
        "cpb_free": (None, [vp]),
        "cpb_index_free": (None, [vp]),
        "cpb_index_key_col": (i32, [vp, i32, P(Str)]),
        "cpb_index_gob_begin": (i32, [vp, vp, vp, u64, P(u64), P(u64), P(Error)]),
        "cpb_index_gob_into": (i32, [vp, vp, i64, i64, vp, u64, P(u64), P(Error)]),
        "cpb_index_load_gob": (i32, [vp, vp, u64, P(vp), P(Error)]),
        "cpb_join": (i32, [vp, vp, vp, P(Str), i32, P(vp), P(Error)]),
        "cpb_except": (i32, [vp, vp, vp, P(Str), i32, P(vp), P(Error)]),
        "cpb_left_join": (i32, [vp, vp, vp, P(Str), i32, P(vp), P(Error)]),
        "cpb_table_to_csv": (i32, [vp, vp, P(Str), i32, P(vp), P(u64), P(Error)]),
        "cpb_table_to_csv_device": (i32, [vp, vp, P(Str), i32, P(vp), P(u64), P(Error)]),
        "cpb_table_to_csv_into": (i32, [vp, vp, P(Str), i32, i32, vp, u64, P(u64), P(Error)]),
        "cpb_table_to_json": (i32, [vp, vp, i32, i32, P(vp), P(u64), P(Error)]),
        "cpb_table_to_json_device": (i32, [vp, vp, i32, i32, P(vp), P(u64), P(Error)]),
        "cpb_table_to_json_into": (i32, [vp, vp, i32, i32, vp, u64, P(u64), P(Error)]),
        "cpb_table_column_as_int64": (i32, [vp, vp, Str, vp, vp, P(u64), P(Error)]),
        "cpb_table_column_as_float64": (i32, [vp, vp, Str, vp, vp, P(u64), P(Error)]),
        "cpb_table_column_as_float32": (i32, [vp, vp, Str, vp, vp, P(u64), P(Error)]),
        "cpb_table_set_int64": (i32, [vp, vp, Str, vp, P(vp), P(Error)]),
        "cpb_table_set_float64": (i32, [vp, vp, Str, vp, C.c_char, i32, P(vp), P(Error)]),
        "cpb_table_set_float32": (i32, [vp, vp, Str, vp, C.c_char, i32, P(vp), P(Error)]),
        "cpb_table_set_literal": (i32, [vp, vp, Str, Str, P(vp), P(Error)]),
        "cpb_table_filter_flags": (i32, [vp, vp, vp, P(vp), P(Error)]),
        "cpb_table_column_codes": (i32, [vp, vp, Str, vp, P(vp), P(Error)]),
        "cpb_table_set_codes": (i32, [vp, vp, Str, vp, vp, P(vp), P(Error)]),
        "cpb_table_set_sprintf": (i32, [vp, vp, Str, Str, P(Str), i32, P(vp), P(Error)]),
        "cpb_table_sprintf_into": (i32, [vp, vp, Str, P(Str), i32, vp, u64, P(u64), P(Error)]),
        "cpb_groups_open": (i32, [vp, P(Str), i32, P(Agg), i32, P(vp)]),
        "cpb_groups_push": (i32, [vp, vp, vp, P(Error)]),
        "cpb_groups_result": (i32, [vp, vp, P(vp), P(u64)]),
        "cpb_groups_values": (i32, [vp, vp, i32, vp]),
        "cpb_groups_free": (i32, [vp, vp]),
        "cpb_table_order_by": (i32, [vp, vp, P(OrderKey), i32, u64, vp, P(vp), P(Error)]),
        "cpb_comm_unique_id": (i32, [vp]),
        "cpb_comm_init_rank": (i32, [vp, i32, i32, vp]),
        "cpb_init_multi": (i32, [P(i32), i32, P(vp)]),
        "cpb_comm_size": (i32, [vp]),
        "cpb_comm_rank": (i32, [vp]),
        "cpb_allgather_table": (i32, [vp, vp, P(vp)]),
        "cpb_allgather_tables": (i32, [P(vp), P(vp), i32, P(vp)]),
        "cpb_allgather_u64": (i32, [vp, P(u64), i32, P(u64)]),
        "cpb_allgather_layout": (i32, [i32, i32, P(u64), P(u64), P(u64)]),
        "cpb_stats_enable": (i32, [vp, i32]),
        "cpb_stats_reset": (i32, [vp]),
        "cpb_stats_get": (i32, [vp, P(KStat), i32, P(i32)]),
        "cpb_kernel_launches": (u64, [vp]),
        "cpb_host_syncs": (u64, [vp]),
        "cpb_gen_csv": (i32, [vp, i32, u64, u64, u64, u64, u64, i32, i32, vp, u64, P(u64)]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L
