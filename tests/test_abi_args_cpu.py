"""The C ABI answers a null context or a null handle with CPB_ERR_ARG (or the accessor's documented -1 / empty value)
instead of dereferencing it.  No device is needed: a null context is refused before anything touches CUDA.  The entry
points come from include/csvplus_b200.h, so a new one is covered without an edit here."""
import ctypes as C
import os
import re

import pytest

from csvplus_b200 import _abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "csvplus_b200.h")).read()
# name -> parameter list of every declaration (a return type at the start of a line, then the name test_abi_cpu.py's
# expression finds; test_entries_cover_the_header checks that the two agree)
ENTRIES = {m.group(1): m.group(2) for m in re.finditer(r"^[a-z][a-z0-9_ ]*\*?\s+(cpb_[a-z0-9_]+)\s*\(([^)]*)\)", HEADER, re.M)}
HANDLE = re.compile(r"^\s*(const\s+)?cpb_(ctx|table|index|stream)\s*\*")
# what an entry that does not return a cpb_status answers for a null handle
NOT_A_STATUS = {"cpb_ctx_stream": None, "cpb_last_error": b"", "cpb_kernel_launches": 0, "cpb_host_syncs": 0, "cpb_comm_size": 1,
                "cpb_comm_rank": 0, "cpb_table_num_rows": -1, "cpb_table_num_cols": -1, "cpb_table_find_col": -1,
                "cpb_table_col_field": -1, "cpb_table_record_fields": -1, "cpb_index_num_rows": -1, "cpb_index_num_keys": -1,
                "cpb_shutdown": None, "cpb_table_free": None, "cpb_index_free": None, "cpb_stream_free": None}


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    return _abi.load()


def null_args(fn) -> list:
    """null / zero for every parameter of a ctypes prototype"""
    return [a() if issubclass(a, C.Structure) else b"\0" if a is C.c_char else None if issubclass(a, (C._Pointer, C.c_void_p)) else 0
            for a in fn.argtypes]


def test_header_enum_values_match_abi_constants():
    values = dict(re.findall(r"\b(CPB_E(?:RR)?_[A-Z_]+)\s*=\s*(\d+)", HEADER))
    for name in ("CPB_ERR_DATA", "CPB_ERR_ARG", "CPB_E_MISSING_COLUMN", "CPB_E_TOO_LARGE"):
        assert getattr(_abi, name) == int(values[name]), name


def test_entries_cover_the_header():
    assert set(ENTRIES) == set(_abi.SYMBOLS)
    with_handle = [n for n, params in ENTRIES.items() if HANDLE.match(params)]
    assert len(with_handle) >= 75 and set(NOT_A_STATUS) <= set(with_handle)


@pytest.mark.parametrize("name", sorted(n for n, params in ENTRIES.items() if HANDLE.match(params)))
def test_null_handle_is_refused(lib, name):
    fn = getattr(lib, name)
    got = fn(*null_args(fn))
    assert got == NOT_A_STATUS.get(name, _abi.CPB_ERR_ARG), (name, got)


@pytest.mark.parametrize("name", ["cpb_init", "cpb_comm_unique_id", "cpb_init_multi", "cpb_allgather_tables", "cpb_allgather_layout"])
def test_null_arguments_without_a_handle_are_refused(lib, name):
    fn = getattr(lib, name)
    assert fn(*null_args(fn)) == _abi.CPB_ERR_ARG


def test_dirty_error_is_cleared_for_a_null_context(lib):
    for name in sorted(ENTRIES):
        fn = getattr(lib, name)
        if not fn.argtypes or fn.argtypes[-1] is not C.POINTER(_abi.Error) or not ENTRIES[name].lstrip().startswith("cpb_ctx"):
            continue
        e = _abi.Error(kind=7, column_index=3, line=99, has_line=1, msg=b"stale")
        assert fn(*null_args(fn)[:-1], C.byref(e)) == _abi.CPB_ERR_ARG, name
        assert (e.kind, e.column_index, e.line, e.has_line, e.msg) == (0, -1, 0, 0, b""), name
