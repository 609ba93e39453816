"""With a live context, every entry point that takes a table, an index or an out-parameter answers a null one with
CPB_ERR_ARG, leaves the reason in cpb_last_error, and never hands back a stale cpb_error.  These are host-side argument
checks: every call here is refused before it reaches the device."""
import ctypes as C
import re

import pytest

import csvplus_b200 as cp
from csvplus_b200 import _abi
from tests.test_abi_args_cpu import ENTRIES, null_args

pytestmark = pytest.mark.gpu

# entries for which null / zero arguments after the context (and the table or index) are a valid call, or that do not
# return a status
VALID_WITH_NULLS = {"cpb_sync", "cpb_pool_reserve", "cpb_host_free", "cpb_device_free", "cpb_memcpy_h2d", "cpb_memcpy_d2h",
                    "cpb_stats_enable", "cpb_stats_reset", "cpb_table_fetch_column", "cpb_index_dedup_apply", "cpb_index_dedup_apply2",
                    "cpb_shutdown", "cpb_ctx_stream", "cpb_last_error", "cpb_comm_size", "cpb_comm_rank", "cpb_kernel_launches",
                    "cpb_host_syncs"}
CTX_ENTRIES = sorted(n for n, params in ENTRIES.items() if params.lstrip().startswith("cpb_ctx*") and n not in VALID_WITH_NULLS)


@pytest.fixture(scope="module")
def ctx():
    c = cp.Context(0)
    yield c
    c.close()


def refused(ctx, name, args):
    """calls the entry with a dirty cpb_error where it takes one; -> the text it left in cpb_last_error"""
    fn = getattr(ctx.lib, name)
    e = None
    if fn.argtypes[-1] is C.POINTER(_abi.Error):
        e = _abi.Error(kind=7, column_index=3, line=99, has_line=1, msg=b"stale")
        args = args[:-1] + [C.byref(e)]
    launches, syncs = ctx.kernel_launches(), ctx.host_syncs()
    assert fn(*args) == _abi.CPB_ERR_ARG, name
    assert (ctx.kernel_launches(), ctx.host_syncs()) == (launches, syncs), name
    text = ctx.lib.cpb_last_error(ctx.h)
    assert text, name
    if e is not None:
        assert (e.kind, e.line, e.has_line) == (0, 0, 0) and e.msg == text, (name, e.msg)
    return text


@pytest.mark.parametrize("name", CTX_ENTRIES)
def test_null_arguments_after_the_context(ctx, name):
    args = null_args(getattr(ctx.lib, name))
    args[0] = ctx.h
    refused(ctx, name, args)


def handle_params(name) -> dict:
    """position -> "table" | "index" of the parameters that are one table or one index handle"""
    found = {}
    for i, param in enumerate(ENTRIES[name].split(",")):
        m = re.fullmatch(r"\s*(?:const\s+)?cpb_(table|index)\*\s*\w+\s*", param)
        if m:
            found[i] = m.group(1)
    return found


@pytest.mark.parametrize("name", [n for n in CTX_ENTRIES if handle_params(n)])
def test_null_out_parameter_beside_live_handles(ctx, name):
    t = cp.Table.from_rows(ctx, [{"k": "1", "v": "a"}, {"k": "2", "v": "b"}], ["k", "v"])
    ix = t.index_on("k")
    live = {"table": t.h, "index": ix.h}
    args = null_args(getattr(ctx.lib, name))
    args[0] = ctx.h
    for i, kind in handle_params(name).items():
        args[i] = live[kind]
    assert refused(ctx, name, args) not in (b"null table", b"null index")
    assert len(t) == 2 and len(ix) == 2


def test_accessors_check_their_out_pointers(ctx):
    t = cp.Table.from_rows(ctx, [{"k": "1"}], ["k"])
    ix = t.index_on("k")
    po = C.c_void_p()
    assert ctx.lib.cpb_table_col_name(t.h, 0, None) == _abi.CPB_ERR_ARG
    assert ctx.lib.cpb_index_key_col(ix.h, 0, None) == _abi.CPB_ERR_ARG
    assert ctx.lib.cpb_table_column_device(t.h, 0, None, C.byref(po)) == _abi.CPB_ERR_ARG
    assert ctx.lib.cpb_table_column_device(t.h, 0, C.byref(po), None) == _abi.CPB_ERR_ARG
    parts = (C.c_void_p * 2)(t.h, None)
    out = C.c_void_p()
    assert ctx.lib.cpb_table_concat(ctx.h, parts, 2, C.byref(out)) == _abi.CPB_ERR_ARG and not out.value
