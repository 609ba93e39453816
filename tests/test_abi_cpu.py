"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads, and exports every
symbol include/csvplus_b200.h declares; without a GPU every compute entry fails loudly (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_build_and_symbols():
    import __graft_entry__ as g
    g.build()
    from csvplus_b200 import _abi
    L = _abi.load()
    hdr = open(os.path.join(ROOT, "include", "csvplus_b200.h")).read()
    declared = set(re.findall(r"\b(cpb_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_abi.SYMBOLS), declared ^ set(_abi.SYMBOLS)
    for s in declared:
        assert hasattr(L, s), s
    assert L.cpb_abi_version() == 1


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import csvplus_b200 as cp
    with pytest.raises(cp.CsvPlusError, match="no CPU fallback"):
        cp.Context(0)
    with pytest.raises(cp.CsvPlusError):
        cp.Take(cp.FromBytes(b"a,b\n1,2\n")).ToRows()


def test_product_never_imports_oracle():
    for root, _, files in os.walk(os.path.join(ROOT, "csvplus_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h")):
                src = open(os.path.join(root, f), errors="replace").read()
                assert "oracle" not in src.lower() or f == "api.py" and "oracle" not in src, f


def test_struct_layouts_match_header():
    from csvplus_b200 import _abi
    assert C.sizeof(_abi.Error) == 512
    assert C.sizeof(_abi.ReaderOpts) == 16
    assert C.sizeof(_abi.HeaderCol) == 24
    assert C.sizeof(_abi.KStat) == 72
    assert C.sizeof(_abi.Pred) == 32


def test_host_mirrors_use_only_declared_abi():
    """The Go package (never compiled: no toolchain in the image) and the C++ mirror may only name entry points, types
    and constants include/csvplus_b200.h declares — the one check a missing compiler leaves possible for go/csvplus."""
    hdr = open(os.path.join(ROOT, "include", "csvplus_b200.h")).read()
    funcs = set(re.findall(r"\b(cpb_[a-z0-9_]+)\s*\(", hdr))
    types = set(re.findall(r"\b(cpb_[a-z0-9_]+)\b", hdr)) - funcs
    consts = set(re.findall(r"\b(CPB_[A-Z0-9_]+)\b", hdr))
    used_f, used_c = set(), set()
    for root, names in ((os.path.join(ROOT, "go", "csvplus"), None), (os.path.join(ROOT, "host"), None)):
        for f in sorted(os.listdir(root)):
            if not f.endswith((".go", ".hpp", ".cpp")):
                continue
            src = open(os.path.join(root, f), errors="replace").read()
            if f.endswith(".go"):
                ids = set(re.findall(r"\bC\.(cpb_[a-z0-9_]+|CPB_[A-Z0-9_]+)\b", src))
                calls = {i for i in ids if i.startswith("cpb_") and re.search(r"\bC\.%s\s*\(" % re.escape(i), src)}
                used_f |= {c for c in calls if c not in types}  # C.cpb_str(...) style conversions name types
                used_c |= {i for i in ids if i.startswith("CPB_")}
                missing_types = {i for i in ids if i.startswith("cpb_") and i not in funcs and i not in types}
                assert not missing_types, (f, missing_types)
            else:
                used_f |= set(re.findall(r"\b(cpb_[a-z0-9_]+)\s*\(", src)) - types
                used_c |= {c for c in re.findall(r"\b(CPB_[A-Z0-9_]+)\b", src) if not c.endswith("_")}  # ("CPB_PRED_*" in a comment)
    assert used_f <= funcs, used_f - funcs
    assert used_c <= consts, used_c - consts
    # and the Go layer reaches every name BASELINE.json's north_star lists
    go = "".join(open(os.path.join(ROOT, "go", "csvplus", f)).read() for f in os.listdir(os.path.join(ROOT, "go", "csvplus")))
    for name in ("FromFile", "SelectColumns", "Take", "Filter", "Map", "Like", "IndexOn", "UniqueIndexOn", "Join", "ToCsv"):
        assert re.search(r"\bfunc\s+(\([^)]*\)\s*)?%s\b" % name, go), name
