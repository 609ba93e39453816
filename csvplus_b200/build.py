"""Builds csvplus_b200/libcsvplus_b200.so (sm_90a only, i.e. H100) in-tree with nvcc.

    python -m csvplus_b200.build [--force]

The .so and the objects under _obj/ are build products and git-ignored.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libcsvplus_b200.so")
SOURCES = ["abi.cu", "parse.cu", "parse_general.cu", "gather.cu", "sort.cu", "join.cu", "write.cu", "json.cu", "gen.cu", "comm.cu", "subst.cu"]
HEADERS = ["core.hpp", "util.cuh", "pred.cuh", "parse_kernels.cuh", "subst.hpp", os.path.join("..", "..", "include", "csvplus_b200.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "--extended-lambda"]


def _mtime(p):
    return os.path.getmtime(p) if os.path.exists(p) else 0.0


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    hdr_time = max(_mtime(os.path.join(CSRC, h)) for h in HEADERS)
    jobs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        if force or _mtime(obj) < max(_mtime(src), hdr_time):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [NVCC, *FLAGS, "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for out in ex.map(compile_one, jobs):
                if verbose and out:
                    print(out)
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or not os.path.exists(LIB):
        r = subprocess.run([NVCC, "-shared", "-cudart", "static", "-o", LIB, *objs, "-ldl"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
