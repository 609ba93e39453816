"""Plain-Python restatement of categorical codes (pandas.factorize(sort=False)) over bytes: each value's code is the
number of distinct values seen before its first appearance, and the dictionary lists the values in that order.  Values
are compared as bytes, nothing else."""
from __future__ import annotations

import numpy as np


def factorize(values: list) -> tuple:
    """values (bytes) -> (codes, dictionary): codes[r] = d.setdefault(values[r], len(d)) over the rows in order"""
    d: dict = {}
    codes = [d.setdefault(bytes(v), len(d)) for v in values]
    return codes, list(d)


def factorize_ids(ids: np.ndarray) -> tuple:
    """the same renumbering of integer value ids (equal ids = equal values; large columns built from a known set of
    distinct values): -> (codes int64[n], the ids of the dictionary rows in code order)"""
    ids = np.asarray(ids, np.int64)
    if ids.size == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    uniq, first = np.unique(ids, return_index=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty(uniq.size, np.int64)
    rank[order] = np.arange(uniq.size)
    return rank[np.searchsorted(uniq, ids)], uniq[order]


def column_of(dict_bytes: list, ids: np.ndarray) -> tuple:
    """(offsets int64[n+1], data uint8[]) of the column whose row r holds dict_bytes[ids[r]], built with numpy"""
    lens_d = np.array([len(v) for v in dict_bytes], np.int64)
    doff = np.zeros(len(dict_bytes) + 1, np.int64)
    np.cumsum(lens_d, out=doff[1:])
    ddata = np.frombuffer(b"".join(dict_bytes) + b"\0", np.uint8)
    ids = np.asarray(ids, np.int64)
    lens = lens_d[ids]
    off = np.zeros(ids.size + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    total = int(off[-1])
    src = np.repeat(doff[ids] - off[:-1], lens) + np.arange(total, dtype=np.int64)
    return off, ddata[src]
