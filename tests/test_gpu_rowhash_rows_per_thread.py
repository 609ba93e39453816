"""GPU parity of the row-carrying hash table's build (rowhash_scatter) and probe (rowhash_probe) where rows meet at a
warp's edges: row counts that are not multiples of the warp or of 128 rows, probes whose rows l, l + 32, l + 64, l + 96
of a block of 128 land in one region (hits, misses and walks past the region's last slot), and duplicate and
overflowing builds whose equal keys or crowded region lie in those rows, against the oracle."""
import random

import numpy as np
import pytest

from oracle import oracle as orc
from tests.hash_ref import first_slots
from tests.test_gpu_rowhash_build import _check, _customers, _index_csv, _layout, _orders, _parse

pytestmark = pytest.mark.gpu

def _by_lane(groups):
    """rows of blocks of 128 in which rows l, l + 32, l + 64, l + 96 are the four keys of groups[l]"""
    out = []
    for b in range(0, len(groups), 32):
        blk = groups[b:b + 32]
        out += [g[u] for u in range(4) for g in blk]
    return out


@pytest.mark.parametrize("n_build,n_probe", [(2, 1), (31, 33), (33, 31), (4097, 4097), (1_000_003, 33), (4097, 1_000_003)])
def test_row_counts(n_build, n_probe):
    # (an index of one row is sorted, not hashed: the smallest build here has two)
    _check(_customers(n_build), _orders(n_probe, n_build + n_build // 10 + 1), key="id", pkey="id")


def _region_keys(n, ncand):
    """keys of an n-row index by region: for each region, keys whose first slot is its last slot (they walk past it to
    the region's first slot) and keys whose first slot is its first"""
    rs, nreg = _layout(n)
    cand = [b"%08d" % i for i in range(ncand)]
    slot = first_slots(cand, rs * nreg)
    last, first = {}, {}
    for i in np.flatnonzero(slot % rs == rs - 1):
        last.setdefault(int(slot[i]) // rs, []).append(cand[i])
    for i in np.flatnonzero(slot % rs == 0):
        first.setdefault(int(slot[i]) // rs, []).append(cand[i])
    return cand, nreg, last, first


def test_probe_rows_of_one_thread_in_one_region():
    n = 5000
    cand, nreg, last, first = _region_keys(n, 1_500_000)
    aimed, missing, groups = [], [], []
    for g in range(nreg):
        assert len(last[g]) >= 7 and len(first[g]) >= 2
        aimed += last[g][:4] + first[g][:2]  # in the index: three of the last-slot keys wrap to the region's first slot
        missing += last[g][4:7]              # not in the index: the same walk to the first empty slot
        hit_wrap, hit_first, miss = last[g][1:4], first[g][:2], last[g][4:7]
        groups += [[hit_wrap[0], miss[0], hit_first[0], hit_wrap[1]], [miss[1], miss[2], hit_wrap[2], miss[0]],
                   [hit_first[1], hit_wrap[0], hit_first[0], miss[1]], [miss[2], hit_first[1], miss[0], hit_wrap[2]]]
    used = set(aimed) | set(missing)
    keys = aimed + [k for k in cand[:3 * n] if k not in used][: n - len(aimed)]
    random.Random(3).shuffle(keys)
    rows = _by_lane(groups)
    # the same rows one row off the warp's boundary, and a tail that is not a multiple of 32
    probe = b"k\n" + b"".join(k + b"\n" for k in rows + [b"x"] + rows + keys[::5][:77])
    _check(_index_csv(keys), probe)


def test_duplicate_rows_of_one_thread():
    import csvplus_b200 as cp
    n = 6000
    base = [b"%07d" % i for i in range(n)]
    cases = []
    for gap in (32, 64, 96):  # rows 1000 and 1000 + gap
        keys = list(base)
        keys[1000 + gap] = keys[1000]
        cases.append(keys)
    keys = list(base)
    for u in range(1, 4):  # one key in rows 1285 + 32u
        keys[1280 + 5 + 32 * u] = keys[1280 + 5]
    cases.append(keys)
    for keys in cases:
        data = _index_csv(keys)
        with pytest.raises(cp.CsvPlusError) as e:
            _parse(data).index_on("k", unique=True)
        with pytest.raises(orc.OracleError) as oe:
            orc.reader_rows(data).unique_index_on("k")
        assert str(e.value) == str(oe.value)
        assert str(e.value).startswith("duplicate value while creating unique index: ")


def test_overflow_from_rows_of_one_thread():
    n = 20000
    rs, nreg = _layout(n)
    cand = [b"%08d" % i for i in range(600_000)]
    region = first_slots(cand, rs * nreg) // rs
    crowd = [cand[i] for i in np.flatnonzero(region == 5)][: rs + 3]  # three more keys than region 5 can take
    assert len(crowd) == rs + 3
    others = [cand[i] for i in np.flatnonzero(region != 5)[: n - len(crowd)]]
    keys = others[:4097] + crowd + others[4097:]  # the crowd in whole warps' rows, starting one row past a warp's
    probe = b"k\n" + b"".join(k + b"\n" for k in crowd[::2] + others[::13] + [b"nope"])
    _check(_index_csv(keys), probe, path="hash16")


def test_region_counts_by_lane():
    # an index whose region 0 holds exactly region - 1 keys (the most a region takes) sent in by whole warps' rows
    n = 6000
    rs, nreg = _layout(n)
    cand = [b"%08d" % i for i in range(400_000)]
    region = first_slots(cand, rs * nreg) // rs
    full = [cand[i] for i in np.flatnonzero(region == 0)][: rs - 1]
    assert len(full) == rs - 1
    others = [cand[i] for i in np.flatnonzero(region != 0)[: n - len(full)]]
    keys = full + others
    probe = b"k\n" + b"".join(k + b"\n" for k in full + others[::7] + [cand[i] for i in np.flatnonzero(region == 0)[rs:rs + 40]])
    _check(_index_csv(keys), probe)
