"""Set terms without a GPU (include/csvplus_b200.h, CPB_PRED_SET_MIN): Predicate.lowerable() takes exactly the trees the
grouping rule allows, trees without a qualifying group are counted as before (tests/pred_ref.count), and a set term is
lowered in bulk onto one keys array."""
import ctypes as C
import os
import random
import re

import pytest

import csvplus_b200 as cp
from csvplus_b200 import _abi
from tests.pred_ref import count, random_tree, to_cp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, O, D, S = _abi.PRED_MAX_TERMS, _abi.PRED_MAX_OPS, _abi.PRED_MAX_DEPTH, _abi.PRED_SET_MIN


def likes(n, keys=("a",), start=0, width=None):
    """n Likes over the column set keys, distinct values (of `width` bytes when given)"""
    out = []
    for i in range(start, start + n):
        v = str(i) if width is None else str(i).rjust(width, "x")
        out.append(cp.Like({k: v + k for k in keys}))
    return out


def test_header_set_min_is_mirrored():
    hdr = open(os.path.join(ROOT, "include", "csvplus_b200.h")).read()
    defs = dict(re.findall(r"#define\s+(CPB_[A-Z_]+)\s+(\d+)", hdr))
    assert int(defs["CPB_PRED_SET_MIN"]) == _abi.PRED_SET_MIN == _abi.PRED_MAX_TERMS + 1


def test_threshold():
    at = cp.Any(*likes(S - 1))
    assert at._set_groups() == [] and at.lowerable()  # 32 Like terms: within the limits, per term
    assert not cp.Any(*likes(S - 1), cp.Like({"b": "x"})).lowerable()  # 33 terms: the group of 32 stays per term
    big = cp.Any(*likes(S))
    assert [m for _, m in big._set_groups()] == [list(range(S))] and big.lowerable()
    assert cp.Any(*likes(S), cp.Like({"b": "x"})).lowerable()
    assert cp.Any(*likes(1_000)).lowerable()


def test_key_sets_and_key_order():
    mixed = [cp.Like({"a": str(i), "b": "x"}) if i % 2 else cp.Like({"b": "y", "a": str(i)}) for i in range(S)]
    p = cp.Any(*mixed)
    assert len(p._set_groups()) == 1 and p.lowerable()  # {a,b} and {b,a} are one set
    assert p._set_groups()[0][0] == ["b", "a"]  # the first Like's key order
    two = cp.Any(*likes(S, ("a",)), *likes(S, ("a", "b")))
    assert len(two._set_groups()) == 2 and two.lowerable()
    # a set of one column and one of two columns that share it are different sets: 40 + 20 Likes, only one group qualifies
    part = cp.Any(*likes(40, ("a",)), *likes(20, ("a", "b")))
    assert len(part._set_groups()) == 1 and not part.lowerable()  # 1 + 40 terms


def test_group_beside_plain_likes():
    plain = [cp.Like({"c%d" % i: "v"}) for i in range(T - 1)]
    assert cp.Any(*plain, *likes(S)).lowerable()  # 31 + 1 terms and 31 ORs: 63 operations
    assert not cp.Any(*plain, cp.Like({"z": "1"}), *likes(S)).lowerable()  # 33 terms
    interleaved = cp.Any(*[x for pair in zip(likes(S), plain + plain) for x in pair])
    assert interleaved._set_groups()[0][1] == list(range(0, 2 * S, 2))


def test_group_under_not_and_all():
    assert cp.Not(cp.Any(*likes(S))).lowerable()
    assert cp.All(cp.Any(*likes(S)), cp.Like({"b": "1"})).lowerable()
    assert not cp.All(*likes(S)).lowerable()  # only the children of an Any form a set
    assert not cp.Not(cp.All(*likes(S))).lowerable()


def test_the_likes_of_a_set_add_no_depth():
    def wrap(p, depth):
        for i in range(depth):
            p = cp.Not(p) if i % 2 else cp.All(p)
        return p
    assert wrap(cp.Any(*likes(S)), D).lowerable()  # the Any at depth 48, its Likes would be at 49
    assert not wrap(cp.Any(*likes(2)), D).lowerable()
    assert not wrap(cp.Any(*likes(S)), D + 1).lowerable()


def test_groups_that_cannot_be_an_index():
    keys16 = tuple("k%d" % i for i in range(16))
    keys17 = keys16 + ("k16",)
    assert cp.Any(*likes(S, keys16)).lowerable()
    p17 = cp.Any(*likes(S, keys17))
    assert p17._set_groups() == [] and not p17.lowerable()
    # one column: w + L(w) <= 4096, L(w) = 2 for 255 <= w < 65535 (the values are width + len("a") bytes)
    assert cp.Any(*likes(S, width=4093)).lowerable()       # 4094 + 2
    assert not cp.Any(*likes(S, width=4094)).lowerable()   # 4095 + 2
    # the longest literal decides, and multi-byte characters count in bytes
    long = likes(S - 1) + [cp.Like({"a": "é" * 2048})]   # 4096 bytes + 2
    assert not cp.Any(*long).lowerable()
    # two columns: (w1 + 2) + (w2 + 2) <= 4096
    assert cp.Any(*likes(S, ("a", "b"), width=2045)).lowerable()      # 2 x (2046 + 2)
    assert not cp.Any(*likes(S, ("a", "b"), width=2046)).lowerable()  # 2 x (2047 + 2)
    assert cp.Any(*likes(S, width=253)).lowerable() and cp.Any(*likes(S, width=254)).lowerable()  # 254 + 1, 255 + 2


def test_duplicates_and_empty_literals_form_a_set():
    p = cp.Any(*[cp.Like({"a": ""}) for _ in range(S)], *[cp.Like({"a": "1"}) for _ in range(S)])
    assert len(p._set_groups()) == 1 and p.lowerable()


@pytest.mark.parametrize("seed", range(3))
def test_trees_without_a_qualifying_group_count_as_before(seed):
    rng = random.Random(seed)
    seen = set()
    for _ in range(300):
        kids = [random_tree(rng, [b"b", b"c"], {}, max_depth=3) for _ in range(rng.randint(0, 10))]
        kids += [("like", {b"a": b"%d" % i}) for i in range(rng.choice([0, 7, 20, S - 1]))]  # groups below the threshold
        rng.shuffle(kids)
        t = ("any", kids)
        for _ in range(rng.choice([0, 0, 45, 47, 48])):
            t = rng.choice([("not", t), ("all", [t])])
        terms, ops, depth = count(t)
        ok = terms <= T and ops <= O and depth <= D
        seen.add(ok)
        assert to_cp(t).lowerable() == ok, t
    assert seen == {True, False}


def _pred(addr):
    return C.cast(C.c_void_p(int(addr)), C.POINTER(_abi.Pred)).contents


def test_a_set_is_lowered_onto_one_keys_array():
    kids = [cp.Like({"b": "y%d" % i, "a": "x%d" % i}) if i % 3 == 0 else cp.Like({"a": "x%d" % i, "b": "y%d" % i}) for i in range(S)]
    p = cp.Any(cp.Like({"c": "1"}), *kids)
    keep = []
    root = p._c(keep)
    assert root.op == 2 and root.n == S + 1
    ptrs = [C.cast(root.children, C.POINTER(C.c_void_p))[i] for i in range(root.n)]
    first = _pred(ptrs[1])
    keys = [C.string_at(first.keys[j].ptr, first.keys[j].len) for j in range(first.n)]
    assert keys == [b"b", b"a"]  # the first Like's order
    for i in range(1, S + 1):
        node = _pred(ptrs[i])
        assert node.op == 0 and node.n == 2
        assert C.cast(node.keys, C.c_void_p).value == C.cast(first.keys, C.c_void_p).value
        vals = [C.string_at(node.values[j].ptr, node.values[j].len) for j in range(2)]
        assert vals == [b"y%d" % (i - 1), b"x%d" % (i - 1)]
    plain = _pred(ptrs[0])
    assert plain.n == 1 and C.string_at(plain.keys[0].ptr, plain.keys[0].len) == b"c"
    assert p._c([]) is root  # lowered once


def test_large_set_lowering_values():
    n = 100_000
    p = cp.Any(*[cp.Like({"id": str(i * 7)}) for i in range(n)], cp.Like({"id": "\udcff"}))  # (surrogateescape bytes)
    root = p._c([])
    ptrs = C.cast(root.children, C.POINTER(C.c_void_p))
    for i in (0, 1, n // 2, n - 1, n):
        node = _pred(ptrs[i])
        assert C.string_at(node.values[0].ptr, node.values[0].len) == (str(i * 7).encode() if i < n else b"\xff")
