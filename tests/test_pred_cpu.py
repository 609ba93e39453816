"""Predicates without a GPU: the plain-Python restatement of Like / All / Any / Not (tests/pred_ref.py), the host
evaluation csvplus_b200.Predicate.__call__ and the oracle agree on random trees; Predicate.lowerable() takes exactly the
trees the device compiler takes (include/csvplus_b200.h's CPB_PRED_MAX_* limits)."""
import os
import random
import re

import pytest

from oracle import oracle as orc
from tests.pred_ref import count, holds, random_tree, str_row, to_cp, to_orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VALUES = [b"", b"a", b"ab", b"abc", b"Ann", b"a\r", b"a\rb", b"x y", "é".encode(), "€uro".encode(), b'say "hi"', b"two\nlines",
          b"\xff\xfe"]


def test_header_limits_are_mirrored():
    from csvplus_b200 import _abi
    hdr = open(os.path.join(ROOT, "include", "csvplus_b200.h")).read()
    defs = dict(re.findall(r"#define\s+(CPB_[A-Z_]+)\s+(\d+)", hdr))
    assert int(defs["CPB_MAX_PARSE_COLS"]) == _abi.MAX_PARSE_COLS
    assert int(defs["CPB_PRED_MAX_TERMS"]) == _abi.PRED_MAX_TERMS
    assert int(defs["CPB_PRED_MAX_OPS"]) == _abi.PRED_MAX_OPS
    assert int(defs["CPB_PRED_MAX_DEPTH"]) == _abi.PRED_MAX_DEPTH


@pytest.mark.parametrize("seed", range(6))
def test_three_evaluators_agree(seed):
    rng = random.Random(seed)
    cols = [b"c0", b"c1", b"c2", b"c3"]
    rows = [{c: rng.choice(VALUES) for c in cols} for _ in range(300)]
    observed = {c: sorted({r[c] for r in rows}) for c in cols}
    table = orc.take_rows(rows)
    matched = 0
    for _ in range(40):
        tree = random_tree(rng, cols + [b"zz"], observed)
        want = [r for r in rows if holds(tree, r)]
        matched += 0 < len(want) < len(rows)
        p = to_cp(tree)
        assert [r for r in rows if p(str_row(r))] == want, tree
        assert table.filter(to_orc(tree)).to_dicts() == want, tree
    assert matched >= 5  # the trees select real subsets, not only everything or nothing


def test_reference_semantics():
    row = {b"a": b"1", b"b": b""}
    assert holds(("like", {b"a": b"1", b"b": b""}), row)
    assert not holds(("like", {b"zz": b""}), row)  # a missing column never matches, not even ""
    assert not holds(("like", {b"a": b"1\r"}), row)
    assert holds(("all", []), row) and not holds(("any", []), row)
    assert holds(("not", ("any", [])), row)


def _chain(depth: int):
    """a Like under `depth` All / Any / Not nodes"""
    t = ("like", {b"c0": b"a"})
    for i in range(depth):
        t = (("all", [t]), ("any", [t]), ("not", t))[i % 3]
    return t


def _terms(n: int, wrap: int = 0):
    t = ("any", [("like", {b"c%d" % (i % 3): b"v%d" % i}) for i in range(n)])
    for _ in range(wrap):
        t = ("not", t)
    return t


def test_lowerable_at_and_past_the_limits():
    from csvplus_b200 import _abi
    T, O, D = _abi.PRED_MAX_TERMS, _abi.PRED_MAX_OPS, _abi.PRED_MAX_DEPTH
    at = {"terms": _terms(T), "ops": _terms(T, wrap=O - (2 * T - 1)), "depth": _chain(D),
          "pairs": ("any", [("like", {b"c%d" % k: b"v" for k in range(4)}) for _ in range(T // 4)])}
    past = {"terms": _terms(T + 1), "ops": _terms(T, wrap=O - (2 * T - 1) + 1), "depth": _chain(D + 1),
            "pairs": ("any", [("like", {b"c%d" % k: b"v" for k in range(4)}) for _ in range(T // 4)] + [("like", {b"c0": b"w"})])}
    assert count(at["terms"])[0] == T and count(at["ops"])[1] == O and count(at["depth"])[2] == D
    assert count(past["terms"])[0] == T + 1 and count(past["ops"])[1] == O + 1 and count(past["depth"])[2] == D + 1
    for name, t in at.items():
        assert to_cp(t).lowerable(), name
    for name, t in past.items():
        assert not to_cp(t).lowerable(), name
    assert to_cp(("all", [])).lowerable() and to_cp(("not", ("any", []))).lowerable()


@pytest.mark.parametrize("seed", range(3))
def test_lowerable_matches_the_compiler_count(seed):
    from csvplus_b200 import _abi
    rng = random.Random(seed)
    seen = set()
    for _ in range(400):  # trees on both sides of each limit
        t = ("any", [random_tree(rng, [b"a", b"b"], {}, max_depth=3) for _ in range(rng.randint(0, 14))])
        for _ in range(rng.choice([0, 0, 44, 46, 47, 48])):
            t = rng.choice([("not", t), ("all", [t])])
        terms, ops, depth = count(t)
        seen |= {("terms", terms > _abi.PRED_MAX_TERMS), ("ops", ops > _abi.PRED_MAX_OPS), ("depth", depth > _abi.PRED_MAX_DEPTH)}
        assert to_cp(t).lowerable() == (terms <= _abi.PRED_MAX_TERMS and ops <= _abi.PRED_MAX_OPS and depth <= _abi.PRED_MAX_DEPTH), t
    assert len(seen) == 6, seen


def test_opaque_functions_are_not_lowerable():
    import csvplus_b200 as cp
    assert not cp.Predicate(1, kids=[lambda r: True]).lowerable()
    assert not isinstance(cp.All(cp.Like({"a": "1"}), lambda r: True), cp.Predicate)


def test_columns_are_distinct_like_keys():
    p = to_cp(("all", [("like", {b"a": b"1", b"b": b"2"}), ("not", ("like", {b"a": b"3"})), ("any", [])]))
    assert p.columns() == {"a", "b"}
