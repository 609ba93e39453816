"""A plain-Python restatement of the reference's predicates Like / All / Any / Not (csvplus.go:1243-1293) over tuple trees,
and seeded random trees for the predicate tests.  It shares no code with csvplus_b200.Predicate, with the CUDA predicate
compiler or with the oracle, so that it can judge all three.

A tree is ("like", {key: value}) | ("all", [tree, ...]) | ("any", [tree, ...]) | ("not", tree), keys and values bytes;
a row is a dict of bytes -> bytes."""
from __future__ import annotations

import random


def holds(tree, row: dict) -> bool:
    op, arg = tree
    if op == "like":  # every (key, value) pair is in the row
        for k, v in arg.items():
            if k not in row or row[k] != v:
                return False
        return True
    if op == "all":
        for t in arg:
            if not holds(t, row):
                return False
        return True
    if op == "any":
        for t in arg:
            if holds(t, row):
                return True
        return False
    if op == "not":
        return not holds(arg, row)
    raise ValueError(op)


def _key(k: bytes) -> str:
    return k.decode("utf-8", "surrogateescape")


def to_cp(tree):
    """the same tree as csvplus_b200 predicates"""
    import csvplus_b200 as cp
    op, arg = tree
    if op == "like":
        return cp.Like({_key(k): v for k, v in arg.items()})
    if op == "not":
        return cp.Not(to_cp(arg))
    return (cp.All if op == "all" else cp.Any)(*[to_cp(t) for t in arg])


def to_orc(tree):
    """the same tree as oracle predicates"""
    from oracle import oracle as orc
    op, arg = tree
    if op == "like":
        return orc.Like(dict(arg))
    if op == "not":
        return orc.Not(to_orc(arg))
    return (orc.All if op == "all" else orc.Any)(*[to_orc(t) for t in arg])


def str_row(row: dict) -> dict:
    """a bytes row as csvplus_b200 rows are: str keys and values (surrogateescape)"""
    return {_key(k): _key(v) for k, v in row.items()}


def bytes_row(row: dict) -> dict:
    return {k.encode("utf-8", "surrogateescape"): v.encode("utf-8", "surrogateescape") for k, v in row.items()}


def literal(rng: random.Random, observed: list) -> bytes:
    """mostly a value that occurs, so that terms match; else one that differs from it at its edges"""
    v = rng.choice(observed) if observed else b""
    r = rng.random()
    if r < 0.55:
        return v
    if r < 0.63:
        return b""
    if r < 0.71:
        return v[:rng.randrange(len(v))] if v else b"a"  # a proper prefix
    if r < 0.79:
        return v + rng.choice([b"a", b" ", b"\xc3", b'"'])  # one byte more
    if r < 0.87:
        return v + b"\r"
    if r < 0.95:
        return v + rng.choice(["é", "€", "\U0001d11e"]).encode()  # multi-byte UTF-8
    return rng.choice([b"\r", b"\n", b"a\nb", b","])


def random_tree(rng: random.Random, keys: list, observed: dict, depth: int = 0, max_depth: int = 4):
    """keys: the column names Like keys are drawn from (selected, unselected and missing ones);
    observed: column name -> values that occur in it"""
    r = rng.random()
    if depth >= max_depth or r < 0.45:
        match = {}
        for _ in range(rng.randint(1, 3)):
            k = rng.choice(keys)
            match[k] = literal(rng, observed.get(k, []))
        return ("like", match)
    if r < 0.6:
        return ("not", random_tree(rng, keys, observed, depth + 1, max_depth))
    kids = [random_tree(rng, keys, observed, depth + 1, max_depth) for _ in range(rng.randint(0, 4))]
    return ("all" if r < 0.8 else "any", kids)


def count(tree) -> tuple:
    """(Like pairs, postfix operations, depth) of a tree as the device compiler counts them"""
    op, arg = tree
    if op == "like":
        return len(arg), 2 * len(arg) - 1, 0
    kids = [arg] if op == "not" else arg
    if not kids:
        return 0, 1, 0
    cs = [count(k) for k in kids]
    return (sum(c[0] for c in cs), sum(c[1] for c in cs) + (1 if op == "not" else len(kids) - 1),
            1 + max(c[2] for c in cs))
