"""Set terms on the GPU (include/csvplus_b200.h, CPB_PRED_SET_MIN): an Any of many Like terms over one column set, on every
route that evaluates a predicate, against the plain-Python restatement of the reference's predicates (tests/pred_ref.py)
over the oracle's rows parsed without a predicate.  Predicate.__call__ raises throughout, so every result comes from the
device; kernel statistics show filter_set (the set-term evaluation) and, on the parse routes, csv_scan."""
import io
import os
import random
import subprocess

import pytest

from oracle import oracle as orc
from tests.helpers import gpu_ctx
from tests.pred_ref import holds, to_cp
from tests.test_gpu_predicates import _limit_trees, _quote, _stats, make_csv, pulled, reference, table_rows

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NASTY = [b"", b"a", b"Ann", "é".encode(), "€uro".encode(), "\U0001d11e".encode(), b"a\rb", b'say "hi"', b"c,d", b"two\nlines",
         b"y" * 300, b"x\r"]
CITIES = [b"Oslo", b"Rome", b"", "Zürich".encode(), b"New York, NY"]


@pytest.fixture(autouse=True)
def device_only(monkeypatch):
    import csvplus_b200 as cp

    def no_host_rows(self, row):
        raise AssertionError("a recognisable predicate was evaluated on host rows")
    monkeypatch.setattr(cp.Predicate, "__call__", no_host_rows)


def make_data(seed, nrows, *, ncols_extra=0, error_at=None, eol=b"\n") -> bytes:
    """id (distinct, in row order), name, city (NASTY / CITIES values, quoted where they need it) and x0.. columns"""
    rng = random.Random(seed)
    head = [b"id", b"name", b"city"] + [b"x%d" % i for i in range(ncols_extra)]
    lines = [b",".join(head)]
    for i in range(nrows):
        f = [b"%d" % (1000 + 7 * i), rng.choice(NASTY), rng.choice(CITIES)] + [b"v%d" % rng.randrange(9) for _ in range(ncols_extra)]
        lines.append(b",".join(_quote(rng, v) if (not v or any(c in v for c in b',"\r\n')) else v for v in f))
        if error_at is not None and i == error_at:
            lines.append(b'1,bad"quote,x' + b",v" * ncols_extra)
    return eol.join(lines) + eol


def matcher(tree):
    """pred_ref.holds as a function of the row, computed as membership for one-column set trees (one lookup instead of one
    Like per literal); every other tree by holds itself"""
    op, arg = tree
    if op == "any" and len(arg) > 1000 and all(t[0] == "like" and len(t[1]) == 1 for t in arg):
        members = {}
        for _, m in arg:
            (k, v), = m.items()
            members.setdefault(k, set()).add(v)
        return lambda row: any(k in row and row[k] in vs for k, vs in members.items())
    return lambda row: holds(tree, row)


def id_set(rows, n, seed):
    """a set of n one-column Likes on id holding about half of the rows' ids; the rest are near misses (one byte shorter
    or longer, another digit) and values longer than every id"""
    rng = random.Random(seed)
    ids = [r[b"id"] for r in rows]
    hit = rng.sample(ids, min(len(ids) // 2, n))
    lits = list(hit)
    while len(lits) < n:
        v = rng.choice(ids)
        lits.append(rng.choice([v[:-1], v + b"0", v + b" ", b"9" + v, v * 4, b"x%d" % len(lits)]))
    rng.shuffle(lits)
    return ("any", [("like", {b"id": v}) for v in lits])


def check_table_and_parse(data, tree, o=None, select=None, table_too=True, kernel="filter_set"):
    import csvplus_b200 as cp
    o = o or orc.Opts()
    rows, err = reference(data, o, select)
    match = matcher(tree)
    want = [r for r in rows if match(r)]
    p = to_cp(tree)
    assert p.lowerable()
    reader = cp.FromBytes(data)
    if o.comment:
        reader = reader.CommentChar(o.comment)
    if o.lazy_quotes:
        reader = reader.LazyQuotes()
    ds = cp.Take(reader.SelectColumns(*[c.decode() for c in select]) if select else reader)
    got, st = _stats(lambda: pulled(ds.Filter(p)))
    assert got == (want, err)
    assert "csv_scan" in st or any(k.startswith("general_rec") for k in st)
    other = "filter_like" if kernel == "filter_set" else "filter_set"
    assert kernel in st and other not in st, sorted(st)
    if table_too and err is None:
        t0, _ = cp.parse_csv(gpu_ctx(), data, spec=[(c.decode(), -1) for c in select] if select else None)
        got, st = _stats(lambda: table_rows(t0.filter(p)))
        assert got == want and kernel in st and other not in st
    return rows, want, st


@pytest.mark.parametrize("n", [33, 1000, 100_000, 1_000_000])
def test_set_sizes(n):
    data = make_data(n, 20_000)
    rows, _ = reference(data, orc.Opts())
    tree = id_set(rows, n, n)
    sample = random.Random(0).sample(rows, min(50, 5_000_000 // n))  # the membership shortcut is holds
    assert [matcher(tree)(r) for r in sample] == [holds(tree, r) for r in sample]
    _, want, _ = check_table_and_parse(data, tree)
    assert 0 < len(want) < len(rows)


def _nasty_lits(rng, rows, cols, n):
    """tuples of cols drawn from the rows, with edits: one byte shorter / longer, longer than every row value, empty; and
    duplicates"""
    out = []
    for _ in range(n):
        r = rng.choice(rows)
        t = {c: r[c] for c in cols}
        c = rng.choice(cols)
        x = rng.random()
        if x < 0.15:
            t[c] = t[c][:-1]
        elif x < 0.3:
            t[c] = t[c] + b"a"
        elif x < 0.4:
            t[c] = b"L" * 400
        elif x < 0.45:
            t[c] = b""
        out.append(t)
    return out + out[:10]


@pytest.mark.parametrize("cols", [[b"name"], [b"name", b"city"], [b"city", b"id", b"name"]])
def test_keys_and_literals(cols):
    rng = random.Random(len(cols))
    data = make_data(7, 3000)
    rows, _ = reference(data, orc.Opts())
    lits = _nasty_lits(rng, rows, cols, 200)
    # Likes with their keys in different orders are one set
    tree = ("any", [("like", dict(sorted(t.items(), reverse=i % 2 == 1))) for i, t in enumerate(lits)])
    _, want, _ = check_table_and_parse(data, tree)
    assert want


def test_absent_column_matches_nothing_and_builds_no_index():
    data = make_data(8, 2000)
    for keys in ([b"zz"], [b"id", b"zz"]):
        tree = ("any", [("like", {k: b"%d" % (1000 + 7 * i) for k in keys}) for i in range(100)])
        # (the set term is a constant false: the plain filter kernel evaluates the rest)
        _, want, st = check_table_and_parse(data, ("any", [tree, ("like", {b"city": b"Oslo"})]), kernel="filter_like")
        assert all(r[b"city"] == b"Oslo" for r in want) and want
        assert "pred_set_upload" not in st and "key_width" not in st


def test_tree_shapes():
    data = make_data(9, 3000)
    rows, _ = reference(data, orc.Opts())
    ids = id_set(rows, 500, 1)
    names = ("any", [("like", {b"name": v, b"city": c}) for v in NASTY for c in CITIES] * 2)
    assert len(names[1]) >= 33
    for tree in [("not", ids), ("all", [ids, ("like", {b"city": b"Rome"})]),
                 ("any", [ids[1][0], ("like", {b"city": b""}), *ids[1][1:], *names[1][:40]]),  # two groups and a plain Like
                 ("all", [("not", ("any", names[1][:40])), ids])]:
        _, want, _ = check_table_and_parse(data, tree)
        assert 0 < len(want) < len(rows), tree[0]


def test_take_while_and_drop_while():
    import csvplus_b200 as cp
    data = make_data(10, 3000)
    rows, _ = reference(data, orc.Opts())
    cut = 1234
    tree = ("any", [("like", {b"id": r[b"id"]}) for r in rows[:cut]] + [("like", {b"id": b"0"})])
    t0, _ = cp.parse_csv(gpu_ctx(), data)
    got, st = _stats(lambda: t0.first_false(to_cp(tree)))
    assert got == cut and "filter_set" in st
    assert pulled(cp.Take(cp.FromBytes(data)).TakeWhile(to_cp(tree))) == (rows[:cut], None)
    assert pulled(cp.Take(cp.FromBytes(data)).DropWhile(to_cp(tree))) == (rows[cut:], None)


def test_streamed_pieces_compile_once(monkeypatch):
    import csvplus_b200 as cp
    data = make_data(11, 6000, eol=b"\r\n")
    rows, _ = reference(data, orc.Opts())
    tree = ("any", [("like", {b"name": v, b"id": r[b"id"]}) for r in rows[::12] for v in (r[b"name"], b"q")])
    want = [r for r in rows if holds(tree, r)]
    monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", 16 << 10)
    got, st = _stats(lambda: pulled(cp.Take(cp.FromReader(io.BytesIO(data))).Filter(to_cp(tree))))
    assert got == (want, None)
    assert st["filter_set"]["launches"] > 5  # one per batch
    assert st["key_width"]["launches"] == 2  # the set's index (two key columns) is built once


@pytest.mark.parametrize("opt", ["comment", "lazy"])
def test_general_path_inputs(opt):
    rng = random.Random(12)
    if opt == "comment":
        o = orc.Opts(comment="#")
        data = make_csv(12, nrows=1500, quote_p=0.1, comment_p=0.05)
    else:
        o = orc.Opts(lazy_quotes=True)
        data = make_csv(13, nrows=1500, quote_p=0.1, extra=(b'x"y', b'a"'))
    rows, _ = reference(data, o)
    tree = ("any", [("like", {b"c1": r[b"c1"], b"c3": r[b"c3"]}) for r in rng.sample(rows, 60)])
    _, want, st = check_table_and_parse(data, tree, o, select=[b"c3", b"c1", b"c0"], table_too=False)
    assert any(k.startswith("general_rec") for k in st) and want


def test_file_wider_than_16_columns():
    data = make_data(14, 2000, ncols_extra=18)
    rows, _ = reference(data, orc.Opts())
    tree = ("any", [("like", {b"x17": b"v%d" % (i % 9), b"name": v}) for i, v in enumerate(NASTY * 4)])
    _, want, _ = check_table_and_parse(data, tree)
    assert 0 < len(want) < len(rows)


def test_data_error_in_the_middle():
    data = make_data(15, 4000, error_at=2500)
    rows, err = reference(data, orc.Opts())
    assert err is not None and len(rows) == 2501
    tree = id_set(rows, 2000, 2)
    check_table_and_parse(data, tree)


@pytest.mark.parametrize("world", [2, 3])
def test_byte_range_shards(world):
    from tests.test_gpu_shards import _run_sharded
    data = make_data(16 + world, 5000)
    rows, _ = reference(data, orc.Opts())
    tree = id_set(rows, 3000, world)
    match = matcher(tree)
    for select in (None, [b"name", b"id"]):
        whole, errs, _ = _run_sharded(data, world, spec=[(c.decode(), -1) for c in select] if select else None, pred=to_cp(tree))
        assert all(e is None for e in errs)
        want = [{k: r[k] for k in (select or r)} for r in rows if match(r)]
        assert table_rows(whole) == want


def test_filter_after_join():
    import csvplus_b200 as cp
    data = make_data(20, 3000)
    labels = b"city,label\n" + b"".join(_quote(random.Random(0), c) + b",L%d\n" % i for i, c in enumerate(CITIES))
    joined = orc.reader_rows(data).join(orc.reader_rows(labels).unique_index_on("city"), "city").to_dicts()
    tree = ("any", [("like", {b"label": b"L%d" % (i % 3), b"id": r[b"id"]}) for i, r in enumerate(joined[::2])])
    want = [r for r in joined if holds(tree, r)]
    assert 0 < len(want) < len(joined)
    idx = cp.Take(cp.FromBytes(labels)).UniqueIndexOn("city")
    got, st = _stats(lambda: pulled(cp.Take(cp.FromBytes(data)).Join(idx, "city").Filter(to_cp(tree))))
    assert got == (want, None) and "filter_set" in st


def test_trees_at_the_limits_take_the_routes_they_took():
    """a tree at CPB_PRED_MAX_TERMS has no set term: the same kernels as before set terms existed, fused into the scan"""
    import csvplus_b200 as cp
    data = make_csv(51, nrows=2000, eol="crlf", quote_p=0.1)
    rows, _ = reference(data, orc.Opts())
    at, _ = _limit_trees(rows)
    t0, _ = cp.parse_csv(gpu_ctx(), data)
    for name, tree in at.items():
        want = [r for r in rows if holds(tree, r)]
        got, st = _stats(lambda: pulled(cp.Take(cp.FromBytes(data)).Filter(to_cp(tree))))
        assert got == (want, None)
        assert {k: v["launches"] for k, v in st.items()} == PARENT_PARSE_LAUNCHES, name
        got, st = _stats(lambda: pulled(cp.TakeTable(t0).Filter(to_cp(tree))))
        assert got == (want, None)
        assert {k: v["launches"] for k, v in st.items()} == PARENT_TABLE_LAUNCHES, name


# kernel launches of those routes before set terms existed (the same at every tree of _limit_trees)
PARENT_PARSE_LAUNCHES = {"csv_header": 1, "csv_scan": 1}
PARENT_TABLE_LAUNCHES = {"compact_ids": 1, "filter_like": 1, "gather_copy": 5, "scan_gather_len": 5, "scan_u32": 1}


def test_cpp_mirror(tmp_path):
    """host/csvplus.hpp: the same lowerable() rule and the bulk lowering, through Filter on a parse and on rows"""
    src = tmp_path / "sets.cpp"
    src.write_text(r'''
#include "csvplus.hpp"
#include <iostream>
using namespace csvplus;
int main(int argc, char** argv) {
    std::vector<Predicate> kids;
    for (int i = 1; i < argc; i++) kids.push_back(Like({{"id", argv[i]}}));
    Predicate p = Any(kids);
    std::vector<Predicate> k32(kids.begin(), kids.begin() + 32);
    std::vector<Predicate> k33(kids.begin(), kids.begin() + 33);
    k32.push_back(Like({{"name", "Ann"}})); k33.push_back(Like({{"name", "Ann"}}));
    std::cout << Any(k32).lowerable() << Any(k33).lowerable() << p.lowerable() << "\n";
    std::string data((std::istreambuf_iterator<char>(std::cin)), std::istreambuf_iterator<char>());
    for (auto& r : Take(FromString(data)).Filter(p).ToRows()) std::cout << r.at("id") << " ";
    std::cout << "\n";
    auto rows = Take(FromString(data)).ToRows();
    for (auto& r : TakeRows(rows).Filter(p).ToRows()) std::cout << r.at("id") << " ";
    std::cout << "\n";
}
''')
    exe = tmp_path / "sets"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "host"), "-o", str(exe), str(src),
                           "-L" + os.path.join(ROOT, "csvplus_b200"), "-lcsvplus_b200", "-Wl,-rpath," + os.path.join(ROOT, "csvplus_b200")])
    data = make_data(21, 3000)
    rows, _ = reference(data, orc.Opts())
    tree = id_set(rows, 1500, 3)
    lits = [m[b"id"].decode() for _, m in tree[1]]
    out = subprocess.run([str(exe)] + lits, input=data, capture_output=True, check=True).stdout.decode().split("\n")
    assert out[0] == "011"  # 32 + 1 terms: declined; a set and one Like: lowered
    want = " ".join(r[b"id"].decode() for r in rows if matcher(tree)(r))
    assert out[1].strip() == want and out[2].strip() == want and want
