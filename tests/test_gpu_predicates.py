"""Filter(Like / All / Any / Not) on every route that evaluates a predicate, against a plain-Python restatement of the
reference's predicates (tests/pred_ref.py) over the oracle's rows parsed WITHOUT a predicate, so that the expected rows
share no code with the CUDA predicate compiler, with Predicate.__call__ or with the oracle's own filter.

Routes of the fused parse (parse_kernels.cuh / parse_general.cu): the fast line path (unquoted records inside a tile
window), the slow record machine (records with quotes, records past the 2 KiB look-ahead, fields longer than a tile), the
dense-tile fallback and the general multi-pass path; padded fields of NumFieldsAny; batches of a streamed input; byte-range
shards.  Then the table filter (Table.filter, TakeWhile / DropWhile, Filter after Join and on TakeRows), and the predicate
size limits of include/csvplus_b200.h.  Every route runs under each line end: LF, CRLF, mixed, no final terminator, a
lone CR at EOF, CR CR LF."""
import io
import random

import pytest

from oracle import oracle as orc
from tests.helpers import gpu_ctx
from tests.pred_ref import bytes_row, holds, random_tree, str_row, to_cp

pytestmark = pytest.mark.gpu

NCOLS = 5
COLS = [b"c%d" % i for i in range(NCOLS)]
PLAIN = [b"", b"a", b"ab", b"Ann", b"a b", b"a\r", b"a\rb", "é".encode(), "€uro".encode(), b"y" * 300]  # written unquoted
QUOTED = [b"a", b"Ann", b"", b"c,d", b'say "hi"', b"two\nlines", b"a\r", b"\r\n"]  # written quoted ("" escapes, \r\n inside)
DENSE = [b"", b"a", b"b", b"ab", "é".encode(), b"a\r"]
EOLS = ["lf", "crlf", "mixed", "noterm", "lone_cr", "crcrlf"]


def _quote(rng, v: bytes) -> bytes:
    return b'"' + v.replace(b'"', b'""').replace(b"\n", rng.choice([b"\n", b"\r\n"])) + b'"'


def make_csv(seed, nrows, *, eol="lf", ncols=NCOLS, values=PLAIN, quote_p=0.0, long_p=0.0, huge=False, short_p=0.0,
             prefixes=(b"",), extra=(), comment_p=0.0, delim=b",") -> bytes:
    """a header c0..c{ncols-1} and nrows records.  quote_p: fields written quoted; long_p: fields of 2.1-3 KB (records
    longer than the look-ahead); huge: one field longer than a 32 KiB tile; short_p: records with fewer fields; prefixes:
    leading white space of fields; extra: more unquoted values; comment_p: '#' lines, some with quotes"""
    rng = random.Random(seed)
    plain = list(values) + list(extra)
    lines = []
    for i in range(nrows):
        if comment_p and rng.random() < comment_p:
            lines.append(b"#" + rng.choice([b' a "quoted, comment', b"", b"c0,c1", b'"']))
        k = ncols if rng.random() >= short_p else rng.randint(1, ncols - 1)
        f = []
        for j in range(k):
            if huge and i == nrows // 2 and j == 1:
                v = b"H" * 40000
            elif long_p and rng.random() < long_p:
                v = (b"L%d-" % j) * rng.randint(700, 1000)
            else:
                v = rng.choice(plain)
            f.append(_quote(rng, rng.choice(QUOTED)) if rng.random() < quote_p else rng.choice(prefixes) + v)
        ln = delim.join(f)
        lines.append(ln if ln else b"a")  # (a line holding one empty field is a blank line)
    out = [delim.join(b"c%d" % i for i in range(ncols)) + (b"\n" if eol == "lf" else b"\r\n")]
    for i, ln in enumerate(lines):
        end = {"lf": b"\n", "crlf": b"\r\n", "crcrlf": b"\r\r\n"}.get(eol) or rng.choice([b"\n", b"\r\n", b"\r\r\n"])
        if i == len(lines) - 1:
            end = {"noterm": b"", "lone_cr": b"\r"}.get(eol, end)
        if ln.endswith(b'"') and end == b"\r\r\n":
            end = b"\r\n"  # (after a closing quote a \r must end the line: keep most of the file free of errors)
        out.append(ln + end)
    return b"".join(out)


def _opts_kw(o: orc.Opts, select):
    return dict(delimiter=o.comma, comment=o.comment, num_fields=o.fields_per_record, lazy_quotes=o.lazy_quotes,
                trim_leading_space=o.trim_leading_space, spec=[(c.decode(), -1) for c in select] if select else None)


def _stats(fn):
    """fn() with kernel statistics on -> (result, {kernel name: stats})"""
    ctx = gpu_ctx()
    ctx.stats(enable=True, reset=True)
    try:
        r = fn()
        return r, ctx.stats()
    finally:
        ctx.stats(enable=False)


def table_rows(t) -> list:
    cols = t.columns
    vals = {c: t.values(c) for c in cols}
    return [{c.encode("utf-8", "surrogateescape"): vals[c][i] for c in cols} for i in range(len(t))]


def pulled(ds):
    """-> (rows as bytes dicts, error text or None) of a DataSource pulled row by row, as the reference's Iterate"""
    import csvplus_b200 as cp
    out = []
    try:
        ds(lambda r: out.append(bytes_row(r)))
    except cp.DataSourceError as e:
        return out, str(e)
    return out, None


def reference(data, o: orc.Opts, select=None):
    r = orc.reader_rows(data, o, select=[c.decode() for c in select] if select else None)
    return r.to_dicts(), r.error


def trees_for(seed, data, o, select, n=10):
    """random trees over the selected columns, one existing but unselected column and one missing column, literals drawn
    from the values of the file; the last one carries a literal of more than 256 bytes"""
    rng = random.Random(seed)
    every, _ = reference(data, o)
    observed = {k: sorted({r[k] for r in every if k in r}) for k in COLS}
    sel = list(select) if select else COLS
    keys = sel + [c for c in COLS if c not in sel][:1] + [b"zz"]
    trees = []
    while len(trees) < n:
        t = random_tree(rng, keys, observed)
        if to_cp(t).lowerable():  # (cpb_parse_csv itself refuses a predicate past the limits)
            trees.append(t)
    if every:  # one term per selected column, on the value a record in the middle holds
        trees += [("like", {k: every[len(every) // 2][k]}) for k in sel if k in every[len(every) // 2]]
    long = rng.choice([v for v in observed[sel[-1]] if len(v) > 256] or [b"z" * 300])
    trees.append(("any", [("like", {sel[0]: rng.choice(observed[sel[0]] or [b""])}), ("like", {sel[-1]: long})]))
    return trees


def check_parse(data, o, select, trees):
    """every tree fused into one cpb_parse_csv call == the reference rows and error; -> True if the general path ran"""
    import csvplus_b200 as cp
    rows, err = reference(data, o, select)
    general, subsets = False, 0
    for tree in trees:
        want = [r for r in rows if holds(tree, r)]
        subsets += 0 < len(want) < len(rows)
        (t, gerr), st = _stats(lambda: cp.parse_csv(gpu_ctx(), data, **_opts_kw(o, select), pred=to_cp(tree)))
        general = general or any(k.startswith("general_rec") for k in st)
        assert (str(gerr) if gerr else None) == err, tree
        assert table_rows(t) == want, tree
    assert len(rows) < 10 or subsets > 0  # some tree selects a real subset
    return general


# ------------------------------------------------------------------ routes of the fused parse x line ends
ROUTES = {
    "fast": (dict(nrows=1500), orc.Opts()),
    "slow": (dict(nrows=1500, quote_p=0.15), orc.Opts()),
    "long": (dict(nrows=120, quote_p=0.05, long_p=0.08, huge=True), orc.Opts()),
    # 5 fields of 0-2 bytes: about 11 bytes per line, so a 32 KiB tile + 2 KiB look-ahead holds about 3000 terminators,
    # more than the 2048 (TILE / 16) the flat index has room for: every tile takes the dense fallback
    "dense": (dict(nrows=9000, values=DENSE), orc.Opts()),
    "comment": (dict(nrows=1500, quote_p=0.1, comment_p=0.05), orc.Opts(comment="#")),
    "lazy": (dict(nrows=1500, quote_p=0.1, extra=(b'x"y', b'a"')), orc.Opts(lazy_quotes=True)),
    "trim": (dict(nrows=1500, quote_p=0.05, prefixes=(b"", b" ", b"\t ", b"\r", b" \r")), orc.Opts(trim_leading_space=True)),
    "runes": (dict(nrows=1500, quote_p=0.1, values=[v for v in PLAIN if "\u20ac".encode() not in v],
                   prefixes=(b"", "\u3000".encode(), "\u2002\u2002".encode()), delim="\u20ac".encode()),
              orc.Opts(comma="\u20ac", trim_leading_space=True)),
}
GENERAL = {"comment": True, "lazy": True, "runes": True, "fast": False, "slow": False, "long": False, "dense": False}


@pytest.mark.parametrize("eol", EOLS)
@pytest.mark.parametrize("route", list(ROUTES))
def test_route_and_line_end(route, eol):
    kw, o = ROUTES[route]
    data = make_csv(100 * list(ROUTES).index(route) + EOLS.index(eol), eol=eol, **kw)
    if route == "dense":
        assert len(data) / data.count(b"\n") < 16
    for select in (None, [b"c4", b"c0", b"c2"]):  # every column, and a selection in another order than the file's
        general = check_parse(data, o, select, trees_for(len(data), data, o, select))
        if route in GENERAL:
            assert general == GENERAL[route], route


@pytest.mark.parametrize("eol", ["lf", "crlf", "lone_cr"])
@pytest.mark.parametrize("route", ["fast", "slow", "dense", "trim"])
def test_padded_fields_of_short_records(route, eol):
    """NumFieldsAny: a selected column past the end of a short record is "" — it matches Like "" and nothing else"""
    kw, o = ROUTES[route]
    o = orc.Opts(**{**o.__dict__, "fields_per_record": -1})
    data = make_csv(7, eol=eol, short_p=0.4, **kw)
    for select in (None, [b"c4", b"c1"]):
        trees = trees_for(11, data, o, select)
        trees += [("like", {b"c4": b""}), ("like", {b"c4": b"a"}), ("all", [("like", {b"c3": b""}), ("not", ("like", {b"c1": b""}))])]
        check_parse(data, o, select, trees)


@pytest.mark.parametrize("eol", ["crlf", "mixed", "lone_cr"])
def test_streamed_batches(monkeypatch, eol):
    """FromReader in small pieces: batch cuts fall inside the data, each batch is parsed with the predicate fused"""
    import csvplus_b200 as cp
    o = orc.Opts()
    data = make_csv(21, nrows=800, eol=eol, quote_p=0.2) + b'9,"bad"x\n1,2,3,4,5\n'
    rows, err = reference(data, o, [b"c4", b"c1"])
    assert err is not None
    for i, tree in enumerate(trees_for(5, data, o, [b"c4", b"c1"])):
        monkeypatch.setattr(cp.api, "STREAM_BATCH_BYTES", (97, 1000, 4096)[i % 3])
        got = pulled(cp.Take(cp.FromReader(io.BytesIO(data)).SelectColumns("c4", "c1")).Filter(to_cp(tree)))
        assert got == ([r for r in rows if holds(tree, r)], err), tree


@pytest.mark.parametrize("world", [2, 3, 4])
def test_byte_range_shards(world):
    from tests.test_gpu_shards import _run_sharded
    o = orc.Opts()
    data = make_csv(world, nrows=3000, eol="mixed", quote_p=0.2)
    for select in (None, [b"c4", b"c0"]):
        rows, err = reference(data, o, select)
        assert err is None
        for tree in trees_for(world, data, o, select, n=4):
            whole, errs, _ = _run_sharded(data, world, spec=[(c.decode(), -1) for c in select] if select else None, pred=to_cp(tree))
            assert all(e is None for e in errs)
            assert table_rows(whole) == [r for r in rows if holds(tree, r)], tree


# ------------------------------------------------------------------ materialised tables (gather.cu filter_flags_kernel)
def _cut_trees(rng, rows, trees):
    """trees whose first false row is somewhere inside: Not(Like(row k's value)) beside a random tree's tautology"""
    out = []
    for t in trees[:4]:
        k = rng.randrange(len(rows))
        key = rng.choice(sorted(rows[k]))
        out.append(("all", [("not", ("like", {key: rows[k][key]})), ("any", [t, ("not", t)])]))
    return out + trees


@pytest.mark.parametrize("eol", ["lf", "crlf", "crcrlf"])
def test_table_filter_and_cuts(eol):
    import csvplus_b200 as cp
    o = orc.Opts()
    data = make_csv(31, nrows=1200, eol=eol, quote_p=0.15)
    rows, err = reference(data, o)
    assert err is None
    t0, e0 = cp.parse_csv(gpu_ctx(), data)
    assert e0 is None
    rng = random.Random(3)
    for tree in _cut_trees(rng, rows, trees_for(13, data, o, None)):
        p = to_cp(tree)
        assert table_rows(t0.filter(p)) == [r for r in rows if holds(tree, r)], tree
        cut = next((i for i, r in enumerate(rows) if not holds(tree, r)), len(rows))
        assert t0.first_false(p) == cut, tree
        assert pulled(cp.Take(cp.FromBytes(data)).TakeWhile(p)) == (rows[:cut], None), tree
        assert pulled(cp.Take(cp.FromBytes(data)).DropWhile(p)) == (rows[cut:], None), tree


def test_filter_after_join_and_on_take_rows():
    import csvplus_b200 as cp
    o = orc.Opts()
    data = make_csv(41, nrows=1500, eol="mixed", quote_p=0.15)
    labels = b"k,label\r\n" + b"".join(_quote(random.Random(0), v) + b",L%d\r\n" % i for i, v in enumerate(PLAIN[:-1] + [b"c,d", b"Ann\r"]))
    joined = orc.reader_rows(data, o).join(orc.reader_rows(labels, o).unique_index_on("k"), "c0").to_dicts()
    assert 0 < len(joined) < 1500
    rng = random.Random(4)
    observed = {k: sorted({r[k] for r in joined}) for k in joined[0]}
    keys = sorted(joined[0]) + [b"zz"]
    idx = cp.Take(cp.FromBytes(labels)).UniqueIndexOn("k")
    for _ in range(10):
        tree = random_tree(rng, keys, observed)
        want = [r for r in joined if holds(tree, r)]
        assert pulled(cp.Take(cp.FromBytes(data)).Join(idx, "c0").Filter(to_cp(tree))) == (want, None), tree
        assert pulled(cp.TakeRows([str_row(r) for r in joined]).Filter(to_cp(tree))) == (want, None), tree


# ------------------------------------------------------------------ size limits (CPB_PRED_MAX_* / CPB_MAX_PARSE_COLS)
def _any_of(values: list, cols: list):
    return ("any", [("like", {cols[i % len(cols)]: v}) for i, v in enumerate(values)])


def _chain(t, depth: int):
    for i in range(depth):
        t = (("all", [t]), ("not", t), ("any", [t]))[i % 3]
    return t


def _limit_trees(rows, ncols=NCOLS):
    from csvplus_b200 import _abi
    cols = [b"c%d" % i for i in range(ncols)]
    vals = [rows[i * 7 % len(rows)][cols[i % ncols]] for i in range(_abi.PRED_MAX_TERMS + 1)]
    terms = _any_of(vals[:_abi.PRED_MAX_TERMS], cols)  # 2 * 32 - 1 = 63 operations
    at = {"terms": terms, "ops": ("not", terms), "depth": _chain(("like", {b"c0": rows[0][b"c0"]}), _abi.PRED_MAX_DEPTH)}
    past = {"terms": _any_of(vals, cols), "ops": ("not", ("not", terms)),
            "depth": _chain(("like", {b"c0": rows[0][b"c0"]}), _abi.PRED_MAX_DEPTH + 1)}
    return at, past


def test_predicates_at_the_limits_run_on_the_device(monkeypatch):
    import csvplus_b200 as cp

    def no_host_rows(self, row):
        raise AssertionError("a recognisable predicate was evaluated on host rows")

    o = orc.Opts()
    data = make_csv(51, nrows=2000, eol="crlf", quote_p=0.1)
    rows, err = reference(data, o)
    t0, _ = cp.parse_csv(gpu_ctx(), data)
    at, _ = _limit_trees(rows)
    monkeypatch.setattr(cp.Predicate, "__call__", no_host_rows)
    for name, tree in at.items():
        want = [r for r in rows if holds(tree, r)]
        got, st = _stats(lambda: pulled(cp.Take(cp.FromBytes(data)).Filter(to_cp(tree))))
        assert got == (want, None) and "csv_scan" in st and "filter_like" not in st, name
        got, st = _stats(lambda: pulled(cp.TakeTable(t0).Filter(to_cp(tree))))
        assert got == (want, None) and "filter_like" in st, name


def test_predicates_past_the_limits_return_the_reference_rows():
    import csvplus_b200 as cp
    o = orc.Opts()
    data = make_csv(52, nrows=2000, eol="mixed", quote_p=0.1)
    rows, _ = reference(data, o)
    _, past = _limit_trees(rows)
    for name, tree in past.items():
        want = [r for r in rows if holds(tree, r)]
        assert want, name
        assert pulled(cp.Take(cp.FromBytes(data)).Filter(to_cp(tree))) == (want, None), name
        cut = next((i for i, r in enumerate(rows) if not holds(tree, r)), len(rows))
        assert pulled(cp.Take(cp.FromBytes(data)).TakeWhile(to_cp(tree))) == (rows[:cut], None), name
        assert not to_cp(tree).lowerable(), name  # (evaluated on host rows)


@pytest.mark.parametrize("npred", [15, 16, 20])
def test_predicate_over_many_columns_of_a_wide_file(npred):
    """a file of 24 columns is parsed 16 columns at a time; a predicate over 16 or more of them filters the parsed table"""
    import csvplus_b200 as cp
    o = orc.Opts()
    data = make_csv(53, nrows=1500, ncols=24, eol="crlf", quote_p=0.1)
    rows, _ = reference(data, o)
    cols = [b"c%d" % i for i in range(npred)]
    tree = ("any", [("like", {c: rows[3 * i][c]}) for i, c in enumerate(cols)] + [("not", ("like", {cols[-1]: b"a"}))])
    want = [r for r in rows if holds(tree, r)]
    assert 0 < len(want) < len(rows)
    got, st = _stats(lambda: pulled(cp.Take(cp.FromBytes(data)).Filter(to_cp(tree))))
    assert got == (want, None)
    assert ("filter_like" in st) == (npred >= 16)


# ------------------------------------------------------------------ Like on the last field of a CRLF record (SlowSink.unput)
def _both(data, tree, o=None, select=None):
    """-> (rows of the fused parse, rows of the DataSource plan), each checked against the reference"""
    import csvplus_b200 as cp
    o = o or orc.Opts()
    rows, err = reference(data, o, select)
    want = [r for r in rows if holds(tree, r)]
    t, gerr = cp.parse_csv(gpu_ctx(), data, **_opts_kw(o, select), pred=to_cp(tree))
    assert (str(gerr) if gerr else None) == err
    assert table_rows(t) == want
    return want


def test_crlf_quoted_record_keeps_like_on_its_last_field():
    want = _both(b'id,q,name\r\n1,"x",Ann\r\n2,y,Ann\r\n', ("like", {b"name": b"Ann"}))
    assert [r[b"id"] for r in want] == [b"1", b"2"]


def test_crlf_dense_tile_keeps_like_on_the_last_field():
    import csvplus_b200 as cp
    data = b"k,v\r\n" + b"".join(b"%d,a\r\n" % (i % 10) for i in range(10000))  # 5-byte lines: the dense fallback
    assert len(_both(data, ("like", {b"v": b"a"}))) == 10000
    assert len(cp.Take(cp.FromBytes(data)).Filter(cp.Like({"v": "a"})).ToRows()) == 10000


def test_crlf_empty_last_field_and_cr_literal():
    assert len(_both(b"k,v\r\n" + b'"1",\r\n' * 3 + b"2,\r\n", ("like", {b"v": b""}))) == 4
    assert len(_both(b"k,v\r\n" + b'"1",a\r\r\n' * 3 + b"2,a\r\r\n", ("like", {b"v": b"a\r"}))) == 4
    assert len(_both(b'k,v\r\n"1",a\r\n"2",a\r', ("like", {b"v": b"a"}))) == 2  # a lone \r before EOF


def test_crlf_general_path_keeps_like_on_the_last_field():
    body = b"".join(b"%d,Ann\r\n" % i for i in range(200))
    cases = [(b"k,v\r\n" + body + b'# "quoted comment\r\n' + body, orc.Opts(comment="#"), 400),  # a comment line holding a quote
             (b"k,v\r\n" + body + b'1"x,Ann\r\n' + body, orc.Opts(lazy_quotes=True), 401),    # a lazy quote
             # the rune delimiter through a stand-in byte (TrimLeadingSpace keeps it off the single-pass scan)
             ("k€v\r\n".encode() + body.replace(b",", "€".encode()), orc.Opts(comma="€", trim_leading_space=True), 200)]
    for data, o, n in cases:
        want, st = _stats(lambda: _both(data, ("like", {b"v": b"Ann"}), o))
        assert len(want) == n, o
        assert any(k.startswith("general_rec") for k in st), o
