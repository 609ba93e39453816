"""The stream cut rule (tests/stream_cut_ref.py) against the oracle: splitting an input at the cut of any of its prefixes
and parsing the second part with the header and field count the first part resolved gives the rows, the first error and
its line of the whole-input parse.  CPU only."""
import itertools
import random

import pytest

from oracle import oracle as orc
import tests.stream_cut_ref as ref
from tests.helpers import random_csv

OPTION_MATRIX = list(itertools.product(["", "#"], [False, True], [False, True], [0, -1, 5]))  # 24 combinations


def soup(seed: int) -> bytes:
    """random_csv with comment lines holding quotes, bare quotes, quotes after spaces and stray CRs mixed in"""
    rng = random.Random(seed)
    data = random_csv(seed, rng.randrange(3, 14), ncols=5, quoted_p=0.35, crlf_p=0.3, blank_p=0.15,
                      ragged_p=0.1 if seed % 3 == 0 else 0.0, trailing_newline=rng.random() < 0.8)
    lines = data.split(b"\n")
    out = []
    for i, ln in enumerate(lines):
        r = rng.random()
        if i and r < 0.12:
            out.append(b'#x"y,' + rng.choice([b'"', b'""', b'a"b']))  # a comment line (or data without CommentChar)
        elif i and r < 0.16:
            ln = ln + b' "q'  # a bare quote; lazily a quote inside a field
        elif i and r < 0.19:
            ln = b' "' + ln  # a quote after a space: a quoted field only under TrimLeadingSpace
        out.append(ln)
    return b"\n".join(out)


def check_split(data: bytes, cut: int, o: orc.Opts):
    whole = orc.reader_rows(data, o)
    first = orc.reader_rows(data[:cut], o)
    if first.error is not None:  # the error is met in the first part: it is the whole input's
        assert (first.error_kind, first.error_line) == (whole.error_kind, whole.error_line), (data, cut)
        assert first.to_dicts() == whole.to_dicts()
        return
    recs, _ = orc.csv_records(data[:cut], orc.Opts(comma=o.comma, comment=o.comment, fields_per_record=-1,
                                                    lazy_quotes=o.lazy_quotes, trim_leading_space=o.trim_leading_space))
    if not recs:  # only blank / comment lines: the second part is the start of the input
        second = orc.reader_rows(data[cut:], o)
        assert second.to_dicts() == whole.to_dicts() and second.error == whole.error, (data, cut)
        return
    header = recs[0]
    spec = {}
    for i, name in enumerate(header):  # later duplicates overwrite earlier ones (csvplus.go:1160-1168)
        spec[name.decode("utf-8", "surrogateescape")] = i
    nf = o.fields_per_record if o.fields_per_record != 0 else len(header)
    o2 = orc.Opts(comma=o.comma, comment=o.comment, fields_per_record=nf, lazy_quotes=o.lazy_quotes,
                  trim_leading_space=o.trim_leading_space)
    second = orc.reader_rows(data[cut:], o2, assume=spec)
    assert first.to_dicts() + second.to_dicts() == whole.to_dicts(), (data, cut)
    if second.error is None:
        assert whole.error is None, (data, cut, whole.error)
    else:
        before = len(recs) - 1  # data records of the first part
        assert (second.error_kind, second.error_line + 1 + before) == (whole.error_kind, whole.error_line), (data, cut)


@pytest.mark.parametrize("comment,lazy,trim,nf", OPTION_MATRIX)
def test_cut_is_a_record_boundary(comment, lazy, trim, nf):
    o = orc.Opts(comment=comment, lazy_quotes=lazy, trim_leading_space=trim, fields_per_record=nf)
    checked = 0
    for seed in range(40):
        data = soup(seed * 7919 + len(comment) * 3 + lazy * 5 + trim * 11 + nf)
        cuts = set()
        for k in range(len(data) + 1):
            cut = ref.stream_cut(data[:k], comment=comment, lazy=lazy, trim=trim)
            assert 0 <= cut <= k and (cut == 0 or data[cut - 1] == 0x0A)
            cuts.add(cut)
        for cut in sorted(cuts - {0}):
            check_split(data, cut, o)
            checked += 1
    assert checked > 100


def test_cut_examples():
    assert ref.stream_cut(b"") == 0
    assert ref.stream_cut(b"a,b") == 0
    assert ref.stream_cut(b"a,b\r\nc") == 5
    assert ref.stream_cut(b'a,"b\nc",d\ne') == 10
    assert ref.stream_cut(b'a,"b\nc') == 0  # ends inside a quoted field
    assert ref.stream_cut(b'h\n#"\nx\n') == 2  # parity: the comment's quote counts
    assert ref.stream_cut(b'h\n#"\nx\n', comment="#") == 7
    assert ref.stream_cut(b'h\na"b\nc\n') == 2
    assert ref.stream_cut(b'h\na"b\nc\n', lazy=True) == 8  # a lazy quote inside a field is data
    assert ref.stream_cut(b'h\n "a\nb\n', lazy=True) == 8  # no TrimLeadingSpace: the quote is data
    assert ref.stream_cut(b'h\n "a\nb\n', lazy=True, trim=True) == 2  # trimmed: it opens a quoted field
    nbsp = "\u00a0".encode()
    assert ref.stream_cut(b'h\n' + nbsp + b'"a\nb\n', lazy=True, trim=True) == 2  # a Unicode space is trimmed too
    assert ref.stream_cut(b'h\n' + nbsp + b'"a\nb\n', lazy=True) == 9
    semi = "\u00a7"  # a two-byte delimiter
    assert ref.stream_cut(b'h\nx' + semi.encode() + b'"a\nb\n', comma=semi, lazy=True) == 2
    assert ref.stream_cut(b'h\nx' + semi.encode() + b'"a\nb\n', lazy=True) == 10
