"""The parse driver's cost per call on every route: host synchronisations, kernel launches and the kernels named in the
statistics, pinned for each route a parse can take (the exact scan, the scan with TrimLeadingSpace / CommentChar /
LazyQuotes checked on the fly, their multi-pass fallback, multi-byte runes, more than 16 columns, byte-range shards, a
streamed input) with and without a data error, together with the rows and the cpb_error each call reports.  A change
to the driver's structure must leave all of it as it is; the numbers were taken on an H100."""
import ctypes as C

import pytest

from tests.helpers import gpu_ctx, people_csv

pytestmark = pytest.mark.gpu


def _err(e) -> tuple:
    return (e.kind, e.column_index, e.line, e.has_line, e.msg.decode("utf-8", "replace"))


def _parse(data: bytes, spec=None, like=None, **opts) -> tuple:
    """cpb_parse_csv -> (status, rows, cpb_error fields)"""
    import csvplus_b200 as cp
    from csvplus_b200 import _abi, api
    ctx, keep = gpu_ctx(), []
    o = api._reader_opts(**opts)
    ptr, n, dev = api._input_ptr(data, None, False, keep)
    sa, nspec, pp = api._spec_and_pred(spec, cp.Like(like) if like else None, keep)
    h, e = C.c_void_p(), _abi.Error()
    st = ctx.lib.cpb_parse_csv(ctx.h, C.c_void_p(ptr), n, int(dev), C.byref(o), sa, nspec, pp, C.byref(h), C.byref(e))
    rows = len(api.Table(ctx, h)) if h.value else None
    return st, rows, _err(e)


def _shards(data: bytes, bad_second: bool) -> tuple:
    """two byte-range shards of one file (cpb_parse_csv_shard): (status, rows, records, cpb_error fields) of each"""
    from csvplus_b200 import _abi, api
    ctx = gpu_ctx()
    cut = data.index(b"\n", len(data) // 2) + 1
    if bad_second:
        data = data[:cut] + data[cut:].replace(b"\n", b",x\n", 1)
    out, spec, nf, hdr = [], None, 0, True
    for i, (lo, own, last) in enumerate([(0, cut, False), (cut, len(data) - cut, True)]):
        keep = []
        o = api._reader_opts(num_fields=nf, header_from_first_row=hdr)
        buf = data[lo:] if last else data[lo:lo + own + 4096]
        ptr, n, dev = api._input_ptr(buf, None, False, keep)
        sa, nspec, pp = api._spec_and_pred(spec, None, keep)
        h, e, recs = C.c_void_p(), _abi.Error(), C.c_uint64()
        st = ctx.lib.cpb_parse_csv_shard(ctx.h, C.c_void_p(ptr), n, int(dev), own, i, int(last), 0, C.byref(o), sa, nspec, pp,
                                         C.byref(h), C.byref(recs), C.byref(e))
        t = api.Table(ctx, h)
        out.append((st, len(t), recs.value, _err(e)))
        if i == 0:
            fields, nf = t.parsed_from()
            spec, hdr = list(fields.items()), False
    return tuple(out)


def _stream(data: bytes, piece: int, **opts) -> tuple:
    """cpb_stream_* over pushes of `piece` bytes: (status, rows, done, cpb_error fields) of every cpb_stream_next"""
    from csvplus_b200 import _abi, api
    ctx = gpu_ctx()
    s = api._Stream(ctx, None, spec=[], **opts)
    out = []
    try:
        for lo in range(0, len(data), piece):
            s.push(data[lo:lo + piece], lo + piece >= len(data))
            h, done, e = C.c_void_p(), C.c_int(), _abi.Error()
            st = ctx.lib.cpb_stream_next(s.h, C.byref(h), C.byref(done), C.byref(e))
            out.append((st, len(api.Table(ctx, h)) if h.value else None, done.value, _err(e)))
            if done.value:
                break
    finally:
        s.free()
    return tuple(out)


def _index_join(data: bytes, key: str, unique: bool, join_on: str) -> tuple:
    """IndexOn / UniqueIndexOn of a parsed table, then Join and Except of it against that index: (status, cpb_error)
    of each call"""
    from csvplus_b200 import _abi, api
    ctx = gpu_ctx()
    t, err = api.parse_csv(ctx, data)
    assert err is None
    out = []
    k, kk = api._strs([key])
    ix, e = C.c_void_p(), _abi.Error()
    out.append((ctx.lib.cpb_index_build(ctx.h, t.h, k, 1, int(unique), C.byref(ix), C.byref(e)), _err(e)))
    if ix.value:
        idx = api.Index(ctx, ix, [key])
        j, jk = api._strs([join_on])
        for fn in (ctx.lib.cpb_join, ctx.lib.cpb_except):
            h, e = C.c_void_p(), _abi.Error()
            out.append((fn(ctx.h, t.h, idx.h, j, 1, C.byref(h), C.byref(e)), _err(e)))
            if h.value:
                api.Table(ctx, h)
    return tuple(out)


def _with(data: bytes, at: int, line: bytes) -> bytes:
    """data with `line` inserted before line `at`"""
    lines = data.split(b"\n")
    return b"\n".join(lines[:at] + [line] + lines[at:])


PEOPLE = people_csv(3000)
SPACED = PEOPLE.replace(b",", b", ")
TABBED = PEOPLE.replace(b",", b"\t ")
COMMENTED = b"\n".join(ln + (b"\n# note %d" % i if i % 97 == 5 else b"") for i, ln in enumerate(PEOPLE.split(b"\n")))
BARE = _with(PEOPLE, 1700, b'9999,Am"elia,Smith,1950')
WIDE = b"\n".join([b",".join(b"c%d" % i for i in range(20))] +
                  [b",".join(b"%d_%d" % (r, c) for c in range(20)) for r in range(2000)]) + b"\n"
SELECT = [("name", -1), ("surname", -1), ("id", -1)]

CASES = {
    "default": lambda: _parse(PEOPLE, SELECT, {"name": "Amelia"}),
    "default_assume": lambda: _parse(PEOPLE, [("a", 0), ("c", 2)], header_from_first_row=False),
    "default_field_count": lambda: _parse(_with(PEOPLE, 2000, b"1,2,3,4,5"), SELECT),
    "default_bare_quote": lambda: _parse(BARE, SELECT),
    "default_misplaced": lambda: _parse(PEOPLE, [("name", 0)]),
    "default_not_found": lambda: _parse(PEOPLE, [("name", -1), ("x", -1), ("y", -1)]),
    "default_bad_delimiter": lambda: _parse(PEOPLE, SELECT, delimiter='"'),
    "default_empty": lambda: _parse(b""),
    "default_header_only": lambda: _parse(b"id,name\n", [("name", -1)]),
    "trim_scan": lambda: _parse(SPACED, SELECT, {"name": "Amelia"}, trim_leading_space=True),
    "trim_scan_field_count": lambda: _parse(_with(SPACED, 2100, b"1, 2"), SELECT, trim_leading_space=True),
    "trim_fallback": lambda: _parse(TABBED, SELECT, {"name": "Amelia"}, delimiter="\t", trim_leading_space=True),
    "trim_fallback_field_count": lambda: _parse(_with(TABBED, 900, b"1\t 2"), SELECT, delimiter="\t", trim_leading_space=True),
    "trim_unicode_space": lambda: _parse(_with(SPACED, 10, "7,\u3000Ava, Smith, 1990".encode()), SELECT, trim_leading_space=True),
    "comment_scan": lambda: _parse(COMMENTED, SELECT, {"name": "Amelia"}, comment="#"),
    "comment_scan_field_count": lambda: _parse(_with(COMMENTED, 2500, b"1,2"), SELECT, comment="#"),
    "comment_fallback": lambda: _parse(_with(COMMENTED, 50, b'# a "quoted note'), SELECT, comment="#"),
    "comment_fallback_field_count": lambda: _parse(_with(_with(COMMENTED, 50, b'# a "note'), 1200, b"1"), SELECT, comment="#"),
    "lazy_scan": lambda: _parse(PEOPLE, SELECT, {"name": "Amelia"}, lazy_quotes=True),
    "lazy_scan_field_count": lambda: _parse(_with(PEOPLE, 1300, b"1,2,3"), SELECT, lazy_quotes=True),
    "lazy_fallback": lambda: _parse(BARE, SELECT, lazy_quotes=True),
    "lazy_fallback_field_count": lambda: _parse(_with(BARE, 2200, b"1,2,3"), SELECT, lazy_quotes=True),
    "multibyte_delimiter": lambda: _parse(PEOPLE.replace(b",", "§".encode()), SELECT, delimiter="§"),
    "multibyte_delimiter_field_count": lambda: _parse(_with(PEOPLE, 800, b"1").replace(b",", "§".encode()), SELECT,
                                                      delimiter="§"),
    "wide": lambda: _parse(WIDE),
    "wide_like": lambda: _parse(WIDE, None, {"c3": "7_3"}),
    "wide_field_count": lambda: _parse(_with(WIDE, 1500, b"1,2")),
    "wide_misplaced": lambda: _parse(WIDE, [("c%d" % i, -1) for i in range(19)] + [("c19", 3)]),
    "shards": lambda: _shards(PEOPLE, False),
    "shards_field_count": lambda: _shards(PEOPLE, True),
    "stream": lambda: _stream(PEOPLE, 16 << 10),
    "stream_field_count": lambda: _stream(_with(PEOPLE, 2400, b"1,2"), 16 << 10),
    "stream_comment_bare_quote": lambda: _stream(_with(COMMENTED, 2400, b'1,"a"b,c,d'), 16 << 10, comment="#"),
    "index_join": lambda: _index_join(PEOPLE, "id", True, "id"),
    "index_missing_column": lambda: _index_join(PEOPLE, "nope", False, "id"),
    "unique_index_duplicate": lambda: _index_join(PEOPLE, "name", True, "name"),
    "join_missing_column": lambda: _index_join(PEOPLE, "id", False, "nope"),
}


def measure(case: str) -> dict:
    """runs the case twice (the first run warms every lazily initialised state up) and counts the second"""
    ctx = gpu_ctx()
    CASES[case]()
    ctx.sync()
    ctx.stats(enable=True, reset=True)
    s0, l0 = ctx.host_syncs(), ctx.kernel_launches()
    result = CASES[case]()
    s1, l1 = ctx.host_syncs(), ctx.kernel_launches()
    kernels = {k: v["launches"] for k, v in sorted(ctx.stats().items())}
    ctx.stats(enable=False, reset=True)
    return {"host_syncs": s1 - s0, "launches": l1 - l0, "kernels": kernels, "result": result}


def _lists(x):
    return [_lists(v) for v in x] if isinstance(x, (tuple, list)) else x


# measured at the commit before the driver was split into steps (H100 80GB HBM3)
EXPECTED = {
    'default': {'host_syncs': 2,
                'launches': 2,
                'kernels': {'csv_header': 1, 'csv_scan': 1, 'h2d_input': 0},
                'result': [0, 288, [0, -1, 0, 0, '']]},
    'default_assume': {'host_syncs': 2,
                       'launches': 2,
                       'kernels': {'csv_header': 1, 'csv_scan': 1, 'h2d_input': 0},
                       'result': [0, 3001, [0, -1, 0, 0, '']]},
    'default_field_count': {'host_syncs': 2,
                            'launches': 2,
                            'kernels': {'csv_header': 1, 'csv_scan': 1, 'h2d_input': 0},
                            'result': [1, 1999, [3, -1, 2001, 1, 'wrong number of fields']]},
    'default_bare_quote': {'host_syncs': 2,
                           'launches': 2,
                           'kernels': {'csv_header': 1, 'csv_scan': 1, 'h2d_input': 0},
                           'result': [1, 1699, [1, -1, 1701, 1, 'bare " in non-quoted-field']]},
    'default_misplaced': {'host_syncs': 1,
                          'launches': 1,
                          'kernels': {'csv_header': 1, 'h2d_input': 0},
                          'result': [1, 0, [7, 0, 1, 1, 'misplaced column "name": expected at pos. 0, but found at pos. 1']]},
    'default_not_found': {'host_syncs': 1,
                          'launches': 1,
                          'kernels': {'csv_header': 1, 'h2d_input': 0},
                          'result': [1, 0, [8, 1, 1, 1, 'columns not found: x, y']]},
    'default_bad_delimiter': {'host_syncs': 0,
                              'launches': 0,
                              'kernels': {'h2d_input': 0},
                              'result': [1, 0, [4, -1, 1, 1, 'csv: invalid field or comment delimiter']]},
    'default_empty': {'host_syncs': 1, 'launches': 1, 'kernels': {'csv_header': 1}, 'result': [1, 0, [5, -1, 1, 1, 'EOF']]},
    'default_header_only': {'host_syncs': 1,
                            'launches': 1,
                            'kernels': {'csv_header': 1, 'h2d_input': 0},
                            'result': [0, 0, [0, -1, 0, 0, '']]},
    'trim_scan': {'host_syncs': 4,
                  'launches': 4,
                  'kernels': {'csv_header': 1, 'csv_header_general': 1, 'csv_scan': 1, 'h2d_input': 0, 'subst_hist': 1},
                  'result': [0, 288, [0, -1, 0, 0, '']]},
    'trim_scan_field_count': {'host_syncs': 4,
                              'launches': 4,
                              'kernels': {'csv_header': 1,
                                          'csv_header_general': 1,
                                          'csv_scan': 1,
                                          'h2d_input': 0,
                                          'subst_hist': 1},
                              'result': [1, 2099, [3, -1, 2101, 1, 'wrong number of fields']]},
    'trim_fallback': {'host_syncs': 7,
                      'launches': 15,
                      'kernels': {'csv_header_general': 1,
                                  'general_boundaries': 6,
                                  'general_rec_count': 1,
                                  'general_rec_emit': 1,
                                  'h2d_input': 0,
                                  'scan_u32': 5,
                                  'subst_hist': 1},
                      'result': [0, 288, [0, -1, 0, 0, '']]},
    'trim_fallback_field_count': {'host_syncs': 7,
                                  'launches': 15,
                                  'kernels': {'csv_header_general': 1,
                                              'general_boundaries': 6,
                                              'general_rec_count': 1,
                                              'general_rec_emit': 1,
                                              'h2d_input': 0,
                                              'scan_u32': 5,
                                              'subst_hist': 1},
                                  'result': [1, 899, [3, -1, 901, 1, 'wrong number of fields']]},
    'trim_unicode_space': {'host_syncs': 8,
                           'launches': 18,
                           'kernels': {'csv_header_general': 1,
                                       'general_boundaries': 6,
                                       'general_rec_count': 1,
                                       'general_rec_emit': 1,
                                       'h2d_input': 0,
                                       'scan_u32': 6,
                                       'subst_count': 1,
                                       'subst_hist': 1,
                                       'subst_write': 1},
                           'result': [0, 3001, [0, -1, 0, 0, '']]},
    'comment_scan': {'host_syncs': 2,
                     'launches': 3,
                     'kernels': {'csv_header': 1, 'csv_header_general': 1, 'csv_scan': 1, 'h2d_input': 0},
                     'result': [0, 288, [0, -1, 0, 0, '']]},
    'comment_scan_field_count': {'host_syncs': 2,
                                 'launches': 3,
                                 'kernels': {'csv_header': 1, 'csv_header_general': 1, 'csv_scan': 1, 'h2d_input': 0},
                                 'result': [1, 2473, [3, -1, 2475, 1, 'wrong number of fields']]},
    'comment_fallback': {'host_syncs': 6,
                         'launches': 16,
                         'kernels': {'csv_header': 1,
                                     'csv_header_general': 1,
                                     'csv_scan': 1,
                                     'general_boundaries': 6,
                                     'general_rec_count': 1,
                                     'general_rec_emit': 1,
                                     'h2d_input': 0,
                                     'scan_u32': 5},
                         'result': [0, 3000, [0, -1, 0, 0, '']]},
    'comment_fallback_field_count': {'host_syncs': 6,
                                     'launches': 16,
                                     'kernels': {'csv_header': 1,
                                                 'csv_header_general': 1,
                                                 'csv_scan': 1,
                                                 'general_boundaries': 6,
                                                 'general_rec_count': 1,
                                                 'general_rec_emit': 1,
                                                 'h2d_input': 0,
                                                 'scan_u32': 5},
                                     'result': [1, 1185, [3, -1, 1187, 1, 'wrong number of fields']]},
    'lazy_scan': {'host_syncs': 2,
                  'launches': 3,
                  'kernels': {'csv_header': 1, 'csv_header_general': 1, 'csv_scan': 1, 'h2d_input': 0},
                  'result': [0, 288, [0, -1, 0, 0, '']]},
    'lazy_scan_field_count': {'host_syncs': 2,
                              'launches': 3,
                              'kernels': {'csv_header': 1, 'csv_header_general': 1, 'csv_scan': 1, 'h2d_input': 0},
                              'result': [1, 1299, [3, -1, 1301, 1, 'wrong number of fields']]},
    'lazy_fallback': {'host_syncs': 6,
                      'launches': 16,
                      'kernels': {'csv_header': 1,
                                  'csv_header_general': 1,
                                  'csv_scan': 1,
                                  'general_boundaries': 6,
                                  'general_rec_count': 1,
                                  'general_rec_emit': 1,
                                  'h2d_input': 0,
                                  'scan_u32': 5},
                      'result': [0, 3001, [0, -1, 0, 0, '']]},
    'lazy_fallback_field_count': {'host_syncs': 6,
                                  'launches': 16,
                                  'kernels': {'csv_header': 1,
                                              'csv_header_general': 1,
                                              'csv_scan': 1,
                                              'general_boundaries': 6,
                                              'general_rec_count': 1,
                                              'general_rec_emit': 1,
                                              'h2d_input': 0,
                                              'scan_u32': 5},
                                  'result': [1, 2199, [3, -1, 2201, 1, 'wrong number of fields']]},
    'multibyte_delimiter': {'host_syncs': 5,
                            'launches': 6,
                            'kernels': {'csv_header': 1,
                                        'csv_scan': 1,
                                        'h2d_input': 0,
                                        'scan_u32': 1,
                                        'subst_count': 1,
                                        'subst_hist': 1,
                                        'subst_write': 1},
                            'result': [0, 3000, [0, -1, 0, 0, '']]},
    'multibyte_delimiter_field_count': {'host_syncs': 5,
                                        'launches': 6,
                                        'kernels': {'csv_header': 1,
                                                    'csv_scan': 1,
                                                    'h2d_input': 0,
                                                    'scan_u32': 1,
                                                    'subst_count': 1,
                                                    'subst_hist': 1,
                                                    'subst_write': 1},
                                        'result': [1, 799, [3, -1, 801, 1, 'wrong number of fields']]},
    'wide': {'host_syncs': 5,
             'launches': 5,
             'kernels': {'csv_header': 3, 'csv_scan': 2, 'h2d_input': 0},
             'result': [0, 2000, [0, -1, 0, 0, '']]},
    'wide_like': {'host_syncs': 5,
                  'launches': 5,
                  'kernels': {'csv_header': 3, 'csv_scan': 2, 'h2d_input': 0},
                  'result': [0, 1, [0, -1, 0, 0, '']]},
    'wide_field_count': {'host_syncs': 5,
                         'launches': 5,
                         'kernels': {'csv_header': 3, 'csv_scan': 2, 'h2d_input': 0},
                         'result': [1, 1499, [3, -1, 1501, 1, 'wrong number of fields']]},
    'wide_misplaced': {'host_syncs': 1,
                       'launches': 1,
                       'kernels': {'csv_header': 1, 'h2d_input': 0},
                       'result': [1, 0, [7, 19, 1, 1, 'misplaced column "c19": expected at pos. 3, but found at pos. 19']]},
    'shards': {'host_syncs': 4,
               'launches': 4,
               'kernels': {'csv_header': 2, 'csv_scan': 2, 'h2d_input': 0},
               'result': [[0, 1527, 1527, [0, -1, 0, 0, '']], [0, 1473, 1473, [0, -1, 0, 0, '']]]},
    'shards_field_count': {'host_syncs': 4,
                           'launches': 4,
                           'kernels': {'csv_header': 2, 'csv_scan': 2, 'h2d_input': 0},
                           'result': [[1, 1526, 1527, [3, -1, 1526, 1, 'wrong number of fields']],
                                      [0, 1473, 1473, [0, -1, 0, 0, '']]]},
    'stream': {'host_syncs': 14,
               'launches': 14,
               'kernels': {'csv_header': 5, 'csv_scan': 5, 'stream_cut': 4},
               'result': [[0, 752, 0, [0, -1, 0, 0, '']], [0, 722, 0, [0, -1, 0, 0, '']], [0, 715, 0, [0, -1, 0, 0, '']],
                          [0, 710, 0, [0, -1, 0, 0, '']], [0, 101, 1, [0, -1, 0, 0, '']]]},
    'stream_field_count': {'host_syncs': 12,
                           'launches': 12,
                           'kernels': {'csv_header': 4, 'csv_scan': 4, 'stream_cut': 4},
                           'result': [[0, 752, 0, [0, -1, 0, 0, '']], [0, 722, 0, [0, -1, 0, 0, '']],
                                      [0, 715, 0, [0, -1, 0, 0, '']], [1, 210, 1, [3, -1, 2401, 1, 'wrong number of fields']]]},
    'stream_comment_bare_quote': {'host_syncs': 14,
                                  'launches': 35,
                                  'kernels': {'csv_header': 5, 'csv_header_general': 5, 'csv_scan': 5, 'stream_cut_dfa': 20},
                                  'result': [[0, 748, 0, [0, -1, 0, 0, '']], [0, 718, 0, [0, -1, 0, 0, '']],
                                             [0, 712, 0, [0, -1, 0, 0, '']], [0, 196, 0, [0, -1, 0, 0, '']],
                                             [1, 0, 1, [2, -1, 2376, 1, 'extraneous or missing " in quoted-field']]]},
    'index_join': {'host_syncs': 7,
                   'launches': 17,
                   'kernels': {'csv_header': 1,
                               'csv_scan': 1,
                               'h2d_input': 0,
                               'hash_build': 1,
                               'join_probe': 3,
                               'key_pack': 4,
                               'key_width': 1,
                               'scan_u32': 5,
                               'unique_check': 1},
                   'result': [[0, [0, -1, 0, 0, '']], [0, [0, -1, 0, 0, '']], [0, [0, -1, 0, 0, '']]]},
    'index_missing_column': {'host_syncs': 2,
                             'launches': 2,
                             'kernels': {'csv_header': 1, 'csv_scan': 1, 'h2d_input': 0},
                             'result': [[1, [11, 0, 2, 1, 'missing column "nope" while creating an index']]]},
    'unique_index_duplicate': {'host_syncs': 10,
                               'launches': 51,
                               'kernels': {'csv_header': 1,
                                           'csv_scan': 1,
                                           'gather_copy': 4,
                                           'h2d_input': 0,
                                           'image_gather': 1,
                                           'key_pack': 1,
                                           'key_width': 1,
                                           'radix_pass': 24,
                                           'rowhash_build': 1,
                                           'rowhash_scatter': 1,
                                           'scan_gather_len': 4,
                                           'scan_u32': 8,
                                           'sort_gather_word': 1,
                                           'sort_hist': 1,
                                           'unique_check': 2},
                               'result': [[1,
                                           [12, -1, 0, 0, 'duplicate value while creating unique index: { "name" : "Amelia" }']]]},
    'join_missing_column': {'host_syncs': 4,
                            'launches': 27,
                            'kernels': {'csv_header': 1,
                                        'csv_scan': 1,
                                        'h2d_input': 0,
                                        'image_gather': 1,
                                        'key_pack': 1,
                                        'key_width': 1,
                                        'radix_pass': 15,
                                        'scan_u32': 5,
                                        'sort_gather_word': 1,
                                        'sort_hist': 1},
                            'result': [[0, [0, -1, 0, 0, '']], [1, [10, 0, 2, 1, 'missing column "nope"']],
                                       [1, [10, 0, 2, 1, 'missing column "nope"']]]},
}


@pytest.mark.parametrize("case", list(CASES))
def test_parse_driver_counts(case):
    got = measure(case)
    got["result"] = _lists(got["result"])
    assert got == EXPECTED[case]
