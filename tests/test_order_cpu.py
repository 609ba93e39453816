"""Known answers of tests/order_ref.py, the restatement OrderBy's GPU results are compared against: NaN, infinities and
signed zeros under cmp.Compare, int64 extremes, byte order of strings, ties in both directions, mixed keys, the
conversion error rule, and the ValueError rules of DataSource.OrderBy (checked when it is called, before anything runs)."""
import pytest

from tests import order_ref as orf


def _col(rows, c="v"):
    return [r[c] for r in rows]


def _rows(*vals, c="v"):
    return [{c: v, "i": b"%d" % i} for i, v in enumerate(vals)]


def test_nan_before_negative_infinity_and_all_nans_equal():
    rows = _rows(b"1", b"-Inf", b"NaN", b"-1e308", b"nan", b"+Inf", b"5e-324", b"0x1p-1074")
    got = orf.order(rows, [("v", "float64", "asc")])
    assert _col(got) == [b"NaN", b"nan", b"-Inf", b"-1e308", b"5e-324", b"0x1p-1074", b"1", b"+Inf"]
    got = orf.order(rows, [("v", "float64", "desc")])
    assert _col(got) == [b"+Inf", b"1", b"5e-324", b"0x1p-1074", b"-1e308", b"-Inf", b"NaN", b"nan"]


def test_signed_zeros_tie_and_keep_plan_order_both_ways():
    rows = _rows(b"0", b"-0", b"+0", b"-0.0", b"0x0p0", b"-1", b"1")
    assert _col(orf.order(rows, [("v", "float64", "asc")])) == [b"-1", b"0", b"-0", b"+0", b"-0.0", b"0x0p0", b"1"]
    assert _col(orf.order(rows, [("v", "float64", "desc")])) == [b"1", b"0", b"-0", b"+0", b"-0.0", b"0x0p0", b"-1"]


def test_int64_extremes():
    rows = _rows(b"0", b"9223372036854775807", b"-9223372036854775808", b"-1", b"+5", b"10", b"9")
    assert _col(orf.order(rows, [("v", "int", "asc")])) == [b"-9223372036854775808", b"-1", b"0", b"+5", b"9", b"10",
                                                            b"9223372036854775807"]
    assert _col(orf.order(rows, [("v", "str", "asc")]))[:3] == [b"+5", b"-1", b"-9223372036854775808"]  # bytes, not numbers


def test_strings_compare_as_unsigned_bytes_with_a_prefix_first():
    rows = _rows(b"ab", b"a", b"", b"\xff", b"\x7f", b"a\x00", b"\x80a", b"b")
    assert _col(orf.order(rows, [("v", "str", "asc")])) == [b"", b"a", b"a\x00", b"ab", b"b", b"\x7f", b"\x80a", b"\xff"]
    assert _col(orf.order(rows, [("v", "str", "desc")])) == [b"\xff", b"\x80a", b"\x7f", b"b", b"ab", b"a\x00", b"a", b""]


def test_mixed_kinds_and_directions_keep_ties_in_plan_order():
    rows = [{"a": a, "b": b, "c": c, "i": b"%d" % i} for i, (a, b, c) in enumerate(
        [(b"x", b"2", b"1.5"), (b"y", b"10", b"NaN"), (b"x", b"10", b"-0"), (b"x", b"2", b"0"), (b"y", b"10", b"2"),
         (b"x", b"10", b"NaN"), (b"y", b"2", b"0")])]
    got = orf.order(rows, [("b", "int", "desc"), ("a", "str", "asc"), ("c", "float64", "desc")])
    assert _col(got, "i") == [b"2", b"5", b"4", b"1", b"0", b"3", b"6"]
    assert _col(orf.order(rows, [("b", "int", "desc"), ("a", "str", "asc")], limit=3), "i") == [b"2", b"5", b"1"]
    assert orf.order(rows, [("a", "str", "asc")], limit=0) == []


def test_conversion_error_lowest_row_then_earlier_key():
    rows = [{"a": b"1", "b": b"x"}, {"a": b"y", "b": b"2"}, {"a": b"z", "b": b"1e999"}]
    assert orf.error(rows, [("a", "int", "asc"), ("b", "float64", "asc")]) == (
        0, 'column "b": cannot convert "x" to float: invalid syntax')
    assert orf.error(rows, [("b", "str", "asc"), ("a", "int", "asc")]) == (
        1, 'column "a": cannot convert "y" to integer: invalid syntax')
    assert orf.error(rows[2:], [("b", "float64", "asc")]) == (0, 'column "b": cannot convert "1e999" to float: value out of range')
    # a missing key column fails at row 0; a conversion error at row 0 of an earlier key wins
    assert orf.error(rows, [("zz", "str", "asc")]) == (0, 'missing column "zz"')
    assert orf.error(rows, [("b", "int", "asc"), ("zz", "int", "asc")])[1].startswith('column "b"')
    assert orf.error(rows, [("a", "str", "asc"), ("b", "str", "asc")]) is None
    assert orf.error([], [("zz", "int", "asc")]) is None


def test_order_by_value_errors_before_anything_runs():
    import csvplus_b200 as cp
    src = cp.TakeRows([{"a": "1", "b": "2"}])
    for keys, msg in (((), "empty key list in OrderBy()"),
                      (("a", ("a", "int")), "duplicate column name(s) in OrderBy()"),
                      ((("a", "float32"),), "unknown kind"),
                      ((("a", "int", "up"),), "unknown direction"),
                      ((("a", "int", "desc", "x"),), "is not a column name"),
                      ((5,), "is not a column name"),
                      (tuple("k%d" % i for i in range(cp.MAX_ORDER_KEYS + 1)), "more than 16 keys")):
        with pytest.raises(ValueError) as e:
            src.OrderBy(*keys)
        assert msg in str(e.value)
    # 16 keys of every form are accepted (nothing runs until a sink pulls the rows)
    ok = src.OrderBy("a", ("b", "int"), ("c", "float64", "desc"), *("k%d" % i for i in range(13)))
    assert ok._src[0] == "ordered" and ok._src[2][:3] == (("a", "str", "asc"), ("b", "int", "asc"), ("c", "float64", "desc"))
    assert cp.ORDER_KINDS == ("str", "int", "float64")
