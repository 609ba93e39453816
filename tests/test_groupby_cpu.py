"""Known answers of tests/groupby_ref.py, the restatement GroupBy's GPU results are compared against: signed zeros and
NaN under sums and math.Min / math.Max, int64 wrap, group identity over empty, NUL and split keys, first / last, the
conversion and missing-column errors."""
import math

from tests import groupby_ref as gr
from tests import strconv_oracle as so

B = so.bits_of
NEG0 = B(-0.0)


def _rows(*vals, col="v", key="k"):
    return [{key: k, col: v} for k, v in vals]


def test_sum_of_negative_zeros_is_positive_zero():
    # acc starts at +0.0 and +0 + -0 = +0, as custAmounts[cid] += amount gives
    _, acc, err = gr.fold(_rows((b"a", b"-0"), (b"a", b"-0.0")), ["k"], {"s": ("sum", "v", "float64")})
    assert err is None and acc["s"] == [0]


def test_float_sum_is_in_row_order_and_rounded_per_addition():
    rows = _rows((b"a", b"1e16"), (b"a", b"1"), (b"a", b"1"), (b"b", b"1"), (b"b", b"1"), (b"b", b"1e16"))
    _, acc, _ = gr.fold(rows, ["k"], {"s": ("sum", "v", "float64")})
    assert acc["s"] == [B(1e16), B(1e16 + 2)]  # 1e16 + 1 rounds back to 1e16; 2 + 1e16 does not


def test_nan_and_infinities_in_sums():
    _, acc, _ = gr.fold(_rows((b"a", b"1"), (b"a", b"NaN"), (b"a", b"2"), (b"b", b"+Inf"), (b"b", b"-Inf"), (b"c", b"-Inf")),
                        ["k"], {"s": ("sum", "v", "float64")})
    assert acc["s"] == [so.NAN_BITS, gr.X86_NAN, gr.NEG_INF]


def test_min_max_signed_zero_and_nan():
    aggs = {"lo": ("min", "v", "float64"), "hi": ("max", "v", "float64")}
    _, acc, _ = gr.fold(_rows((b"z", b"0"), (b"z", b"-0"), (b"y", b"-0"), (b"y", b"0"), (b"n", b"1"), (b"n", b"NaN"), (b"n", b"-5"),
                              (b"i", b"NaN"), (b"i", b"-Inf"), (b"i", b"+Inf")), ["k"], aggs)
    assert acc["lo"] == [NEG0, NEG0, so.NAN_BITS, gr.NEG_INF]
    assert acc["hi"] == [0, 0, so.NAN_BITS, gr.POS_INF]


def test_go_min_max_special_cases():
    assert gr.go_min(gr.NEG_INF, so.NAN_BITS) == gr.NEG_INF and gr.go_max(gr.POS_INF, so.NAN_BITS) == gr.POS_INF
    assert gr.go_min(0, NEG0) == NEG0 and gr.go_min(NEG0, 0) == NEG0
    assert gr.go_max(0, NEG0) == 0 and gr.go_max(NEG0, 0) == 0
    assert gr.go_min(B(2.5), B(-1.0)) == B(-1.0) and gr.go_max(B(2.5), B(-1.0)) == B(2.5)
    # the identities the folds start from
    for x in (B(1.5), NEG0, 0, so.NAN_BITS, gr.NEG_INF, gr.POS_INF):
        assert gr.go_min(gr.POS_INF, x) == (so.NAN_BITS if gr.is_nan(x) else x)
        assert gr.go_max(gr.NEG_INF, x) == (so.NAN_BITS if gr.is_nan(x) else x)


def test_int64_sum_wraps():
    m = str(so.INT64_MAX).encode()
    _, acc, _ = gr.fold(_rows((b"a", m), (b"a", b"1"), (b"b", b"-9223372036854775808"), (b"b", b"-1")), ["k"],
                        {"s": ("sum", "v", "int"), "lo": ("min", "v", "int"), "hi": ("max", "v", "int")})
    assert acc["s"] == [so.INT64_MIN, so.INT64_MAX]
    assert acc["lo"] == [1, so.INT64_MIN] and acc["hi"] == [so.INT64_MAX, -1]


def test_empty_and_nul_key_values_are_values():
    rows = [{"k": b"", "v": b"1"}, {"k": b"\x00", "v": b"2"}, {"k": b"", "v": b"3"}, {"k": b"\x00\x00", "v": b"4"}]
    order, acc, _ = gr.fold(rows, ["k"], {"n": ("count",), "s": ("sum", "v", "int")})
    assert order == [(b"",), (b"\x00",), (b"\x00\x00",)]
    assert acc["n"] == [2, 1, 1] and acc["s"] == [4, 2, 4]


def test_split_keys_are_different_groups():
    rows = [{"a": b"ab", "b": b"c"}, {"a": b"a", "b": b"bc"}, {"a": b"ab", "b": b"c"}]
    order, acc, _ = gr.fold(rows, ["a", "b"], {"n": ("count",)})
    assert order == [(b"ab", b"c"), (b"a", b"bc")] and acc["n"] == [2, 1]


def test_first_and_last():
    rows = _rows((b"x", b"5"), (b"y", b"7"), (b"x", b"-3"), (b"x", b"9"), (b"y", b"1"))
    order, acc, _ = gr.fold(rows, ["k"], {"f": ("first", "v", "int"), "l": ("last", "v", "int"), "fl": ("first", "v", "float64")})
    assert order == [(b"x",), (b"y",)]
    assert acc["f"] == [5, 7] and acc["l"] == [9, 1] and acc["fl"] == [B(5.0), B(7.0)]


def test_conversion_error_stops_before_its_row():
    rows = _rows((b"a", b"1"), (b"b", b"2"), (b"a", b"x"), (b"a", b"4"))
    order, acc, err = gr.fold(rows, ["k"], {"s": ("sum", "v", "int")})
    assert order == [(b"a",), (b"b",)] and acc["s"] == [1, 2]
    assert err == (2, 'column "v": cannot convert "x" to integer: invalid syntax')


def test_conversion_error_ties_go_to_the_earlier_aggregate():
    rows = [{"k": b"a", "p": b"1", "q": b"2"}, {"k": b"a", "p": b"?", "q": b"!"}]
    _, _, err = gr.fold(rows, ["k"], {"x": ("sum", "q", "float64"), "y": ("sum", "p", "int")})
    assert err == (1, 'column "q": cannot convert "!" to float: invalid syntax')


def test_missing_columns():
    _, _, err = gr.fold([{"k": b"a"}], ["k", "j"], {"n": ("count",)})
    assert err == (0, 'missing column "j"')
    _, _, err = gr.fold([{"k": b"a"}], ["k"], {"s": ("max", "w", "int")})
    assert err == (0, 'missing column "w"')


def test_float_sum_equals_python_sequential_sum():
    vals = [0.1, 0.2, 0.3, 1e-17, -0.6, 1e300, -1e300]
    rows = _rows(*[(b"g", repr(v).encode()) for v in vals])
    _, acc, _ = gr.fold(rows, ["k"], {"s": ("sum", "v", "float64")})
    s = 0.0
    for v in vals:
        s += v
    assert acc["s"] == [B(s)] and not math.isnan(s)
