"""tests/parse_sizing_ref.py against hand-computed samples and capacities, and its builders against the caps they claim
to meet.  No GPU: the GPU side of these inputs is tests/test_gpu_scan_matrix.py."""
import pytest

from tests import parse_sizing_ref as ref


def _records(data: bytes) -> list:
    """the lines after the header, '#' lines dropped (the builders write no quotes)"""
    return [ln for ln in data.split(b"\n")[1:-1] if not ln.startswith(b"#")]


def test_tiny_file():
    """8 bytes: the windows are [0, 8), [4, 8) and [0, 8), none holds an aligned 16-byte block.  Thread 0 of the first
    and last window splits "1,2"; the middle one's thread 0 starts inside "1,2", whose newline is the last byte."""
    s = ref.sample(b"a,b\n1,2\n")
    assert (s.bytes, s.newlines, s.lines) == (0, 0, 2)
    assert s.field_bytes[:3] == [2, 2, 0]
    # avg falls back to n = 8; row_cap = min(4 / 8 * 1.1 + 4096, 4 / 2 + 2) = 4 -> 1 MiB rows; 2 lines < 16: body
    c = ref.estimate(s, 8, 4, [1, 0])
    assert (c.row_cap, c.data_cap) == (1 << 20, [4, 4])


def test_overlapping_windows():
    """100 000 bytes of 100-byte lines: windows [0, 65536), [50000, 100000) and [34464, 100000) overlap.
    Newlines at 100k + 99: 655 + 500 + 656 in 65536 + 50000 + 65536 aligned bytes.  Lines: 256 threads in the first and
    last window; in the middle one only t <= 194 (t = 195 starts at 99920, whose next line start is the end of input)."""
    data = (b"x" * 99 + b"\n") * 1000
    s = ref.sample(data)
    assert (s.bytes, s.newlines) == (65536 + 50000 + 65536, 655 + 500 + 656)
    assert s.lines == 256 + 195 + 256
    assert s.field_bytes[0] == 99 * s.lines and s.field_bytes[1] == 0
    c = ref.estimate(s, len(data), 0, [0])
    # body / avg * 1.1 + 4096 = 5196 -> 1 MiB rows; mean 99: 1 MiB * 99 * 1.25 + 4 MiB -> 128 MiB > body
    assert c.row_cap == 1 << 20
    assert int(float(1 << 20) * 99.0 * 1.25) + (4 << 20) == 133955584
    assert c.data_cap == [len(data)]


def test_field_past_the_sampled_ones():
    """fields 64 and up are not sampled: their cap is the body even when every sampled field has a small one"""
    b = ref.column_input(70, 63, 0)
    assert b.caps.data_cap[63] == ref.DATA_CLASS
    assert b.caps.data_cap[:64] == [ref.DATA_CLASS] * 64
    body = len(b.data) - b.data_start
    assert b.caps.data_cap[64:] == [body] * 6
    s = ref.sample(b.data)
    assert s.lines >= ref.MIN_SAMPLED_LINES and s.field_bytes[63] == s.lines  # one byte each in the window lines


def test_fewer_than_16_sampled_lines():
    """5001-byte lines never end within 4096 bytes of their start: no line counts, but the 10-byte field 0 their comma
    closes does.  With < 16 lines every field's cap is the body."""
    data = (b"x" * 10 + b"," + b"y" * 4989 + b"\n") * 20
    s = ref.sample(data)
    assert s.lines == 0
    assert s.field_bytes[0] > 0 and s.field_bytes[0] % 10 == 0 and s.field_bytes[1] == 0
    c = ref.estimate(s, len(data), 0, [0, 1])
    assert c.data_cap == [len(data)] * 2


def test_no_newline_in_the_windows():
    """no newline sampled: avg is the input size, so the row estimate is 4096 before the 1 MiB class"""
    data = b"z" * 300000
    s = ref.sample(data)
    assert (s.newlines, s.lines) == (0, 0)
    assert ref.estimate(s, len(data), 0, [0]) == ref.Caps(1 << 20, [300000])


@pytest.mark.parametrize("extra", [0, 1])
@pytest.mark.parametrize("variant", ["plain", "trim", "comment"])
def test_rows_builder_meets_row_cap(extra, variant):
    b = ref.rows_input(extra, trim=variant == "trim", comment=variant == "comment")
    assert b.caps.row_cap == 1 << 20
    assert len(_records(b.data)) == b.rows == b.caps.row_cap + extra
    assert ref.caps(b.data, b.data_start, [0, 1]) == b.caps


@pytest.mark.parametrize("error_at", [1000, -10])
def test_rows_builder_error_ordinal(error_at):
    b = ref.rows_input(5000, error_at=error_at)
    recs = _records(b.data)
    bad = [i for i, ln in enumerate(recs) if ln.count(b",") != 1]
    assert bad == [b.error_row]
    assert (b.error_row < b.caps.row_cap) == (error_at >= 0)


@pytest.mark.parametrize("extra", [0, 1])
def test_column_builder_meets_data_cap(extra):
    b = ref.column_input(3, 0, extra)
    recs = _records(b.data)
    assert b.caps.row_cap == 1 << 20 and len(recs) == b.rows < b.caps.row_cap
    tot = [sum(len(ln.split(b",")[f]) for ln in recs) for f in range(3)]
    assert tot == b.col_bytes
    assert tot[0] == b.caps.data_cap[0] + extra == ref.DATA_CLASS + extra
    assert tot[1] < b.caps.data_cap[1] // 4 and tot[2] < b.caps.data_cap[2] // 4


def test_wide_builder_overflows_field_63_only():
    b = ref.column_input(70, 63, 1)
    over = [f for f in range(70) if b.col_bytes[f] > b.caps.data_cap[f]]
    assert over == [63]
    assert b.col_bytes[63] == b.caps.data_cap[63] + 1


def test_flood_builder_far_over_both_caps():
    b = ref.flood_input()
    recs = _records(b.data)
    assert len(recs) == b.rows > 6 * b.caps.row_cap
    assert sum(len(ln) - 1 - len(ln.split(b",")[1]) for ln in recs) == b.col_bytes[0] > b.caps.data_cap[0]
    assert b.caps.data_cap[0] == ref.DATA_CLASS and b.col_bytes[1] < b.caps.data_cap[1]
