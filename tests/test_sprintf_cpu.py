"""The Sprintf restatement (sprintf_ref.py) against answers derived from Go's fmt rules, and against a second,
independent route: Python's % operator over text decoded with surrogateescape, which gives one code point per Go rune
(invalid bytes included), so its precision and width count what Go's truncateString and padString count."""
import random

import pytest

from tests import sprintf_ref as ref

ALPHABET = b"abcdefghijklmnopqrstuvwxyz"
NIHON = "日本語日本語".encode()


@pytest.mark.parametrize("fmt,values,want", [
    (b"%5s", [b"abc"], b"  abc"),
    (b"%-5s|", [b"abc"], b"abc  |"),
    (b"%.5s", [ALPHABET], b"abcde"),
    (b"%.0s", [NIHON], b""),
    (b"%.5s", [NIHON], "日本語日本".encode()),
    (b"%4s", ["日本".encode()], "  日本".encode()),
    (b"%.2s", [b"\xe2\x82a"], b"\xe2\x82"),
    (b"%6s|", [b"\xf4\x90\x80\x80"], b"  \xf4\x90\x80\x80|"),
    (b"%.s|", [b"abc"], b"|"),
    (b"%--5s|", [b"ab"], b"ab   |"),
    (b"%5.1s|", [b"xyz"], b"    x|"),
    (b"100%%", [], b"100%"),
    (b"%v-%s", [b"a", b"b"], b"a-b"),
    (b"%s%s", [b"", b""], b""),
    (b"\x00\xff%s\xc2", [b"\x00"], b"\x00\xff\x00\xc2"),
    (b"%3s", [b"\xed\xa0\x80"], b"\xed\xa0\x80"),  # a surrogate's bytes: three runes
    (b"%3s", [b"\xc0\x80"], b" \xc0\x80"),         # an overlong NUL: two runes
    (b"%.1s", [b"\xf0\x9f\x98\x80!"], b"\xf0\x9f\x98\x80"),
    (b"literal only", [], b"literal only"),
])
def test_known_answers(fmt, values, want):
    assert ref.sprintf(fmt, values) == want


def test_width_needs_no_count_at_four_bytes_per_rune():
    v = "😀".encode() * 3  # 12 bytes, 3 runes
    assert ref.sprintf(b"%3s", [v]) == v and ref.sprintf(b"%4s", [v]) == b" " + v


@pytest.mark.parametrize("fmt,nargs", ref.REFUSED)
def test_refused(fmt, nargs):
    with pytest.raises(ref.Refused):
        ref.parse(fmt, nargs)


EDGE_VALUES = [b"", b"\x00", b"a", b"\xe2\x82", b"\xe2\x82a", b"\xed\xa0\x80", b"\xc0\x80", b"\xf4\x90\x80\x80", b"\x80\x80",
               b"\xf0\x9f\x98", "😀".encode(), "é".encode(), "日本".encode(), b"\xff\xfe", b"%s", b"a b"]


def random_value(rng: random.Random) -> bytes:
    parts = [rng.choice(EDGE_VALUES) if rng.random() < 0.6 else bytes(rng.randrange(256) for _ in range(rng.randrange(4)))
             for _ in range(rng.randrange(6))]
    return b"".join(parts)


def random_format(rng: random.Random, nverbs: int) -> tuple:
    """(format bytes, the same format as Python %-text with every verb s)"""
    go, py = [], []
    for k in range(nverbs + 1):
        lit = rng.choice([b"", b" ", b"|", b"\xc2\xa3", b"\xff", b"\x00", b"%%", b"ab%%c"])
        go.append(lit); py.append(lit.decode("utf-8", "surrogateescape"))
        if k == nverbs:
            break
        spec = "-" * rng.choice([0, 0, 1, 2])
        if rng.random() < 0.5:
            spec += str(rng.choice([1, 2, 3, 5, 8, 13]))
        if rng.random() < 0.5:
            spec += "." + rng.choice(["", "0", "1", "2", "4", "07"])
        verb = rng.choice("sv")
        go.append(("%" + spec + verb).encode()); py.append("%" + spec + "s")
    return b"".join(go), "".join(py)


def test_fuzz_against_python_percent():
    rng = random.Random(20261017)
    for _ in range(4000):
        nverbs = rng.randrange(5)
        fmt, pyfmt = random_format(rng, nverbs)
        values = [random_value(rng) for _ in range(nverbs)]
        want = (pyfmt % tuple(v.decode("utf-8", "surrogateescape") for v in values)).encode("utf-8", "surrogateescape")
        assert ref.sprintf(fmt, values) == want, (fmt, values)


def test_rune_table_against_python_decoder():
    """every 1- to 4-byte sequence's first rune, as Python's strict decoder sees it, over a grid of lead and next bytes"""
    conts = [0x00, 0x41, 0x7F, 0x80, 0x8F, 0x90, 0x9F, 0xA0, 0xBF, 0xC0, 0xFF]
    for lead in range(256):
        for b1 in conts:
            for b2 in conts:
                s = bytes([lead, b1, b2, 0x80])
                want = 1
                for n in (4, 3, 2, 1):
                    try:
                        if len(s[:n].decode("utf-8")) == 1:
                            want = n
                            break
                    except UnicodeDecodeError:
                        continue
                assert ref.rune_size(s, 0) == want, s.hex()
