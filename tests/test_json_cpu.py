"""ToJSON's text without a GPU: known answers of the restated encoder (tests/json_oracle.py) for every byte class of
encoding/json's string encoding, a differential fuzz of that restatement against the host encoder of csvplus_b200.api,
and the committed fixture."""
import os
import random

from oracle import oracle as orc
from tests import json_oracle as jo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_control_bytes():
    short = {0x08: b"\\b", 0x09: b"\\t", 0x0A: b"\\n", 0x0C: b"\\f", 0x0D: b"\\r"}
    for c in range(0x20):
        assert jo.enc(bytes([c])) == b'"' + short.get(c, b"\\u00%02x" % c) + b'"', c
    assert jo.enc(b"\x1f\x0b") == b'"\\u001f\\u000b"'  # lowercase hex


def test_ascii_and_html():
    assert jo.enc(b'"') == b'"\\""'
    assert jo.enc(b"\\") == b'"\\\\"'
    assert jo.enc(b"\x7f") == b'"\x7f"'
    assert jo.enc(b"<a href='x'>&amp;</a>") == b"\"<a href='x'>&amp;</a>\""  # SetEscapeHTML(false)
    assert jo.enc(b"") == b'""'


def test_utf8_valid_and_separators():
    assert jo.enc("\u00e9\u20ac\U0001F642\U0010FFFF\ufffd".encode()) == b'"' + "\u00e9\u20ac\U0001F642\U0010FFFF\ufffd".encode() + b'"'
    assert jo.enc("a\u2028b\u2029c".encode()) == b'"a\\u2028b\\u2029c"'
    assert jo.enc("\u202a\u2027".encode()) == b'"' + "\u202a\u2027".encode() + b'"'


def test_utf8_invalid_classes():
    R = b"\\ufffd"
    cases = {
        b"\x80": R, b"\xbf": R,                                        # lone continuation bytes
        b"\xc0\xaf": R + R, b"\xc1\xbf": R + R,                        # C0 / C1 leads (overlong 2-byte)
        b"\xe0\x80\x80": R * 3, b"\xe0\x9f\xbf": R * 3,               # E0 overlong
        b"\xed\xa0\x80": R * 3, b"\xed\xbf\xbf": R * 3,               # surrogates
        b"\xf0\x80\x80\x80": R * 4,                                    # F0 overlong
        b"\xf4\x90\x80\x80": R * 4,                                    # above U+10FFFF
        b"\xf5\x80\x80\x80": R * 4, b"\xff": R, b"\xfe": R,            # F5-FF never start a rune
        b"a\xe2\x82": b"a" + R + R,                                    # truncated at the end of the value
        b"\xf0\x9f\x99": R * 3,
        b"\xe2\x28\xa1": R + b"(" + R,                                 # a bad continuation re-starts at the next byte
        b"\xc3\xa9\xc3": "\u00e9".encode() + R,
        b"\xed\x9f\xbf": "\ud7ff".encode(),                            # last code point before the surrogates
        b"\xf4\x8f\xbf\xbf": "\U0010ffff".encode(),
    }
    for raw, want in cases.items():
        assert jo.enc(raw) == b'"' + want + b'"', raw


def test_document_shapes():
    assert jo.document([]) == b"[]"
    assert jo.document([{}]) == b"[{}\n]"
    assert jo.document([{b"a": b"1"}, {b"b": b"2", b"a": b""}]) == b'[{"a":"1"}\n,{"a":"","b":"2"}\n]'  # heterogeneous rows
    # bytewise key order: "B" < "a" < "\u00e9"
    assert jo.document([{"\u00e9".encode(): b"3", b"a": b"2", b"B": b"1"}]) == ('[{"B":"1","a":"2","\u00e9":"3"}\n]').encode()
    rows = [{b"a": b"x"}, {b"a": b"y"}, {b"a": b"z"}]
    assert jo.document(rows[:1], True, False) + jo.document(rows[1:], False, True) == jo.document(rows)
    assert jo.columns_document([b"b", b"a"], [[b"1", b"2"], [b"3", b"4"]]) == jo.document([{b"b": b"1", b"a": b"3"}, {b"b": b"2", b"a": b"4"}])


def test_host_encoder_b_and_f():
    from csvplus_b200.api import _go_json_string
    assert _go_json_string(b"\x08\x0c") == b'"\\b\\f"'
    assert _go_json_string(b"a\x08b\x0cc\x07") == b'"a\\bb\\fc\\u0007"'


def test_host_encoder_differential_fuzz():
    """the restated encoder and the host encoder agree on 20 000 seeded random byte strings, biased towards the bytes
    that take the escape / UTF-8 paths"""
    from csvplus_b200.api import _go_json_string
    rng = random.Random(0x15011)
    pool = list(range(0x20)) + [0x22, 0x5C, 0x7F, 0x41, 0x20] + [0x80, 0x8F, 0x90, 0x9F, 0xA0, 0xA8, 0xA9, 0xBF] + \
        [0xC0, 0xC1, 0xC2, 0xC3, 0xDF, 0xE0, 0xE1, 0xE2, 0xEC, 0xED, 0xEE, 0xEF, 0xF0, 0xF1, 0xF3, 0xF4, 0xF5, 0xFF]
    for i in range(20_000):
        n = rng.randrange(0, 24)
        if i % 3 == 0:
            s = bytes(rng.randrange(256) for _ in range(n))
        else:
            s = bytes(rng.choice(pool) for _ in range(n))
        assert jo.enc(s) == _go_json_string(s), s
    for ch in ("\u2028", "\u2029", "\U0001F642", "\u00e9", "\u07ff", "\u0800", "\uffff", "\U00010000"):
        assert jo.enc(ch.encode()) == _go_json_string(ch)


def test_json_fixture():
    csv = open(os.path.join(GOLDEN, "json_escapes.csv"), "rb").read()
    want = open(os.path.join(GOLDEN, "json_escapes.json"), "rb").read()
    rows = orc.reader_rows(csv, select=["a", "B", "\u00e9", 'k"\\<'])
    assert rows.error is None
    assert jo.document(rows.to_dicts()) == want
    # the fixture holds every byte class: all control bytes, quote, backslash, 0x7f, separators, invalid UTF-8
    for needle in [b"\\u%04x" % c for c in range(0x20) if c not in (8, 9, 10, 12, 13)] + \
            [b"\\b", b"\\t", b"\\n", b"\\f", b"\\r", b'\\"', b"\\\\", b"\x7f", b"\\u2028", b"\\u2029", b"\\ufffd", b'"k\\"\\\\<":']:
        assert needle in want, needle
