"""The restated encoding/gob rules of tests/gob_oracle.py (the index file of Index.WriteTo / LoadIndex) against the
known answers of the gob package documentation, hand-derived type definitions, and a fuzzed round trip."""
import os
import random

from tests import gob_oracle as g

HERE = os.path.dirname(os.path.abspath(__file__))


def test_documentation_answers():
    # type Point struct{X, Y int}; Point{22, 33}: the definition message, then the value message
    point = g.enc_int(-65) + g.struct({2: g.struct({0: g.common_type(b"Point", 65), 1: g.enc_uint(2) + g.struct({0: g.enc_str(b"X"), 1: g.enc_int(2)})
                                                                                        + g.struct({0: g.enc_str(b"Y"), 1: g.enc_int(2)})})})
    assert g.message(point).hex(" ") == ("1f ff 81 03 01 01 05 50 6f 69 6e 74 01 ff 82 00 01 02 01 01 58 01 04 00 01 01 59 01 04 00 00 00")
    assert g.message(g.enc_int(65) + g.struct({0: g.enc_int(22), 1: g.enc_int(33)})).hex(" ") == "07 ff 82 01 2c 01 42 00"


def test_uint_int_edges():
    assert g.enc_uint(0) == b"\x00" and g.enc_uint(127) == b"\x7f"
    assert g.enc_uint(128) == b"\xff\x80" and g.enc_uint(255) == b"\xff\xff"
    assert g.enc_uint(256) == b"\xfe\x01\x00"
    assert g.enc_uint(1 << 16) == b"\xfd\x01\x00\x00"
    assert g.enc_uint(1 << 32) == b"\xfb\x01\x00\x00\x00\x00"
    assert g.enc_int(-129) == b"\xfe\x01\x01" and g.enc_int(-1) == b"\x01" and g.enc_int(63) == b"\x7e" and g.enc_int(64) == b"\xff\x80"
    for x in (0, 1, 127, 128, 255, 256, 1 << 16, (1 << 32) - 1, 1 << 32, (1 << 64) - 1):
        b = g._Buf(g.enc_uint(x))
        assert b.uint() == x and b.i == len(b.b)
    for x in (0, -1, 1, -129, 128, -(1 << 40), (1 << 62)):
        assert g._Buf(g.enc_int(x)).int() == x


def test_type_definitions():
    # []string: wireType{SliceT: sliceType{CommonType{Id: 65}, Elem: string}}
    assert g.message(g.slice_def(65, g.STRING)).hex(" ") == "0c ff 81 02 01 02 ff 82 00 01 0c 00 00"
    # []Row: wireType{SliceT: sliceType{CommonType{Id: 67}, Elem: 66}}
    assert g.message(g.slice_def(67, 66)).hex(" ") == "0d ff 85 02 01 02 ff 86 00 01 ff 84 00 00"
    # Row: wireType{MapT: mapType{CommonType{Name: "Row", Id: 66}, Key: string, Elem: string}}
    assert g.message(g.map_def(b"Row", 66, g.STRING, g.STRING)).hex(" ") == "13 ff 83 04 01 01 03 52 6f 77 01 ff 84 00 01 0c 01 0c 00 00"
    # a whole file: the columns value and one row
    f = g.encode_index([b"id"], [{b"id": b"7", b"name": b"Ann"}])
    assert f.hex(" ") == ("0c ff 81 02 01 02 ff 82 00 01 0c 00 00 "
                          "07 ff 82 00 01 02 69 64 "
                          "0d ff 85 02 01 02 ff 86 00 01 ff 84 00 00 "
                          "13 ff 83 04 01 01 03 52 6f 77 01 ff 84 00 01 0c 01 0c 00 00 "
                          "13 ff 86 00 01 02 02 69 64 01 37 04 6e 61 6d 65 03 41 6e 6e")
    assert g.decode_index(f) == ([b"id"], [{b"id": b"7", b"name": b"Ann"}])


def test_golden_file_matches_the_restatement():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_gob_golden", os.path.join(HERE, "golden", "make_gob_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    with open(os.path.join(HERE, "golden", "people_index.gob"), "rb") as f:
        assert f.read() == mk.golden_bytes()


def test_fuzzed_round_trip():
    rng = random.Random(11)
    for trial in range(200):
        k = rng.randrange(1, 6)
        names = list({bytes(rng.randrange(256) for _ in range(rng.randrange(0, 5))) for _ in range(k)})
        n = rng.choice([0, 1, 2, 5, 127, 128, 300])
        rows = []
        for _ in range(n):
            rows.append({c: bytes(rng.randrange(256) for _ in range(rng.choice([0, 1, 5, 127, 128, 300]))) for c in names})
        keys = names[:rng.randrange(1, len(names) + 1)]
        order = g.random_order(trial)
        ids = rng.choice([(65, 66, 67), (70, 90, 80), (100, 101, 300)])
        data = g.encode_index(keys, rows, order=order, ids=ids, row_def_first=rng.random() < 0.5)
        assert g.decode_index(data) == (keys, rows)
        # and the pair order written is the one asked for
        vals = g.decode_stream(data)
        assert [dict(r) for r in vals[1]] == rows
    try:
        g.decode_index(b"")
    except g.GobError as e:
        assert str(e) == "EOF"
    else:
        raise AssertionError("empty stream decoded")
