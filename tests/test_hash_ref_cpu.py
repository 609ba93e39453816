"""tests/hash_ref.py on its own: the inverses undo the hashes, crafted values and rows collide where they are meant to
and nowhere else, and keys aimed at a join table slot start there.  (tests/test_gpu_hash_collisions.py checks the
restatement against the device.)"""
import random

import pytest

from tests import hash_ref as hr

M = hr.MASK


def test_inverses_round_trip():
    rng = random.Random(1)
    for _ in range(2000):
        w, i = rng.getrandbits(64), rng.randrange(600)
        assert hr.unfmix64(hr.fmix64(w)) == w and hr.fmix64(hr.unfmix64(w)) == w
        assert hr.unword_mix(hr.word_mix(w, i), i) == w
        n = rng.randrange(1 << 32)
        assert hr.unhash_finish(hr.hash_finish(w, n), n) == w
    for w in (0, 1, M, 1 << 63, hr.GOLDEN):
        assert hr.unfmix64(hr.fmix64(w)) == w


def test_empty_value_hashes_to_zero():
    assert hr.fmix64(0) == 0 and hr.value_hash(b"") == 0


def test_value_hash_by_definition():
    # words little-endian, the last zero-padded, the length folded in last
    assert hr.words(b"\x01\x02") == [0x0201]
    assert hr.value_hash(b"ab") == hr.hash_finish(hr.word_mix(0x6261, 0), 2)
    assert hr.value_hash(b"a") != hr.value_hash(b"a\0")  # the same words, another length
    v = bytes(range(20))
    s = sum(hr.word_mix(w, i) for i, w in enumerate(hr.words(v))) & M
    assert hr.value_hash(v) == hr.hash_finish(s, 20)


LENGTHS = [8, 9, 15, 16, 128, 129, 136, 4097]


@pytest.mark.parametrize("H", [M, 0, 0x0123456789ABCDEF], ids=["ones", "zero", "other"])
def test_crafted_values_collide(H):
    # (an 8-byte value is all word 0: one value per hash; 9 bytes leave one free byte)
    seeds = {8: 1, 9: 6}
    vals = [hr.collide(H, n, (H, n, s)) for n in LENGTHS for s in range(seeds.get(n, 6))]
    assert len(set(vals)) == len(vals)
    assert [len(v) for v in vals] == [n for n in LENGTHS for _ in range(seeds.get(n, 6))]
    assert {hr.value_hash(v) for v in vals} == {H}
    assert hr.collide(H, 40, 7) == hr.collide(H, 40, 7)  # deterministic in the seed
    # a rejected byte is drawn again
    v = hr.collide(H, 300, 3, reject=b"\r\n")
    assert b"\r" not in v and b"\n" not in v and hr.value_hash(v) == H


def test_ones_start_in_the_last_slot_of_every_table():
    for bits in range(6, 30):
        nslots = 1 << bits
        assert M & (nslots - 1) == nslots - 1 and 0 & (nslots - 1) == 0
        assert hr.codes_slots(nslots // 2) == nslots
    assert [hr.codes_slots(n) for n in (0, 1, 32, 33, 1000)] == [64, 64, 64, 128, 2048]
    assert [hr.groupby_slots(g) for g in (0, 32, 33, 64, 65, 3000)] == [64, 64, 128, 128, 256, 8192]
    assert hr.chain_crosses_end([63, 63], 64) and not hr.chain_crosses_end([63, 0, 1], 64)


@pytest.mark.parametrize("lengths", [[3, 16], [6, 12], [20, 5, 136], [4, 4, 8]])
def test_crafted_rows_collide_only_as_rows(lengths):
    R = 0xFEDCBA9876543210
    rows = [hr.collide_row(R, lengths, s) for s in range(40)]
    assert len(set(rows)) == len(rows) and all([len(v) for v in r] == lengths for r in rows)
    assert {hr.row_hash(r) for r in rows} == {R}
    for k in range(len(lengths)):  # no two different values of a column share a hash
        assert len({hr.value_hash(r[k]) for r in rows}) == len({r[k] for r in rows}), k
    assert len({hr.value_hash(r[-1]) for r in rows}) > 1  # the rows collide, their last columns do not
    assert hr.row_hash([b"a"]) == hr.row_hash_step(0, hr.value_hash(b"a"), 0)
    v = hr.collide(hr.row_target(R), 20, 1)  # one column: the value hash that gives the row hash R
    assert hr.row_hash([v]) == R and hr.value_hash(v) != R


def test_key_image():
    # width 7: value, zero padding, one length byte; over the width: cut, length all ones
    assert hr.key_image([b"ab"], [7]) == b"ab\0\0\0\0\0\x02"
    assert hr.key_image([b"abcdefghi"], [7]) == b"abcdefg\xff"
    assert hr.key_image([b"x", b""], [1, 300]) == b"x\x01" + b"\0" * 300 + b"\0\0"
    assert hr.key_image([b"x" * 70000], [65535]) == b"x" * 65535 + b"\xff\xff\xff\xff"
    assert [hr.len_bytes(w) for w in (0, 254, 255, 65534, 65535)] == [1, 1, 2, 2, 4]
    assert hr.image_bytes([7, 15]) == 8 + 16
    assert hr.image_words(b"\x01" + b"\0" * 7 + b"\x02") == [1 << 56, 2 << 56]


def test_probe_kinds_and_slots():
    assert hr.ordinal_slots(0) == 16 and hr.ordinal_slots(3000) == 8192 and hr.ordinal_slots(16384) == 32768
    assert hr.probe_kind(3000, 8, 5000) == "smem" and hr.probe_kind(16384, 25, 20000) == "smem"
    assert hr.probe_kind(20000, 12, 20000) == "unique16" and hr.probe_kind(20000, 12, 20001) == "run32"
    assert hr.probe_kind(17000, 24, 20000) == "run32" and hr.probe_kind(17000, 25, 20000) == "global"
    assert hr.probe_slots("unique16", 20000) == 40016 and hr.probe_slots("run32", 17000) == 25516
    assert hr.probe_slots("global", 17000) == 65536


@pytest.mark.parametrize("kind,width", [("smem", 7), ("global", 24), ("unique16", 11), ("run32", 23), ("unique16", 3)])
def test_aimed_keys_start_where_intended(kind, width):
    nslots = {"smem": 8192, "global": 65536, "unique16": 40016, "run32": 25516}[kind]
    rng = random.Random(width)
    cand = [b"%0*d" % (width, rng.randrange(10 ** width)) for _ in range(3000)]
    starts = hr.np_probe_start(kind, cand, width, nslots)
    for k, s in zip(cand[:300], starts[:300]):
        assert int(s) == hr.probe_start(kind, [k], [width], nslots)
        assert 0 <= s < nslots
    if kind == "unique16":
        assert list(hr.first_slots(cand[:50], nslots)) == list(starts[:50])
    # a short key (shorter than the width) by the scalar definition
    short = b"ab"
    img = hr.key_image([short], [width])
    ws = hr.image_words(img, 4)
    want = hr.hash_prefix(ws, len(img)) & (nslots - 1) if kind in ("smem", "global") else \
        hr.slot_of(hr.hash3(ws[0], ws[1], 0 if kind == "unique16" else ws[2]), nslots)
    assert hr.probe_start(kind, [short], [width], nslots) == want
    assert list(hr.np_probe_start(kind, [short, b"cd"], width, nslots))[0] == want


def test_hash_prefix_masks_the_partial_word():
    ws = [0x0102030405060708, 0xAABBCCDDEEFF0011, 0x1234]
    assert hr.hash_prefix(ws, 9) == hr.hash_prefix([ws[0], 0xAA00000000000000, 99], 9)
    assert hr.hash_prefix(ws, 8) == hr.mix64(hr.GOLDEN ^ ws[0]) and hr.hash_prefix([], 0) == hr.GOLDEN
    assert hr.slot_of(M, 40016) == 40015 and hr.slot_of(0, 40016) == 0
