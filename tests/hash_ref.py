"""Every hash of the CUDA hash tables, restated in plain Python, with the inverses that aim keys at chosen hashes.

keyhash.cuh (codes.cu, groupby.cu): the hash of a value is hash_finish(sum of word_mix(word i, i), length) over its 8-byte
little-endian words (the last one zero-padded).  fmix64 is a bijection (an xor-shift by 33 undoes itself, and both
multipliers are odd), so word_mix is one in the word: for any target hash H and any length >= 8, word 0 of a value can be
solved so that the value hashes to H (collide).  GroupBy chains the column hashes hk of a row as h = row_hash_step(h, hk, k)
from h = 0, which inverts the same way (collide_row).  Codes and GroupBy probe from hash & (nslots - 1).

rowhash.cuh / join.cu (Join, Except, LeftJoin, Filter set terms): a key is the order-preserving image of sort.cu (each
column's value cut or zero-padded to its width, then a big-endian length field; 0xff.. when the value is longer than
the width), read as big-endian 8-byte words.  The ordinal tables (smem, global) probe from hash_prefix & (nslots - 1), the
embedded-key tables from slot_of(hash3(w0, w1, 0)) (unique16) and slot_of(hash3(w0, w1, w2)) (run32).  Those inputs are
constrained, so keys are aimed at a slot by search over candidates (first_slots and friends, in numpy).

tests/hash_harness.cu checks this module against the device functions themselves."""
from __future__ import annotations

import random

import numpy as np

MASK = (1 << 64) - 1
C1, C2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53
C1_INV, C2_INV = pow(C1, -1, 1 << 64), pow(C2, -1, 1 << 64)
GOLDEN = 0x9E3779B97F4A7C15
LEN_MUL = 0xC2B2AE3D27D4EB4F
LONG_BYTES = 128  # keyhash.cuh: longer values are hashed and compared by a whole warp


# ------------------------------------------------------------------ keyhash.cuh
def fmix64(k: int) -> int:
    k ^= k >> 33
    k = k * C1 & MASK
    k ^= k >> 33
    k = k * C2 & MASK
    return k ^ (k >> 33)


def unfmix64(k: int) -> int:
    k ^= k >> 33
    k = k * C2_INV & MASK
    k ^= k >> 33
    k = k * C1_INV & MASK
    return k ^ (k >> 33)


def word_mix(w: int, i: int) -> int:
    return fmix64(w ^ ((i + 1) * GOLDEN & MASK))


def unword_mix(m: int, i: int) -> int:
    return unfmix64(m) ^ ((i + 1) * GOLDEN & MASK)


def hash_finish(s: int, length: int) -> int:
    return fmix64((s + length * LEN_MUL) & MASK)


def unhash_finish(h: int, length: int) -> int:
    """the word sum that hash_finish(., length) takes to h"""
    return (unfmix64(h) - length * LEN_MUL) & MASK


def words(b: bytes) -> list:
    """the 8-byte little-endian words of b, the last one zero-padded"""
    return [int.from_bytes(b[i:i + 8], "little") for i in range(0, len(b), 8)]


def value_hash(b: bytes) -> int:
    s = 0
    for i, w in enumerate(words(b)):
        s = (s + word_mix(w, i)) & MASK
    return hash_finish(s, len(b))


def row_hash_step(h: int, hk: int, k: int) -> int:
    return fmix64((h + word_mix(hk, k)) & MASK)


def row_hash(values) -> int:
    """GroupBy's hash of a row whose key columns hold `values`"""
    h = 0
    for k, v in enumerate(values):
        h = row_hash_step(h, value_hash(v), k)
    return h


def collide(H: int, length: int, seed, reject: bytes = b"") -> bytes:
    """a value of `length` >= 8 bytes with value_hash H: bytes 8.. drawn from random.Random(seed), word 0 solved (so the
    zero padding of a partial last word stays as it is).  Drawn again while it holds a byte of `reject`.  (There is one
    8-byte value per hash, and 256 ** (length - 8) values of a longer length.)"""
    assert length >= 8
    rng = random.Random(str(seed))
    while True:
        tail = rng.randbytes(length - 8)
        s = unhash_finish(H, length)
        for i, w in enumerate(words(tail)):
            s = (s - word_mix(w, i + 1)) & MASK
        v = unword_mix(s, 0).to_bytes(8, "little") + tail
        if not any(c in v for c in reject):
            return v


def row_target(R: int, h: int = 0, k: int = 0) -> int:
    """the column hash hk with row_hash_step(h, hk, k) == R: for k = h = 0, the value hash that makes a one-column row
    hash to R"""
    return unword_mix((unfmix64(R) - h) & MASK, k)


def collide_row(R: int, lengths: list, seed, reject: bytes = b"") -> tuple:
    """a row of len(lengths) key values with row_hash R: the columns before the last drawn from random.Random(seed) (empty
    for length 0), the last one (length >= 8) solved with collide"""
    rng = random.Random(str(seed))
    vals = []
    for n in lengths[:-1]:
        while True:
            v = rng.randbytes(n)
            if not any(c in v for c in reject):
                break
        vals.append(v)
    h = 0
    for k, v in enumerate(vals):
        h = row_hash_step(h, value_hash(v), k)
    return tuple(vals) + (collide(row_target(R, h, len(vals)), lengths[-1], rng.getrandbits(64), reject),)


def codes_slots(n: int) -> int:
    """codes.cu: slots of the table over n rows (a power of two >= 2n, at least 64)"""
    s = 64
    while s < 2 * n:
        s <<= 1
    return s


def groupby_first_slots(m: int) -> int:
    """groupby.cu: slots of the temporary first-appearance table over a push's m misses (as codes_slots)"""
    return codes_slots(m)


def groupby_slots(ngroups: int) -> int:
    """groupby.cu: slots of the persistent table once it holds ngroups groups: 64, doubled while 2 ngroups exceed it"""
    s = 64
    while 2 * ngroups > s:
        s *= 2
    return s


def chain_crosses_end(starts, nslots: int) -> bool:
    """whether linear probing from these start slots (one key each, in any insert order) fills slot nslots - 1 and wraps
    into slot 0: the keys starting at the last slot are more than the slot can hold"""
    return sum(1 for s in starts if s == nslots - 1) >= 2


# ------------------------------------------------------------------ rowhash.cuh / join.cu
mix64 = fmix64


def hash3(a: int, b: int, c: int) -> int:
    return mix64(mix64(mix64(GOLDEN ^ a) ^ b) ^ c)


def slot_of(h: int, nslots: int) -> int:
    return (h * nslots) >> 64


def len_bytes(w: int) -> int:
    """bytes of the length field after a key column of width w (core.hpp: len_field_bytes)"""
    return 1 if w < 255 else 2 if w < 65535 else 4


def image_bytes(widths) -> int:
    return sum(w + len_bytes(w) for w in widths)


def key_image(values, widths) -> bytes:
    """the key image of one row (sort.cu's packer, rowhash.cuh: pack3): per column the value cut or zero-padded to its
    width, then its length big-endian in len_bytes(width) bytes, all ones when the value is longer than the width"""
    out = b""
    for v, w in zip(values, widths):
        lb = len_bytes(w)
        lf = (1 << 32) - 1 if len(v) > w else len(v)
        out += v[:w].ljust(w, b"\0") + (lf & ((1 << (8 * lb)) - 1)).to_bytes(lb, "big")
    return out


def image_words(img: bytes, nwords: int | None = None) -> list:
    """big-endian 8-byte words of an image, zero-padded to nwords"""
    n = (len(img) + 7) // 8 if nwords is None else nwords
    img = img.ljust(8 * n, b"\0")
    return [int.from_bytes(img[8 * i:8 * i + 8], "big") for i in range(n)]


def hash_prefix(ws: list, pbytes: int) -> int:
    """the hash of the first pbytes bytes of an image given as words"""
    full, rem = pbytes >> 3, pbytes & 7
    h = GOLDEN
    for w in ws[:full]:
        h = mix64(h ^ w)
    if rem:
        h = mix64(h ^ (ws[full] & (MASK << (8 * (8 - rem)) & MASK)))
    return h


def ordinal_slots(nheads: int) -> int:
    """slots of the smem / global tables: a power of two, load factor at most 1/2"""
    s = 1
    while s < max(16, nheads * 2):
        s <<= 1
    return s


def unique16_slots(nheads: int) -> int:
    return nheads * 2 + 16


def run32_slots(nheads: int) -> int:
    return nheads + nheads // 2 + 16


def probe_kind(nheads: int, pbytes: int, nrows: int) -> str:
    """join.cu: probe_kind"""
    if (ordinal_slots(nheads) + nheads + 1) * 4 <= 200 * 1024:
        return "smem"
    if pbytes <= 12 and nheads == nrows:
        return "unique16"
    if pbytes <= 24:
        return "run32"
    return "global"


def probe_slots(kind: str, nheads: int) -> int:
    return {"smem": ordinal_slots, "global": ordinal_slots, "unique16": unique16_slots, "run32": run32_slots}[kind](nheads)


def probe_start(kind: str, values, widths, nslots: int) -> int:
    """the first slot of the probe sequence of a key (all the index's key columns) in a table of this kind"""
    img = key_image(values, widths)
    ws = image_words(img, max(3, (len(img) + 7) // 8))
    if kind in ("smem", "global"):
        return hash_prefix(ws, len(img)) & (nslots - 1)
    return slot_of(hash3(ws[0], ws[1], 0 if kind == "unique16" else ws[2]), nslots)


# ------------------------------------------------------------------ the same in numpy, over many candidate keys
U64 = np.uint64


def np_mix64(h):
    with np.errstate(over="ignore"):
        h = h ^ (h >> U64(33)); h = h * U64(C1)
        h = h ^ (h >> U64(33)); h = h * U64(C2)
        return h ^ (h >> U64(33))


def np_slot_of(h, nslots: int):
    """the high 64 bits of h * nslots (nslots < 2^32)"""
    with np.errstate(over="ignore"):
        lo, hi = h & U64(0xffffffff), h >> U64(32)
        return (hi * U64(nslots) + ((lo * U64(nslots)) >> U64(32))) >> U64(32)


def np_image_words(keys: list, width: int, nwords: int):
    """(len(keys), nwords) big-endian image words of equal-length one-column keys (length <= width < 255)"""
    n, length = len(keys), len(keys[0])
    img = np.zeros((n, 8 * nwords), np.uint8)
    if length:
        img[:, :length] = np.frombuffer(b"".join(keys), np.uint8).reshape(n, length)
    img[:, width] = length
    return img.reshape(n, nwords, 8)[:, :, ::-1].copy().view("<u8").reshape(n, nwords)


def np_probe_start(kind: str, keys: list, width: int, nslots: int):
    """probe_start of equal-length one-column keys, vectorised"""
    pbytes = width + 1
    ws = np_image_words(keys, width, max(3, (pbytes + 7) // 8))
    with np.errstate(over="ignore"):
        if kind in ("smem", "global"):
            full, rem = pbytes >> 3, pbytes & 7
            h = np.full(len(keys), GOLDEN, np.uint64)
            for w in range(full):
                h = np_mix64(h ^ ws[:, w])
            if rem:
                h = np_mix64(h ^ (ws[:, full] & U64(MASK << (8 * (8 - rem)) & MASK)))
            return h & U64(nslots - 1)
        h = np_mix64(np_mix64(np_mix64(U64(GOLDEN) ^ ws[:, 0]) ^ ws[:, 1]) ^ (U64(0) if kind == "unique16" else ws[:, 2]))
        return np_slot_of(h, nslots)


def first_slots(keys: list, nslots: int):
    """first slot of each key (equal-length byte strings of at most 11 bytes) as the one key column of a unique index on
    the row-carrying table (rowhash.cuh: rh_start), whose width is their length"""
    return np_probe_start("unique16", keys, len(keys[0]), nslots)
