"""An independent restatement of the encoding/gob stream of an index file (Index.WriteTo / LoadIndex, csvplus.go:655-705),
written from the format's rules: a stream of messages `uint(len) int(type id) ...`, type definitions under negative ids
(wireType structs), values under positive ids; struct fields as (delta, value) pairs ending in 0; a top-level non-struct
value behind a 0 byte; slices and maps as a count then their elements.

encode_index() writes what WriteTo writes for key columns and rows, with the pair order of every row given explicitly
(the reference's is Go's random map order); decode_stream() is a generic decoder of such streams."""
from __future__ import annotations

import random

STRING = 6
ID_STRINGS, ID_ROW, ID_ROWS = 65, 66, 67
TOO_BIG = 8 << 30


class GobError(Exception):
    pass


def enc_uint(x: int) -> bytes:
    if x < 128:
        return bytes([x])
    b = x.to_bytes((x.bit_length() + 7) // 8, "big")
    return bytes([256 - len(b)]) + b


def enc_int(x: int) -> bytes:
    return enc_uint((~x << 1) | 1 if x < 0 else x << 1)


def enc_str(s: bytes) -> bytes:
    return enc_uint(len(s)) + s


def message(body: bytes) -> bytes:
    return enc_uint(len(body)) + body


def struct(fields: dict) -> bytes:
    """fields: {field number: encoded value}; zero values are left out by the caller"""
    out, last = b"", -1
    for f in sorted(fields):
        out += enc_uint(f - last) + fields[f]
        last = f
    return out + b"\0"


def common_type(name: bytes, tid: int) -> bytes:
    return struct({**({0: enc_str(name)} if name else {}), 1: enc_int(tid)})


def slice_def(tid: int, elem: int) -> bytes:
    return enc_int(-tid) + struct({1: struct({0: common_type(b"", tid), 1: enc_int(elem)})})


def map_def(name: bytes, tid: int, key: int, elem: int) -> bytes:
    return enc_int(-tid) + struct({3: struct({0: common_type(name, tid), 1: enc_int(key), 2: enc_int(elem)})})


def enc_row(pairs: list) -> bytes:
    return enc_uint(len(pairs)) + b"".join(enc_str(k) + enc_str(v) for k, v in pairs)


def encode_index(columns: list, rows: list, order=None, ids=(ID_STRINGS, ID_ROW, ID_ROWS), row_def_first=False) -> bytes:
    """columns: the key columns (bytes); rows: list of {bytes: bytes}; order(row) -> the row's (key, value) pairs in the order
    to write (default: bytewise by key, what WriteTo writes); ids / row_def_first: other legal type numberings and
    definition orders"""
    sid, rid, rsid = ids
    order = order or (lambda r: sorted(r.items()))
    out = message(slice_def(sid, STRING))
    out += message(enc_int(sid) + b"\0" + enc_uint(len(columns)) + b"".join(enc_str(c) for c in columns))
    defs = [message(slice_def(rsid, rid)), message(map_def(b"Row", rid, STRING, STRING))]
    out += b"".join(defs[::-1] if row_def_first else defs)
    out += message(enc_int(rsid) + b"\0" + enc_uint(len(rows)) + b"".join(enc_row(order(r)) for r in rows))
    return out


def random_order(seed: int):
    rng = random.Random(seed)

    def order(r):
        items = list(r.items())
        rng.shuffle(items)
        return items
    return order


# ------------------------------------------------------------------ decoding
class _Buf:
    def __init__(self, b: bytes):
        self.b, self.i = b, 0

    def uint(self) -> int:
        if self.i >= len(self.b):
            raise GobError("unexpected EOF")
        c = self.b[self.i]
        self.i += 1
        if c < 128:
            return c
        n = 256 - c
        if n > 8 or self.i + n > len(self.b):
            raise GobError("bad uint")
        v = int.from_bytes(self.b[self.i:self.i + n], "big")
        self.i += n
        return v

    def int(self) -> int:
        u = self.uint()
        return ~(u >> 1) if u & 1 else u >> 1

    def bytes_(self) -> bytes:
        n = self.uint()
        if self.i + n > len(self.b):
            raise GobError("string beyond the message")
        s = self.b[self.i:self.i + n]
        self.i += n
        return s


def _struct(buf: _Buf, field) -> dict:
    """a struct: field(number, buf) decodes one field's value"""
    out, f = {}, -1
    while True:
        d = buf.uint()
        if d == 0:
            return out
        f += d
        out[f] = field(f, buf)


def _wire_type(buf: _Buf) -> dict:
    def common(f, b):
        return b.bytes_() if f == 0 else b.int()

    def inner(f, b):
        return _struct(b, common) if f == 0 else b.int()

    return _struct(buf, lambda f, b: (f, _struct(b, inner)))


def decode_stream(data: bytes) -> list:
    """-> the values of the stream in order: [] of strings for slices of string, [] of [(key, value)] for slices of maps of
    string to string (the pairs in file order).  Raises GobError("EOF") when it ends between messages."""
    i, types, values = 0, {}, []
    while i < len(data):
        head = _Buf(data[i:])
        n = head.uint()
        if n >= TOO_BIG or head.i + n > len(head.b):
            raise GobError("unexpected EOF")
        body = _Buf(data[i + head.i:i + head.i + n])
        i += head.i + n
        tid = body.int()
        if tid < 0:
            types[-tid] = _wire_type(body)
            continue
        kind, t = types[tid][next(iter(types[tid]))]
        if kind != 1:
            raise GobError("top-level value is not a slice")
        elem = t[1]
        if body.uint() != 0:
            raise GobError("non-zero singleton delta")
        count = body.uint()
        if elem == STRING:
            values.append([body.bytes_() for _ in range(count)])
        else:
            mk, mt = types[elem][next(iter(types[elem]))]
            if mk != 3 or mt.get(1) != STRING or mt.get(2) != STRING:
                raise GobError("not a map[string]string")
            rows = []
            for _ in range(count):
                k = body.uint()
                rows.append([(body.bytes_(), body.bytes_()) for _ in range(k)])
            values.append(rows)
        if body.i != len(body.b):
            raise GobError("extra data in message")
    return values


def decode_index(data: bytes) -> tuple:
    """-> (key columns, rows as dicts in file order) of an index file"""
    vals = decode_stream(data)
    if len(vals) < 2:
        raise GobError("EOF")
    return vals[0], [dict(r) for r in vals[1]]
