"""ToJSON restated for the tests (csvplus.go:446-474 with encoding/json's appendString, go 1.23), written from the rules,
not from the product code: json.Encoder with SetEscapeHTML(false) and no indent, Encode's trailing newline, map keys in
bytewise order.  Rows are dicts of bytes -> bytes and may have different column sets."""
from __future__ import annotations

import re

_SPECIAL = re.compile(rb'[\x00-\x1f"\\\x80-\xff]')
_SHORT = {0x22: b'\\"', 0x5C: b"\\\\", 0x0A: b"\\n", 0x0D: b"\\r", 0x09: b"\\t", 0x08: b"\\b", 0x0C: b"\\f"}
# second-byte range of each valid UTF-8 lead byte and the number of continuation bytes (utf8.DecodeRune's table)
_LEAD = {}
for _c in range(0xC2, 0xE0): _LEAD[_c] = (0x80, 0xBF, 1)
_LEAD[0xE0] = (0xA0, 0xBF, 2)
for _c in range(0xE1, 0xED): _LEAD[_c] = (0x80, 0xBF, 2)
_LEAD[0xED] = (0x80, 0x9F, 2)
for _c in (0xEE, 0xEF): _LEAD[_c] = (0x80, 0xBF, 2)
_LEAD[0xF0] = (0x90, 0xBF, 3)
for _c in (0xF1, 0xF2, 0xF3): _LEAD[_c] = (0x80, 0xBF, 3)
_LEAD[0xF4] = (0x80, 0x8F, 3)


def enc(s: bytes) -> bytes:
    if not _SPECIAL.search(s):
        return b'"' + s + b'"'
    out = bytearray(b'"')
    i, n = 0, len(s)
    while i < n:
        c = s[i]
        if c < 0x80:
            if c in _SHORT: out += _SHORT[c]
            elif c < 0x20: out += b"\\u00%02x" % c
            else: out.append(c)
            i += 1
            continue
        lead = _LEAD.get(c)
        ok = lead is not None and i + lead[2] < n and lead[0] <= s[i + 1] <= lead[1] and \
            all(0x80 <= s[i + j] <= 0xBF for j in range(2, lead[2] + 1))
        if not ok:
            out += b"\\ufffd"; i += 1
        elif s[i:i + 3] in (b"\xe2\x80\xa8", b"\xe2\x80\xa9"):
            out += b"\\u2028" if s[i + 2] == 0xA8 else b"\\u2029"; i += 3
        else:
            out += s[i:i + lead[2] + 1]; i += lead[2] + 1
    out += b'"'
    return bytes(out)


def row_json(row: dict) -> bytes:
    return b"{" + b",".join(enc(k) + b":" + enc(row[k]) for k in sorted(row)) + b"}\n"


def document(rows, first: bool = True, last: bool = True) -> bytes:
    parts = [b"[" if first else b""]
    for i, r in enumerate(rows):
        if i or not first:
            parts.append(b",")
        parts.append(row_json(r))
    if last:
        parts.append(b"]")
    return b"".join(parts)


def columns_document(names, columns, first: bool = True, last: bool = True) -> bytes:
    """document() of a table given as names + per-column value lists (every row has every column)"""
    order = sorted(range(len(names)), key=lambda k: names[k])
    keys = [enc(names[k]) + b":" for k in order]
    cols = [columns[k] for k in order]
    n = len(cols[0]) if cols else 0
    parts = [b"[" if first else b""]
    for i in range(n):
        if i or not first:
            parts.append(b",")
        parts.append(b"{" + b",".join(keys[j] + enc(cols[j][i]) for j in range(len(cols))) + b"}\n")
    if last:
        parts.append(b"]")
    return b"".join(parts)

