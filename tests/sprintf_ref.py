"""A plain-Python restatement of fmt.Sprintf(format, v...) for string operands over bytes, for the subset of Go's fmt
the library accepts (Table.with_column(Sprintf), DataSource.ToText).

Go's doPrintf reads a '%', then flags (# 0 + - space), an optional [n] argument index, a width (* or digits), an optional
'.' and precision (* or digits, none meaning 0), another optional [n], and the verb rune.  For a string operand, %s and
%v call fmtS: truncateString keeps the first prec runes (`for i := range s`), then padString pads with spaces to width
runes (utf8.RuneCountInString), on the right when '-' was given.  Runes are utf8.DecodeRune's; every byte that does not
start a valid sequence is one rune of one byte.

Accepted: literal bytes, a bare %%, and %s / %v whose only flag is '-' and whose width and precision are at most
1000000, with exactly one verb per column, at most 64 verbs and at most 4096 format bytes.  Everything else is Refused.
"""
from __future__ import annotations

MAX_VERBS = 64
MAX_FORMAT = 4096
MAX_NUM = 1_000_000

# utf8.DecodeRune's accepting ranges: lead byte -> (sequence length, range of the second byte); later bytes 80..BF
_LEADS = {}
for _b in range(0xC2, 0xE0):
    _LEADS[_b] = (2, 0x80, 0xBF)
_LEADS[0xE0] = (3, 0xA0, 0xBF)
for _b in list(range(0xE1, 0xED)) + [0xEE, 0xEF]:
    _LEADS[_b] = (3, 0x80, 0xBF)
_LEADS[0xED] = (3, 0x80, 0x9F)
_LEADS[0xF0] = (4, 0x90, 0xBF)
for _b in (0xF1, 0xF2, 0xF3):
    _LEADS[_b] = (4, 0x80, 0xBF)
_LEADS[0xF4] = (4, 0x80, 0x8F)


class Refused(ValueError):
    def __init__(self, offset: int, what: str):
        super().__init__(f"{what} at byte {offset}")
        self.offset = offset


def rune_size(s: bytes, i: int) -> int:
    """bytes of the rune at s[i] as utf8.DecodeRune reads it"""
    lead = _LEADS.get(s[i])
    if lead is None:
        return 1
    n, lo, hi = lead
    if i + n > len(s) or not lo <= s[i + 1] <= hi:
        return 1
    if any(not 0x80 <= s[k] <= 0xBF for k in range(i + 2, i + n)):
        return 1
    return n


def runes(s: bytes) -> list:
    """the start offsets of s's runes (`for i := range s`)"""
    out, i = [], 0
    while i < len(s):
        out.append(i)
        i += rune_size(s, i)
    return out


def truncate(s: bytes, prec) -> bytes:  # fmt.truncateString
    if prec is None:
        return s
    starts = runes(s)
    return s if prec >= len(starts) else s[: starts[prec]]


def pad(s: bytes, width, left: bool) -> bytes:  # fmt.padString
    if width is None:
        return s
    n = width - len(runes(s))
    if n <= 0:
        return s
    return s + b" " * n if left else b" " * n + s


def parse(fmt: bytes, nargs: int) -> list:
    """the pieces of an accepted format: bytes (a literal) or (width | None, prec | None, left); Refused otherwise"""
    if len(fmt) > MAX_FORMAT:
        raise Refused(MAX_FORMAT, "format too long")
    pieces, i, end, nverbs = [], 0, len(fmt), 0
    while i < end:
        j = fmt.find(b"%", i)
        j = end if j < 0 else j
        if j > i:
            pieces.append(fmt[i:j])
        if j >= end:
            break
        start = j
        i = j + 1
        if i >= end:
            raise Refused(start, "lone %")
        left = False
        while i < end and fmt[i] in b"#0+- ":
            if fmt[i] != ord("-"):
                raise Refused(i, "flag")
            left = True
            i += 1

        def number(i):
            k = i
            while k < end and 0x30 <= fmt[k] <= 0x39:
                k += 1
            if k == i:
                return None, i
            v = int(fmt[i:k])
            if v > MAX_NUM:
                raise Refused(i, "number too large")
            return v, k
        if i < end and fmt[i] in b"[*":
            raise Refused(i, "index or star")
        width, i = number(i)
        prec = None
        if i < end and fmt[i] == ord("."):
            i += 1
            if i < end and fmt[i] in b"[*":
                raise Refused(i, "index or star")
            prec, i = number(i)
            prec = 0 if prec is None else prec
        if i < end and fmt[i] == ord("["):
            raise Refused(i, "index")
        if i >= end:
            raise Refused(start, "no verb")
        verb = fmt[i]
        i += 1
        if verb == ord("%"):
            if left or width is not None or prec is not None:
                raise Refused(start, "flags on %%")
            pieces.append(b"%")
        elif verb in b"sv":
            nverbs += 1
            if nverbs > MAX_VERBS:
                raise Refused(start, "too many verbs")
            if nverbs > nargs:
                raise Refused(start, "missing operand")
            pieces.append((width if width else None, prec, left))
        else:
            raise Refused(i - 1, "verb")
    if nverbs != nargs:
        raise Refused(end, "operand count")
    return pieces


def sprintf(fmt: bytes, values: list) -> bytes:
    """fmt.Sprintf(fmt, values...) of string values given as bytes"""
    out, k = [], 0
    for p in parse(fmt, len(values)):
        if isinstance(p, bytes):
            out.append(p)
        else:
            width, prec, left = p
            out.append(pad(truncate(values[k], prec), width, left))
            k += 1
    return b"".join(out)


def text(fmt: bytes, rows: list) -> bytes:
    """what DataSource.ToText writes: every row's text (rows: lists of value bytes in column order)"""
    return b"".join(sprintf(fmt, r) for r in rows)


# formats the library must refuse, with the number of columns they are given
REFUSED = [
    (b"%d", 1), (b"%q", 1), (b"%x", 1), (b"%S", 1), (b"%V", 1), (b"%T", 1), (b"%\xc3\xa9", 1), (b"%\xff", 1),
    (b"abc%", 0), (b"%s%", 1), (b"%", 0),
    (b"%0s", 1), (b"%05s", 1), (b"%-0s", 1), (b"%+s", 1), (b"%#s", 1), (b"%#v", 1), (b"% s", 1),
    (b"%*s", 1), (b"%.*s", 1), (b"%[1]s", 1), (b"%.[1]s", 1), (b"%5[1]s", 1), (b"%[2]*s", 1),
    (b"%5%", 0), (b"%-%", 0), (b"%.2%", 0), (b"%.%", 0),
    (b"%5", 0), (b"%-", 0), (b"%.", 0), (b"%5.", 0),
    (b"%s", 0), (b"%s %s", 1), (b"%s", 2), (b"plain", 1), (b"", 1),
    (b"%1000001s", 1), (b"%.1000001s", 1), (b"%99999999999999999999s", 1),
    (b"%s" * 65, 65), (b"a" * 4097, 0),
]
