"""Go 1.23 strconv.Atoi and strconv.ParseFloat(s, 64), restated from their rules for the numeric tests (csrc/numeric.cu).

Both take bytes and return (value, status) with status 0 ok, 1 ErrSyntax, 2 ErrRange, and the value Go returns alongside
the error.  The grammar is restated here; the values come from Python: int() once the digits are validated, float() of a
rebuilt decimal string, float.fromhex for hex.  Python's decimal conversion and fromhex are correctly rounded, as Go's
are.  The exponent keeps Go's cap (digits beyond the value 10000 still parse but stop growing it), so the strings are
rebuilt from the parsed digits rather than passed through.  Go cannot run here: baseline/go/numeric/main.go regenerates
tests/golden/numeric_kat.expected with the real strconv on a machine that has Go."""
from __future__ import annotations

import struct

OK, SYNTAX, RANGE = 0, 1, 2
INT64_MAX, INT64_MIN = (1 << 63) - 1, -(1 << 63)
NAN_BITS = 0x7FF8000000000001  # math.NaN()


def atoi(s: bytes) -> tuple[int, int]:
    """strconv.Atoi (= ParseInt(s, 10, 0) on a 64-bit int): optional sign, one or more ASCII digits; the first problem met
    left to right decides, so an overflow before a bad byte is ErrRange"""
    if not s:
        return 0, SYNTAX
    neg = s[:1] == b"-"
    body = s[1:] if s[:1] in (b"+", b"-") else s
    if not body:
        return 0, SYNTAX
    v = 0
    for c in body:
        if not 0x30 <= c <= 0x39:
            return 0, SYNTAX
        v = v * 10 + (c - 0x30)
        if v >= 1 << 64:  # ParseUint's range error, at the first digit that overflows uint64
            return (INT64_MIN if neg else INT64_MAX), RANGE
    if not neg and v > INT64_MAX:
        return INT64_MAX, RANGE
    if neg and v > 1 << 63:
        return INT64_MIN, RANGE
    return (-v if neg else v), OK


def _lower(c: int) -> int:
    return c | 0x20


def _special(s: bytes):
    """strconv.special: (bits, consumed) or None"""
    if not s:
        return None
    sign = 0
    i = 0
    c = _lower(s[0])
    if s[0] in b"+-":
        sign = 1 << 63 if s[0] == 0x2D else 0
        i, c = 1, ord("i")
    if c == ord("i"):
        k = 0
        while k < 8 and i + k < len(s) and _lower(s[i + k]) == b"infinity"[k]:
            k += 1
        if 3 < k < 8:
            k = 3
        if k in (3, 8):
            return sign | 0x7FF0000000000000, i + k
    elif c == ord("n"):
        if len(s) >= 3 and _lower(s[1]) == ord("a") and _lower(s[2]) == ord("n"):
            return NAN_BITS, 3
    return None


def underscore_ok(s: bytes) -> bool:
    """strconv.underscoreOK: '_' only between digits, or between a base prefix and a digit"""
    saw = "^"
    i = 0
    if s[:1] in (b"+", b"-"):
        s = s[1:]
    hexa = False
    if len(s) >= 2 and s[0] == 0x30 and _lower(s[1]) in b"box":
        i, saw, hexa = 2, "0", _lower(s[1]) == ord("x")
    while i < len(s):
        c = s[i]
        if 0x30 <= c <= 0x39 or (hexa and ord("a") <= _lower(c) <= ord("f")):
            saw = "0"
        elif c == 0x5F:
            if saw != "0":
                return False
            saw = "_"
        else:
            if saw == "_":
                return False
            saw = "!"
        i += 1
    return saw != "_"


def read_float(s: bytes):
    """strconv.readFloat + ParseFloat's whole-string rule: None (ErrSyntax) or (neg, hex, digits, dp) where the value is
    0.<digits> * base^dp for decimal (base 10) and 0.<hex digits> * 2^dp for hex (dp already in bits)"""
    n = len(s)
    i = 0
    if n == 0:
        return None
    neg = False
    if s[0] == 0x2B:
        i += 1
    elif s[0] == 0x2D:
        neg, i = True, 1
    hexa = i + 2 < n and s[i] == 0x30 and _lower(s[i + 1]) == ord("x")
    if hexa:
        i += 2
    underscores = False
    sawdot = sawdigits = False
    digits = []
    dp = 0
    while i < n:
        c = s[i]
        if c == 0x5F:
            underscores = True
        elif c == 0x2E:
            if sawdot:
                break
            sawdot, dp = True, len(digits)
        elif 0x30 <= c <= 0x39 or (hexa and ord("a") <= _lower(c) <= ord("f")):
            sawdigits = True
            if c == 0x30 and not digits:
                dp -= 1  # leading zero
            else:
                digits.append(chr(_lower(c)) if c > 0x39 else chr(c))
        else:
            break
        i += 1
    if not sawdigits:
        return None
    if not sawdot:
        dp = len(digits)
    if hexa:
        dp *= 4
    exp_char = ord("p") if hexa else ord("e")
    if i < n and _lower(s[i]) == exp_char:
        i += 1
        if i >= n:
            return None
        esign = 1
        if s[i] == 0x2B:
            i += 1
        elif s[i] == 0x2D:
            i, esign = i + 1, -1
        if i >= n or not 0x30 <= s[i] <= 0x39:
            return None
        e = 0
        while i < n and (0x30 <= s[i] <= 0x39 or s[i] == 0x5F):
            if s[i] == 0x5F:
                underscores = True
            elif e < 10000:
                e = e * 10 + s[i] - 0x30
            i += 1
        dp += e * esign
    elif hexa:
        return None
    if underscores and not underscore_ok(s[:i]):
        return None
    if i != n:
        return None
    return neg, hexa, "".join(digits), dp


def bits_of(f: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", f))[0]


def float_of(b: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def parse_float(s: bytes) -> tuple[int, int]:
    """strconv.ParseFloat(s, 64) -> (IEEE bits of the value, status)"""
    sp = _special(s)
    if sp is not None:
        return (sp[0], OK) if sp[1] == len(s) else (0, SYNTAX)
    r = read_float(s)
    if r is None:
        return 0, SYNTAX
    neg, hexa, digits, dp = r
    sign = 1 << 63 if neg else 0
    if not digits.strip("0"):
        return sign, OK
    try:
        f = float.fromhex(f"0x0.{digits}p{dp}") if hexa else float(f"0.{digits}e{dp}")
    except OverflowError:
        f = float("inf")
    b = bits_of(f)
    if b == 0x7FF0000000000000:
        return sign | b, RANGE
    return sign | b, OK


def go_quote(s: bytes) -> bytes:
    """the project's go_quote (csrc/abi.cu): Go's %q for printable ASCII, \\n \\r \\t, \\xNN for other control bytes
    and 0x7f; other bytes pass through (Go's %q differs for \\a \\b \\f \\v and bytes >= 0x80: DESIGN §7)"""
    out = bytearray(b'"')
    for ch in s:
        if ch in (0x22, 0x5C):
            out += bytes([0x5C, ch])
        elif ch == 0x0A:
            out += b"\\n"
        elif ch == 0x0D:
            out += b"\\r"
        elif ch == 0x09:
            out += b"\\t"
        elif ch < 0x20 or ch == 0x7F:
            out += b"\\x%02x" % ch
        else:
            out.append(ch)
    return bytes(out + b'"')


def message(column: str, value: bytes, is_float: bool, status: int) -> str:
    """Row.ValueAsInt / ValueAsFloat64's error text (csvplus.go:176, :198) as the Python layer reports it: the C ABI's
    bytes, cut to cpb_error.msg (487 bytes) and decoded as UTF-8 with replacement"""
    m = (b"column " + go_quote(column.encode()) + b": cannot convert " + go_quote(value) + b" to " + (b"float" if is_float else b"integer")
         + b": " + (b"value out of range" if status == RANGE else b"invalid syntax"))
    return m[:487].decode("utf-8", "replace")
