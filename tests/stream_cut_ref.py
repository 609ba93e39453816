"""The stream cut rule (csvplus_b200/csrc/stream.cu, DESIGN.md §3.7) restated in plain Python.  TEST INFRASTRUCTURE ONLY.

A buffer starts at a record start.  Its cut is the end of its last complete record: 1 + the position of the last '\\n'
that ends a line of encoding/csv's readRecord (0 when there is none).  [0, cut) is then a CSV input of its own and
[cut, n) starts at a record start.

  * no CommentChar, no LazyQuotes: in valid input every '"' opens or closes a quoted field or is half of an escaped
    pair, so a '\\n' ends a line exactly when the quotes before it are even in number;
  * CommentChar or LazyQuotes: a quote in a comment line does not count and a lazy quote inside a field is data, so the
    line structure is followed rune by rune with readRecord's rules (the machine below, written from the Go source's
    cases: line start, comment line, field start, unquoted field, quoted field, a quote inside a quoted field).
Multi-byte Delimiter / CommentChar runes and the multi-byte Unicode spaces TrimLeadingSpace trims are matched as their
UTF-8 byte sequences."""

UNICODE_SPACES = [0x85, 0xA0, 0x1680, 0x2000, 0x2001, 0x2002, 0x2003, 0x2004, 0x2005, 0x2006, 0x2007, 0x2008, 0x2009,
                  0x200A, 0x2028, 0x2029, 0x202F, 0x205F, 0x3000]
ASCII_SPACES = b" \t\v\f\r"


def cut_parity(buf: bytes) -> int:
    even, cut = True, 0
    for i, b in enumerate(buf):
        if b == 0x22:
            even = not even
        elif b == 0x0A and even:
            cut = i + 1
    return cut


def _tokens(buf: bytes, comma: str, comment: str, trim: bool):
    """-> (kind, position of the token's last byte) per rune-level token: 'comma', 'comment', 'space', or the byte itself"""
    seqs = []
    if ord(comma) >= 0x80:
        seqs.append((comma.encode(), "comma"))
    if comment and ord(comment) >= 0x80:
        seqs.append((comment.encode(), "comment"))
    if trim:
        seqs += [(chr(r).encode(), "space") for r in UNICODE_SPACES if chr(r) not in (comma, comment)]
    i, n = 0, len(buf)
    while i < n:
        b = buf[i]
        hit = None
        if b >= 0x80:
            for seq, kind in seqs:
                if buf.startswith(seq, i):
                    hit = (seq, kind)
                    break
        if hit:
            yield hit[1], i + len(hit[0]) - 1
            i += len(hit[0])
            continue
        if b == 0x22:
            kind = "quote"
        elif b == 0x0A:
            kind = "nl"
        elif ord(comma) < 0x80 and b == ord(comma):
            kind = "comma"
        elif b == 0x0D:
            kind = "cr"
        elif comment and ord(comment) < 0x80 and b == ord(comment):
            kind = "comment"
        elif trim and b in ASCII_SPACES:
            kind = "space"
        else:
            kind = "other"
        yield kind, i
        i += 1


def cut_lines(buf: bytes, comma=",", comment="", lazy=False, trim=False) -> int:
    state, cut = "line", 0
    for kind, pos in _tokens(buf, comma, comment, trim):
        if kind == "nl" and state not in ("quoted",):
            # every state but "inside a quoted field" ends the line here ("\r\n" and '"' + "\r\n" included)
            state, cut = "line", pos + 1
            continue
        if state == "line":  # the first rune of a line
            if kind == "comment":
                state = "comment"
            elif kind == "cr":
                state = "line_cr"
            else:
                state = _field_start(kind, trim)
        elif state == "line_cr":  # "\r" then not "\n": the \r is the line's first data byte
            state = _field_start(kind, trim) if trim else _unquoted(kind)
        elif state == "comment":
            pass
        elif state == "field":
            state = _field_start(kind, trim)
        elif state == "unquoted":
            state = _unquoted(kind)
        elif state == "quoted":
            state = "quote" if kind == "quote" else "quoted"
        elif state in ("quote", "quote_cr"):  # after a '"' inside a quoted field (and a '\r' after it)
            if kind == "quote":
                state = "quoted" if state == "quote" else "quote"  # "" is an escaped quote; lazy "\r" then a new quote
            elif kind == "comma" and state == "quote":
                state = "field"
            elif kind == "cr" and state == "quote":
                state = "quote_cr"
            else:
                state = "quoted"  # lazy: the quote was data (strict: an error was met already)
    return cut


def _field_start(kind, trim):
    if kind == "quote":
        return "quoted"
    if kind == "comma":
        return "field"
    if trim and kind in ("space", "cr"):
        return "field"
    return "unquoted"


def _unquoted(kind):
    return "field" if kind == "comma" else "unquoted"


def stream_cut(buf: bytes, comma=",", comment="", lazy=False, trim=False) -> int:
    if comment or lazy:
        return cut_lines(buf, comma, comment, lazy, trim)
    return cut_parity(buf)
