"""Regenerates the ToJSON fixture of tests/golden/ from the CPU oracle's CSV reader and tests/json_oracle.py:

    python tests/golden/make_json_golden.py

json_escapes.csv holds every byte class encoding/json's string encoder treats differently (all 32 control bytes, '"',
'\\', 0x7f, HTML characters, U+2028 / U+2029, valid 2-, 3- and 4-byte sequences, and each kind of invalid UTF-8), in
values and in column names; json_escapes.json is what ToJSON writes for it.  The other fixtures are left untouched."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import oracle as orc  # noqa: E402
from tests import json_oracle  # noqa: E402

NAMES = [b"a", b"B", "\u00e9".encode(), b'k"\\<']
VALUES = [
    bytes(range(0x00, 0x20)),                                   # every control byte (\n \r \t \b \f and \u00xx)
    b'say "hi" \\ back\\slash \x7f <b>&amp;</b>',
    "\u2028line\u2029para \u00e9 \u20ac \U0001F642 \ufffd".encode(),  # escaped separators, valid 2/3/4-byte runes
    b"\x80lone \xbf\xc0\xaf\xc1\xbf C0/C1",                       # lone continuations, C0 / C1 leads
    b"\xe0\x80\x80 overlong \xed\xa0\x80 surrogate",
    b"\xf4\x90\x80\x80 above \xf5\x80 \xfe\xff",
    b"cut \xe2\x82",                                           # truncated at the end of the value
    b"cut4 \xf0\x9f\x99",
    b"",
    b"plain ascii value",
    b"\xe2\x80\xa8\xe2\x80\xa9\xe2\x80\xaa",                   # U+202A is copied
    b"\xc3\xa9\xc3",                                           # valid then truncated
]


def _field(v: bytes) -> bytes:
    return b'"' + v.replace(b'"', b'""') + b'"'


def fixture_csv() -> bytes:
    lines = [b",".join(_field(n) for n in NAMES)]
    for i in range(len(VALUES)):
        lines.append(b",".join(_field(VALUES[(i + k) % len(VALUES)]) for k in range(len(NAMES))))
    return b"\n".join(lines) + b"\n"


def expected_json(csv: bytes) -> bytes:
    rows = orc.reader_rows(csv, select=[n.decode("utf-8") for n in NAMES])
    assert rows.error is None and len(rows) == len(VALUES)
    return json_oracle.document(rows.to_dicts())


def main():
    csv = fixture_csv()
    with open(os.path.join(HERE, "json_escapes.csv"), "wb") as f:
        f.write(csv)
    with open(os.path.join(HERE, "json_escapes.json"), "wb") as f:
        f.write(expected_json(csv))


if __name__ == "__main__":
    main()
