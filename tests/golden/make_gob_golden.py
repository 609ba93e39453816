"""Regenerates the index-file fixture of tests/golden/ (oracle-pinned: written by the restatement tests/gob_oracle.py, not
by an execution of the reference; baseline/go/gob pins it to encoding/gob on a machine with Go):

    python tests/golden/make_gob_golden.py

people_index.gob is what Index.WriteTo writes for IndexOn("id") over SelectColumns("id", "name", "surname") of
people.csv (TestIndexStore, csvplus_test.go:960-1014): the key columns, then the rows in key order, the pairs of every
row in bytewise column-name order.  The other fixtures are left untouched."""
import csv
import io
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import gob_oracle  # noqa: E402


def golden_rows() -> list:
    with open(os.path.join(HERE, "people.csv"), "rb") as f:
        recs = list(csv.reader(io.TextIOWrapper(f, encoding="utf-8", newline="")))
    head = recs[0]
    rows = [{c: r[head.index(c)].encode() for c in ("id", "name", "surname")} for r in recs[1:] if r]
    rows.sort(key=lambda r: r["id"])  # IndexOn("id"): bytewise order of the key, ties in input order
    return [{k.encode(): v for k, v in r.items()} for r in rows]


def golden_bytes() -> bytes:
    return gob_oracle.encode_index([b"id"], golden_rows())


if __name__ == "__main__":
    with open(os.path.join(HERE, "people_index.gob"), "wb") as f:
        f.write(golden_bytes())
