"""Regenerates the golden fixtures of tests/golden/ from the CPU oracle (oracle/):

    python tests/golden/make_golden.py

The reference itself (Go) cannot run in this image, so these files pin the ORACLE's behaviour (and through the parity
tests the CUDA path's) on fixed inputs: any later change of either side that alters an output shows up as a diff of a
committed file.  Inputs are committed next to the expected outputs; nothing here reads the reference's sources."""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import oracle as orc  # noqa: E402
from tests.helpers import people_csv, random_csv  # noqa: E402


def orders_csv(n, ncust, nprod, seed=3):
    rng = random.Random(seed)
    rows = [b"order_id,cust_id,prod_id,qty,ts"]
    for i in range(n):
        rows.append(b"%d,%d,%d,%d,2016-09-14T08:%02d:%02d+01:00" % (i, rng.randrange(ncust), rng.randrange(nprod), 1 + rng.randrange(100),
                                                                    rng.randrange(60), rng.randrange(60)))
    return b"\n".join(rows) + b"\n"


def write(name, data: bytes):
    with open(os.path.join(HERE, name), "wb") as f:
        f.write(data)


def main():
    people = people_csv(300, seed=7)
    orders = orders_csv(2000, 330, 8, seed=5)   # cust ids 300..329 have no customer
    nasty = random_csv(23, nrows=400, ncols=4, quoted_p=0.5, crlf_p=0.3)
    write("people.csv", people); write("orders.csv", orders); write("nasty.csv", nasty)
    meta = {}
    # configs[1] shape: parse + SelectColumns + Filter(Like)
    r = orc.reader_rows(people, select=["name", "surname", "id"], pred=orc.Like({"name": "Amelia"}))
    out, err = r.to_csv("name", "surname", "id")
    assert err is None
    write("people_amelia.csv", out); meta["people_amelia_rows"] = len(r)
    # configs[2] shape: UniqueIndexOn + Join, then ToCsv of the merged rows
    idx = orc.reader_rows(people, select=["id", "name", "surname"]).unique_index_on("id")
    j = orc.reader_rows(orders, select=["order_id", "cust_id", "qty"]).join(idx, "cust_id")
    out, err = j.to_csv("order_id", "cust_id", "qty", "id", "name", "surname")
    assert err is None
    write("orders_join_people.csv", out); meta["join_rows"] = len(j)
    # sorted index order (stable) on a non-unique two-column key
    oidx = orc.reader_rows(orders).index_on("prod_id", "qty")
    out, err = oidx.rows().to_csv("prod_id", "qty", "order_id")
    assert err is None
    write("orders_sorted_prod_qty.csv", out)
    # anti-join
    ex = orc.reader_rows(orders, select=["order_id", "cust_id"]).except_(idx, "cust_id")
    out, err = ex.to_csv("order_id", "cust_id")
    assert err is None
    write("orders_without_customer.csv", out); meta["except_rows"] = len(ex)
    # quoting / CRLF / blank-line handling of the reader, re-serialised by the writer
    rn = orc.reader_rows(nasty)
    out, err = rn.to_csv("c0", "c1", "c2", "c3")
    assert err is None and rn.error is None
    write("nasty_roundtrip.csv", out); meta["nasty_rows"] = len(rn)
    with open(os.path.join(HERE, "meta.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True); f.write("\n")
    print(meta)


if __name__ == "__main__":
    main()
