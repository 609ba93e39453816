"""LeftJoin against Join on BASELINE configs[3]'s shapes, at 0 / 1 / 10 / 50 % missing keys:

    python tools/time_left_join.py [orders]      (default 125 000 000)

orders x customers (100 M ids, UniqueIndexOn("id"): the row-carrying table) on cust_id, and orders x products (1 M ids,
UniqueIndexOn("prod_id"): the unique16 table) on prod_id.  Misses are made by generating only the first (1 - f) of the
customer / product ids the orders draw from.  Also timed: what a user would run without LeftJoin, Join + Except +
with_column("") per index-only column + concat (plan order not restored).  Device time per call (CUDA events, median of
5 after 2 warm-ups); the card's name and power limit are printed with the numbers."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import csvplus_b200 as cp
from csvplus_b200.api import Table

SEED = 12345
CUST, PROD = 100_000_000, 1_000_000


def timed(ctx, fn, reps=5, warm=2):
    for _ in range(warm):
        r = fn()
        del r
    ctx.sync()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ctx.sync()
        a.record(torch.cuda.current_stream())
        r = fn()
        ctx.sync()
        b.record(torch.cuda.current_stream())
        b.synchronize()
        ms.append(a.elapsed_time(b))
        n = len(r)
        del r
    ms.sort()
    return ms[len(ms) // 2], n


def join_except_concat(t, ix, col, fill):
    j = t.join(ix, col)
    e = t.join(ix, col, anti=True)
    for name in fill:
        e = e.with_column(name, "")
    return Table.concat([j, e.select(*j.columns)])


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 125_000_000
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", card)
    ctx = cp.Context(0)
    orders, err = cp.parse_csv(ctx, ctx.gen_csv("orders", (0, n), seed=SEED, n_cust=CUST, n_prod=PROD, header=True),
                               spec=[("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)])
    assert err is None
    for side, total, kind, key, spec in (("customers", CUST, "customers", "id", [("id", -1), ("name", -1), ("surname", -1)]),
                                         ("products", PROD, "products", "prod_id", [("prod_id", -1), ("product", -1), ("price", -1)])):
        col = "cust_id" if side == "customers" else "prod_id"
        for f in (0.0, 0.01, 0.10, 0.50):
            k = int(round(total * (1 - f)))
            kw = {"n_cust": k} if side == "customers" else {"n_prod": k}
            t, err = cp.parse_csv(ctx, ctx.gen_csv(kind, (0, k), seed=SEED, permute=True, header=True, **kw), spec=spec)
            assert err is None
            ix = t.index_on(key, unique=True)
            ctx.stats(enable=True, reset=True)
            orders.slice(0, 1000).join(ix, col)
            route = "rowhash" if "rowhash_probe" in ctx.stats() else "probe table"
            ctx.stats(enable=False)
            ms_j, nj = timed(ctx, lambda: orders.join(ix, col))
            ms_l, nl = timed(ctx, lambda: orders.join(ix, col, left=True))
            fill = [c for c in t.columns if c not in orders.columns]
            ms_b, nb = timed(ctx, lambda: join_except_concat(orders, ix, col, fill), reps=3, warm=1)
            assert nl == nb == n, (nl, nb, n)
            print("%s %s x %d index rows (%s), %.2f %% of orders missing: Join %.1f ms (%d rows), LeftJoin %.1f ms (%d rows), "
                  "Join+Except+with_column+concat %.1f ms" % (side, n, k, route, 100.0 * (n - nj) / n, ms_j, nj, ms_l, nl, ms_b),
                  flush=True)
            del ix, t
            ctx.sync()
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
