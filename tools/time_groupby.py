"""GroupBy timing: python tools/time_groupby.py [rows]

  orders generated on the GPU (rows, default 100 M) and parsed into one device table (cust_id, prod_id, qty).  Cases:
  grouped by cust_id with 10 M and 100 M customers, by prod_id (1000 products) and by one constant column (a single
  group of every row: the serial float fold at its longest).  Aggregates: count, sum of qty as "int" and sum of qty as
  "float64".  Per case: DataSource.GroupBy of the table (one push), wall time around the call after warm-up, with the
  per-kernel times of one call; beside it the route without GroupBy, ToTensors({key: "category", qty: int, qty: float64})
  + torch index_add_ (not bit-exact for float sums: atomic order), timed the same way.  Then the host RowFunc (a Python
  dict fold over ToRows) at 1 M rows.  The card's name and power limit are printed first."""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import csvplus_b200 as cp  # noqa: E402

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000_000
REPS = 3
ctx = cp.Context(0)
dev = torch.device("cuda", ctx.device)
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
except OSError:
    print("nvidia-smi not available", flush=True)

AGGS = {"n": ("count",), "qty_int": ("sum", "qty", "int"), "qty_float": ("sum", "qty", "float64")}


def orders(n_cust: int) -> cp.Table:
    buf = ctx.gen_csv("orders", (0, rows), n_cust=n_cust, n_prod=1000)
    t, err = cp.parse_csv(ctx, buf, on_device=True, spec=[("cust_id", -1), ("prod_id", -1), ("qty", -1)])
    assert err is None
    ctx.sync()
    buf.free()
    return t.with_column("one", "x")


def wall(fn, reps=REPS):
    fn()
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize(dev)
    return (time.perf_counter() - t0) / reps, out


def tensors_route(t: cp.Table, key: str):
    d = cp.TakeTable(t).ToTensors({key: "category", "qty": "int"})
    codes, q = d[key].codes, d["qty"]
    ng = len(d[key].dictionary)
    n = torch.zeros(ng, dtype=torch.int64, device=dev).index_add_(0, codes, torch.ones_like(q))
    s = torch.zeros(ng, dtype=torch.int64, device=dev).index_add_(0, codes, q)
    f = torch.zeros(ng, dtype=torch.float64, device=dev).index_add_(0, codes, cp.TakeTable(t).ToTensors({"qty": "float64"})["qty"])
    return n, s, f


def case(label: str, t: cp.Table, key: str):
    s, g = wall(lambda: cp.TakeTable(t).GroupBy([key], AGGS))
    n = len(t)
    print(f"{label}: {n} rows, {len(g)} groups", flush=True)
    print(f"  GroupBy                    {s * 1e3:9.2f} ms  {n / s / 1e9:6.3f} G rows/s", flush=True)
    ctx.stats(enable=True, reset=True)
    cp.TakeTable(t).GroupBy([key], AGGS)
    st = ctx.stats(); ctx.stats(enable=False)
    print("    " + "  ".join(f"{k} {v['ms']:.2f}" for k, v in sorted(st.items(), key=lambda kv: -kv[1]["ms"])) + " (ms)", flush=True)
    del g
    s2, out = wall(lambda: tensors_route(t, key))
    print(f"  ToTensors + index_add_     {s2 * 1e3:9.2f} ms  {n / s2 / 1e9:6.3f} G rows/s  (GroupBy takes {s / s2:.2f}x this time)",
          flush=True)
    del out


for n_cust, label in ((10_000_000, "orders by cust_id, 10 M customers"), (100_000_000, "orders by cust_id, 100 M customers")):
    t = orders(n_cust)
    case(label, t, "cust_id")
    if n_cust == 10_000_000:
        case("orders by prod_id, 1000 products", t, "prod_id")
        case("orders in one group", t, "one")
    del t
    torch.cuda.empty_cache()

# the host RowFunc at 1 M rows: what a Python closure folding the delivered rows costs
small = orders(1000).slice(0, min(rows, 1_000_000))


def rowfunc():
    n, qi, qf = {}, {}, {}
    for r in cp.TakeTable(small).ToRows():
        k = r["cust_id"]
        n[k] = n.get(k, 0) + 1
        qi[k] = qi.get(k, 0) + int(r["qty"])
        qf[k] = qf.get(k, 0.0) + float(r["qty"])
    return n


s, _ = wall(rowfunc, reps=1)
sg, _ = wall(lambda: cp.TakeTable(small).GroupBy(["cust_id"], AGGS))
print(f"host RowFunc at {len(small)} rows: {s * 1e3:.1f} ms ({len(small) / s / 1e6:.2f} M rows/s); GroupBy {sg * 1e3:.2f} ms", flush=True)
