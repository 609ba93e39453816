"""OrderBy timing: python tools/time_order.py [rows]

  orders generated on the GPU (rows, default 100 M), parsed into one device table (cust_id, prod_id, qty, ts) and joined
  with the products' unique index for price.  Cases, wall time around the call after warm-up:
    - Table.order_by of every row by price float64 descending, and by (cust_id, ts) as strings, with the per-kernel times
      of one call;
    - the first k rows by price descending, k = 10 .. rows / 2: order_by(limit=k) (the radix select up to rows / 2, the
      full sort above) against the full sort and a slice; run with CPB_LIB set to a library built with
      -DORDER_SELECT_RATIO=1 (tools/build_variant.sh) to time the select on both sides of the crossover;
    - for scale, torch.sort(stable=True) and torch.topk of the ToTensors price values;
    - a streamed FromBytes of the orders CSV (several GiB) .OrderBy(("ts", "str", "desc")).Top(100), against the same
      stream parsed and filtered to no rows;
    - the host route, ToRows() + Python sorted, at 1 M rows.
  The card's name and power limit are printed first."""
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
print("library:", os.environ.get("CPB_LIB", "default"), flush=True)


def wall(fn, reps=REPS):
    fn()
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize(dev)
    return (time.perf_counter() - t0) / reps, out


def kernels(fn):
    ctx.stats(enable=True, reset=True)
    fn()
    st = ctx.stats()
    ctx.stats(enable=False)
    return "  ".join(f"{k} {v['ms']:.2f}" for k, v in sorted(st.items(), key=lambda kv: -kv[1]["ms"])[:8]) + " (ms)"


buf = ctx.gen_csv("orders", (0, rows), n_cust=rows // 10, n_prod=1000)
o, err = cp.parse_csv(ctx, buf, on_device=True, spec=[("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)])
assert err is None
ctx.sync()
buf.free()
pbuf = ctx.gen_csv("products", (0, 1000), n_prod=1000)
prods, err = cp.parse_csv(ctx, pbuf, on_device=True, spec=[("prod_id", -1), ("price", -1)])
assert err is None
t = o.join(prods.index_on("prod_id", unique=True), "prod_id")
del o
n = len(t)
PRICE = ("price", "float64", "desc")
print(f"orders: {n} rows, columns {t.columns}", flush=True)

for label, keys in (("price float64 desc", (PRICE,)), ("(cust_id, ts) str", ("cust_id", "ts"))):
    s, r = wall(lambda: t.order_by(*keys))
    del r
    print(f"order_by {label:22s} {s * 1e3:9.2f} ms  {n / s / 1e9:6.3f} G rows/s", flush=True)
    print("    " + kernels(lambda: t.order_by(*keys)), flush=True)

full_s, _ = wall(lambda: t.order_by(PRICE).slice(0, 10))
for k in (10, 1000, 100_000, 1_000_000, n // 32, n // 8, n // 4, n // 2, 3 * n // 4, 9 * n // 10):
    s, r = wall(lambda: t.order_by(PRICE, limit=k))
    del r
    print(f"first {k:>10} by price: order_by(limit=k) {s * 1e3:9.2f} ms   full sort + slice {full_s * 1e3:9.2f} ms", flush=True)
    if k in (10, 1_000_000):
        print("    " + kernels(lambda: t.order_by(PRICE, limit=k)), flush=True)

v = cp.TakeTable(t).ToTensors({"price": "float64"})["price"]
s, _ = wall(lambda: torch.sort(v, descending=True, stable=True))
print(f"torch.sort(stable=True) of ToTensors price {s * 1e3:9.2f} ms", flush=True)
for k in (10, 1_000_000):
    s, _ = wall(lambda: torch.topk(v, k))
    print(f"torch.topk k={k:<8} {s * 1e3:9.2f} ms", flush=True)
del v, t
torch.cuda.empty_cache()

# streamed: the orders CSV on the host, pushed in STREAM_BATCH_BYTES batches
stream_rows = min(rows, 80_000_000)
sbuf = ctx.gen_csv("orders", (0, stream_rows), n_cust=stream_rows // 10, n_prod=1000)
data = sbuf.to_host()
sbuf.free()
gib = data.size / 2 ** 30
s, top = wall(lambda: cp.Take(cp.FromBytes(data, ctx)).OrderBy(("ts", "str", "desc")).Top(100).ToRows(), reps=1)
assert len(top) == 100
s0, _ = wall(lambda: cp.Take(cp.FromBytes(data, ctx)).Filter(cp.Like({"cust_id": "none"})).ToRows(), reps=1)
print(f"streamed FromBytes {gib:.2f} GiB ({stream_rows} rows) .OrderBy(ts desc).Top(100): {s * 1e3:9.1f} ms "
      f"({gib / s:.2f} GiB/s); parse + Filter to no rows {s0 * 1e3:9.1f} ms", flush=True)
ctx.pool_used_high(reset=True)
cp.Take(cp.FromBytes(data, ctx)).OrderBy(("ts", "str", "desc")).Top(100).ToRows()
print(f"    device pool high-water mark {ctx.pool_used_high() / 2 ** 20:.0f} MiB", flush=True)
del data

# the host route at 1 M rows
small = cp.Take(cp.FromBytes(ctx.gen_csv("orders", (0, 1_000_000), n_cust=100_000, n_prod=1000).to_host(), ctx))
s, _ = wall(lambda: sorted(small.ToRows(), key=lambda r: r["ts"], reverse=True)[:100], reps=1)
sg, _ = wall(lambda: small.OrderBy(("ts", "str", "desc")).Top(100).ToRows(), reps=1)
print(f"host route ToRows() + sorted at 1 M rows: {s * 1e3:.1f} ms; OrderBy(...).Top(100) {sg * 1e3:.2f} ms", flush=True)
