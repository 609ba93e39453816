"""ValueAsInt / ValueAsFloat64 / ParseFloat(s, 32) timing: python tools/time_numeric.py [rows]

  columns: qty, cust_id, order_id of generated orders (int), price of products and score of people (float64, then the
  same column as float32 beside it), and a hard-float column of 17-25-digit values (float64, then float32);
  per column: kernel ms per call (numeric_int / numeric_float + numeric_rare, numeric_float32 + numeric_rare32),
  algorithmic bytes (offsets + value bytes + 8 B of output (4 B for float32) + 1 B of status per row) over kernel time
  against the H100 SXM data-sheet 3.35 TB/s, rows that took the exact path, and host synchronisations per call;
  then the host path the conversion replaces (Table.rows() + int() / float()) at 1 M rows."""
import os
import random
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import csvplus_b200 as cp  # noqa: E402

PEAK = 3.35e12
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 20_000_000
ctx = cp.Context(0)
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
except OSError:
    print("nvidia-smi not available", flush=True)


def timed(t, name, kind, reps=5):
    conv = {"int": t.values_as_int, "float64": t.values_as_float64, "float32": t.values_as_float32}[kind]
    for _ in range(2):
        conv(name, strict=False)
    ctx.stats(enable=True, reset=True)
    s0 = ctx.host_syncs()
    for _ in range(reps):
        conv(name, strict=False)
    syncs = (ctx.host_syncs() - s0) / reps
    st = ctx.stats(); ctx.stats(enable=False)
    return {k: (v["ms"] / reps, v["algo_bytes"] / reps) for k, v in st.items()}, syncs


def report(label, t, name, kind):
    st, syncs = timed(t, name, kind)
    total = sum(ms for ms, _ in st.values())
    print(f"{label}: {len(t)} rows, {total:.3f} ms of kernels per call, {syncs:.0f} host sync(s) per call", flush=True)
    for k, (ms, b) in sorted(st.items()):
        extra = f"  algo {b / 1e9:.3f} GB -> {b / (ms * 1e-3) / 1e9:.0f} GB/s = {b / (ms * 1e-3) / PEAK:.1%} of 3.35 TB/s" if b and ms else ""
        print(f"  {k:14s} {ms:8.3f} ms{extra}", flush=True)


orders = ctx.gen_csv("orders", (0, rows), n_cust=rows // 10, n_prod=1000)
to, _ = cp.parse_csv(ctx, orders, spec=[("order_id", -1), ("cust_id", -1), ("qty", -1)])
for c in ("qty", "cust_id", "order_id"):
    report(f"orders.{c} (int)", to, c, "int")
products = ctx.gen_csv("products", (0, rows), n_prod=rows)
tp, _ = cp.parse_csv(ctx, products, spec=[("price", -1)])
report("products.price (float64)", tp, "price", "float64")
report("products.price (float32)", tp, "price", "float32")
people = ctx.gen_csv("people", (0, rows))
tq, _ = cp.parse_csv(ctx, people, spec=[("score", -1)])
report("people.score (float64)", tq, "score", "float64")
report("people.score (float32)", tq, "score", "float32")
# hard floats: 17-25 significant digits with exponents across the range
rng = random.Random(5)
nh = min(rows, 2_000_000)
hard = [f"{rng.randint(1, 9)}.{rng.randrange(10 ** 24):024d}"[: rng.randint(18, 26)] + f"e{rng.randint(-300, 300)}" for _ in range(nh)]
th = cp.Table.from_rows(ctx, [{"h": v} for v in hard], columns=["h"])
report(f"hard floats, 17-25 digits (float64, {nh} rows)", th, "h", "float64")
hard32 = [v[: v.index("e")] + f"e{rng.randint(-40, 35)}" for v in hard]  # the same digits inside float32's range
th32 = cp.Table.from_rows(ctx, [{"h": v} for v in hard32], columns=["h"])
report(f"hard floats, 17-25 digits, exponents -40..35 (float64, {nh} rows)", th32, "h", "float64")
report(f"hard floats, 17-25 digits, exponents -40..35 (float32, {nh} rows)", th32, "h", "float32")

n1 = min(rows, 1_000_000)
small = to.slice(0, n1)
t0 = time.perf_counter()
rs = small.rows()
host = [int(r["qty"]) for r in rs]
host_s = time.perf_counter() - t0
t0 = time.perf_counter()
dev = small.values_as_int("qty").cpu().tolist()
dev_s = time.perf_counter() - t0
assert dev == host
sp = tp.slice(0, n1)
t0 = time.perf_counter()
hostf = [float(r["price"]) for r in sp.rows()]
hostf_s = time.perf_counter() - t0
assert sp.values_as_float64("price").cpu().tolist() == hostf
print(f"host path at {n1} rows: qty via rows() + int() {host_s:.2f} s, price via rows() + float() {hostf_s:.2f} s; "
      f"GPU values_as_int incl. the copy to the host {dev_s * 1e3:.1f} ms; outputs identical", flush=True)
