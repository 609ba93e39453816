"""ToJSON timing: python tools/time_json.py [rows]

  1. orders parse (4 columns), ToJSON of the table with the bytes left in HBM, against ToCsv of the same table and columns
     in the same run (the yardstick);
  2. the same on an orders x customers join result (6 columns);
  3. the host encoder the GPU path replaces (TakeTable(t).ToRows() + api._go_json_string) at 1 M rows.
Per kernel: ms per call, and algorithmic bytes (value bytes + offsets [+ lengths] + output bytes) over kernel time against
the H100 SXM data-sheet 3.35 TB/s.  Output GB/s = output bytes / the sum of the call's kernel times."""
import ctypes as C
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import csvplus_b200 as cp  # noqa: E402
from csvplus_b200 import api  # noqa: E402

PEAK = 3.35e12
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 20_000_000
ctx = cp.Context(0)
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
except OSError:
    print("nvidia-smi not available", flush=True)


def value_bytes(t):
    tot = 0
    for i in range(len(t.columns)):
        nb = C.c_uint64()
        ctx.lib.cpb_table_col_bytes(ctx.h, t.h, i, 0, len(t), C.byref(nb))
        tot += nb.value
    return tot


def timed(fn, reps=5):
    for _ in range(2):
        b = fn(); n = b.nbytes; b.free()
    ctx.stats(enable=True, reset=True)
    for _ in range(reps):
        fn().free()
    st = ctx.stats(); ctx.stats(enable=False)
    return n, {k: v["ms"] / reps for k, v in st.items()}


def report(label, t, cols):
    n, nc, vb = len(t), len(t.columns), value_bytes(t)
    jn, jms = timed(lambda: t.to_json_device())
    cn, cms = timed(lambda: t.to_csv_device(*cols))
    algo = {"json_row_len": vb + n * 4 * (nc + 1) + n * 4, "json_write": vb + n * 4 * (nc + 1) + jn}
    print(f"{label}: {n} rows, {nc} columns, {vb} value bytes", flush=True)
    for k, ms in sorted(jms.items()):
        extra = f"  algo {algo[k] / 1e9:.2f} GB -> {algo[k] / (ms * 1e-3) / 1e9:.0f} GB/s = {algo[k] / (ms * 1e-3) / PEAK:.1%} of 3.35 TB/s" if k in algo else ""
        print(f"  ToJSON {k:14s} {ms:8.3f} ms{extra}", flush=True)
    jt, ct = sum(jms.values()), sum(cms.values())
    print(f"  ToJSON {jn} bytes in {jt:.3f} ms of kernels: {jn / (jt * 1e-3) / 1e9:.1f} GB/s of output", flush=True)
    print(f"  ToCsv  {cn} bytes in {ct:.3f} ms of kernels: {cn / (ct * 1e-3) / 1e9:.1f} GB/s of output  {dict((k, round(v, 3)) for k, v in cms.items())}",
          flush=True)
    print(f"  ToCsv / ToJSON output rate: {(cn / ct) / (jn / jt):.2f}x", flush=True)


orders = ctx.gen_csv("orders", (0, rows), n_cust=rows // 10, n_prod=1000)
t, _ = cp.parse_csv(ctx, orders, spec=[("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)])
report("orders", t, ["cust_id", "prod_id", "qty", "ts"])

cust = ctx.gen_csv("customers", (0, rows // 10), n_cust=rows // 10, permute=True)
tc, _ = cp.parse_csv(ctx, cust, spec=[("id", -1), ("name", -1), ("surname", -1)])
tp, _ = cp.parse_csv(ctx, orders, spec=[("cust_id", -1), ("prod_id", -1), ("qty", -1)])
j = tp.join(tc.index_on("id", unique=True), "cust_id")
report("orders x customers", j, sorted(j.columns))

n1 = min(rows, 1_000_000)
small = t.slice(0, n1)
t0 = time.perf_counter()
rs = cp.TakeTable(small).ToRows()
doc = b"[" + b",".join(b"{" + b",".join(api._go_json_string(k) + b":" + api._go_json_string(r[k]) for k in sorted(r)) + b"}\n" for r in rs) + b"]"
host_s = time.perf_counter() - t0
t0 = time.perf_counter()
dev = small.to_json()
dev_s = time.perf_counter() - t0
assert dev == doc
print(f"host encoder at {n1} rows: {host_s:.2f} s ({len(doc) / host_s / 1e6:.1f} MB/s); GPU to_json of the same rows incl. the copy to "
      f"the host: {dev_s * 1e3:.1f} ms; outputs identical", flush=True)
