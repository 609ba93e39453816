"""Kernel times of the customers index and join on the row-carrying hash table: python tools/prof_rowhash.py [orders_rows]
[customers_rows]; prints one line of ms per repetition (5 repetitions after 2 warm-ups, from the library's CUDA-event
stats) for rowhash_scatter, rowhash_build (rowhash_region_kernel) and rowhash_probe.

Run it against a library built with a diagnostic switch (CPB_LIB=csvplus_b200/_var/<name>.so, built by
SOURCES="join.cu gather.cu" tools/build_variant.sh <name> - -D<switch>) to see where a kernel's time goes:
RH_DIAG_NO_ATOMIC (scatter: the position from the row number instead of the fill-count atomic), RH_DIAG_NO_PAYLOAD
(scatter: the key alone), RH_DIAG_NO_STORE (scatter: no image store), RH_DIAG_SEQ_SLOT (probe: the slot at row % nslots
instead of the key's, so the random sector read becomes a sequential one), RH_DIAG_L2_FETCH32 (probe: L2 fills of 32
bytes).  Such a build makes wrong tables: an index or join it fails is reported and its kernel times still count."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import csvplus_b200 as cp

KERNELS = ("rowhash_scatter", "rowhash_build", "rowhash_probe")
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 125_000_000
ncust = int(sys.argv[2]) if len(sys.argv) > 2 else 100_000_000
ctx = cp.Context(0)
cust = ctx.gen_csv("customers", (0, ncust), n_cust=ncust, permute=True)
orders = ctx.gen_csv("orders", (0, rows), n_cust=ncust, n_prod=1_000_000)
tc, _ = cp.parse_csv(ctx, cust, spec=[("id", -1), ("name", -1), ("surname", -1)])
to, _ = cp.parse_csv(ctx, orders, spec=[("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)])
errors = set()


def step():
    try:
        idx = tc.index_on("id", unique=True)
        return len(to.join(idx, "cust_id"))
    except cp.CsvPlusError as e:
        errors.add(str(e)[:80])
        return -1


for _ in range(2):
    step()
ctx.sync()
reps = 5
ctx.stats(enable=True, reset=True)
t0 = time.perf_counter()
for _ in range(reps):
    n = step()
ctx.sync()
dt = (time.perf_counter() - t0) / reps * 1e3
st = ctx.stats()
ctx.stats(enable=False)
out = {"lib": os.path.basename(os.environ.get("CPB_LIB", "libcsvplus_b200.so")), "rows": n, "wall_ms": round(dt, 2)}
out.update({k: round(st[k]["ms"] / reps, 3) if k in st else None for k in KERNELS})
out["three_ms"] = round(sum(out[k] or 0.0 for k in KERNELS), 3)
if errors:
    out["errors"] = sorted(errors)
print(json.dumps(out), flush=True)
