"""ToText timing: python tools/time_sprintf.py [orders]

On bench.py's shapes (customers = orders / 1.25, 1 M products, both permuted, UniqueIndexOn("id") / ("prod_id")), N orders
joined with both as bench.py joins them, then:
  1. ToText of the README's Printf line ("%s %s bought %s %ss for £%s each on %s\\n" of name, surname, qty, product,
     price, ts) through Table.sprintf_into into one pinned buffer, against to_csv_into of the same six columns (the e2e
     sink today) in the same run;
  2. with_column(Sprintf) of the same line, the bytes left in HBM;
  3. the host RowFunc the GPU path replaces (ToRows + %-formatting per row) at 1 M rows.
Per kernel: ms per call.  Output GB/s = output bytes / the sum of the call's kernel times (copies to the host excluded);
wall ms per call includes them."""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import csvplus_b200 as cp  # noqa: E402

SEED = 0xC5B200
FMT = "%s %s bought %s %ss for £%s each on %s\n"
COLS = ("name", "surname", "qty", "product", "price", "ts")
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 20_000_000
ctx = cp.Context(0)
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
except OSError:
    print("nvidia-smi not available", flush=True)

n_cust, n_prod = max(1, rows * 4 // 5), 1_000_000
cust = ctx.gen_csv("customers", (0, n_cust), seed=SEED, n_cust=n_cust, permute=True)
prod = ctx.gen_csv("products", (0, n_prod), seed=SEED, n_prod=n_prod, permute=True)
orders = ctx.gen_csv("orders", (0, rows), seed=SEED, n_cust=n_cust, n_prod=n_prod)
tc, _ = cp.parse_csv(ctx, cust, spec=[("id", -1), ("name", -1), ("surname", -1)])
tp, _ = cp.parse_csv(ctx, prod, spec=[("prod_id", -1), ("product", -1), ("price", -1)])
to, _ = cp.parse_csv(ctx, orders, spec=[("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)])
j = to.join(tc.index_on("id", unique=True), "cust_id").join(tp.index_on("prod_id", unique=True))
del cust, prod, orders
print(f"joined rows: {len(j)}", flush=True)


def timed(call, reps=5):
    """(output bytes, {kernel: ms per call}, wall ms per call) of call(), after two warm-up calls"""
    for _ in range(2):
        n = call()
    ctx.sync()
    ctx.stats(enable=True, reset=True)
    t0 = time.perf_counter()
    for _ in range(reps):
        call()
    ctx.sync()
    wall = (time.perf_counter() - t0) * 1e3 / reps
    st = ctx.stats(); ctx.stats(enable=False)
    return n, {k: v["ms"] / reps for k, v in st.items()}, wall


def report(label, n, kms, wall):
    kt = sum(v for k, v in kms.items() if k != "d2h_output")
    per = ", ".join(f"{k} {v:.3f} ms" for k, v in sorted(kms.items()))
    print(f"{label}: {n} bytes; kernels {kt:.3f} ms -> {n / (kt * 1e-3) / 1e9:.1f} GB/s of output; wall {wall:.2f} ms per call  [{per}]",
          flush=True)


size = j.sprintf_into(None, 0, FMT, *COLS)
csv_size = j.to_csv_into(None, 0, *COLS, header=False)
buf = ctx.host_alloc(max(size, csv_size) + 64)
report("ToText (sprintf_into)", *timed(lambda: j.sprintf_into(buf, 0, FMT, *COLS)))
report("ToCsv  (to_csv_into) ", *timed(lambda: j.to_csv_into(buf, 0, *COLS, header=False)))
buf.free()
report("with_column(Sprintf) ", *timed(lambda: (j.with_column("line", cp.Sprintf(FMT, *COLS)), size)[1]))

n1 = min(len(j), 1_000_000)
small = j.slice(0, n1)
t0 = time.perf_counter()
host = "".join(FMT % tuple(r[c] for c in COLS) for r in cp.TakeTable(small).ToRows()).encode("utf-8", "surrogateescape")
host_s = time.perf_counter() - t0
b = ctx.host_alloc(small.sprintf_into(None, 0, FMT, *COLS) + 64)
t0 = time.perf_counter()
nb = small.sprintf_into(b, 0, FMT, *COLS)
dev_s = time.perf_counter() - t0
assert bytes(b.array()[:nb]) == host
b.free()
print(f"host RowFunc at {n1} rows: {host_s:.2f} s ({n1 / host_s:.0f} rows/s); GPU sprintf_into of the same rows incl. the copy to the "
      f"host: {dev_s * 1e3:.1f} ms; outputs identical", flush=True)
