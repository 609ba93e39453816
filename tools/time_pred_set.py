"""Set-term timing: python tools/time_pred_set.py [orders_rows]

Filter(Any(Like{cust_id: v1}, Like{cust_id: v2}, ...)) over generated orders in device memory (FromBytes(DeviceBuffer):
one cpb_parse_csv call), with sets of 33, 10^3, 10^5 and 10^6 literals.  Each set holds every second customer id of
2 x its size customers, so about half of the rows match.  Per set size:
  - the whole call: ms and input GB/s (host clock around the call, which ends in a host synchronisation);
  - per kernel (CUDA events): the literal table upload (pred_set_upload), the index build (key_width, key_pack, the radix
    sort, image_gather, hash_heads, hash_build), the probe (join_probe), the evaluation (filter_set), and the parse and
    compaction around them;
  - the host compile (cpb_table_filter on a table with no rows: the predicate is compiled, nothing runs);
  - the same input filtered with a single Like (fused into csv_scan): the ceiling.
Then the Python lowering time of the 10^6-literal tree, and the host-row route a tree past the limits took before set
terms existed (every row a dict, Predicate.__call__, Table.from_rows) at 1 M rows with the 33-literal set.
The card's name and power limit are printed first."""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import csvplus_b200 as cp  # noqa: E402

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 50_000_000
SIZES = [33, 1_000, 100_000, 1_000_000]
SPEC = [("cust_id", -1), ("prod_id", -1), ("qty", -1), ("ts", -1)]
ctx = cp.Context(0)
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
except OSError:
    print("nvidia-smi not available", flush=True)


def literals(k):
    cust = ctx.gen_csv("customers", (0, 2 * k), n_cust=2 * k)
    t, _ = cp.parse_csv(ctx, cust, spec=[("id", -1)])
    return [v.decode() for v in t.values("id")[::2]]


def timed(fn, reps=3):
    """-> (result, best wall ms, per-kernel ms of the best repetition)"""
    fn()
    ctx.sync()
    best = None
    for _ in range(reps):
        ctx.stats(enable=True, reset=True)
        t0 = time.perf_counter()
        r = fn()
        ctx.sync()
        ms = (time.perf_counter() - t0) * 1e3
        st = ctx.stats(); ctx.stats(enable=False)
        if best is None or ms < best[1]:
            best = (r, ms, {k: v["ms"] for k, v in st.items()})
    return best


BUILD = ("key_width", "key_pack", "radix", "image_gather", "hash_heads", "hash_build")
for k in SIZES:
    buf = ctx.gen_csv("orders", (0, rows), n_cust=2 * k, n_prod=1000)
    nb = buf.nbytes
    lits = literals(k)
    pred = cp.Any(*[cp.Like({"cust_id": v}) for v in lits])
    t0 = time.perf_counter()
    pred._c([])
    lower_ms = (time.perf_counter() - t0) * 1e3
    assert pred.lowerable()
    empty, _ = cp.parse_csv(ctx, b"cust_id,prod_id,qty,ts\n", spec=SPEC)
    _, compile_ms, _ = timed(lambda: empty.filter(pred))
    (t, err), ms, st = timed(lambda: cp.parse_csv(ctx, buf, spec=SPEC, pred=pred))
    assert err is None
    kept = len(t)
    build = sum(v for name, v in st.items() if name.startswith(BUILD))
    print(f"set of {k:>9,} literals: {kept:,} of {rows:,} rows kept; {ms:8.2f} ms = {nb / ms / 1e6:6.1f} GB/s over {nb / 1e9:.2f} GB; "
          f"host compile {compile_ms:.2f} ms, Python lowering {lower_ms:.1f} ms", flush=True)
    print(f"    upload {st.get('pred_set_upload', 0):.3f} ms, index build {build:.3f} ms, probe {st.get('join_probe', 0):.3f} ms, "
          f"filter_set {st.get('filter_set', 0):.3f} ms, csv_scan {st.get('csv_scan', 0):.3f} ms", flush=True)
    print("    every kernel (ms):", {name: round(v, 3) for name, v in sorted(st.items(), key=lambda kv: -kv[1])}, flush=True)
    one = cp.Like({"cust_id": lits[0]})
    (t1, _), ms1, st1 = timed(lambda: cp.parse_csv(ctx, buf, spec=SPEC, pred=one))
    print(f"    single Like (fused): {len(t1):,} rows, {ms1:8.2f} ms = {nb / ms1 / 1e6:6.1f} GB/s; csv_scan {st1.get('csv_scan', 0):.3f} ms",
          flush=True)
    del t, t1, buf

# the route of a tree past the limits before set terms: host rows, Predicate.__call__, the kept rows uploaded again
n1 = 1_000_000
buf = ctx.gen_csv("orders", (0, n1), n_cust=2 * SIZES[0], n_prod=1000)
pred = cp.Any(*[cp.Like({"cust_id": v}) for v in literals(SIZES[0])])
t, _ = cp.parse_csv(ctx, buf, spec=SPEC)
t0 = time.perf_counter()
kept = [r for r in t.rows() if pred(r)]
back = cp.Table.from_rows(ctx, kept, [c for c, _ in SPEC])
ctx.sync()
host_ms = (time.perf_counter() - t0) * 1e3
(td, _), dev_ms, _ = timed(lambda: cp.parse_csv(ctx, buf, spec=SPEC, pred=pred))
assert len(td) == len(back)
print(f"1 M rows, set of 33: host rows {host_ms:.0f} ms ({buf.nbytes / host_ms / 1e6:.3f} GB/s) vs the device {dev_ms:.2f} ms "
      f"({buf.nbytes / dev_ms / 1e6:.1f} GB/s, parse included)", flush=True)
