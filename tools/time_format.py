"""FormatInt / FormatFloat timing: python tools/time_format.py [rows]

  shapes (values already in HBM): FormatInt of ids, FormatFloat(price*qty, 'f', 2) and FormatFloat(x, 'g', -1) of random
  finite doubles, each float shape followed by its float32 leg (the same prices as float32 with bitSize 32; random
  finite float32 bits);
  per shape: kernel ms per call (format_int / format_float / format_float32, format_rare / format_rare32 when rows took
  the exact path, the offset scan, format_write), algorithmic bytes (8 B of value per row (4 B for float32) + 4 B of
  offset per row + the output bytes) over the sum of
  kernel times against the H100 SXM data-sheet 3.35 TB/s, each kernel's own bytes over its time, the call's wall time
  and host synchronisations per call;
  then a MapTensors step end to end against the host Transform closure it replaces, at 1 M rows, both through ToCsv."""
import ctypes as C
import io
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import csvplus_b200 as cp  # noqa: E402

PEAK = 3.35e12
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 20_000_000
ctx = cp.Context(0)
dev = torch.device("cuda", ctx.device)
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
except OSError:
    print("nvidia-smi not available", flush=True)


def base(n):
    off = torch.zeros(n + 1, dtype=torch.int32, device=dev)
    data = torch.zeros(16, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    return cp.Table.from_device_columns(ctx, ["k"], [(off.data_ptr(), data.data_ptr())], n)


def report(label, t, values, fmt=None, prec=-1, reps=5):
    if isinstance(values, cp.FormatFloat):  # the format is in the marker
        vbytes, kw = values.values.element_size(), {}
    else:
        vbytes, kw = values.element_size(), {"fmt": fmt, "prec": prec}
    for _ in range(2):
        out = t.with_column("v", values, **kw)
    ctx.stats(enable=True, reset=True)
    s0 = ctx.host_syncs()
    torch.cuda.synchronize(dev)
    w0 = time.perf_counter()
    for _ in range(reps):
        out = t.with_column("v", values, **kw)
    wall = (time.perf_counter() - w0) / reps
    syncs = (ctx.host_syncs() - s0) / reps
    st = ctx.stats(); ctx.stats(enable=False)
    n = len(t)
    nb = C.c_uint64()
    ctx.lib.cpb_table_col_bytes(ctx.h, out.h, out.columns.index("v"), 0, n, C.byref(nb))
    out_total = nb.value
    algo = vbytes * n + 4 * (n + 1) + out_total
    kms = sum(v["ms"] for k, v in st.items()) / reps
    print(f"{label}: {n} rows, {out_total / n:.1f} B per row, {kms:.3f} ms of kernels per call, wall {wall * 1e3:.3f} ms per call, "
          f"{syncs:.0f} host sync(s) per call; algo {algo / 1e9:.3f} GB -> {algo / (kms * 1e-3) / 1e9:.0f} GB/s = "
          f"{algo / (kms * 1e-3) / PEAK:.1%} of 3.35 TB/s", flush=True)
    for k, v in sorted(st.items()):
        ms, b = v["ms"] / reps, v["algo_bytes"] / reps
        extra = f"  algo {b / 1e9:.3f} GB -> {b / (ms * 1e-3) / 1e9:.0f} GB/s = {b / (ms * 1e-3) / PEAK:.1%} of 3.35 TB/s" if b and ms else ""
        print(f"  {k:14s} {ms:8.3f} ms{extra}", flush=True)


g = torch.Generator(device=dev).manual_seed(1)
t = base(rows)
report("FormatInt(id)", t, torch.arange(rows, dtype=torch.int64, device=dev) * 7919 % (10 ** 9))
price = torch.randint(1, 100_000, (rows,), device=dev, generator=g).to(torch.float64) / 100
qty = torch.randint(1, 50, (rows,), device=dev, generator=g).to(torch.float64)
report("FormatFloat(price*qty, 'f', 2)", t, price * qty, "f", 2)
report("FormatFloat(price*qty, 'f', 2, 32)", t, cp.FormatFloat((price * qty).float(), "f", 2, bit_size=32))
x = torch.randint(-2**63, 2**63 - 1, (rows,), dtype=torch.int64, device=dev, generator=g).view(torch.float64)
x = torch.where(torch.isfinite(x), x, torch.zeros_like(x))
report("FormatFloat(x, 'g', -1), random bits", t, x, "g", -1)
x32 = torch.randint(-2**31, 2**31 - 1, (rows,), dtype=torch.int32, device=dev, generator=g).view(torch.float32)
x32 = torch.where(torch.isfinite(x32), x32, torch.zeros_like(x32))
report("FormatFloat(x, 'g', -1, 32), random bits", t, cp.FormatFloat(x32, "g", -1, bit_size=32))
del t, price, qty, x, x32

# a MapTensors step against the host Transform closure, end to end through ToCsv, at 1 M rows
n1 = 1_000_000
rng = np.random.default_rng(3)
p1, q1 = rng.integers(1, 100_000, n1) / 100, rng.integers(1, 50, n1)
data = ("id,price,qty\n" + "".join(f"{i},{p!r},{q}\n" for i, (p, q) in enumerate(zip(p1.tolist(), q1.tolist())))).encode()


def dev_plan():
    return cp.Take(cp.FromBytes(data, ctx)).MapTensors(
        {"price": "float64", "qty": "int"}, lambda v: {"amount": cp.FormatFloat(v["price"] * v["qty"].to(torch.float64), "f", 2)})


def host_tr(row):
    row["amount"] = "%.2f" % (float(row["price"]) * int(row["qty"]))  # strconv.FormatFloat(x, 'f', 2, 64) for these values
    return row


def host_plan():
    return cp.Take(cp.FromBytes(data, ctx)).Transform(host_tr)


res = {}
for name, plan in (("MapTensors", dev_plan), ("host Transform", host_plan)) * 2:
    out = io.BytesIO()
    t0 = time.perf_counter()
    plan().ToCsv(out, "id", "amount")
    res.setdefault(name, []).append((time.perf_counter() - t0, out.getvalue()))
assert res["MapTensors"][-1][1] == res["host Transform"][-1][1]
print(f"1 M rows through ToCsv(id, amount): MapTensors {min(s for s, _ in res['MapTensors']) * 1e3:.1f} ms, host Transform "
      f"{min(s for s, _ in res['host Transform']) * 1e3:.1f} ms (best of 2 each, alternating); outputs identical", flush=True)
