"""Streamed input timing: python tools/time_stream.py [orders_rows[,orders_rows...]] [batch_MiB]

  1. stream_cut at a 1 GiB batch on generated orders and on a quote-heavy input, quote-parity kernel and the DFA variant
     (CommentChar set): ms per call and algorithmic GB/s (each input byte read once) against the H100 SXM data-sheet
     3.35 TB/s;
  2. end to end: FromFile(orders).SelectColumns(cust_id, prod_id, qty, ts).Join(custIdx, "cust_id").Join(prodIdx)
     .ToCsv(...) from the page cache into a writer that keeps a CRC of the bytes, streamed in batches of
     STREAM_BATCH_BYTES against the same file pushed as one piece in the same run (alternating, best of three):
     input GB/s, rows/s, batches, host synchronisations, and the peak device memory of the context's pool during the run
     (cpb_pool_used_high; it includes the two indices).  The two outputs are compared by length and CRC-32.  By default at 30 M rows and
     at 125 M rows, where the one-piece path fails (a ToCsv batch output above 4 GiB) and the streamed path runs alone.
The card's name and power limit are printed first."""
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import csvplus_b200 as cp  # noqa: E402
from csvplus_b200 import api  # noqa: E402

PEAK = 3.35e12
rows = [int(x) for x in sys.argv[1].split(",")] if len(sys.argv) > 1 else [30_000_000, 125_000_000]
batch_mib = int(sys.argv[2]) if len(sys.argv) > 2 else api.STREAM_BATCH_BYTES >> 20
ctx = cp.Context(0)
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
except OSError:
    print("nvidia-smi not available", flush=True)


def time_cut(label, buf, n, reps=20, **opts):
    for _ in range(3):
        cut = cp.csv_stream_cut(ctx, buf, nbytes=n, on_device=True, **opts)
    ctx.stats(enable=True, reset=True)
    for _ in range(reps):
        assert cp.csv_stream_cut(ctx, buf, nbytes=n, on_device=True, **opts) == cut
    st = ctx.stats(); ctx.stats(enable=False)
    name = "stream_cut_dfa" if opts else "stream_cut"
    ms = st[name]["ms"] / reps
    print(f"  {label:28s} {name:15s} {ms:8.3f} ms  {n / (ms * 1e-3) / 1e9:7.1f} GB/s = {n / (ms * 1e-3) / PEAK:5.1%} of 3.35 TB/s"
          f"  (cut at {cut})", flush=True)


GIB = 1 << 30
print("stream_cut at a 1 GiB batch", flush=True)
orders_1g = ctx.gen_csv("orders", (0, 24_000_000), n_cust=1_000_000, n_prod=1000)
assert orders_1g.nbytes >= GIB
time_cut("orders", orders_1g, GIB)
time_cut("orders", orders_1g, GIB, comment="#")
orders_1g.free()
block = (b'"a ""quoted"" field,\nwith a newline",' * 40 + b'x,"y"\n') * 64
quoted = ctx.device_alloc(GIB)
hb = cp.HostBuffer(ctx, GIB)
a = hb.array()
rep = bytes(block) * (GIB // len(block) + 1)
a[:] = np.frombuffer(rep, np.uint8, GIB)
ctx.lib.cpb_memcpy_h2d(ctx.h, api.C.c_void_p(quoted.ptr), api.C.c_void_p(hb.ptr), GIB)
hb.free()
del rep
time_cut("quote-heavy", quoted, GIB)
time_cut("quote-heavy", quoted, GIB, comment="#")
quoted.free()

# ---------------------------------------------------------------- end to end
n_cust, n_prod = 10_000_000, 1_000_000
cust = ctx.gen_csv("customers", (0, n_cust), n_cust=n_cust, permute=True)
prod = ctx.gen_csv("products", (0, n_prod), n_prod=n_prod)
cust_idx = cp.Take(cp.FromBytes(cust, ctx).SelectColumns("id", "name", "surname")).UniqueIndexOn("id")
prod_idx = cp.Take(cp.FromBytes(prod, ctx).SelectColumns("prod_id", "product", "price")).UniqueIndexOn("prod_id")
cust.free(); prod.free()


class Sink:
    """a file-like output that keeps a CRC of everything written (the outputs of both paths are compared by it and by
    length) instead of storing gigabytes"""

    def __init__(self):
        import zlib
        self.zlib, self.crc, self.n = zlib, 0, 0

    def write(self, b):
        self.crc = self.zlib.crc32(b, self.crc)
        self.n += len(b)
        return len(b)


def run(path, size, streamed: bool):
    api.STREAM_BATCH_BYTES = (batch_mib << 20) if streamed else size + 1
    out = Sink()
    ctx.pool_used_high(reset=True)
    s0, t0 = ctx.host_syncs(), time.perf_counter()
    batches = [0]
    ds = cp.Take(cp.FromFile(path, ctx).SelectColumns("cust_id", "prod_id", "qty", "ts")).Join(cust_idx, "cust_id").Join(prod_idx)
    orig = api.Reader._batches

    def counting(self, pred=None):
        for b in orig(self, pred):
            batches[0] += 1
            yield b
    api.Reader._batches = counting
    try:
        ds.ToCsv(out, "cust_id", "name", "prod_id", "product", "qty", "ts")
    except cp.CsvPlusError as e:
        return None, str(e)
    finally:
        api.Reader._batches = orig
    ctx.sync()
    dt = time.perf_counter() - t0
    return (dt, out, batches[0], ctx.host_syncs() - s0, ctx.pool_used_high()), None


def compare(rows):
    tmp = tempfile.mkdtemp()
    path = os.path.join(tmp, "orders.csv")
    with open(path, "wb") as f:
        step = 20_000_000
        for lo in range(0, rows, step):
            b = ctx.gen_csv("orders", (lo, min(rows, lo + step)), n_cust=n_cust, n_prod=n_prod, header=lo == 0)
            f.write(memoryview(b.to_host()))
            b.free()
    size = os.path.getsize(path)
    print(f"orders file: {rows} rows, {size / 1e9:.2f} GB (page cache)", flush=True)
    res, fail = {True: [], False: []}, {}
    for _ in range(3):
        for streamed in (True, False):
            if streamed in fail:
                continue
            r, err = run(path, size, streamed)
            if err is not None:
                fail[streamed] = err
            else:
                res[streamed].append(r)
    for streamed in (True, False):
        name = "streamed" if streamed else "one piece"
        if streamed in fail:
            print(f"  {name:11s} fails: {fail[streamed]}", flush=True)
            continue
        dt, out, nb, syncs, peak = min(res[streamed], key=lambda r: r[0])
        print(f"  {name:11s} best of 3: {dt:6.2f} s  {size / dt / 1e9:5.2f} GB/s of input  {rows / dt / 1e6:6.1f} M rows/s  "
              f"batches {nb}  host syncs {syncs}  peak device memory {peak / 2**30:.2f} GiB  output {out.n} bytes", flush=True)
    if res[True] and res[False]:
        a, b = res[True][0][1], res[False][0][1]
        assert (a.n, a.crc) == (b.n, b.crc), "streamed and one-piece outputs differ"
        print(f"  outputs identical: {a.n} bytes, crc32 {a.crc:08x}; batch {batch_mib} MiB", flush=True)
    os.remove(path)
    os.rmdir(tmp)


print(f"device memory of the two indices: {ctx.pool_used_high(reset=True) / 2**30:.2f} GiB", flush=True)
for r in rows:
    compare(r)
