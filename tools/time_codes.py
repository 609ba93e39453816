"""Categorical codes timing: python tools/time_codes.py [rows]

  columns generated on the GPU: rows (default 100 M) fixed-width 12-digit decimal values with 10, 10 k, 1 M distinct
  values and all rows distinct; then values of 2-8 KiB (uniform lengths) with 1000 distinct values and all distinct, as
  many rows as fit one column below 4 GiB (700 k).  Per column: Table.values_as_codes (cpb_table_column_codes: codes
  and dictionary) and the round trip with_column(c, codes) (cpb_table_set_codes), each as wall time around the call
  (which ends in a host synchronisation) after warm-up, in rows/s and input GB/s (offsets + value bytes), with the
  per-kernel times of one call; and beside them the route a user has without codes, IndexOn(column) + dup_groups()
  (runs of equal values, no codes), timed the same way.  IndexOn refuses values longer than its 4096-byte key image."""
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


def table_of(off64: torch.Tensor, data: torch.Tensor, n: int) -> cp.Table:
    """a device table of one column "v" from int64 offsets[n+1] and uint8 bytes (copied by cpb_table_from_device)"""
    off32 = off64.contiguous().view(torch.int32)[::2].contiguous()  # the low words: uint32 offsets
    torch.cuda.synchronize(dev)
    t = cp.Table.from_device_columns(ctx, ["v"], [(off32.data_ptr(), data.data_ptr())], n)
    ctx.sync()
    return t


def decimal_column(ids: torch.Tensor) -> cp.Table:
    """row r = ids[r] as 12 zero-padded decimal digits"""
    n = ids.numel()
    p = torch.tensor([10 ** (11 - k) for k in range(12)], dtype=torch.int64, device=dev)
    data = ((ids[:, None] // p[None, :]) % 10 + 48).to(torch.uint8).reshape(-1)
    off = torch.arange(n + 1, dtype=torch.int64, device=dev) * 12
    return table_of(off, data, n)


def long_column(n: int, ndistinct: int | None, gen: torch.Generator) -> cp.Table:
    """n values of 2048..8192 bytes: ndistinct random values picked at random, or (None) every row its own bytes"""
    if ndistinct is None:
        lens = torch.randint(2048, 8193, (n,), device=dev, generator=gen)
        off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        torch.cumsum(lens, 0, out=off[1:])
        data = torch.randint(0, 256, (int(off[-1]),), dtype=torch.uint8, device=dev, generator=gen)
        return table_of(off, data, n)
    dlens = torch.randint(2048, 8193, (ndistinct,), device=dev, generator=gen)
    doff = torch.zeros(ndistinct + 1, dtype=torch.int64, device=dev)
    torch.cumsum(dlens, 0, out=doff[1:])
    dd = torch.randint(0, 256, (int(doff[-1]),), dtype=torch.uint8, device=dev, generator=gen)
    ids = torch.randint(0, ndistinct, (n,), device=dev, generator=gen)
    lens = dlens[ids]
    off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    torch.cumsum(lens, 0, out=off[1:])
    data = torch.empty(int(off[-1]), dtype=torch.uint8, device=dev)
    step = 20_000
    for a in range(0, n, step):  # gathered in pieces: the byte index of a whole column would not fit in memory
        b = min(n, a + step)
        ln = lens[a:b]
        src = torch.repeat_interleave(doff[ids[a:b]] - (off[a:b] - off[a]), ln) + torch.arange(int(ln.sum()), device=dev)
        data[int(off[a]):int(off[b])] = dd[src]
    return table_of(off, data, n)


def wall(fn, reps=REPS):
    fn()
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize(dev)
    return (time.perf_counter() - t0) / reps, out


def report(label, t):
    n = len(t)
    nbytes = 4 * (n + 1) + _col_bytes(t)
    s, cat = wall(lambda: t.values_as_codes("v"))
    print(f"{label}: {n} rows, {nbytes / 1e9:.2f} GB of input, {len(cat.dictionary)} distinct", flush=True)
    print(f"  values_as_codes      {s * 1e3:9.2f} ms  {n / s / 1e9:6.2f} G rows/s  {nbytes / s / 1e9:7.1f} GB/s", flush=True)
    ctx.stats(enable=True, reset=True)
    t.values_as_codes("v")
    st = ctx.stats(); ctx.stats(enable=False)
    print("    " + "  ".join(f"{k} {v['ms']:.2f}" for k, v in sorted(st.items(), key=lambda kv: -kv[1]["ms"])) + " (ms)", flush=True)
    s2, _ = wall(lambda: t.with_column("v", cat))
    print(f"  with_column(codes)   {s2 * 1e3:9.2f} ms  {n / s2 / 1e9:6.2f} G rows/s  {nbytes / s2 / 1e9:7.1f} GB/s", flush=True)
    del cat
    try:
        s3, (lo, _) = wall(lambda: t.index_on("v").dup_groups(), reps=1)
        print(f"  IndexOn + dup_groups {s3 * 1e3:9.2f} ms  {n / s3 / 1e9:6.2f} G rows/s  {nbytes / s3 / 1e9:7.1f} GB/s"
              f"  ({len(lo)} groups of >= 2 rows; {s3 / s:.1f}x the time of values_as_codes)", flush=True)
    except cp.CsvPlusError as e:
        print(f"  IndexOn + dup_groups: refused ({e})", flush=True)


def _col_bytes(t):
    import ctypes as C
    nb = C.c_uint64()
    t.ctx._call("cpb_table_col_bytes", t.h, 0, 0, len(t), C.byref(nb))
    return nb.value


gen = torch.Generator(device=dev)
gen.manual_seed(1)
for k in (10, 10_000, 1_000_000):
    t = decimal_column(torch.randint(0, k, (rows,), device=dev, generator=gen))
    report(f"{k} distinct, 12-byte values", t)
    del t
t = decimal_column(torch.randperm(rows, device=dev, generator=gen))
report("all distinct, 12-byte values", t)
del t
nl = min(rows, 700_000)
t = long_column(nl, 1000, gen)
report("1000 distinct, 2-8 KiB values", t)
del t
t = long_column(nl, None, gen)
report("all distinct, 2-8 KiB values", t)
