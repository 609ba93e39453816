"""Index.WriteTo / LoadIndex timing: python tools/time_gob.py [rows]

  1. a customers index (id, name, surname; UniqueIndexOn("id")) of `rows` rows is written to a temporary file with
     WriteTo and loaded back with LoadIndex, end to end (file system included), three times each;
  2. per kernel of the encode (gob_row_len, gob_write) and of the decode (gob_cand, gob_path, gob_mark, gob_extract,
     gob_copy): ms per call and algorithmic bytes over kernel time against the H100 SXM data-sheet 3.35 TB/s;
  3. the host path they replace at min(rows, 1 M) rows: Table.rows() to Python objects + the gob encoder restated in
     tests/gob_oracle.py, and that encoder's generic decoder."""
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import csvplus_b200 as cp  # noqa: E402
from tests import gob_oracle  # noqa: E402

PEAK = 3.35e12
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
ctx = cp.Context(0)
try:
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
except OSError:
    print("nvidia-smi not available", flush=True)

cust = ctx.gen_csv("customers", (0, rows), n_cust=rows, permute=True)
t, _ = cp.parse_csv(ctx, cust, spec=[("id", -1), ("name", -1), ("surname", -1)])
ix = t.index_on("id", unique=True)
len(ix.table())  # materialise the sorted rows outside the timed region

with tempfile.TemporaryDirectory() as d:
    path = os.path.join(d, "customers.gob")
    ix.WriteTo(path)
    size = os.path.getsize(path)
    ctx.stats(enable=True, reset=True)
    w = []
    for _ in range(3):
        t0 = time.perf_counter(); ix.WriteTo(path); w.append(time.perf_counter() - t0)
    wst = ctx.stats(); ctx.stats(enable=True, reset=True)
    lt = []
    for _ in range(3):
        t0 = time.perf_counter(); ix2 = cp.LoadIndex(path, ctx); lt.append(time.perf_counter() - t0)
    lst = ctx.stats(); ctx.stats(enable=False)
    assert len(ix2) == rows and ix2.columns == ["id"]
print(f"customers index: {rows} rows, file {size} bytes", flush=True)
print(f"WriteTo end to end: {', '.join('%.1f ms' % (x * 1e3) for x in w)}  ({size / min(w) / 1e9:.2f} GB/s)", flush=True)
print(f"LoadIndex end to end: {', '.join('%.1f ms' % (x * 1e3) for x in lt)}  ({size / min(lt) / 1e9:.2f} GB/s)", flush=True)
for label, st in (("encode", wst), ("decode", lst)):
    for k, v in sorted(st.items()):
        if not k.startswith("gob_"):
            continue
        ms = v["ms"] / 3
        gb = v["algo_bytes"] / 3
        print(f"  {label} {k:12s} {ms:8.3f} ms  algo {gb / 1e9:.2f} GB -> {gb / (ms * 1e-3) / 1e9:.0f} GB/s = "
              f"{gb / (ms * 1e-3) / PEAK:.1%} of 3.35 TB/s", flush=True)

n1 = min(rows, 1_000_000)
small = ix.table().slice(0, n1)
t0 = time.perf_counter()
rs = [{k.encode("utf-8", "surrogateescape"): v.encode("utf-8", "surrogateescape") for k, v in r.items()} for r in small.rows()]
data = gob_oracle.encode_index([b"id"], rs)
host_w = time.perf_counter() - t0
t0 = time.perf_counter()
cols, back = gob_oracle.decode_index(data)
host_r = time.perf_counter() - t0
assert back == rs
print(f"host path at {n1} rows ({len(data)} bytes): rows() + encode {host_w:.2f} s ({len(data) / host_w / 1e6:.1f} MB/s), "
      f"decode {host_r:.2f} s ({len(data) / host_r / 1e6:.1f} MB/s)", flush=True)
