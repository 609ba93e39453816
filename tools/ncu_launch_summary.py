"""Summarise an ncu launch list (--metrics gpu__time_duration.sum --csv) per kernel:
python tools/ncu_launch_summary.py launches.csv "<command line that was profiled>" > launches_summary.csv"""
import csv, re, sys, collections
rows = [r for r in csv.reader(open(sys.argv[1])) if len(r) > 14]
hdr = rows[0]
ki, mi, ui, vi = (hdr.index(x) for x in ("Kernel Name", "Metric Name", "Metric Unit", "Metric Value"))
agg = collections.OrderedDict()
for r in rows[1:]:
    if r[mi] != "gpu__time_duration.sum":
        continue
    name = re.sub(r"\(.*$", "", r[ki]).replace("void ", "").replace("cpb::", "").strip()
    scale = {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(r[ui], 1e-6)
    a = agg.setdefault(name, [0, 0.0]); a[0] += 1; a[1] += float(r[vi].replace(",", "")) * scale
tot = sum(a[1] for a in agg.values())
print(f"# ncu launch list summary — {sys.argv[2] if len(sys.argv) > 2 else ''}")
print("# per-launch times are cold-cache and serialised: compare SHARES, not absolutes")
print("kernel,launches,total_ms,share_pct,avg_us")
for k, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"{k},{a[0]},{a[1]:.3f},{100 * a[1] / tot:.1f},{1e3 * a[1] / a[0]:.1f}")
