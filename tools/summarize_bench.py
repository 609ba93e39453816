"""Markdown summary of bench.py JSON lines: python tools/summarize_bench.py bench_n1.json [more.json ...]"""
import json
import sys


def load(path):
    lines = [l for l in open(path) if l.startswith("{")]
    return json.loads(lines[-1])


for path in sys.argv[1:]:
    d = load(path)
    print(f"### `{path}` — N = {d['n_gpus']}, steps {d['steps']}, warm-up {d['warmup']}, clocks {d['clocks']['sm_mhz'] if d.get('clocks') else '?'} MHz "
          f"(throttle reasons: {d['clocks']['reasons'] if d.get('clocks') else '?'})\n")
    print("| quantity | value |\n|---|---|")
    print(f"| three-way join, CSV resident in HBM (`value`) | {d['ms_per_step']:.1f} ms/step = {d['value'] / 1e9:.2f} G probe rows/s |")
    if d.get("e2e"):
        e = d["e2e"]
        print(f"| same from pinned host CSV to CSV text in pinned host memory (`e2e`) | {e['ms_per_step']:.0f} ms/step = {e['value'] / 1e9:.3f} G rows/s; "
              f"H2D {e['h2d_bytes_per_step'] / 1e9:.2f} GB + D2H {e['d2h_bytes_per_step'] / 1e9:.2f} GB per step |")
    r = d.get("roofline")
    if r:
        print(f"| `csv_scan` in the join step (roofline) | {r['achieved']:.0f} GB/s algorithmic = {r['frac']:.3f} of {r['peak']:.0f} GB/s ({r['peak_kind']}); "
              f"{r['ms_per_launch']:.2f} ms/launch |")
    p = d.get("csv_parse")
    if p:
        print(f"| configs[1] parse + select 3 + `Like` | {p['value']:.0f} GB/s of input, {p['ms_per_step']:.2f} ms/step; roofline frac {p['roofline']['frac']:.3f} |")
    ix = d.get("index_on")
    if ix:
        print(f"| configs[4] `IndexOn(cust_id,prod_id)` + sorted rows, 10 M rows | {ix['ms_per_step']:.2f} ms = {ix['value'] / 1e9:.2f} G rows/s; roofline frac {ix['roofline']['frac']:.3f} |")
        for s in ix.get("resolve_duplicates", []):
            m = s["ms"]
            print(f"| `ResolveDuplicates`, last sorted row {'in a group' if s['last_row_in_group'] else 'a singleton'} | {s['rows']} → {s['rows_after']} rows, {s['groups']} groups; "
                  f"dup_groups {m['dup_groups']:.1f} ms, host resolver {m['resolver_host_callback']:.0f} ms, dedup_apply {m['dedup_apply']:.1f} ms |")
    c = d.get("cpu_baseline")
    if c:
        print(f"| CPU port of the reference, {c['cores']} thread ({c['sample']}) | {c['value'] / 1e3:.0f} k rows/s; parse {c['csv_parse']['value']:.3f} GB/s; "
              f"IndexOn {c['index_on']['value'] / 1e3:.0f} k rows/s |")
    print(f"| host gap / blocking host waits per step | {d.get('host_gap_ms_per_step', 0):.2f} ms / {d.get('host_syncs_per_step', '?')} |")
    ks = sorted(d["kernels"].items(), key=lambda kv: -kv[1]["ms"])
    print("| kernels per step (ms) | " + ", ".join(f"{k} {v['ms'] / d['steps']:.2f}" for k, v in ks if v["ms"] > 0) + " |")
    print()
