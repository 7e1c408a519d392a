#!/usr/bin/env python
"""Turn bench.py JSON lines (the b200 arm and, optionally, the reference arm) into a markdown table.
usage: tools/bench_table.py <b200.json> [reference.json]"""
import json
import sys


def last_line(p):
    return json.loads([l for l in open(p).read().strip().splitlines() if l.startswith("{")][-1])


d = last_line(sys.argv[1])
ref = last_line(sys.argv[2]) if len(sys.argv) > 2 else None
rows = [("c2", d)] + [(k, d["configs"][k]) for k in ("c3", "c1", "c4", "c5") if k in d.get("configs", {})]
print("| config | metric | value (device-timed) | e2e (host buffers) | ms / step | roofline | cpu_baseline | parity |")
print("|---|---|---:|---:|---:|---|---|---|")
for k, c in rows:
    if "error" in c:
        print("| %s | FAILED: %s |" % (k, c["error"]))
        continue
    rf, cb, pa = c.get("roofline", {}), c.get("cpu_baseline", {}), c.get("parity", {})
    print("| %s | %s | %.4g %s | %.4g | %.3f | %s %.4g / %.4g %s = %.3f | %s | %s |" % (
        k, c["metric"], c["value"], c["unit"], c.get("e2e", {}).get("value", float("nan")), c["ms_per_step"], rf.get("bound", "?"), rf.get("achieved", 0), rf.get("peak", 0),
        rf.get("unit", ""), rf.get("frac", 0), ("%.4g %s (%s, %s threads)" % (cb["value"], cb["unit"], cb["kind"], cb["cores"])) if cb else "-", "ok" if pa.get("ok") else str(pa)[:40]))
print()
print("n_gpus %d, clocks %s" % (d["n_gpus"], json.dumps(d.get("clocks"))))
if "host_driven" in d:
    print("\nhost-driven seam: `%s`" % json.dumps(d["host_driven"]))
if ref:
    print("\nreference arm (`bench.py --impl reference`): %.4g %s, %s threads, recall@10 %s — `%s`" % (
        ref["value"], ref["unit"], ref["cpu_baseline"]["cores"], ref.get("recall_at_10"), ref["cpu_baseline"]["sample"]))
