#!/usr/bin/env python
"""Summarise an .ncu-rep (raw page + SASS source page) into markdown.
usage: tools/ncu_summary.py <rep> <title> [algorithmic_bytes]   (NCU_INDEX=i picks the i-th profiled launch of the report, default 0)"""
import csv
import io
import os
import subprocess
import sys

rep, title = sys.argv[1], sys.argv[2]
algo = float(sys.argv[3]) if len(sys.argv) > 3 else None
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
IDX = int(os.environ.get("NCU_INDEX", "0"))
hdr, units, vals = rows[0], rows[1], rows[2 + IDX]
m = {h: (v, u) for h, u, v in zip(hdr, units, vals)}


def g(name):
    v = m.get(name, ("", ""))[0].replace(",", "")
    try:
        return float(v)
    except ValueError:
        return None


print("# %s\n" % title)
print("source: `%s` (ncu --set full --clock-control none --import-source on, one launch, ~39 replay passes; durations under the profiler are not bench values)\n" % rep)
print("kernel: `%s`\n" % m.get("Kernel Name", ("?",))[0])
dur = g("gpu__time_duration.sum")
unit = m.get("gpu__time_duration.sum", ("", ""))[1]
dur_ms = dur / 1e6 if unit in ("ns", "nsecond") else (dur / 1e3 if unit in ("us", "usecond") else dur)
rd, wr = g("dram__bytes_read.sum"), g("dram__bytes_write.sum")


def tobytes(name):
    v, u = m.get(name, ("0", "byte"))
    v = float(v.replace(",", ""))
    return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}.get(u, 1)


traffic = tobytes("dram__bytes_read.sum") + tobytes("dram__bytes_write.sum")
print("| metric | value |\n|---|---|")
print("| duration | %.3f ms |" % dur_ms)
print("| grid x block | %s x %s |" % (m.get("launch__grid_size", ("?",))[0], m.get("launch__block_size", ("?",))[0]))
print("| registers / thread | %s |" % m.get("launch__registers_per_thread", ("?",))[0])
print("| dynamic smem / block | %s %s |" % m.get("launch__shared_mem_per_block_dynamic", ("?", "")))
print("| occupancy limit (regs / smem / warps) blocks | %s / %s / %s |" % (m.get("launch__occupancy_limit_registers", ("?",))[0],
      m.get("launch__occupancy_limit_shared_mem", ("?",))[0], m.get("launch__occupancy_limit_warps", ("?",))[0]))
print("| warps active (%% of peak) | %s |" % m.get("sm__warps_active.avg.pct_of_peak_sustained_active", ("?",))[0])
print("| DRAM traffic (dram__bytes_read.sum + dram__bytes_write.sum) | %.3f GB (read %.3f, write %.3f) |" % (traffic / 1e9, tobytes("dram__bytes_read.sum") / 1e9, tobytes("dram__bytes_write.sum") / 1e9))
print("| DRAM throughput = traffic / duration | %.1f GB/s (%.1f%% of the measured 6579.6 GB/s copy peak) |" % (traffic / dur_ms / 1e6, 100 * traffic / dur_ms / 1e6 / 6579.6))
print("| gpu__dram_throughput %% of ncu's theoretical peak | %s |" % m.get("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", ("?",))[0])
if algo:
    print("| algorithmic bytes of this launch | %.3f GB -> %.1f GB/s, frac %.3f of measured peak; traffic / algorithmic = %.3f |" % (algo / 1e9, algo / dur_ms / 1e6, algo / dur_ms / 1e6 / 6579.6, traffic / algo))
print("| L2 sector hit rate | %s %% |" % m.get("lts__t_sector_hit_rate.pct", ("?",))[0])
print("| L1 sector hit rate | %s %% |" % m.get("l1tex__t_sector_hit_rate.pct", ("?",))[0])
print("| SM throughput %% | %s |" % m.get("sm__throughput.avg.pct_of_peak_sustained_elapsed", ("?",))[0])
print("| issue slots busy %% | %s |" % m.get("smsp__issue_active.avg.pct_of_peak_sustained_active", ("?",))[0])
print("| shared-memory bank conflicts | %s |" % m.get("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", ("?",))[0])
print("| L2 throughput %% (lts__throughput) | %s |" % m.get("lts__throughput.avg.pct_of_peak_sustained_elapsed", ("?",))[0])
print("| tensor pipe active %% (sm__pipe_tensor_cycles_active_realtime) | %s |" % m.get("TPC.TriageCompute.sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed", ("?",))[0])
print()
src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--launch-skip", str(IDX), "--launch-count", "1"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(src)))
hdr = rows[1]
ci, cs = hdr.index("Source"), hdr.index("Warp Stall Sampling (All Samples)")
names = ["stall_barrier", "stall_long_sb", "stall_short_sb", "stall_wait", "stall_lg", "stall_mio", "stall_math", "stall_branch_resolving",
         "stall_not_selected", "stall_selected", "stall_no_inst", "stall_membar", "stall_dispatch"]
idx = {n: hdr.index(n) for n in names if n in hdr}
tot, agg, st = 0.0, [], {n: 0.0 for n in idx}
for r in rows[2:]:
    if len(r) <= cs:
        continue
    try:
        v = float(r[cs])
    except ValueError:
        continue
    tot += v
    top = max(idx, key=lambda n: float(r[idx[n]] or 0))
    agg.append((v, r[ci].strip()[:80], top))
    for n in idx:
        st[n] += float(r[idx[n]] or 0)
print("warp stall sampling (%d samples): " % tot + ", ".join("%s %.1f%%" % (n.replace("stall_", ""), 100 * st[n] / tot) for n in sorted(st, key=lambda n: -st[n])[:7]))
print("\ntop SASS instructions by stall samples:\n\n| share | dominant stall | instruction |\n|---:|---|---|")
for v, s, t in sorted(agg, reverse=True)[:10]:
    print("| %.2f%% | %s | `%s` |" % (100 * v / tot, t.replace("stall_", ""), s))
mn = set()
for r in rows[2:]:
    if len(r) > ci:
        op = r[ci].strip().split(" ")[0].lstrip("@!P0123456789 ").split(".")[0]
        s_ = r[ci]
        for key in ("UBLKPF", "UBLKCP", "SYNCS", "POPC", "LDG", "ATOMG", "ATOMS", "SHFL", "UTMALDG", "CCTL"):
            if key in s_:
                mn.add(key)
print("\nSASS mnemonics present: " + ", ".join(sorted(mn)))
