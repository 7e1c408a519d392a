#!/usr/bin/env python
"""Merging graph segments: jv_graph_compact against a fresh build of the live rows.

  python tools/compact_bench.py                          # 1M x 768 latent rows in 4 segments of 250k, DOT_PRODUCT, 10 % dead
  python tools/compact_bench.py --n 40000 --nq 1000      # a smaller world for a rehearsal
  python tools/compact_bench.py --pq fused               # segments with PQ of their own, FusedPQ records (jv_graph_compact_pq)
  python tools/compact_bench.py --pq sidecar             # the same codes beside the graphs instead of inside them

Every segment is built with M = 32, beam 100 and hierarchy; 10 % of each segment's nodes are dead (a fixed seed). It reports the
compaction's device time and counters, the device time of its kernels by part (graph_search_kernel: the cross-segment searches;
compact_assemble_kernel: the candidate assembly; prune_*: the prune; the rest: row gathers and scatters) from a second, profiled
call, the device time of a fresh build over the live rows, both graphs' recall@10 at rerankK 100 against brute force over the live
rows, and the ratio of compaction to rebuild time. One JSON line on stdout, with the card's name and power limit read in the same
run.

With --pq every segment also gets a PQ of its own (ProductQuantization.compute, --pq-m sub-spaces, 256 clusters), fused into its graph
for --pq fused. The compaction then retrains PQ and encodes the merged rows (and fuses the merged graph): retrain, encode and fuse are
reported beside the merge's parts, and recall is that of the c3-shaped search (the fused PQ walk with an fp32 rerank for --pq fused, a
plain PQ walk with the rerank for --pq sidecar) on the merged graph and on a fresh build with a fresh PQ of the live rows."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, limit = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:  # the numbers still stand; say why the card is unknown
        return {"name": None, "power_limit": None, "error": str(e)}


def recall(nodes, truth):
    k = truth.shape[1]
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / k for i in range(len(nodes))]))


def kernel_ms(torch, fn):
    """fn() under torch.profiler: device milliseconds of its kernels by part"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    parts = {"search": 0.0, "assembly": 0.0, "prune": 0.0, "retrain": 0.0, "encode": 0.0, "fuse": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / 1000.0
        if ev.key.startswith("cuda") or ev.key.startswith("Memcpy") or ev.key.startswith("Memset") or t == 0:
            continue
        k = ev.key
        key = ("search" if "graph_search_kernel" in k else "assembly" if "compact_assemble" in k else "prune" if "prune" in k
               else "encode" if ("pq_encode" in k or "pq_self" in k) else "fuse" if "fuse_pq" in k else "retrain" if "pq_train" in k else "other")
        parts[key] += t
    return parts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--segments", type=int, default=4)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--dead", type=float, default=0.1)
    ap.add_argument("--pq", choices=["fused", "sidecar"], default=None)
    ap.add_argument("--pq-m", type=int, default=96)
    a = ap.parse_args()
    import torch

    import jvector_b200 as jv
    from bench import SEED, gen_unit_rows_device
    jv.init(0)
    DOT = jv.VectorSimilarityFunction.DOT_PRODUCT
    host = gen_unit_rows_device(torch, SEED, a.n, a.dim).cpu().numpy()
    queries = gen_unit_rows_device(torch, SEED + 1, a.nq, a.dim).cpu().numpy()
    kw = dict(M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=SEED)
    rng = np.random.default_rng(SEED + 5)
    parts = np.array_split(np.arange(a.n), a.segments)
    sources, live, seg_ms = [], [], []
    for i, p in enumerate(parts):
        vec = jv.F32Vectors(np.ascontiguousarray(host[p]))
        b = jv.GraphIndexBuilder(DOT, **kw)
        g = b.build(vec)
        seg_ms.append(b.device_ms)
        if a.pq:
            pqv = jv.ProductQuantization.compute(vec, a.pq_m, 256, seed=SEED + i).encodeAll(vec)
            if a.pq == "fused":
                g.fuse_pq(pqv)
            sources.append((g, vec, pqv))
        else:
            sources.append((g, vec))
        live.append(rng.random(len(p)) >= a.dead)
    keep = np.concatenate([p[m] for p, m in zip(parts, live)])  # new id i = row keep[i]
    comp = jv.GraphIndexCompactor(sources, live, None, DOT)
    out_handles = comp.compact()
    merged, rows = out_handles[:2]
    codes = out_handles[2] if a.pq else None
    stats = dict(comp.stats)
    again = jv.GraphIndexCompactor(sources, live, None, DOT)
    by_part = kernel_ms(torch, lambda: [h.close() for h in again.compact()])
    sub = jv.F32Vectors(np.ascontiguousarray(host[keep]))
    fb = jv.GraphIndexBuilder(DOT, **kw)
    fresh = fb.build(sub)
    fresh_ms = fb.device_ms
    fresh_pq = None
    if a.pq:
        pq = jv.ProductQuantization.compute(sub, a.pq_m, 256, seed=SEED)
        fresh_pq = pq.encodeAll(sub)
        if a.pq == "fused":
            fresh.fuse_pq(fresh_pq)
    truth, _, _ = jv.topk_bruteforce(sub, DOT, queries, 10)
    if a.pq:
        rm = jv.GraphSearcher(merged).search(codes, queries, DOT, 10, 100, reranker=rows)
        rf = jv.GraphSearcher(fresh).search(fresh_pq, queries, DOT, 10, 100, reranker=sub)
    else:
        rm = jv.GraphSearcher(merged).search(rows, queries, DOT, 10, 100)
        rf = jv.GraphSearcher(fresh).search(sub, queries, DOT, 10, 100)
    total_ms = stats["device_ms"] + stats.get("retrain_ms", 0.0) + stats.get("encode_ms", 0.0) + stats.get("fuse_ms", 0.0)
    out = {"world": {"n": a.n, "dim": a.dim, "segments": a.segments, "metric": "DOT_PRODUCT", "M": 32, "beam": 100, "hierarchy": True,
                     "dead_fraction": a.dead, "live": int(len(keep)), "nq": a.nq, "rerankK": 100, "segment_build_ms": seg_ms,
                     "pq": a.pq, "pq_m": a.pq_m if a.pq else None},
           "card": card(),
           "compact": stats, "compact_total_ms": total_ms, "compact_kernel_ms_by_part": by_part, "fresh_build_ms": fresh_ms,
           "compact_over_fresh_build": total_ms / fresh_ms if fresh_ms else None,
           "recall10": {"compacted": recall(rm.nodes, truth), "fresh": recall(rf.nodes, truth)},
           "visited_per_query": {"compacted": rm.visitedCount / a.nq, "fresh": rf.visitedCount / a.nq}}
    print(json.dumps(out))
    for h in [merged, rows, fresh, sub] + ([codes, fresh_pq] if a.pq else []) + [x for s in sources for x in s]:
        h.close()


if __name__ == "__main__":
    main()
