#!/usr/bin/env python
"""The refine pass (jv_graph_refine) on the two worlds it serves.

  python tools/refine_bench.py                              # both workloads at full size
  python tools/refine_bench.py --n 40000 --nq 1000          # a smaller world for a rehearsal
  python tools/refine_bench.py --workload build             # one of them

build   : an n x dim latent-row build, DOT_PRODUCT, M = 32, beam 100, with hierarchy; then GraphIndexBuilder.refine (the builder form).
          Reports the build's and the refine's device time, the refine's counters, and recall@10 at rerankK 100 on nq queries against
          brute force, before and after.
compact : the same rows in `segments` segments, each built as above, 10 % of each segment's nodes dead (a fixed seed); the compaction,
          then the compactor's refine pass (refineAfterCompaction). Reports both device times and the recall of the merged graph before
          and after the refine.
One JSON line on stdout, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from compact_bench import card, recall  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--segments", type=int, default=4)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--dead", type=float, default=0.1)
    ap.add_argument("--workload", default="all", choices=["all", "build", "compact"])
    a = ap.parse_args()
    import torch

    import jvector_b200 as jv
    from bench import SEED, gen_unit_rows_device
    jv.init(0)
    DOT = jv.VectorSimilarityFunction.DOT_PRODUCT
    host = gen_unit_rows_device(torch, SEED, a.n, a.dim).cpu().numpy()
    queries = gen_unit_rows_device(torch, SEED + 1, a.nq, a.dim).cpu().numpy()
    kw = dict(M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=SEED)
    out = {"world": {"n": a.n, "dim": a.dim, "metric": "DOT_PRODUCT", "M": 32, "beam": 100, "hierarchy": True, "nq": a.nq, "topK": 10, "rerankK": 100},
           "card": card()}
    if a.workload in ("all", "build"):
        vec = jv.F32Vectors(host)
        b = jv.GraphIndexBuilder(DOT, **kw)
        g = b.build(vec)
        build_ms = b.device_ms
        r = b.refine(g, vec)
        truth, _, _ = jv.topk_bruteforce(vec, DOT, queries, 10)
        before = recall(jv.GraphSearcher(g).search(vec, queries, DOT, 10, 100).nodes, truth)
        after = recall(jv.GraphSearcher(r).search(vec, queries, DOT, 10, 100).nodes, truth)
        out["build"] = {"build_ms": build_ms, "refine": r.refine_stats, "refine_over_build": r.refine_stats["device_ms"] / build_ms,
                        "recall10": {"built": before, "refined": after}}
        for h in (g, r, vec):
            h.close()
    if a.workload in ("all", "compact"):
        rng = np.random.default_rng(SEED + 5)
        parts = np.array_split(np.arange(a.n), a.segments)
        sources, live = [], []
        for p in parts:
            vec = jv.F32Vectors(np.ascontiguousarray(host[p]))
            sources.append((jv.GraphIndexBuilder(DOT, **kw).build(vec), vec))
            live.append(rng.random(len(p)) >= a.dead)
        keep = np.concatenate([p[m] for p, m in zip(parts, live)])
        plain = jv.GraphIndexCompactor(sources, live, None, DOT)
        merged, rows = plain.compact()
        comp = jv.GraphIndexCompactor(sources, live, None, DOT, refineAfterCompaction=True)
        refined, rows2 = comp.compact()
        sub = jv.F32Vectors(np.ascontiguousarray(host[keep]))
        truth, _, _ = jv.topk_bruteforce(sub, DOT, queries, 10)
        out["compact"] = {"segments": a.segments, "dead_fraction": a.dead, "live": int(len(keep)), "compact_ms": plain.stats["device_ms"],
                          "refine": comp.refine_stats, "refine_over_compact": comp.refine_stats["device_ms"] / plain.stats["device_ms"],
                          "recall10": {"compacted": recall(jv.GraphSearcher(merged).search(rows, queries, DOT, 10, 100).nodes, truth),
                                       "refined": recall(jv.GraphSearcher(refined).search(rows2, queries, DOT, 10, 100).nodes, truth)}}
        for h in [merged, rows, refined, rows2, sub] + [x for s in sources for x in s]:
            h.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
