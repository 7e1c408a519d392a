#!/usr/bin/env python
"""Deleting nodes from the c2 world: jv_graph_remove_deleted against a fresh build of the survivors.

  python tools/delete_repair_bench.py            # 1M x 768 latent rows, DOT_PRODUCT, M = 32, beam 100, with hierarchy
  python tools/delete_repair_bench.py --n 50000  # a smaller world for a rehearsal

For 1 %, 10 % and 30 % of the nodes deleted (a fixed seed) it reports the counters and device time of the repair, how many level-0
rows each prune tier takes (distinct candidates per row: <= 64, <= 128 tensor-core Gram kernels; <= 256, <= 1024, more: the
incremental kernel at growing capacity), the device time of a fresh build over the survivors' rows, and recall@10 / visited per
query at rerankK 100, against brute force over the survivors, for (a) the original graph searched with acceptOrds = live, (b) the
repaired graph, (c) the fresh build. One JSON line on stdout, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TIERS = (64, 128, 256, 1024)


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, limit = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:  # the numbers still stand; say why the card is unknown
        return {"name": None, "power_limit": None, "error": str(e)}


def tier_histogram(torch, adj, dead, chunk=65536):
    """level 0: distinct candidates per repaired row (live neighbours + live 2-hop ids through deleted neighbours), by prune tier;
    rows whose deleted neighbours offer nothing (random fallback) are counted apart"""
    n, deg = adj.shape
    hist = [0] * (len(TIERS) + 1)
    fallback = 0
    for lo in range(0, n, chunk):
        a = adj[lo:lo + chunk]
        v = torch.arange(lo, lo + a.shape[0], device=adj.device)[:, None]
        ok = a >= 0
        ac = a.clamp(min=0)
        nd = ok & dead[ac]
        rows = nd.any(1) & ~dead[v[:, 0]]
        if not rows.any():
            continue
        a, ac, ok, nd, v = a[rows], ac[rows], ok[rows], nd[rows], v[rows]
        live = torch.where(ok & ~nd, a, -1)
        two = adj[ac]                                     # [r][deg][deg]
        keep = nd[:, :, None] & (two >= 0) & (two != v[:, :, None]) & ~dead[two.clamp(min=0)]
        two = torch.where(keep, two, -1).reshape(two.shape[0], -1)
        fb = (two < 0).all(1)
        fallback += int(fb.sum())
        allc = torch.cat([live, two], 1).sort(1).values
        distinct = ((allc[:, 1:] != allc[:, :-1]) & (allc[:, 1:] >= 0)).sum(1) + (allc[:, 0] >= 0).long()
        distinct = distinct[~fb]
        edges = torch.tensor(TIERS, device=adj.device)
        idx = torch.bucketize(distinct, edges, right=False)
        for t, c in enumerate(torch.bincount(idx, minlength=len(TIERS) + 1).tolist()):
            hist[t] += c
    return {"le64": hist[0], "le128": hist[1], "le256": hist[2], "le1024": hist[3], "gt1024": hist[4], "random_fallback": fallback}


def recall(nodes, truth):
    k = truth.shape[1]
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / k for i in range(len(nodes))]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--fractions", default="0.01,0.1,0.3")
    a = ap.parse_args()
    import torch

    import jvector_b200 as jv
    from bench import SEED, gen_unit_rows_device
    jv.init(0)
    DOT = jv.VectorSimilarityFunction.DOT_PRODUCT
    base = gen_unit_rows_device(torch, SEED, a.n, a.dim)
    queries = gen_unit_rows_device(torch, SEED + 1, a.nq, a.dim).cpu().numpy()
    host = base.cpu().numpy()
    vec = jv.F32Vectors(host)
    kw = dict(M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=SEED)
    builder = jv.GraphIndexBuilder(DOT, **kw)
    gi = builder.build(vec)
    out = {"world": {"n": a.n, "dim": a.dim, "metric": "DOT_PRODUCT", "M": 32, "beam": 100, "hierarchy": True, "nq": a.nq,
                     "rerankK": 100, "build_ms": builder.device_ms},
           "card": card(), "cases": []}
    _, adj0 = gi.level(0)
    adj_dev = torch.from_numpy(adj0).to("cuda").long()
    rng = np.random.default_rng(SEED + 3)
    for frac in [float(x) for x in a.fractions.split(",")]:
        deleted = rng.random(a.n) < frac
        live = np.flatnonzero(~deleted)
        rep = jv.GraphIndexBuilder(DOT, **kw).removeDeletedNodes(gi, vec, deleted)
        hist = tier_histogram(torch, adj_dev, torch.from_numpy(deleted).to("cuda"))
        sub = jv.F32Vectors(host[live])
        fb = jv.GraphIndexBuilder(DOT, **kw)
        fresh = fb.build(sub)
        truth_local, _, _ = jv.topk_bruteforce(sub, DOT, queries, 10)
        truth = live[truth_local]
        ra = jv.GraphSearcher(gi).search(vec, queries, DOT, 10, 100, acceptOrds=~deleted)
        rb = jv.GraphSearcher(rep).search(vec, queries, DOT, 10, 100)
        rc = jv.GraphSearcher(fresh).search(sub, queries, DOT, 10, 100)
        case = {"deleted_fraction": frac, "repair": dict(rep.remove_stats), "level0_rows_by_tier": hist, "fresh_build_ms": fb.device_ms,
                "recall10": {"original_accept_live": recall(ra.nodes, truth), "repaired": recall(rb.nodes, truth), "fresh": recall(live[rc.nodes], truth)},
                "visited_per_query": {"original_accept_live": ra.visitedCount / a.nq, "repaired": rb.visitedCount / a.nq, "fresh": rc.visitedCount / a.nq}}
        case["repair_over_fresh_build"] = case["repair"]["device_ms"] / fb.device_ms if fb.device_ms else None
        out["cases"].append(case)
        print(json.dumps(case), file=sys.stderr, flush=True)
        for h in (rep, fresh, sub):
            h.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
