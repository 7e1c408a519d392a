#!/usr/bin/env python
"""Maintaining a graph over PQ codes on the c2 world of bench.py: jv_graph_add_nodes_pq and jv_graph_remove_deleted_pq against a fresh
jv_graph_build_pq.

  python tools/pq_maintain_bench.py             # 1M x 768 latent rows, DOT_PRODUCT, M = 32, beam 100, hierarchy, c3's codebooks
  python tools/pq_maintain_bench.py --n 50000   # a smaller world for a rehearsal

Adds: a PQ graph over the first 99 / 90 / 50 % of the rows, then the rest added; against the PQ build over all the rows.
Removals: 1 / 10 / 30 % of the nodes (a fixed seed) removed from that build; against a PQ build over the survivors, and against the
original graph searched with acceptOrds = live. A build, an add and a heavy removal at 20 000 rows run first, so that every kernel's
module is loaded; each timed call then runs once at full size (seconds of device work), and its time is the call's own CUDA-event time. Per case: device time, the removal's counters and
its level-0 rows per prune tier, recall@10 of the PQ walk at rerankK 100 with an fp32 rerank (the fp32 rows serve the brute-force
truth and the rerank only). One JSON line on stdout with the card's name and the power limit it reports, and a table on stderr."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402
import jvector_b200 as jv  # noqa: E402
from jvector_b200 import _native as nat  # noqa: E402
from pq_build_bench import DEGREE, BEAM, DIM, K, PQ_M, card, train_codebooks  # noqa: E402

TIERS = (64, 128, 256, 1024, 2048)  # build.cu PQ_REPAIR_TIER_MAX; anything larger runs at 8192


def recall(nodes, truth):
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / truth.shape[1] for i in range(len(nodes))]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--add", default="0.01,0.1,0.5")
    ap.add_argument("--remove", default="0.01,0.1,0.3")
    a = ap.parse_args()
    import torch
    jv.init(0)
    lib = nat.init()
    n = a.n
    vsf = jv.VectorSimilarityFunction.DOT_PRODUCT
    base_dev = bench.gen_unit_rows_device(torch, bench.SEED, n, DIM)
    queries = bench.gen_unit_rows_device(torch, bench.SEED + 1, a.nq, DIM).cpu().numpy()
    h = C.c_void_p()
    nat.check(lib.jv_dataset_adopt_f32_device(C.c_void_p(base_dev.data_ptr()), n, DIM, DIM, C.byref(h)))
    f32 = jv.api._Vectors(h, base_dev)
    cb = train_codebooks(torch, base_dev, n)
    codes = jv.pq_encode_all(f32, cb, PQ_M, K)
    pqv = jv.PQVectors(codes, cb, DIM, K)
    kw = dict(M=DEGREE, beamWidth=BEAM, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=bench.SEED)

    def build(vec):
        b = jv.GraphIndexBuilder(vsf, **kw)
        return b.build(vec), b.device_ms

    def pq_walk(g, approx, rerank, **sk):
        return jv.GraphSearcher(g).search(approx, queries, vsf, 10, 100, reranker=rerank, **sk).nodes

    # warm-up at small shapes: every kernel of the build, the add and the removal (each prune tier's module) is loaded before timing
    w = min(n, 20000)
    wpq = jv.PQVectors(codes[:w], cb, DIM, K)
    wsmall = jv.PQVectors(codes[:w // 2], cb, DIM, K)
    wb = jv.GraphIndexBuilder(vsf, **kw)
    wg = wb.build(wsmall)
    wa = wb.addGraphNodes(wg, wpq)
    wr = wb.removeDeletedNodes(wa, wpq, np.random.default_rng(1).random(w) < 0.4)
    for x in (wg, wa, wr, wpq, wsmall):
        x.close()

    truth, _, _ = jv.topk_bruteforce(f32, vsf, queries, 10)
    fresh, fresh_ms = build(pqv)
    r_fresh = recall(pq_walk(fresh, pqv, f32), truth)
    out = {"world": {"n": n, "dim": DIM, "metric": "DOT_PRODUCT", "M": DEGREE, "beam": BEAM, "hierarchy": True, "pq_M": PQ_M, "pq_k": K,
                     "nq": a.nq, "rerankK": 100, "fresh_build_pq_ms": fresh_ms, "fresh_recall10": r_fresh},
           "card": card(), "adds": [], "removals": []}
    for frac in [float(x) for x in a.add.split(",")]:
        n0 = n - int(round(frac * n))
        small = jv.PQVectors(codes[:n0], cb, DIM, K)
        part, part_ms = build(small)
        b = jv.GraphIndexBuilder(vsf, **kw)
        grown = b.addGraphNodes(part, pqv)
        case = {"added_fraction": frac, "n0": n0, "build_n0_ms": part_ms, "add_ms": b.device_ms, "batches": b.batches,
                "dropped_backlinks": b.dropped_backlinks, "add_over_fresh_build": b.device_ms / fresh_ms,
                "recall10": {"added": recall(pq_walk(grown, pqv, f32), truth), "fresh": r_fresh}}
        out["adds"].append(case)
        print(json.dumps(case), file=sys.stderr, flush=True)
        for x in (part, grown, small):
            x.close()
    adj_dev = torch.from_numpy(fresh.level(0)[1]).to("cuda").long()
    rng = np.random.default_rng(bench.SEED + 3)
    for frac in [float(x) for x in a.remove.split(",")]:
        deleted = rng.random(n) < frac
        live = np.flatnonzero(~deleted)
        rep = jv.GraphIndexBuilder(vsf, **kw).removeDeletedNodes(fresh, pqv, deleted)
        d = torch.from_numpy(deleted).to("cuda")
        hist = tier_histogram(torch, adj_dev, d)
        live_dev = torch.from_numpy(live).cuda()
        sub_rows = base_dev[live_dev]
        hs = C.c_void_p()
        nat.check(lib.jv_dataset_adopt_f32_device(C.c_void_p(sub_rows.data_ptr()), len(live), DIM, DIM, C.byref(hs)))
        sub_f32 = jv.api._Vectors(hs, sub_rows)
        sub_pq = jv.PQVectors(codes[live], cb, DIM, K)
        surv, surv_ms = build(sub_pq)
        t = live[jv.topk_bruteforce(sub_f32, vsf, queries, 10)[0]]
        case = {"deleted_fraction": frac, "repair": dict(rep.remove_stats), "level0_rows_by_tier": hist, "fresh_build_survivors_ms": surv_ms,
                "remove_over_fresh_build": rep.remove_stats["device_ms"] / surv_ms,
                "recall10": {"removed": recall(pq_walk(rep, pqv, f32), t), "original_accept_live": recall(pq_walk(fresh, pqv, f32, acceptOrds=~deleted), t),
                             "fresh": recall(live[pq_walk(surv, sub_pq, sub_f32)], t)}}
        out["removals"].append(case)
        print(json.dumps(case), file=sys.stderr, flush=True)
        for x in (rep, surv, sub_pq, sub_f32):
            x.close()
        del sub_rows
    print("| case | device s | over fresh PQ build | recall@10 maintained / fresh / original + acceptOrds |", file=sys.stderr)
    for c in out["adds"]:
        print("| add %g %% | %.3f | %.3f | %.4f / %.4f / - |" % (100 * c["added_fraction"], c["add_ms"] / 1e3, c["add_over_fresh_build"],
                                                             c["recall10"]["added"], c["recall10"]["fresh"]), file=sys.stderr)
    for c in out["removals"]:
        r = c["recall10"]
        print("| remove %g %% | %.3f | %.3f | %.4f / %.4f / %.4f |" % (100 * c["deleted_fraction"], c["repair"]["device_ms"] / 1e3, c["remove_over_fresh_build"],
                                                                   r["removed"], r["fresh"], r["original_accept_live"]), file=sys.stderr)
    print(json.dumps(out))


def tier_histogram(torch, adj, dead, chunk=65536):
    """level 0: distinct candidates per repaired row (live neighbours + live 2-hop ids through deleted neighbours) by PQ prune tier, as
    delete_repair_bench counts them for the fp32 tiers; rows that take the random fallback are counted apart"""
    n, deg = adj.shape
    hist = [0] * (len(TIERS) + 1)
    fallback = 0
    edges = torch.tensor(TIERS, device=adj.device)
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
        two = adj[ac]
        keep = nd[:, :, None] & (two >= 0) & (two != v[:, :, None]) & ~dead[two.clamp(min=0)]
        two = torch.where(keep, two, -1).reshape(two.shape[0], -1)
        fb = (two < 0).all(1)
        fallback += int(fb.sum())
        allc = torch.cat([live, two], 1).sort(1).values
        distinct = ((allc[:, 1:] != allc[:, :-1]) & (allc[:, 1:] >= 0)).sum(1) + (allc[:, 0] >= 0).long()
        for t, c in enumerate(torch.bincount(torch.bucketize(distinct[~fb], edges, right=False), minlength=len(TIERS) + 1).tolist()):
            hist[t] += c
    names = ["le%d" % t for t in TIERS] + ["gt%d" % TIERS[-1]]
    return dict(zip(names, hist), random_fallback=fallback)


if __name__ == "__main__":
    main()
