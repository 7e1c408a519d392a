#!/usr/bin/env python
"""Filtered search: jv_exhaustive_search_batch (every accepted row scored) against the graph walk with the same filter.

  python tools/filtered_bench.py                         # 1M x 768 latent rows (the c2 world), fp32 / PQ (M = 96) / BQ, 10 000 queries
  python tools/filtered_bench.py --n 40000 --nq 500      # a smaller world for a rehearsal
  python tools/filtered_bench.py --no-graph              # skip the graph build and the walk

Filters: a random acceptOrds at 10 %, 1 % and 0.1 % density, shared by the batch and one per query. For each storage kind and filter
it reports the exhaustive search's queries/s and device time (topK 10, rerankK 100; PQ and BQ rerank against the fp32 rows, DOT_PRODUCT
for fp32 and PQ, the BQ score for BQ), its recall@10 against a numpy DOT_PRODUCT top-10 over the accepted rows (shared filters, the
first 200 queries), and,
where the walk over an M = 32 beam 100 graph succeeds with the same filter, the walk's device time and recall; and the wall time of
the unfiltered jv_topk_bruteforce at k = rerankK on each kind. One JSON line on stdout,
with the card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, limit = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:
        return {"name": None, "power_limit": None, "error": str(e)}


def random_bits(rng, rows, n, density):
    """[rows][ceil(n / 32)] accept words, each bit set with probability `density` (packed a block of rows at a time)"""
    words = (n + 31) // 32
    out = np.empty((rows, words), np.uint32)
    for r0 in range(0, rows, 256):
        r1 = min(rows, r0 + 256)
        m = rng.random((r1 - r0, words * 32), dtype=np.float32) < density
        m[:, n:] = False
        out[r0:r1] = np.packbits(m, axis=1, bitorder="little").view(np.uint32)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nq", type=int, default=10000)
    ap.add_argument("--pq-m", type=int, default=96)
    ap.add_argument("--no-graph", action="store_true")
    a = ap.parse_args()
    import torch

    import jvector_b200 as jv
    from bench import SEED, gen_unit_rows_device
    from jvector_b200 import _native as nat
    jv.init(0)
    lib = nat.load()
    DOT, COS = int(jv.VectorSimilarityFunction.DOT_PRODUCT), int(jv.VectorSimilarityFunction.COSINE)
    host = gen_unit_rows_device(torch, SEED, a.n, a.dim).cpu().numpy()
    queries = gen_unit_rows_device(torch, SEED + 1, a.nq, a.dim).cpu().numpy()
    f32 = jv.F32Vectors(host)
    pq = jv.ProductQuantization.compute(f32, a.pq_m, 256, seed=SEED).encodeAll(f32)
    bq = jv.BQVectors(jv.bq_encode_all(host), a.dim)
    kinds = {"f32": (f32, None, DOT), "pq": (pq, f32, DOT), "bq": (bq, f32, COS)}
    graph = None
    if not a.no_graph:
        b = jv.GraphIndexBuilder(jv.VectorSimilarityFunction.DOT_PRODUCT, M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=SEED)
        graph = b.build(f32)
    rng = np.random.default_rng(SEED + 11)
    topK, rerankK = 10, 100

    def run(fn, approx, rr, metric, opts, nodes, scores):
        st = nat.SearchStats()
        t0 = time.perf_counter()
        rc = fn(approx._h, rr._h if rr is not None else None, metric, nat.fp(queries), a.nq, topK, rerankK, C.byref(opts), nat.ip(nodes), nat.fp(scores), C.byref(st))
        wall = time.perf_counter() - t0
        return rc, st, wall

    def exhaustive(*args):
        return lib.jv_exhaustive_search_batch(*args)

    def walk(approx, rr, *rest):
        return lib.jv_graph_search_batch_ex(graph._h, approx, rr, *rest)

    unfiltered = {}
    for kind, (approx, _, metric) in kinds.items():  # the unfiltered brute force at k = rerankK, the cost the filters scale
        jv.topk_bruteforce(approx, metric, queries, rerankK)
        t0 = time.perf_counter()
        jv.topk_bruteforce(approx, metric, queries, rerankK)
        unfiltered[kind] = {"wall_s": time.perf_counter() - t0}
    results = []
    for density in (0.1, 0.01, 0.001):
        for form in ("shared", "per_query"):
            bits = random_bits(rng, 1 if form == "shared" else a.nq, a.n, density)
            if form == "shared":
                bits = bits[0]
            opts = nat.SearchOptions(bits.ctypes.data, 0 if form == "shared" else bits.shape[1], 0.0, 0.0)
            acc = np.unpackbits(bits.view(np.uint8), bitorder="little")[:a.n].astype(bool) if form == "shared" else None
            truth = None
            if form == "shared":  # numpy ground truth over the accepted rows, a sample of the queries
                ids = np.flatnonzero(acc)
                s = queries[:200] @ host[ids].T
                truth = ids[np.argsort(-s, axis=1, kind="stable")[:, :topK]]
            for kind, (approx, rr, metric) in kinds.items():
                nodes = np.empty((a.nq, topK), np.int32)
                scores = np.empty((a.nq, topK), np.float32)
                run(exhaustive, approx, rr, metric, opts, nodes, scores)  # warm-up: scratch, module load
                rc, st, wall = run(exhaustive, approx, rr, metric, opts, nodes, scores)
                row = {"density": density, "filter": form, "kind": kind, "exhaustive": {"rc": rc, "device_ms": st.device_ms, "wall_s": wall,
                                                                                         "qps": a.nq / wall if rc == 0 else None,
                                                                                         "visited_per_query": st.visited / a.nq}}
                if truth is not None and rc == 0:
                    row["exhaustive"]["recall10"] = float(np.mean([len(set(nodes[i]) & set(truth[i])) / topK for i in range(len(truth))]))
                if graph is not None and kind != "bq":
                    gn = np.empty((a.nq, topK), np.int32)
                    gs = np.empty((a.nq, topK), np.float32)
                    grc, gst, gwall = run(walk, approx, rr, metric, opts, gn, gs)
                    g = {"rc": grc, "error": lib.jv_last_error().decode() if grc else None}
                    if grc == 0:
                        grc, gst, gwall = run(walk, approx, rr, metric, opts, gn, gs)
                        g.update({"device_ms": gst.device_ms, "wall_s": gwall, "qps": a.nq / gwall, "visited_per_query": gst.visited / a.nq})
                        if truth is not None:
                            g["recall10"] = float(np.mean([len(set(gn[i]) & set(truth[i])) / topK for i in range(len(truth))]))
                    row["graph"] = g
                results.append(row)
                print(json.dumps(row), file=sys.stderr, flush=True)
    print(json.dumps({"world": {"n": a.n, "dim": a.dim, "nq": a.nq, "topK": topK, "rerankK": rerankK, "pq_m": a.pq_m, "graph": graph is not None},
                      "card": card(), "unfiltered_topk": unfiltered, "results": results}))


if __name__ == "__main__":
    main()
