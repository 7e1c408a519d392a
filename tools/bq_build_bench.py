#!/usr/bin/env python
"""The graph build over BQ codes on the c4 world of bench.py: jv_graph_build_bq against jv_graph_build, and its maintenance
(jv_graph_add_nodes_bq, jv_graph_remove_deleted_bq) against a rebuild.

  python tools/bq_build_bench.py              # 1M x 1536 latent unit rows, their BQ words, degree 32, beam 100, hierarchy
  python tools/bq_build_bench.py --n 50000    # a smaller world for a rehearsal

Builds: jv_graph_build over the fp32 rows (DOT_PRODUCT) and jv_graph_build_bq over the words from jv_bq_encode_dataset, each timed
with CUDA events (the call's own device_ms). Footprint: the builder's HBM computed as tools/pq_build_bench.py's builder_bytes computes
it (rows or words, adjacency, per-batch scratch), not measured. Recall@10 of both graphs, under the fp32 walk and under the BQ walk with
an fp32 rerank at rerankK 100, against the fp32 brute force. Maintenance: a BQ graph over 99 % / 90 % of the rows with the rest added,
and 1 % / 10 % of the nodes removed from the full BQ graph, each against the full BQ build's time. A build, an add and a removal at
20 000 rows run first so that every kernel's module is loaded. One JSON line on stdout with the card's name and the power limit it
reports, and a table on stderr."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402
import jvector_b200 as jv  # noqa: E402
from jvector_b200 import _native as nat  # noqa: E402
from pq_build_bench import card  # noqa: E402

DIM, DEGREE, BEAM = 1536, 32, 100


def recall(nodes, truth):
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / truth.shape[1] for i in range(len(nodes))]))


def builder_bytes(n, bq):
    """pq_build_bench.builder_bytes for this world: what builder_create holds at the default max_batch (a BQ builder also holds the
    insert queries, max_batch x dim floats), the data set (fp32 rows or BQ words) and the finished level-0 adjacency"""
    hard_max = int(np.float32(1.2) * np.float32(DEGREE))
    row_cap = max(2 * DEGREE, hard_max + 1)
    mb = 16384
    builder = n * row_cap * 4 + n * (4 + 4 + 4 + 4 + 1) + mb * BEAM * 8 + mb * DEGREE * (8 + 8 + 1 + 4 + 4) + mb * 5
    if bq:
        builder += mb * DIM * 4
    data = n * 8 * ((DIM + 63) // 64) if bq else n * DIM * 4
    return {"builder": builder, "data": data, "adjacency": n * DEGREE * 4, "total": builder + data + n * DEGREE * 4}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--add", default="0.01,0.1")
    ap.add_argument("--remove", default="0.01,0.1")
    a = ap.parse_args()
    import ctypes as C

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
    words = jv.bq_encode_all(f32)
    bqv = jv.BQVectors(words, DIM)
    kw = dict(M=DEGREE, beamWidth=BEAM, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=bench.SEED)

    def build(vec):
        b = jv.GraphIndexBuilder(vsf, **kw)
        g = b.build(vec)
        return g, b.device_ms

    def walks(g):
        s = jv.GraphSearcher(g)
        return {"f32_walk": recall(s.search(f32, queries, vsf, 10, 100).nodes, truth),
                "bq_walk_f32_rerank": recall(s.search(bqv, queries, vsf, 10, 100, reranker=f32).nodes, truth)}

    # warm-up at small shapes: the build, the add and the removal (every prune capacity a removal reaches) are loaded before timing
    w = min(n, 20000)
    wbq, whalf = jv.BQVectors(words[:w], DIM), jv.BQVectors(words[:w // 2], DIM)
    wb = jv.GraphIndexBuilder(vsf, **kw)
    wg = wb.build(whalf)
    wa = wb.addGraphNodes(wg, wbq)
    wr = wb.removeDeletedNodes(wa, wbq, np.random.default_rng(1).random(w) < 0.4)
    wf = wb.build(jv.F32Vectors(queries[:min(len(queries), 500)]))
    for x in (wg, wa, wr, wf, wbq, whalf):
        x.close()

    truth, _, _ = jv.topk_bruteforce(f32, vsf, queries, 10)
    g_f32, f32_ms = build(f32)
    r_f32 = walks(g_f32)
    g_f32.close()
    g_bq, bq_ms = build(bqv)
    r_bq = walks(g_bq)
    out = {"world": {"n": n, "dim": DIM, "metric": "DOT_PRODUCT (the BQ build ignores it)", "M": DEGREE, "beam": BEAM, "hierarchy": True,
                     "nq": a.nq, "rerankK": 100},
           "card": card(),
           "build_ms": {"fp32": f32_ms, "bq": bq_ms},
           "builder_bytes": {"fp32": builder_bytes(n, False), "bq": builder_bytes(n, True)},
           "recall10": {"fp32_graph": r_f32, "bq_graph": r_bq},
           "adds": [], "removals": []}
    print(json.dumps({k: out[k] for k in ("build_ms", "builder_bytes", "recall10")}), file=sys.stderr, flush=True)
    for frac in [float(x) for x in a.add.split(",")]:
        n0 = n - int(round(frac * n))
        small = jv.BQVectors(words[:n0], DIM)
        part, part_ms = build(small)
        b = jv.GraphIndexBuilder(vsf, **kw)
        grown = b.addGraphNodes(part, bqv)
        case = {"added_fraction": frac, "n0": n0, "build_n0_ms": part_ms, "add_ms": b.device_ms, "add_over_rebuild": b.device_ms / bq_ms,
                "recall10": walks(grown)}
        out["adds"].append(case)
        print(json.dumps(case), file=sys.stderr, flush=True)
        for x in (part, grown, small):
            x.close()
    rng = np.random.default_rng(bench.SEED + 3)
    for frac in [float(x) for x in a.remove.split(",")]:
        deleted = rng.random(n) < frac
        rep = jv.GraphIndexBuilder(vsf, **kw).removeDeletedNodes(g_bq, bqv, deleted)
        st = dict(rep.remove_stats)
        case = {"deleted_fraction": frac, "repair": st, "remove_over_rebuild": st["device_ms"] / bq_ms}
        out["removals"].append(case)
        print(json.dumps(case), file=sys.stderr, flush=True)
        rep.close()
    g_bq.close()
    print("| case | device s | over the BQ build | recall@10 fp32 walk / BQ walk + rerank |", file=sys.stderr)
    print("| fp32 build | %.3f | %.3f | %.4f / %.4f |" % (f32_ms / 1e3, f32_ms / bq_ms, r_f32["f32_walk"], r_f32["bq_walk_f32_rerank"]), file=sys.stderr)
    print("| BQ build | %.3f | 1 | %.4f / %.4f |" % (bq_ms / 1e3, r_bq["f32_walk"], r_bq["bq_walk_f32_rerank"]), file=sys.stderr)
    for c in out["adds"]:
        r = c["recall10"]
        print("| add %g %% | %.3f | %.3f | %.4f / %.4f |" % (100 * c["added_fraction"], c["add_ms"] / 1e3, c["add_over_rebuild"], r["f32_walk"],
                                                          r["bq_walk_f32_rerank"]), file=sys.stderr)
    for c in out["removals"]:
        print("| remove %g %% | %.3f | %.3f | - |" % (100 * c["deleted_fraction"], c["repair"]["device_ms"] / 1e3, c["remove_over_rebuild"]), file=sys.stderr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
