#!/usr/bin/env python
"""Adding nodes to the c2 world: jv_graph_add_nodes against a fresh build of all rows.

  python tools/add_nodes_bench.py            # 1M x 768 latent rows, DOT_PRODUCT, M = 32, beam 100, with hierarchy
  python tools/add_nodes_bench.py --n 50000  # a smaller world for a rehearsal

For f = 1 %, 10 % and 50 % it builds a graph over the first (1 - f) N rows, then adds the last f N rows to it, and reports the
add's device time, its inserts per second and counters, against the device time of a fresh build of all N rows; and recall@10
at rerankK 100 over the queries, against brute force, for the added graph and for the fresh one. The data sets borrow prefixes
of one device buffer (jv_dataset_adopt_f32_device), so growing the data set copies nothing. One JSON line on stdout, with the
card's name and power limit read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from delete_repair_bench import card, recall  # noqa: E402


def adopt(jv, tensor, rows):
    """F32Vectors over the first `rows` rows of a device tensor, borrowed"""
    from jvector_b200 import _native as nat
    h = C.c_void_p()
    nat.check(nat.load().jv_dataset_adopt_f32_device(C.c_void_p(tensor.data_ptr()), rows, tensor.shape[1], tensor.shape[1], C.byref(h)))
    return jv.api._Vectors(h, tensor)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nq", type=int, default=1000)
    ap.add_argument("--fractions", default="0.01,0.1,0.5")
    a = ap.parse_args()
    import torch

    import jvector_b200 as jv
    from bench import SEED, gen_unit_rows_device
    jv.init(0)
    DOT = jv.VectorSimilarityFunction.DOT_PRODUCT
    base = gen_unit_rows_device(torch, SEED, a.n, a.dim)
    queries = gen_unit_rows_device(torch, SEED + 1, a.nq, a.dim).cpu().numpy()
    vec = adopt(jv, base, a.n)
    kw = dict(M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=SEED)
    fb = jv.GraphIndexBuilder(DOT, **kw)
    fresh = fb.build(vec)
    truth, _, _ = jv.topk_bruteforce(vec, DOT, queries, 10)
    r_fresh = recall(jv.GraphSearcher(fresh).search(vec, queries, DOT, 10, 100).nodes, truth)
    out = {"world": {"n": a.n, "dim": a.dim, "metric": "DOT_PRODUCT", "M": 32, "beam": 100, "hierarchy": True, "nq": a.nq, "rerankK": 100},
           "card": card(), "fresh": {"build_ms": fb.device_ms, "inserts_per_s": a.n / fb.device_ms * 1e3, "recall10": r_fresh},
           "cases": []}
    print(json.dumps(out["fresh"]), file=sys.stderr, flush=True)
    for frac in [float(x) for x in a.fractions.split(",")]:
        n0 = a.n - int(round(frac * a.n))
        small = adopt(jv, base, n0)
        bb = jv.GraphIndexBuilder(DOT, **kw)
        g = bb.build(small)
        ab = jv.GraphIndexBuilder(DOT, **kw)
        added = ab.addGraphNodes(g, vec)
        res = jv.GraphSearcher(added).search(vec, queries, DOT, 10, 100)
        case = {"added_fraction": frac, "n0": n0, "added": a.n - n0, "base_build_ms": bb.device_ms,
                "add": {"device_ms": ab.device_ms, "inserts_per_s": (a.n - n0) / ab.device_ms * 1e3, "batches": ab.batches,
                        "dropped_backlinks": ab.dropped_backlinks, "levels": added.info()["levels"]},
                "add_over_fresh_build": ab.device_ms / fb.device_ms,
                "recall10": {"added": recall(res.nodes, truth), "fresh": r_fresh},
                "visited_per_query": res.visitedCount / a.nq}
        out["cases"].append(case)
        print(json.dumps(case), file=sys.stderr, flush=True)
        for h in (g, added, small):
            h.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
