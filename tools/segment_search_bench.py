#!/usr/bin/env python
"""Multi-segment search: S single jv_graph_search_batch_ex calls merged in numpy, against one jv_segments_search_batch.

  python tools/segment_search_bench.py                               # 1M x 768 latent rows, S in {4, 16, 64}, nq in {1, 16, 256, 10 000}
  python tools/segment_search_bench.py --n 100000 --segments 4 16    # a smaller world

The rows (bench.py's latent distribution) are split into S contiguous segments of equal size, each built alone with jv_graph_build
(DOT_PRODUCT, M = 16, beam 100, hierarchy). Per (S, nq) the two arms run alternately in the same process, --reps times each after one
warm-up call of each: the single calls (one per segment, then the stable merge on the host) and the one segment call. Each arm
reports the host wall time around its synchronised calls (median, ms) and the summed device_ms; the merged outputs of both arms must
be identical on every run. topK 10, rerankK 40, no reranker. One JSON line on stdout, with the card's name and power limit read in the
same run."""
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


def host_merge(lists, topK):
    """the stable merge of jv_segments_search_batch over per-segment (nodes, scores) [nq][topK]: score descending as the top-k key's
    sortable score, equal scores in segment order, then list order; padding (node -1) dropped, output padded with -1 / -1 / 0"""
    S = len(lists)
    nq = lists[0][0].shape[0]
    nodes = np.stack([l[0] for l in lists], 1).reshape(nq, S * topK)
    scores = np.stack([l[1] for l in lists], 1).reshape(nq, S * topK)
    b = scores.view(np.int32)
    key = (b ^ ((b >> 31) & 0x7fffffff)).astype(np.int64)
    key = np.where(nodes >= 0, key, -(1 << 40))  # below every sortable score
    order = np.argsort(-key, axis=1, kind="stable")[:, :topK]  # (segment, position) order among equal keys
    take = lambda a: np.take_along_axis(a, order, 1)
    valid = take(nodes) >= 0
    seg = np.where(valid, (order // topK).astype(np.int32), -1)
    return seg, np.where(valid, take(nodes), -1).astype(np.int32), np.where(valid, take(scores), 0).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--segments", type=int, nargs="+", default=[4, 16, 64])
    ap.add_argument("--nq", type=int, nargs="+", default=[1, 16, 256, 10000])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch

    import jvector_b200 as jv
    from bench import SEED, gen_unit_rows_device
    from jvector_b200 import _native as nat
    jv.init(0)
    lib = nat.load()
    DOT = int(jv.VectorSimilarityFunction.DOT_PRODUCT)
    topK, rerankK = 10, 40
    host = gen_unit_rows_device(torch, SEED, a.n, a.dim).cpu().numpy()
    queries = gen_unit_rows_device(torch, SEED + 1, max(a.nq), a.dim).cpu().numpy()
    out = {"card": card(), "n": a.n, "dim": a.dim, "topK": topK, "rerankK": rerankK, "reps": a.reps, "runs": []}
    for S in a.segments:
        bounds = np.linspace(0, a.n, S + 1).astype(np.int64)
        segs = []
        t0 = time.perf_counter()
        for s in range(S):
            v = jv.F32Vectors(host[bounds[s]:bounds[s + 1]])
            g = jv.GraphIndexBuilder(jv.VectorSimilarityFunction.DOT_PRODUCT, M=16, beamWidth=100, addHierarchy=True, seed=SEED + s).build(v)
            segs.append((g, v))
        build_s = time.perf_counter() - t0
        arr = (nat.SearchSegment * S)(*[nat.SearchSegment(g._h, v._h, None, None) for g, v in segs])
        for nq in a.nq:
            q = np.ascontiguousarray(queries[:nq])
            fq = q.ctypes.data_as(C.POINTER(C.c_float))

            def singles():
                lists, ms = [], 0.0
                for g, v in segs:
                    nodes = np.empty((nq, topK), np.int32)
                    scores = np.empty((nq, topK), np.float32)
                    st = nat.SearchStats()
                    rc = lib.jv_graph_search_batch_ex(g._h, v._h, None, DOT, fq, nq, topK, rerankK, None, nodes.ctypes.data_as(C.POINTER(C.c_int32)),
                                                      scores.ctypes.data_as(C.POINTER(C.c_float)), C.byref(st))
                    assert rc == 0, lib.jv_last_error()
                    lists.append((nodes, scores))
                    ms += st.device_ms
                return host_merge(lists, topK), ms

            def together():
                seg = np.empty((nq, topK), np.int32)
                nodes = np.empty((nq, topK), np.int32)
                scores = np.empty((nq, topK), np.float32)
                st = nat.SearchStats()
                rc = lib.jv_segments_search_batch(arr, S, DOT, fq, nq, topK, rerankK, 0.0, 0.0, seg.ctypes.data_as(C.POINTER(C.c_int32)),
                                                  nodes.ctypes.data_as(C.POINTER(C.c_int32)), scores.ctypes.data_as(C.POINTER(C.c_float)), C.byref(st), None)
                assert rc == 0, lib.jv_last_error()
                return (seg, nodes, scores), st.device_ms

            wall = {"singles": [], "segments": []}
            dev = {"singles": [], "segments": []}
            for rep in range(a.reps + 1):  # rep 0 warms both arms up
                for name, fn in (("singles", singles), ("segments", together)):
                    lib.jv_device_synchronize()
                    t = time.perf_counter()
                    res, ms = fn()
                    w = (time.perf_counter() - t) * 1e3
                    if name == "singles":
                        want = res
                    else:
                        assert all(np.array_equal(x, y) for x, y in zip(res[:2], want[:2])), (S, nq, "the arms disagree")
                        assert np.array_equal(res[2].view(np.int32), want[2].view(np.int32)), (S, nq, "the arms disagree on score bits")
                    if rep:
                        wall[name].append(w)
                        dev[name].append(ms)
            run = {"S": S, "nq": nq, "build_s": round(build_s, 1)}
            for name in wall:
                run[name + "_wall_ms"] = round(float(np.median(wall[name])), 3)
                run[name + "_device_ms"] = round(float(np.median(dev[name])), 3)
            run["speedup_wall"] = round(run["singles_wall_ms"] / run["segments_wall_ms"], 2)
            out["runs"].append(run)
            print(json.dumps(run), file=sys.stderr, flush=True)
        for g, v in segs:
            g.close()
            v.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
