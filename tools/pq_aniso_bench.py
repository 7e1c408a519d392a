"""PQ with an anisotropic threshold on the device (jv_pq_train_anisotropic, jv_pq_encode_dataset_anisotropic) on the c3 world.

1M x 768 latent unit rows (bench.gen_unit_rows_device), M = 96, k = 256, no centring, DOT, for T in {UNWEIGHTED, 0.2, 0.5}. For each T:
training device time (CUDA events) at the default cap (128 000 rows), split into the unweighted phase (the T = -1 call on the same
seed runs exactly that phase) and the anisotropic rounds; encoding of all rows with the call's device time (codebook upload and code
download included), its rows/s and kernel time (torch.profiler, a run of its own), moves and sweeps; the quantisation MSE, the mean
squared parallel error <x - x_hat, x>^2, ADC brute-force recall@10 with an fp32 rerank of the best 100 over 1000 queries, and the PQ
walk + fp32 rerank recall@10 (rerankK 100) on the c2 graph (degree 32, beam 100, hierarchy). Prints a table and one JSON line.

usage: python tools/pq_aniso_bench.py [--n 1000000] [--nq 1000]"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
import jvector_b200 as jv  # noqa: E402
from jvector_b200 import _native as nat  # noqa: E402
from pq_build_bench import card  # noqa: E402
from pq_train_bench import decode  # noqa: E402

DIM, PQ_M, K = 768, 96, 256
THRESHOLDS = (-1.0, 0.2, 0.5)


def train(lib, vec, T):
    p = nat.PQTrainParams(PQ_M, K, 0, 6, 0, bench.SEED)
    cb = np.empty(K * DIM, np.float32)
    st = nat.PQAnisotropicStats()
    nat.check(lib.jv_pq_train_anisotropic(vec._h, C.byref(p), T, nat.fp(cb), None, C.byref(st)))
    return cb, st


def encode(lib, vec, n, cb, T):
    codes = np.empty((n, PQ_M), np.uint8)
    st = nat.PQEncodeStats()
    nat.check(lib.jv_pq_encode_dataset_anisotropic(vec._h, PQ_M, K, nat.fp(cb), None, T, nat.bp(codes), C.byref(st)))
    return codes, st


def encode_kernel_ms(lib, vec, n, cb, T):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        encode(lib, vec, n, cb, T)
    return sum(ev.device_time_total for ev in prof.key_averages() if "pq_encode" in ev.key) / 1e3


def quality(torch, base, q, truth, codes, codebooks):
    rec = decode(torch, codes, codebooks)
    err = base - rec
    mse = float((err ** 2).sum(1).mean())
    par = float(((err * base).sum(1) ** 2).mean())
    cand = torch.topk(q @ rec.T, 100, dim=1).indices
    exact = torch.gather(q @ base.T, 1, cand)
    top = torch.gather(cand, 1, torch.topk(exact, 10, dim=1).indices).cpu().numpy()
    del rec, err
    return mse, par, float(np.mean([len(set(top[i]) & set(truth[i])) / 10 for i in range(len(truth))]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--nq", type=int, default=1000)
    a = ap.parse_args()
    import torch
    lib = nat.init(0)
    base = bench.gen_unit_rows_device(torch, bench.SEED, a.n, DIM)
    q = bench.gen_unit_rows_device(torch, bench.SEED + 1, a.nq, DIM)
    h = C.c_void_p()
    nat.check(lib.jv_dataset_adopt_f32_device(C.c_void_p(base.data_ptr()), a.n, DIM, DIM, C.byref(h)))
    vec = jv.api._Vectors(h, base)
    truth = torch.topk(q @ base.T, 10, dim=1).indices.cpu().numpy()
    res = {"workload": "c3 world %d x %d, PQ M=%d k=%d, no centring, DOT" % (a.n, DIM, PQ_M, K)}
    res.update(card())

    vsf = jv.VectorSimilarityFunction.DOT_PRODUCT
    g = jv.GraphIndexBuilder(vsf, M=32, beamWidth=100, addHierarchy=True, seed=bench.SEED).build(vec)
    s = jv.GraphSearcher(g)
    qh = q.cpu().numpy()
    cb0, _ = train(lib, vec, -1.0)  # warm-up: module load, allocations
    encode(lib, vec, a.n, cb0, -1.0)
    encode(lib, vec, a.n, cb0, 0.2)
    unweighted_ms = None
    rows = []
    for T in THRESHOLDS:
        cb, st = train(lib, vec, T)
        total = st.lloyd.device_ms
        if T == -1.0:
            unweighted_ms = total
        r = {"T": T, "train_ms": total, "train_unweighted_ms": unweighted_ms, "train_anisotropic_ms": total - unweighted_ms,
             "max_lloyd_updates": st.lloyd.max_lloyd_updates, "max_anisotropic_updates": st.max_anisotropic_updates,
             "anisotropic_reseeds": st.anisotropic_reseeds}
        codes, est = encode(lib, vec, a.n, cb, T)
        r.update({"encode_call_ms": est.device_ms, "encode_rows_per_s": a.n / (est.device_ms / 1e3),
                  "encode_kernel_ms": encode_kernel_ms(lib, vec, a.n, cb, T), "moves": est.moves, "rows_moved": est.rows_moved,
                  "max_sweeps": est.max_sweeps})
        mse, par, adc = quality(torch, base, q, truth, codes, cb)
        pqv = jv.PQVectors(codes, cb, DIM, K)
        sr = s.search(pqv, qh, vsf, 10, 100, reranker=vec)
        walk = float(np.mean([len(set(sr.nodes[i]) & set(truth[i])) / 10 for i in range(a.nq)]))
        pqv.close()
        r.update({"mse": mse, "parallel_sq_err": par, "adc_recall_at_10": adc, "pq_walk_fp32_rerank_recall_at_10": walk})
        rows.append(r)
    g.close()
    res["runs"] = rows
    cols = ("T", "train_ms", "train_anisotropic_ms", "encode_call_ms", "encode_kernel_ms", "encode_rows_per_s", "moves", "max_sweeps", "mse",
            "parallel_sq_err", "adc_recall_at_10", "pq_walk_fp32_rerank_recall_at_10")
    print(" | ".join(cols))
    for r in rows:
        print(" | ".join(("%.4g" % r[c]) if isinstance(r[c], float) else str(r[c]) for c in cols))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
