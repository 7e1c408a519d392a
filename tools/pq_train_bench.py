"""PQ training on the device (jv_pq_train) against bench.py c3's numpy recipe, on the c3 world.

1M x 768 latent unit rows (bench.gen_unit_rows_device), M = 96, k = 256, no centring. Device training at the default cap (128 000
rows): device time (CUDA events), split into sampling, seeding and Lloyd by a torch.profiler run of its own (kernel time summed by
name). For the device codebooks and for c3's (train_pq_numpy on 20 000 sampled rows, 6 iterations, with its CPU wall time): the
quantisation MSE over all rows, ADC brute-force recall@10 with an fp32 rerank of the best 100 over 1000 queries, and the PQ walk +
fp32 rerank recall@10 (rerankK 100) on the c2 graph (degree 32, beam 100, hierarchy). Prints one JSON line.

usage: python tools/pq_train_bench.py [--n 1000000] [--nq 1000]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
import jvector_b200 as jv  # noqa: E402
import oracle_lib as o  # noqa: E402
from jvector_b200 import _native as nat  # noqa: E402
from pq_build_bench import card, train_codebooks  # noqa: E402

DIM, PQ_M, K = 768, 96, 256
PHASES = {"sampling": ("gather", "colsum", "mean"), "seeding": ("seed_kernel", "seed_finish"), "lloyd": ("assign", "update", "finalize")}


def decode(torch, codes, codebooks):
    """reconstructed rows [n][DIM] on the device"""
    sizes, offsets = o.pq_layout(DIM, PQ_M)
    cb = torch.from_numpy(codebooks).cuda()
    codes = torch.from_numpy(codes.astype(np.int64)).cuda()
    out = torch.empty((codes.shape[0], DIM), device="cuda")
    for m in range(PQ_M):
        book = cb[K * offsets[m]:K * (offsets[m] + sizes[m])].view(K, int(sizes[m]))
        out[:, offsets[m]:offsets[m] + sizes[m]] = book[codes[:, m]]
    return out


def quality(torch, base, q, truth, codes, codebooks):
    rec = decode(torch, codes, codebooks)
    mse = float(((base - rec) ** 2).sum(1).mean())
    cand = torch.topk(q @ rec.T, 100, dim=1).indices
    exact = torch.gather(q @ base.T, 1, cand)
    top = torch.gather(cand, 1, torch.topk(exact, 10, dim=1).indices).cpu().numpy()
    del rec
    return mse, float(np.mean([len(set(top[i]) & set(truth[i])) / 10 for i in range(len(truth))]))


def device_train(lib, vec):
    p = nat.PQTrainParams(PQ_M, K, 0, 6, 0, bench.SEED)
    cb = np.empty(K * DIM, np.float32)
    st = nat.PQTrainStats()
    nat.check(lib.jv_pq_train(vec._h, C.byref(p), nat.fp(cb), None, C.byref(st)))
    return cb, {name: getattr(st, name) for name, _ in nat.PQTrainStats._fields_}


def phases(torch, lib, vec):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        device_train(lib, vec)
    out = {k: 0.0 for k in PHASES}
    for ev in prof.key_averages():
        if "pq_train" not in ev.key:
            continue
        for phase, keys in PHASES.items():
            if any(("pq_train_" + k) in ev.key for k in keys):
                out[phase] += ev.device_time_total / 1e3
    return {k + "_ms": v for k, v in out.items()}


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
    res = {"workload": "c3 world %d x %d, PQ M=%d k=%d, no centring" % (a.n, DIM, PQ_M, K)}
    res.update(card())

    device_train(lib, vec)  # warm-up: module load, allocations
    cb_dev, st = device_train(lib, vec)
    res["device"] = {"train_rows": st["train_rows"], "device_ms": st["device_ms"], "max_lloyd_updates": st["max_lloyd_updates"],
                     "empty_reseeds": st["empty_reseeds"], "seeding_fallbacks": st["seeding_fallbacks"]}
    res["device"].update(phases(torch, lib, vec))
    t0 = time.time()
    cb_np = train_codebooks(torch, base, a.n)
    res["numpy"] = {"train_rows": min(a.n, 20000), "cpu_wall_s": time.time() - t0}

    vsf = jv.VectorSimilarityFunction.DOT_PRODUCT
    g = jv.GraphIndexBuilder(vsf, M=32, beamWidth=100, addHierarchy=True, seed=bench.SEED).build(vec)
    s = jv.GraphSearcher(g)
    qh = q.cpu().numpy()
    for name, cb in (("device", cb_dev), ("numpy", cb_np)):
        codes = jv.pq_encode_all(vec, cb, PQ_M, K)
        mse, adc = quality(torch, base, q, truth, codes, cb)
        pqv = jv.PQVectors(codes, cb, DIM, K)
        r = s.search(pqv, qh, vsf, 10, 100, reranker=vec)
        walk = float(np.mean([len(set(r.nodes[i]) & set(truth[i])) / 10 for i in range(a.nq)]))
        res[name].update({"mse": mse, "adc_recall_at_10": adc, "pq_walk_fp32_rerank_recall_at_10": walk})
        pqv.close()
    g.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
