"""The graph build over PQ codes (jv_graph_build_pq) against the fp32 build, on the c2 world of bench.py.

Default: 1M x 768 latent unit rows (bench.gen_unit_rows_device), DOT_PRODUCT, M = 32, beam 100, hierarchy, c3's codebooks
(M = 96, k = 256, trained on 20 000 sampled rows). Both graphs are built, timed with CUDA events (the PQ build's time includes its
centroid-pair table), and searched with the fp32 walk and with the PQ walk + fp32 rerank at rerankK 100. Prints one JSON line.

--n N: the PQ build alone at N rows, for sizes whose fp32 rows would not fit in HBM: the rows are generated on the device and encoded
chunk by chunk, only the codes are kept; time and footprint only.

usage: python tools/pq_build_bench.py [--n N] [--nq 1000]"""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import jvector_b200 as jv  # noqa: E402
import oracle_lib as o  # noqa: E402
from jvector_b200 import _native as nat  # noqa: E402

DIM, PQ_M, K = 768, 96, 256
DEGREE, BEAM = 32, 100


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        name, limit = [x.strip() for x in q.stdout.strip().split(",")[:2]]
        return {"card": name, "power_limit": limit}
    except Exception:
        return {"card": None, "power_limit": None}


def builder_bytes(n, dim, pq):
    """HBM the builder itself holds (build.cu builder_create at the default max_batch), plus what the build needs of the data set
    (fp32 rows, or codes + the centroid-pair table) and the finished level-0 adjacency"""
    hard_max = int(np.float32(1.2) * np.float32(DEGREE))
    row_cap = max(2 * DEGREE, hard_max + 1)
    mb = 16384
    builder = n * row_cap * 4 + n * (4 + 4 + 4 + 4 + 1) + mb * BEAM * 8 + mb * DEGREE * (8 + 8 + 1 + 4 + 4) + mb * 5
    if pq:
        builder += mb * dim * 4
        data = n * ((PQ_M + 3) & ~3) + PQ_M * (K * (K + 1) // 2) * 4
    else:
        data = n * dim * 4
    return {"builder": builder, "data": data, "adjacency": n * DEGREE * 4, "total": builder + data + n * DEGREE * 4}


def train_codebooks(torch, base_dev, n):
    rs = np.random.default_rng(bench.SEED + 99)  # c3's codebooks
    sel = np.sort(rs.choice(n, min(n, 20000), replace=False))
    sample = base_dev[torch.from_numpy(sel).cuda()].cpu().numpy()
    cb, _, _ = o.train_pq_numpy(rs, sample, PQ_M, K, iters=6)
    return cb


def recall(res, truth):
    return float(np.mean([len(set(res.nodes[i]) & set(truth[i])) / 10 for i in range(len(truth))]))


def compare(torch, n, nq):
    base_dev = bench.gen_unit_rows_device(torch, bench.SEED, n, DIM)
    q = bench.gen_unit_rows_device(torch, bench.SEED + 1, nq, DIM).cpu().numpy()
    lib = nat.init()
    h = C.c_void_p()
    nat.check(lib.jv_dataset_adopt_f32_device(C.c_void_p(base_dev.data_ptr()), n, DIM, DIM, C.byref(h)))
    f32 = jv.api._Vectors(h, base_dev)
    cb = train_codebooks(torch, base_dev, n)
    pqv = jv.PQVectors(jv.pq_encode_all(f32, cb, PQ_M, K), cb, DIM, K)
    vsf = jv.VectorSimilarityFunction.DOT_PRODUCT
    truth, _, _ = jv.topk_bruteforce(f32, vsf, q, 10)
    out = {}
    for name, vec in (("fp32", f32), ("pq", pqv)):
        b = jv.GraphIndexBuilder(vsf, M=DEGREE, beamWidth=BEAM, addHierarchy=True, seed=bench.SEED)
        g = b.build(vec)
        s = jv.GraphSearcher(g)
        out[name] = {"device_s": b.device_ms / 1e3, "inserts_per_s": n / (b.device_ms / 1e3), "batches": b.batches,
                     "dropped_backlinks": b.dropped_backlinks, "hbm_bytes": builder_bytes(n, DIM, name == "pq"),
                     "recall_at_10": {"fp32_walk": recall(s.search(f32, q, vsf, 10, 100), truth),
                                      "pq_walk_fp32_rerank": recall(s.search(pqv, q, vsf, 10, 100, reranker=f32), truth)}}
        g.close()
    pqv.close()
    return out


def pq_only(torch, n, chunk=1 << 20):
    """the PQ build at n rows: rows generated and encoded chunk by chunk on the device, only the codes kept"""
    lib = nat.init()
    first = bench.gen_unit_rows_device(torch, bench.SEED, min(n, chunk), DIM)
    cb = train_codebooks(torch, first, first.shape[0])
    codes = np.empty((n, PQ_M), np.uint8)
    for i in range(0, n, chunk):
        j = min(n, i + chunk)
        rows = first if i == 0 else bench.gen_unit_rows_device(torch, bench.SEED + i // chunk, j - i, DIM)
        h = C.c_void_p()
        nat.check(lib.jv_dataset_adopt_f32_device(C.c_void_p(rows.data_ptr()), j - i, DIM, DIM, C.byref(h)))
        v = jv.api._Vectors(h, rows)
        codes[i:j] = jv.pq_encode_all(v, cb, PQ_M, K)
        v.close()
        del rows
    del first
    torch.cuda.empty_cache()
    pqv = jv.PQVectors(codes, cb, DIM, K)
    del codes
    b = jv.GraphIndexBuilder(jv.VectorSimilarityFunction.DOT_PRODUCT, M=DEGREE, beamWidth=BEAM, addHierarchy=True, seed=bench.SEED)
    t0 = time.time()
    g = b.build(pqv)
    wall = time.time() - t0
    free, total = torch.cuda.mem_get_info()
    out = {"n": n, "device_s": b.device_ms / 1e3, "wall_s": wall, "inserts_per_s": n / (b.device_ms / 1e3), "batches": b.batches,
           "hbm_bytes": builder_bytes(n, DIM, True), "fp32_rows_bytes": n * DIM * 4, "hbm_total": total}
    g.close()
    pqv.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=0, help="PQ build alone at this many rows (time and footprint only)")
    ap.add_argument("--nq", type=int, default=1000)
    a = ap.parse_args()
    import torch
    jv.init(0)
    res = {"workload": "c2 world %s x %d, DOT_PRODUCT, M=%d beam=%d hierarchy, PQ M=%d k=%d (c3 codebooks)" % (a.n or 1000000, DIM, DEGREE, BEAM, PQ_M, K)}
    res.update(card())
    if a.n:
        res["pq_only"] = pq_only(torch, a.n)
    else:
        res.update(compare(torch, 1000000, a.nq))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
