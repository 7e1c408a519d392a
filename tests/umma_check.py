"""Run by tests/test_gpu_parity.py::test_bq_bruteforce_filter_kernels_exact (argument: umma | imma) in a SUBPROCESS (a faulting wgmma pipeline traps and
poisons the CUDA context; it must not take the other tests with it): BQ top-k with the filter pass on wgmma (JV_BQ_FILTER=umma)
against the oracle's scalar popcount restatement, bit for bit."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
os.environ["JV_BQ_FILTER"] = sys.argv[1] if len(sys.argv) > 1 else "umma"
import jvector_b200 as jv  # noqa: E402
import oracle_lib as o  # noqa: E402
from oracle_lib import fp, lp, wp  # noqa: E402

jv.init()
L = o.load()
for dim, n, nq, k in ((1536, 20000, 130, 100), (256, 9000, 7, 10), (128, 60000, 300, 100), (2048, 5000, 3, 1), (1000, 4100, 257, 33)):
    rng = np.random.default_rng(dim + n)
    data = rng.standard_normal((n, dim)).astype(np.float32)
    data[n - 64:] = data[:64]
    words = jv.bq_encode_all(data)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    queries[0] = data[3]
    qw = np.zeros((nq, words.shape[1]), np.uint64)
    for i in range(nq):
        L.jvo_bq_encode(fp(queries[i]), dim, wp(qw[i]))
    bqv = jv.BQVectors(words, dim)
    t0 = time.time()
    _, _, keys = jv.topk_bruteforce(bqv, o.COSINE, queries, k)
    dt = time.time() - t0
    want = np.empty((nq, k), np.int64)
    L.jvo_bq_bruteforce_batch(wp(words), n, dim, wp(qw), nq, k, 8, lp(want))
    bad = np.flatnonzero((keys != want).any(axis=1))
    print("dim=%d n=%d nq=%d k=%d: %d queries differ (%.3f s)" % (dim, n, nq, k, len(bad), dt), flush=True)
    if len(bad):
        print("first bad query", bad[0], keys[bad[0]][:5], want[bad[0]][:5])
        sys.exit(1)
    bqv.close()
print("UMMA_OK")
