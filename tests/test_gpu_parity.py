"""Parity tests proper: the sm_90a kernels, called through the C ABI, against the CPU oracle on the same seeded inputs.
Bar (BASELINE.json north_star): bit-exact for BQ/Hamming, code bytes and integer top-k ordering; within 1e-5 relative
for float32 similarity scores. Run on an H100: pytest -m gpu."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as o
from oracle_lib import bp, fp, ip, lp, wp

pytestmark = pytest.mark.gpu

REL = 1e-5  # north_star tolerance for float32 similarities
METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)


@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


def close(got, want, scale=None):
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    # scores live in [0, 1]; (1 + cos) / 2 near 0 is a cancellation, so relative error is floored at |want| = 1e-2
    s = np.maximum(np.abs(want), 1e-2 if scale is None else scale)
    bad = np.abs(got - want) > REL * s
    assert not bad.any(), (np.flatnonzero(bad)[:5], got[bad][:5], want[bad][:5])


def oracle_f32_scores(L, metric, data, q, ids):
    return np.array([L.jvo_compare_f32(metric, fp(q), fp(data[i]), data.shape[1]) for i in ids], dtype=np.float32)


# ------------------------------------------------------------------------------------------------ fp32
@pytest.mark.parametrize("dim", [1, 3, 4, 5, 7, 8, 33, 100, 128, 255, 768, 1021])
def test_f32_score_batch(jv, oracle, dim):
    rng = np.random.default_rng(dim)
    n = 300
    data = o.random_unit_vectors(rng, n, dim) if dim > 1 else rng.standard_normal((n, 1)).astype(np.float32)
    data[5] = o.make_vec(dim, 0.7)
    q = o.make_vec(dim, 1.3) if dim < 64 else o.random_unit_vectors(rng, 1, dim)[0]
    vec = jv.F32Vectors(data)
    ids = rng.permutation(n).astype(np.int32)
    for metric in METRICS:
        sf = vec.score_function_for(q, metric)
        got = sf.similarityToBatch(ids)
        want = oracle_f32_scores(oracle, metric, data, q, ids)
        # (1 + dot) / 2 of NON-unit test vectors cancels: the natural scale of the dot product is |q| |row| / 2
        sc = max(1e-2, 0.5 * float(np.linalg.norm(q)) * float(np.linalg.norm(data, axis=1).max())) if metric == o.DOT_PRODUCT else None
        close(got, want, sc)
        close([sf.similarityTo(int(ids[0]))], want[:1], sc)
        # empty batch and a ragged tail
        assert len(sf.similarityToBatch(np.zeros(0, np.int32))) == 0
        close(sf.similarityToBatch(ids[:37]), want[:37], sc)
        sf.close()
    vec.close()


def test_f32_identities(jv, oracle):
    # native-c:tests/test_similarity.cpp:150-219: L2(a,a) ~ 0, cosine(a, 2a) = 1, orthogonal -> 0
    dim = 128
    a = o.make_vec(dim, 0.7)
    e0 = np.zeros(dim, np.float32); e0[0] = 1
    e1 = np.zeros(dim, np.float32); e1[1] = 1
    vec = jv.F32Vectors(np.stack([a, 2 * a, e0, e1]))
    l2 = vec.score_function_for(a, o.EUCLIDEAN).similarityToBatch([0])
    assert abs(1.0 / l2[0] - 1.0) <= 1e-6 * dim
    cs = vec.score_function_for(a, o.COSINE).similarityToBatch([1])
    assert abs((2 * cs[0] - 1) - 1.0) <= 1e-5
    oc = vec.score_function_for(e0, o.COSINE).similarityToBatch([3])
    assert abs(2 * oc[0] - 1) <= 1e-4


def test_f32_multi_and_pairs(jv, oracle):
    rng = np.random.default_rng(2)
    n, dim, nq = 500, 96, 17
    data = o.random_unit_vectors(rng, n, dim)
    queries = o.random_unit_vectors(rng, nq, dim)
    vec = jv.F32Vectors(data)
    counts = rng.integers(0, 200, nq)
    counts[3] = 0
    counts[5] = 300
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    ids = rng.integers(0, n, offsets[-1]).astype(np.int32)
    for metric in METRICS:
        got = jv.score_multi(vec, metric, queries, ids, offsets)
        want = np.concatenate([oracle_f32_scores(oracle, metric, data, queries[i], ids[offsets[i]:offsets[i + 1]]) for i in range(nq)])
        close(got, want)
        a = rng.integers(0, n, 257).astype(np.int32)
        b = rng.integers(0, n, 257).astype(np.int32)
        got = vec.diversity_scores(a, b, metric)
        want = np.array([oracle.jvo_compare_f32(metric, fp(data[x]), fp(data[y]), dim) for x, y in zip(a, b)], np.float32)
        close(got, want, scale=1e-3)
    vec.close()


# ------------------------------------------------------------------------------------------------ PQ
def _pq(rng, oracle, n, dim, M, centered):
    k = 256
    data = o.random_unit_vectors(rng, n, dim)
    cb, sizes, offsets = o.train_pq_numpy(rng, data[: min(n, 1500)], M, k, iters=2)
    cen = data.mean(0).astype(np.float32) if centered else None
    codes = o.encode_pq(oracle, cb, sizes, offsets, M, k, cen, data)
    return data, cb, sizes, offsets, cen, codes, k


@pytest.mark.parametrize("dim,M,centered", [(64, 8, False), (100, 7, True), (768, 96, False), (33, 33, False), (128, 30, True)])
def test_pq_lut_and_adc(jv, oracle, dim, M, centered):
    rng = np.random.default_rng(dim + M)
    n = 400
    data, cb, sizes, offsets, cen, codes, k = _pq(rng, oracle, n, dim, M, centered)
    q = o.random_unit_vectors(rng, 1, dim)[0]
    pqv = jv.PQVectors(codes, cb, dim, k, cen)
    ids = rng.permutation(n).astype(np.int32)
    mag = np.empty(M * k, np.float32)
    oracle.jvo_pq_self_magnitudes(fp(cb), ip(sizes), ip(offsets), M, k, fp(mag))
    cq = (q - cen).astype(np.float32) if centered else q
    bmag = oracle.jvo_dot_f32(fp(cq), fp(cq), dim)
    for metric in METRICS:
        lm = o.EUCLIDEAN if metric == o.EUCLIDEAN else o.DOT_PRODUCT
        lut = np.empty(M * k, np.float32)
        oracle.jvo_pq_lut(fp(cb), ip(sizes), ip(offsets), M, k, fp(cen), fp(q), dim, lm, fp(lut))
        sf = pqv.score_function_for(q, metric)
        np.testing.assert_allclose(sf.partial_sums(), lut, rtol=1e-5, atol=1e-6)  # calculatePartialSums
        got = sf.similarityToBatch(ids)
        want = np.array([oracle.jvo_pq_score_lut(metric, fp(lut), fp(mag), bmag, k, bp(codes[i]), M) for i in ids], np.float32)
        close(got, want)
        # LUT path == direct path (tests:quantization/TestCompressedVectors.java:230-256), here against the device scores
        direct = np.array([oracle.jvo_pq_score_direct(fp(cb), ip(sizes), ip(offsets), M, k, fp(cen), fp(q), dim, metric, bp(codes[i])) for i in ids[:40]], np.float32)
        assert np.abs(got[:40] - direct).max() <= 5e-6
        sf.close()
        # code-vs-code diversity scores (PQVectors.diversityFunctionFor)
        a = rng.integers(0, n, 64).astype(np.int32)
        b = rng.integers(0, n, 64).astype(np.int32)
        gotp = pqv.diversity_scores(a, b, metric)
        wantp = np.array([oracle.jvo_pq_diversity_direct(fp(cb), ip(sizes), ip(offsets), M, k, metric, bp(codes[x]), bp(codes[y])) for x, y in zip(a, b)], np.float32)
        close(gotp, wantp, scale=1e-3)
    pqv.close()


def test_pq_encode_exact(jv, oracle):
    rng = np.random.default_rng(4)
    for dim, M, centered in ((64, 8, False), (100, 7, True), (768, 96, False)):
        data, cb, sizes, offsets, cen, codes, k = _pq(rng, oracle, 200, dim, M, centered)
        got = jv.pq_encode_all(data, cb, M, k, cen)
        assert np.array_equal(got, codes)  # code bytes: bit-exact


@pytest.mark.parametrize("dim,M", [(64, 8), (100, 7), (768, 96)])
def test_pq_pair_table_and_assemble_and_sum_pq(jv, oracle, dim, M):
    # a-9: ProductQuantization.createCodebookPartialSums (triangular table, ProductQuantization.java:609-628) built on the device and
    # ImmutablePQVectors' code-vs-code scores summed from it (assembleAndSumPQ, ImmutablePQVectors.java:63-105)
    rng = np.random.default_rng(dim)
    n, k = 400, 256
    data, cb, sizes, offsets, cen, codes, _ = _pq(rng, oracle, n, dim, M, False)
    pqv = jv.PQVectors(codes, cb, dim, k)
    a = rng.integers(0, n, 300).astype(np.int32)
    b = rng.integers(0, n, 300).astype(np.int32)
    b[:10] = a[:10]
    for metric in METRICS:
        tm = o.EUCLIDEAN if metric == o.EUCLIDEAN else o.DOT_PRODUCT
        want_t = np.empty(M * (k * (k + 1) // 2), np.float32)
        oracle.jvo_pq_pair_table(fp(cb), ip(sizes), ip(offsets), M, k, tm, fp(want_t))
        pqv.build_pair_table(metric)
        got_t = pqv.pair_table(metric)
        np.testing.assert_allclose(got_t, want_t, rtol=1e-5, atol=1e-6)
        got = pqv.diversity_scores(a, b, metric)
        want = np.array([oracle.jvo_pq_diversity_table(metric, fp(want_t), M, k, bp(codes[x]), bp(codes[y])) for x, y in zip(a, b)], np.float32)
        close(got, want, scale=1e-2)
    pqv.close()


def test_kmeans_assignment_step(jv, oracle):
    # f-4: KMeansPlusPlusClusterer.getNearestCluster for a batch of points; first minimum wins, so duplicated centroids tie to the lower index
    rng = np.random.default_rng(4)
    for dim, k, n in ((8, 256, 5000), (3, 17, 1000), (96, 40, 700)):
        pts = rng.standard_normal((n, dim)).astype(np.float32)
        cen = rng.standard_normal((k, dim)).astype(np.float32)
        cen[k - 1] = cen[2]
        pts[:5] = cen[2]
        want = np.empty(n, np.int32)
        oracle.jvo_kmeans_assign(fp(pts), n, dim, fp(cen), k, ip(want))
        got = jv.kmeans_assign(pts, cen)
        assert np.array_equal(got, want), np.flatnonzero(got != want)[:5]
        assert (got[:5] == 2).all()


# ------------------------------------------------------------------------------------------------ BQ
# dims 2049 / 3000 / 4096: more than 32 words, so brute force takes the generic topk_filter_kernel<BQ>
@pytest.mark.parametrize("dim", [1, 63, 64, 65, 128, 1000, 1536, 2049, 3000, 4096])
def test_bq_exact(jv, oracle, dim):
    rng = np.random.default_rng(dim)
    n = 700
    data = rng.standard_normal((n, dim)).astype(np.float32)
    data[0, : min(dim, 3)] = 0.0
    W = (dim + 63) // 64
    words = np.zeros((n, W), np.uint64)
    for i in range(n):
        oracle.jvo_bq_encode(fp(data[i]), dim, wp(words[i]))
    got_words = jv.bq_encode_all(data)
    assert np.array_equal(got_words, words)
    q = rng.standard_normal(dim).astype(np.float32)
    qw = np.zeros(W, np.uint64)
    oracle.jvo_bq_encode(fp(q), dim, wp(qw))
    bqv = jv.BQVectors(words, dim)
    ids = rng.permutation(n).astype(np.int32)
    got = bqv.score_function_for(q, o.COSINE).similarityToBatch(ids)
    want = np.array([oracle.jvo_bq_score(wp(qw), wp(words[i]), W, dim) for i in ids], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))  # bit-exact
    a, b = ids[:100], ids[100:200]
    gp = bqv.diversity_scores(a, b, o.COSINE)
    wp_ = np.array([oracle.jvo_bq_score(wp(words[x]), wp(words[y]), W, dim) for x, y in zip(a, b)], np.float32)
    assert np.array_equal(gp.view(np.uint32), wp_.view(np.uint32))
    # brute-force first pass: integer top-k ordering must be identical (ties -> smaller node id)
    k = 25
    nodes, scores, keys = jv.topk_bruteforce(bqv, o.COSINE, q[None, :], k)
    allk = o.keys_of(np.array([oracle.jvo_bq_score(wp(qw), wp(words[i]), W, dim) for i in range(n)], np.float32), np.arange(n))
    wantk = np.sort(allk)[::-1][:k]
    assert np.array_equal(keys[0], wantk)
    bqv.close()


def _bq_world(jv, oracle, rng, n, dim, nq, dup=0):
    data = rng.standard_normal((n, dim)).astype(np.float32)
    if dup:
        data[n - dup:] = data[:dup]  # duplicated rows: identical distances for every query, order decided by node id alone
    words = jv.bq_encode_all(data)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    queries[0] = data[3]
    W = words.shape[1]
    qw = np.zeros((nq, W), np.uint64)
    for i in range(nq):
        oracle.jvo_bq_encode(fp(queries[i]), dim, wp(qw[i]))
    return words, queries, qw


@pytest.mark.parametrize("dim,n,nq,k", [(1536, 20000, 130, 100), (256, 9000, 7, 10), (128, 60000, 40, 100), (2048, 5000, 3, 1), (1000, 4100, 129, 33),
                                        (256, 20000, 5, 2048),   # k = 2048 = BQ_IMMA_CAP / 4: the largest k the tensor-core path takes
                                        (256, 5000, 4097, 10),   # nq = 4097: two IMMA_QUERY_CHUNK launches, status words summed
                                        # odd W (or n < 4096): the popcount filter topk_filter_bq_kernel<MAXW>, sampled at n = 20 000;
                                        # W = 3 / 7 / 15 / 23 / 31 reach MAXW = 4 / 8 / 16 / 24 / 32. k = 1: the best sampled row (row 3 for
                                        # query 0, which equals it) is the threshold key itself and must pass the filter
                                        (150, 20000, 9, 50), (420, 20000, 9, 1), (960, 20000, 9, 50), (1470, 20000, 9, 1), (1984, 20000, 9, 50),
                                        (128, 3000, 9, 50)])     # W = 2 with n < 4096: whole, MAXW = 4
def test_bq_bruteforce_tensor_core_contraction_exact(jv, oracle, dim, n, nq, k):
    # csrc/bq_imma.cu (n >= 4096, even word count): Hamming top-k as a u8 contraction on IMMA + integer thresholds. Integer work:
    # every key must equal the scalar popcount restatement, ties to the smaller node id. dim 128 over 60 000 rows makes Hamming
    # bins of thousands of rows (the capture buffer overflows and the redo / fallback paths run); the duplicated tail makes exact
    # key ties; nq 129 / 130 crosses a query tile.
    rng = np.random.default_rng(dim + n)
    words, queries, qw = _bq_world(jv, oracle, rng, n, dim, nq, dup=64)
    bqv = jv.BQVectors(words, dim)
    _, _, keys = jv.topk_bruteforce(bqv, o.COSINE, queries, k)
    want = np.empty((nq, k), np.int64)
    oracle.jvo_bq_bruteforce_batch(wp(words), n, dim, wp(qw), nq, k, 8, lp(want))
    bad = np.flatnonzero((keys != want).any(axis=1))
    assert len(bad) == 0, (len(bad), bad[:5], keys[bad[:1]], want[bad[:1]])
    # the popcount kernels of round 1 stay reachable (JV_BQ_BRUTEFORCE=popc) and must agree as well
    import os
    os.environ["JV_BQ_BRUTEFORCE"] = "popc"
    try:
        _, _, keys2 = jv.topk_bruteforce(bqv, o.COSINE, queries[:5], k)
    finally:
        del os.environ["JV_BQ_BRUTEFORCE"]
    assert np.array_equal(keys2, want[:5])
    bqv.close()


@pytest.mark.parametrize("filter_kernel", ["umma", "imma"])
def test_bq_bruteforce_filter_kernels_exact(jv, filter_kernel):
    # the same top-k with the filter pass forced onto wgmma (u8, register accumulators, csrc/bq_umma.cu: the default where the
    # shape allows) and onto the legacy-MMA kernel (csrc/bq_imma.cu: the fallback), each in its own process
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    out = subprocess.run([sys.executable, os.path.join(here, "umma_check.py"), filter_kernel], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "UMMA_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]


def test_bq_bruteforce_giant_tie_bin_falls_back_exactly(jv, oracle):
    # 11 000 copies of one row: for the query equal to that row, Hamming bin 0 alone is wider than the capture buffer, the
    # integer-threshold path reports the query unresolved and the key-threshold kernels must produce the exact answer
    rng = np.random.default_rng(77)
    n, dim, nq, k = 30000, 256, 6, 50
    data = rng.standard_normal((n, dim)).astype(np.float32)
    data[5000:16000] = data[3]
    words = jv.bq_encode_all(data)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    queries[0] = data[3]
    qw = np.zeros((nq, words.shape[1]), np.uint64)
    for i in range(nq):
        oracle.jvo_bq_encode(fp(queries[i]), dim, wp(qw[i]))
    bqv = jv.BQVectors(words, dim)
    _, _, keys = jv.topk_bruteforce(bqv, o.COSINE, queries, k)
    want = np.empty((nq, k), np.int64)
    oracle.jvo_bq_bruteforce_batch(wp(words), n, dim, wp(qw), nq, k, 8, lp(want))
    assert np.array_equal(keys, want)
    bqv.close()


def test_bq_bruteforce_stream_ordered_shards(jv, oracle):
    # the multi-process path's building blocks on ONE device: two range shards -> stream-ordered local top-k (global ids) ->
    # shard-major gather -> stream-ordered merge, no host synchronisation in between; must equal the unsharded oracle, bit for bit
    import torch

    from jvector_b200 import parallel as par
    rng = np.random.default_rng(19)
    n, dim, nq, k = 16000, 512, 50, 20
    words, queries, qw = _bq_world(jv, oracle, rng, n, dim, nq, dup=16)
    halves = [jv.BQVectors(words[:7000], dim), jv.BQVectors(words[7000:], dim)]
    qd = torch.from_numpy(queries).cuda()
    sbs = [par.gpu_sharded_bruteforce(None, halves[0], o.COSINE, 0), par.gpu_sharded_bruteforce(None, halves[1], o.COSINE, 7000)]
    parts = [sb.local_topk(qd, k) for sb in sbs]
    merged = sbs[0].merge(torch.stack(parts), k)
    torch.cuda.synchronize()
    assert sbs[0].status() == 0 and sbs[1].status() == 0
    want = np.empty((nq, k), np.int64)
    oracle.jvo_bq_bruteforce_batch(wp(words), n, dim, wp(qw), nq, k, 8, lp(want))
    assert np.array_equal(merged.cpu().numpy(), want)
    for v in halves:
        v.close()


def test_multi_device_in_one_process(jv, oracle):
    # one process driving several GPUs through the C ABI alone (what a single JVM needs): range-sharded brute force with peer
    # copies + device merge, and replica graph search with the batch split across devices. With one visible device the same
    # entry points run as their 1-shard / 1-replica degenerate.
    import ctypes as C

    from jvector_b200 import _native as nat
    lib = nat.load()
    ndev = min(lib.jv_gpu_device_count(), 8)
    nat.check(lib.jv_gpu_init_mask((1 << ndev) - 1))
    rng = np.random.default_rng(29)
    n, dim, nq, k = 30000, 1536, 33, 50
    words, queries, qw = _bq_world(jv, oracle, rng, n, dim, nq, dup=8)
    m = C.c_void_p()
    nat.check(lib.jv_multi_register_bq(wp(words), n, dim, C.byref(m)))
    assert lib.jv_multi_shard_count(m) == ndev
    keys = np.empty((nq, k), np.int64)
    nat.check(lib.jv_multi_topk_bruteforce(m, o.COSINE, fp(queries), nq, k, lp(keys)))
    want = np.empty((nq, k), np.int64)
    oracle.jvo_bq_bruteforce_batch(wp(words), n, dim, wp(qw), nq, k, 8, lp(want))
    assert np.array_equal(keys, want)
    nat.check(lib.jv_multi_free(m))
    # replica graph search
    gn, gdim = 3000, 48
    data = o.random_unit_vectors(rng, gn, gdim)
    adj = np.empty((gn, 12), np.int32)
    entry = oracle.jvo_graph_build_f32(o.DOT_PRODUCT, fp(data), gn, gdim, 12, 60, 1.2, 1.2, ip(adj))
    gq = o.random_unit_vectors(rng, 41, gdim)
    graphs, vecs = [], []
    for d in range(ndev):
        nat.check(lib.jv_gpu_set_device(d))
        vecs.append(jv.F32Vectors(data))
        graphs.append(jv.GraphIndex(adj, entry))
        assert lib.jv_dataset_device(vecs[-1]._h) == d
    nat.check(lib.jv_gpu_set_device(0))
    GA = (C.c_void_p * ndev)(*[g._h for g in graphs])
    VA = (C.c_void_p * ndev)(*[v._h for v in vecs])
    nodes = np.empty((41, 10), np.int32)
    scores = np.empty((41, 10), np.float32)
    st = nat.SearchStats()
    nat.check(lib.jv_multi_graph_search_batch(ndev, GA, VA, None, o.DOT_PRODUCT, fp(gq), 41, 10, 40, None, ip(nodes), fp(scores), C.byref(st)))
    g = o.make_graph(adj, entry)
    wn, ws, wv, wr = _oracle_search(oracle, g, lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), gn, gdim, fp(q)), gq, 10, 40)
    assert np.array_equal(nodes, wn) and np.array_equal(scores.view(np.int32), ws.view(np.int32)) and st.visited == wv
    for x in graphs + vecs:
        x.close()


# ------------------------------------------------------------------------------------------------ NVQ
@pytest.mark.parametrize("dim,nsub", [(64, 1), (65, 2), (256, 4), (768, 2), (100, 3)])
def test_nvq_scores(jv, oracle, dim, nsub):
    rng = np.random.default_rng(dim * 7 + nsub)
    n = 300
    data = o.random_unit_vectors(rng, n, dim)
    mean = data.mean(0).astype(np.float32)
    params = np.empty((n, nsub, 4), np.float32)
    bys = np.empty((n, dim), np.uint8)
    for i in range(n):
        oracle.jvo_nvq_encode(fp(data[i]), fp(mean), dim, nsub, i % 2, fp(params[i]), bp(bys[i]))
    nv = jv.NVQVectors(bys, params, mean, nsub)
    q = o.random_unit_vectors(rng, 1, dim)[0]
    ids = rng.permutation(n).astype(np.int32)
    for metric in METRICS:
        got = nv.score_function_for(q, metric).similarityToBatch(ids)
        want = np.array([oracle.jvo_nvq_score(metric, fp(q), fp(mean), dim, nsub, fp(params[i]), bp(bys[i])) for i in ids], np.float32)
        close(got, want)
    nv.close()


def test_nvq_encode(jv, oracle):
    # the growth-rate grid search compares loss sums, so parameters are bit-exact only under ONE summation order: the kernel sums
    # with 32 strided accumulators + a xor butterfly, and the oracle restates exactly that order (jvo_nvq_encode_lanes, lanes = 32;
    # the order is pinned against the reference's kernels in tests/test_oracle.py::test_nvq_loss_lane_orders_vs_ref)
    rng = np.random.default_rng(8)
    for dim, nsub in ((64, 1), (768, 2), (100, 3), (1536, 2), (33, 2)):
        n = 120
        data = o.random_unit_vectors(rng, n, dim)
        mean = data.mean(0).astype(np.float32)
        for learn in (False, True):
            params, bys = jv.nvq_encode_all(data, mean, nsub, learn)
            wp_ = np.empty((n, nsub, 4), np.float32)
            wb = np.empty((n, dim), np.uint8)
            for i in range(n):
                oracle.jvo_nvq_encode_lanes(fp(data[i]), fp(mean), dim, nsub, 1 if learn else 0, 32, fp(wp_[i]), bp(wb[i]))
            assert np.array_equal(params, wp_), np.argwhere(params != wp_)[:5]  # min / max / growth rate / midpoint: all exact
            assert np.array_equal(bys, wb)                                       # bytes: unconditionally bit-exact


# ------------------------------------------------------------------------------------------------ brute force / siftsmall (C1)
def test_siftsmall_bruteforce_matches_ground_truth(jv, sift):
    base, queries, gt = sift
    vec = jv.F32Vectors(base)
    nodes, scores, keys = jv.topk_bruteforce(vec, o.EUCLIDEAN, queries, 100)
    assert (np.diff(keys, axis=1) < 0).all()  # strictly descending keys
    exact = 0
    for qi in range(100):
        if np.array_equal(nodes[qi], gt[qi]):
            exact += 1
        else:
            d_mine = ((base[nodes[qi]] - queries[qi]) ** 2).sum(1)
            d_gt = ((base[gt[qi]] - queries[qi]) ** 2).sum(1)
            assert np.array_equal(d_mine, d_gt)  # only tie order may differ from the shipped file
    assert exact >= 80
    vec.close()


def test_bruteforce_vs_oracle_keys(jv, oracle):
    # keys EQUAL to the oracle's warp-order top-k: the scores are its bits and ties go to the smaller id, so there is no tolerance
    # (every other dispatch tier of the brute force: tests/test_topk_tiers.py)
    rng = np.random.default_rng(12)
    n, dim = 3000, 64
    data = o.random_unit_vectors(rng, n, dim)
    queries = o.random_unit_vectors(rng, 5, dim)
    vec = jv.F32Vectors(data)
    for metric in METRICS:
        _, _, keys = jv.topk_bruteforce(vec, metric, queries, 10)
        want = np.stack([o.scorer_topk(oracle, oracle.jvo_scorer_f32(metric, fp(data), n, dim, fp(q)), 10) for q in queries])
        assert np.array_equal(keys, want), metric
    # k larger than n pads with -1 (key INT64_MIN)
    small = jv.F32Vectors(data[:7])
    nodes, _, keys = jv.topk_bruteforce(small, o.DOT_PRODUCT, queries[:1], 10)
    want = o.scorer_topk(oracle, oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), 7, dim, fp(queries[0])), 10)
    assert np.array_equal(keys[0], want)
    assert (nodes[0, 7:] == -1).all() and (nodes[0, :7] >= 0).all()
    small.close()
    vec.close()


# ------------------------------------------------------------------------------------------------ graph search
# Traversal parity is asserted as EQUALITY: identical id lists, bit-identical scores, identical visited / reranked counters, for
# every query. That needs both sides to produce the same float bits, so the oracle scorers run in warp order (the summation
# order of the kernels, oracle/jv_oracle.c "WARP-ORDER restatements"; order 0 vs order 1 agree to 1e-6, test_oracle.py).
def _oracle_search(oracle, g, scorer_factory, queries, topK, rerankK, rerank_factory=None, threshold=0.0, rerank_floor=0.0, accept=None, order=1):
    nq = len(queries)
    nodes = np.full((nq, topK), -1, np.int32)
    scores = np.zeros((nq, topK), np.float32)
    visited = reranked = 0
    st = o.Stats()
    for i in range(nq):
        sf = scorer_factory(queries[i])
        rr = rerank_factory(queries[i]) if rerank_factory else None
        oracle.jvo_scorer_set_order(sf, order)
        if rr:
            oracle.jvo_scorer_set_order(rr, order)
        bits = None
        if accept is not None:
            a = accept if accept.ndim == 1 else accept[i]
            bits = np.packbits(np.concatenate([a, np.zeros((-len(a)) % 32, bool)]), bitorder="little").view(np.uint32)
        oracle.jvo_graph_search_ex(C.byref(g), sf, rr, topK, rerankK, threshold, rerank_floor,
                                   bits.ctypes.data_as(C.POINTER(C.c_uint32)) if bits is not None else None, ip(nodes[i]), fp(scores[i]), C.byref(st))
        visited += st.visited
        reranked += st.reranked
        oracle.jvo_scorer_free(sf)
        if rr:
            oracle.jvo_scorer_free(rr)
    return nodes, scores, visited, reranked


def _assert_same_search(res, want, what):
    wn, ws, wv, wr = want
    same = (res.nodes == wn).all(axis=1)
    assert same.all(), (what, "id lists differ for queries", np.flatnonzero(~same)[:8].tolist(), float(same.mean()))
    assert np.array_equal(res.scores.view(np.int32), ws.view(np.int32)), (what, "score bits differ", float(np.abs(res.scores - ws).max()))
    assert res.visitedCount == wv, (what, res.visitedCount, wv)
    assert res.rerankedCount == wr, (what, res.rerankedCount, wr)


def test_scores_bit_identical_to_warp_order_oracle(jv, oracle):
    # the premise of the equality tests: through the C ABI, every scorer returns the bits of the oracle's warp-order restatement
    rng = np.random.default_rng(44)
    for dim, M, nsub in ((64, 16, 2), (100, 7, 3), (768, 96, 2), (33, 33, 1)):
        n = 300
        data = o.random_unit_vectors(rng, n, dim)
        q = o.random_unit_vectors(rng, 1, dim)[0]
        ids = rng.permutation(n).astype(np.int32)
        cb, sizes, offsets = o.train_pq_numpy(rng, data, M, 256, iters=1)
        cen = data.mean(0).astype(np.float32)
        codes = o.encode_pq(oracle, cb, sizes, offsets, M, 256, cen, data)
        params = np.empty((n, nsub, 4), np.float32)
        bys = np.empty((n, dim), np.uint8)
        for i in range(n):
            oracle.jvo_nvq_encode(fp(data[i]), fp(cen), dim, nsub, 1, fp(params[i]), bp(bys[i]))
        f32v, pqv, nvv = jv.F32Vectors(data), jv.PQVectors(codes, cb, dim, 256, cen), jv.NVQVectors(bys, params, cen, nsub)
        for metric in METRICS:
            for name, vec, mk in (("f32", f32v, lambda: oracle.jvo_scorer_f32(metric, fp(data), n, dim, fp(q))),
                                  ("pq", pqv, lambda: oracle.jvo_scorer_pq(metric, fp(cb), M, 256, dim, fp(cen), bp(codes), n, fp(q))),
                                  ("nvq", nvv, lambda: oracle.jvo_scorer_nvq(metric, fp(cen), dim, nsub, fp(params), bp(bys), n, fp(q)))):
                sf = mk()
                oracle.jvo_scorer_set_order(sf, 1)
                want = np.array([oracle.jvo_scorer_score(sf, int(i)) for i in ids], np.float32)
                oracle.jvo_scorer_free(sf)
                h = vec.score_function_for(q, metric)
                got = h.similarityToBatch(ids)
                h.close()
                bad = np.flatnonzero(got.view(np.int32) != want.view(np.int32))
                assert len(bad) == 0, (name, dim, metric, len(bad), got[bad][:3], want[bad][:3])
        for v in (f32v, pqv, nvv):
            v.close()


@pytest.fixture(scope="module")
def sift_graph(oracle, sift):
    base, queries, gt = sift
    n = 3000
    b = np.ascontiguousarray(base[:n])
    adj = np.empty((n, 16), np.int32)
    entry = oracle.jvo_graph_build_f32(o.EUCLIDEAN, fp(b), n, 128, 16, 100, 1.2, 1.2, ip(adj))
    return b, queries, adj, entry


def test_graph_search_matches_oracle_f32(jv, oracle, sift_graph):
    # SIFT has integer-valued distances: exact score ties are common, including at the result-queue boundary
    b, queries, adj, entry = sift_graph
    n = b.shape[0]
    g = o.make_graph(adj, entry)
    vec = jv.F32Vectors(b)
    gi = jv.GraphIndex(adj, entry)
    searcher = jv.GraphSearcher(gi)
    for topK, rerankK in ((10, 10), (10, 50), (100, 100), (1, 1), (7, 33)):
        res = searcher.search(vec, queries, o.EUCLIDEAN, topK, rerankK)
        want = _oracle_search(oracle, g, lambda q: oracle.jvo_scorer_f32(o.EUCLIDEAN, fp(b), n, 128, fp(q)), queries, topK, rerankK)
        _assert_same_search(res, want, ("sift", topK, rerankK))
    gi.close()
    vec.close()


def _hier_world(oracle, rng, n, dim, deg, metric=None):
    data = o.random_unit_vectors(rng, n, dim)
    adj = np.empty((n, deg), np.int32)
    entry = oracle.jvo_graph_build_f32(o.DOT_PRODUCT, fp(data), n, dim, deg, 60, 1.2, 1.2, ip(adj))
    ids1 = np.sort(rng.choice(n, 200, replace=False)).astype(np.int32)
    a1 = np.empty((200, deg), np.int32)
    oracle.jvo_graph_build_f32(o.DOT_PRODUCT, fp(np.ascontiguousarray(data[ids1])), 200, dim, deg, 60, 1.2, 1.2, ip(a1))
    a1 = np.where(a1 >= 0, ids1[np.clip(a1, 0, None)], -1).astype(np.int32)
    ids2 = ids1[:10].copy()
    a2 = np.empty((10, deg), np.int32)
    oracle.jvo_graph_build_f32(o.DOT_PRODUCT, fp(np.ascontiguousarray(data[ids2])), 10, dim, deg, 60, 1.2, 1.2, ip(a2))
    a2 = np.where(a2 >= 0, ids2[np.clip(a2, 0, None)], -1).astype(np.int32)
    return data, adj, entry, [(ids1, a1), (ids2, a2)], int(ids2[0])


def test_graph_search_continuous_scores_exact_ids(jv, oracle):
    rng = np.random.default_rng(5)
    n, dim = 2500, 48
    data, adj, entry, upper_levels, entry_top = _hier_world(oracle, rng, n, dim, 12)
    queries = o.random_unit_vectors(rng, 64, dim)
    for upper in (None, upper_levels):
        e = entry if upper is None else entry_top
        g = o.make_graph(adj, e, upper)
        gi = jv.GraphIndex(adj, e, upper)
        searcher = jv.GraphSearcher(gi)
        vec = jv.F32Vectors(data)
        for metric in METRICS:
            res = searcher.search(vec, queries, metric, 10, 40)
            want = _oracle_search(oracle, g, lambda q: oracle.jvo_scorer_f32(metric, fp(data), n, dim, fp(q)), queries, 10, 40)
            _assert_same_search(res, want, ("continuous", metric, upper is not None))
        vec.close()
        gi.close()


def test_graph_search_pq_rerank_and_nvq_bq(jv, oracle):
    rng = np.random.default_rng(6)
    n, dim, M, k, nsub = 2000, 64, 16, 256, 2
    data, adj, entry, upper_levels, entry_top = _hier_world(oracle, rng, n, dim, 16)
    data[500:520] = data[40:60]  # duplicated vectors: equal approximate AND equal exact scores (rerank tie order matters)
    queries = o.random_unit_vectors(rng, 40, dim)
    queries[0] = data[40]
    cb, sizes, offsets = o.train_pq_numpy(rng, data[:1500], M, k, iters=2)
    codes = o.encode_pq(oracle, cb, sizes, offsets, M, k, None, data)
    mean = data.mean(0).astype(np.float32)
    params = np.empty((n, nsub, 4), np.float32)
    bys = np.empty((n, dim), np.uint8)
    for i in range(n):
        oracle.jvo_nvq_encode(fp(data[i]), fp(mean), dim, nsub, 1, fp(params[i]), bp(bys[i]))
    words = np.zeros((n, 1), np.uint64)
    for i in range(n):
        oracle.jvo_bq_encode(fp(data[i]), dim, wp(words[i]))
    f32v, pqv, nvv, bqv = jv.F32Vectors(data), jv.PQVectors(codes, cb, dim, k), jv.NVQVectors(bys, params, mean, nsub), jv.BQVectors(words, dim)
    mk_f32 = lambda metric: (lambda q: oracle.jvo_scorer_f32(metric, fp(data), n, dim, fp(q)))
    mk_pq = lambda metric: (lambda q: oracle.jvo_scorer_pq(metric, fp(cb), M, k, dim, None, bp(codes), n, fp(q)))
    mk_nvq = lambda metric: (lambda q: oracle.jvo_scorer_nvq(metric, fp(mean), dim, nsub, fp(params), bp(bys), n, fp(q)))
    mk_bq = lambda q: oracle.jvo_scorer_bq(wp(words), n, dim, fp(q))
    for upper in (None, upper_levels):
        e = entry if upper is None else entry_top
        g = o.make_graph(adj, e, upper)
        gi = jv.GraphIndex(adj, e, upper)
        searcher = jv.GraphSearcher(gi)
        for metric in (o.DOT_PRODUCT, o.EUCLIDEAN, o.COSINE):
            # config 3 shape: PQ ADC first pass + fp32 rerank
            res = searcher.search(pqv, queries, metric, 10, 50, reranker=f32v)
            _assert_same_search(res, _oracle_search(oracle, g, mk_pq(metric), queries, 10, 50, mk_f32(metric)), ("pq+f32", metric))
            # NVQ as the reranker (feature/NVQ.rerankerFor)
            res = searcher.search(pqv, queries, metric, 10, 50, reranker=nvv)
            _assert_same_search(res, _oracle_search(oracle, g, mk_pq(metric), queries, 10, 50, mk_nvq(metric)), ("pq+nvq", metric))
            # NVQ walking the graph itself
            res = searcher.search(nvv, queries, metric, 10, 30)
            _assert_same_search(res, _oracle_search(oracle, g, mk_nvq(metric), queries, 10, 30), ("nvq", metric))
        # BQ first pass: at most dim + 1 distinct scores, ties everywhere — the case the reference's boundary rule exists for
        for topK, rerankK in ((10, 60), (10, 10), (1, 1), (25, 25)):
            res = searcher.search(bqv, queries, o.COSINE, topK, rerankK, reranker=f32v)
            _assert_same_search(res, _oracle_search(oracle, g, mk_bq, queries, topK, rerankK, mk_f32(o.COSINE)), ("bq+f32", topK, rerankK))
            res = searcher.search(bqv, queries, o.COSINE, topK, rerankK)
            _assert_same_search(res, _oracle_search(oracle, g, mk_bq, queries, topK, rerankK), ("bq", topK, rerankK))
        gi.close()
    for v in (f32v, pqv, nvv, bqv):
        v.close()


def test_fused_pq_layout_and_walk(jv, oracle):
    # FusedPQ feature (FusedPQ.java:122-141, FusedPQDecoder.java:84-114, OnDiskGraphIndex.java:639-651): records packed on the device
    # must equal the reference's writeInline layout byte for byte, and the walk that reads them must equal the oracle's
    # edge-loading traversal — and therefore the plain PQ walk — id for id, score bit for score bit
    rng = np.random.default_rng(73)
    n, dim, k = 2500, 64, 256
    data, adj, entry, upper_levels, entry_top = _hier_world(oracle, rng, n, dim, 16)
    queries = o.random_unit_vectors(rng, 32, dim)
    for M in (16, 10):  # M = 10: code rows padded to 12 bytes inside the record
        cb, sizes, offsets = o.train_pq_numpy(rng, data[:1500], M, k, iters=2)
        codes = o.encode_pq(oracle, cb, sizes, offsets, M, k, None, data)
        packed = np.empty((n, 16, M), np.uint8)
        oracle.jvo_fused_pq_pack(ip(adj), n, 16, bp(codes), M, bp(packed))
        pqv, f32v = jv.PQVectors(codes, cb, dim, k), jv.F32Vectors(data)
        for upper in (None, upper_levels):
            e = entry if upper is None else entry_top
            g = o.make_graph(adj, e, upper)
            gi = jv.GraphIndex(adj, e, upper).fuse_pq(pqv)
            rec = gi.fused_records()
            cs = (M + 3) & ~3
            assert np.array_equal(rec[:, :64].copy().view(np.int32), adj)
            got_codes = rec[:, 64:64 + 16 * cs].reshape(n, 16, cs)
            assert np.array_equal(got_codes[:, :, :M], packed) and not got_codes[:, :, M:].any()
            for metric in METRICS:
                def mk(q):
                    sf = oracle.jvo_scorer_pq(metric, fp(cb), M, k, dim, None, bp(codes), n, fp(q))
                    oracle.jvo_scorer_set_packed_neighbors(sf, bp(packed), 16)
                    return sf
                res = jv.GraphSearcher(gi).search(pqv, queries, metric, 10, 40, reranker=f32v)
                want = _oracle_search(oracle, g, mk, queries, 10, 40, lambda q: oracle.jvo_scorer_f32(metric, fp(data), n, dim, fp(q)))
                _assert_same_search(res, want, ("fused pq", M, metric, upper is not None))
                plain = _oracle_search(oracle, g, lambda q: oracle.jvo_scorer_pq(metric, fp(cb), M, k, dim, None, bp(codes), n, fp(q)), queries, 10, 40,
                                       lambda q: oracle.jvo_scorer_f32(metric, fp(data), n, dim, fp(q)))
                assert np.array_equal(want[0], plain[0])  # the fused layout changes where codes are read from, never a score
            gi.close()
        pqv.close()
        f32v.close()


def test_graph_search_accept_threshold_rerank_floor(jv, oracle):
    # GraphSearcher.search(sp, topK, rerankK, threshold, rerankFloor, acceptOrds): GraphSearcher.java:166-181,427-431, NodeQueue.java:168-230
    rng = np.random.default_rng(61)
    n, dim = 2000, 64
    data, adj, entry, upper_levels, entry_top = _hier_world(oracle, rng, n, dim, 16)
    queries = o.random_unit_vectors(rng, 24, dim)
    words = np.zeros((n, 1), np.uint64)
    for i in range(n):
        oracle.jvo_bq_encode(fp(data[i]), dim, wp(words[i]))
    f32v, bqv = jv.F32Vectors(data), jv.BQVectors(words, dim)
    mk_f32 = lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q))
    mk_bq = lambda q: oracle.jvo_scorer_bq(wp(words), n, dim, fp(q))
    shared = rng.random(n) < 0.3
    per_query = rng.random((24, n)) < 0.5
    for upper in (None, upper_levels):
        e = entry if upper is None else entry_top
        g = o.make_graph(adj, e, upper)
        gi = jv.GraphIndex(adj, e, upper)
        s = jv.GraphSearcher(gi)
        for acc in (shared, per_query):
            res = s.search(f32v, queries, o.DOT_PRODUCT, 10, 20, acceptOrds=acc)
            _assert_same_search(res, _oracle_search(oracle, g, mk_f32, queries, 10, 20, accept=acc), "accept f32")
            allowed = acc if acc.ndim == 1 else None
            if allowed is not None:
                assert allowed[res.nodes[res.nodes >= 0]].all()
            res = s.search(bqv, queries, o.COSINE, 10, 20, reranker=f32v, acceptOrds=acc, rerankFloor=0.55)
            _assert_same_search(res, _oracle_search(oracle, g, mk_bq, queries, 10, 20, lambda q: oracle.jvo_scorer_f32(o.COSINE, fp(data), n, dim, fp(q)),
                                                    accept=acc, rerank_floor=0.55), "accept bq + floor")
        res = s.search(f32v, queries, o.DOT_PRODUCT, 10, 20, threshold=0.58)
        _assert_same_search(res, _oracle_search(oracle, g, mk_f32, queries, 10, 20, threshold=0.58), "threshold")
        assert (res.scores[res.nodes >= 0] >= 0.58).all()
        res = s.search(bqv, queries, o.COSINE, 5, 15, reranker=f32v, rerankFloor=2.0)  # nothing above the floor: the best one is reranked alone
        _assert_same_search(res, _oracle_search(oracle, g, mk_bq, queries, 5, 15, lambda q: oracle.jvo_scorer_f32(o.COSINE, fp(data), n, dim, fp(q)),
                                                rerank_floor=2.0), "floor above everything")
        assert res.rerankedCount == 24 and (res.nodes[:, 1:] == -1).all()
        gi.close()
    f32v.close()
    bqv.close()


def test_graph_search_tie_tail_overflow_retry(jv, oracle):
    # JV_LIST_CAP = rerankK leaves no room for a tie tail: BQ walks must report overflow code 2, be re-run with a 4x list and
    # still equal the reference traversal exactly
    import os
    rng = np.random.default_rng(62)
    n, dim = 3000, 64
    data = o.random_unit_vectors(rng, n, dim)
    adj = np.empty((n, 16), np.int32)
    entry = oracle.jvo_graph_build_f32(o.DOT_PRODUCT, fp(data), n, dim, 16, 60, 1.2, 1.2, ip(adj))
    queries = o.random_unit_vectors(rng, 32, dim)
    words = np.zeros((n, 1), np.uint64)
    for i in range(n):
        oracle.jvo_bq_encode(fp(data[i]), dim, wp(words[i]))
    bqv = jv.BQVectors(words, dim)
    g = o.make_graph(adj, entry)
    gi = jv.GraphIndex(adj, entry)
    os.environ["JV_LIST_CAP"] = "20"
    try:
        res = jv.GraphSearcher(gi).search(bqv, queries, o.COSINE, 10, 20)
    finally:
        del os.environ["JV_LIST_CAP"]
    assert res.retried > 0, "the tight list was expected to overflow on Hamming ties"
    _assert_same_search(res, _oracle_search(oracle, g, lambda q: oracle.jvo_scorer_bq(wp(words), n, dim, fp(q)), queries, 10, 20), "tie tail retry")
    gi.close()
    bqv.close()


# ------------------------------------------------------------------------------------------------ build (C5 shape, small)
def test_graph_build_recall_siftsmall(jv, sift):
    base, queries, gt = sift
    vec = jv.F32Vectors(base)
    for hier in (False, True):
        b = jv.GraphIndexBuilder(o.EUCLIDEAN, M=16, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=hier, seed=7)
        gi = b.build(vec)
        inf = gi.info()
        assert inf["n"] == 10000 and inf["degree"] == 16 and (inf["levels"] > 1) == hier
        ids, adj = gi.level(0)
        deg = (adj >= 0).sum(1)
        assert deg.max() <= 16 and deg.mean() > 6 and (adj < 10000).all()
        # no self loops, no duplicate neighbours
        assert not (adj == np.arange(10000)[:, None]).any()
        srt = np.sort(adj, axis=1)
        assert not ((srt[:, 1:] == srt[:, :-1]) & (srt[:, 1:] >= 0)).any()
        res = jv.GraphSearcher(gi).search(vec, queries, o.EUCLIDEAN, 10, 100)
        recall = np.mean([len(set(res.nodes[i]) & set(gt[i, :10])) / 10.0 for i in range(100)])
        assert recall > 0.9, (hier, recall)  # tests:graph/TestVectorGraph.java:672
        gi.close()
    vec.close()


def test_stepwise_builder_equals_one_call_build(jv):
    # the build is deterministic (sorted back-links, exact traversal): the batch-by-batch driver a sharded build uses
    # (jvector_b200/parallel.py sharded_build, here with one rank) must produce the adjacency of jv_graph_build, bit for bit
    from jvector_b200 import parallel as par
    rng = np.random.default_rng(88)
    n, dim = 12000, 64
    A = rng.standard_normal((10, dim)).astype(np.float32)
    x = rng.standard_normal((n, 10)).astype(np.float32) @ A + 0.3 * rng.standard_normal((n, dim)).astype(np.float32)
    data = np.ascontiguousarray(x / np.linalg.norm(x, axis=1, keepdims=True), dtype=np.float32)
    vec = jv.F32Vectors(data)
    kw = dict(M=16, beamWidth=60, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=5, max_batch=1024)
    g1 = jv.GraphIndexBuilder(o.DOT_PRODUCT, **kw).build(vec)
    g1b = jv.GraphIndexBuilder(o.DOT_PRODUCT, **kw).build(vec)
    g2, ms, _ = par.sharded_build(None, vec, o.DOT_PRODUCT, **kw)
    for lvl in range(g1.info()["levels"]):
        i1, a1 = g1.level(lvl)
        i1b, a1b = g1b.level(lvl)
        i2, a2 = g2.level(lvl)
        assert np.array_equal(a1, a1b), "the one-call build is not reproducible"
        assert np.array_equal(i1, i2) and np.array_equal(a1, a2), (lvl, int((a1 != a2).any(axis=1).sum()))
    # in-batch visibility: with the in-progress window some neighbours come from the same batch as the node
    _, adj = g1.level(0)
    g0 = jv.GraphIndexBuilder(o.DOT_PRODUCT, concurrent_window=0, **kw).build(vec)
    _, adj0 = g0.level(0)
    assert not np.array_equal(adj, adj0)
    for g in (g1, g1b, g2, g0):
        g.close()
    vec.close()


def test_errors(jv):
    rows = np.zeros((4, 8), np.float32)
    vec = jv.F32Vectors(rows)
    with pytest.raises(jv.JVectorB200Error):
        jv.GraphSearcher(jv.GraphIndex(np.full((5, 4), -1, np.int32), 0)).search(vec, rows[:1], o.DOT_PRODUCT, 2, 2)  # size mismatch
    with pytest.raises(jv.JVectorB200Error):
        jv.topk_bruteforce(vec, o.DOT_PRODUCT, rows[:1], 0)
    vec.close()


# ------------------------------------------------------------------------------------------------ specialised brute force
def test_pq_bruteforce_tma_lut(jv, oracle):
    # PQ ADC brute force: LUT staged into shared memory by one TMA bulk copy (M = 16), whole path (n <= 16384); keys EQUAL to the
    # oracle's warp-order top-k (the other shapes and the sampled path: tests/test_topk_tiers.py::test_pq_shared_memory_lut)
    rng = np.random.default_rng(31)
    n, dim, M, k = 5000, 64, 16, 256
    data, cb, sizes, offsets, cen, codes, _ = _pq(rng, oracle, n, dim, M, False)
    queries = o.random_unit_vectors(rng, 6, dim)
    pqv = jv.PQVectors(codes, cb, dim, k)
    for metric in METRICS:
        _, _, keys = jv.topk_bruteforce(pqv, metric, queries, 20)
        want = np.stack([o.scorer_topk(oracle, oracle.jvo_scorer_pq(metric, fp(cb), M, k, dim, None, bp(codes), n, fp(q)), 20) for q in queries])
        assert np.array_equal(keys, want), metric
    pqv.close()


def test_sharded_bruteforce_single_rank_device(jv, oracle):
    # the N = 1 degenerate of the multi-GPU path: device-resident queries/keys, global id rebasing, device merge kernel
    import torch

    from jvector_b200 import parallel as par
    rng = np.random.default_rng(9)
    n, dim, W = 4000, 256, 4
    data = rng.standard_normal((n, dim)).astype(np.float32)
    queries = rng.standard_normal((5, dim)).astype(np.float32)
    words = jv.bq_encode_all(data)
    halves = [jv.BQVectors(words[:2000], dim), jv.BQVectors(words[2000:], dim)]
    qd = torch.from_numpy(queries).cuda()
    parts = [par.gpu_sharded_bruteforce(None, halves[i], o.COSINE, 2000 * i).local_topk(qd, 15) for i in range(2)]
    merged = par.gpu_sharded_bruteforce(None, halves[0], o.COSINE, 0).merge(torch.stack(parts), 15).cpu().numpy()
    full = jv.BQVectors(words, dim)
    _, _, want = jv.topk_bruteforce(full, o.COSINE, queries, 15)
    assert np.array_equal(merged, want)  # integer ordering: bit-exact across the shard boundary
    for v in halves + [full]:
        v.close()


def test_device_builder_quality_vs_reference_builder(jv, oracle):
    # the batched device builder must give a graph as searchable as the reference's sequential insert (oracle restatement)
    rng = np.random.default_rng(17)
    n, dim, lat = 6000, 64, 12
    A = rng.standard_normal((lat, dim)).astype(np.float32)
    def gen(m):
        x = rng.standard_normal((m, lat)).astype(np.float32) @ A + 0.3 * rng.standard_normal((m, dim)).astype(np.float32)
        return np.ascontiguousarray(x / np.linalg.norm(x, axis=1, keepdims=True), dtype=np.float32)
    data, queries = gen(n), gen(200)
    vec = jv.F32Vectors(data)
    gt, _, _ = jv.topk_bruteforce(vec, o.DOT_PRODUCT, queries, 10)
    adj = np.empty((n, 16), np.int32)
    entry = oracle.jvo_graph_build_f32(o.DOT_PRODUCT, fp(data), n, dim, 16, 60, 1.2, 1.2, ip(adj))
    g_ref = jv.GraphIndex(adj, entry)
    g_dev = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, neighborOverflow=1.2, alpha=1.2).build(vec)
    rec = {}
    for name, g in (("ref", g_ref), ("dev", g_dev)):
        res = jv.GraphSearcher(g).search(vec, queries, o.DOT_PRODUCT, 10, 30)
        rec[name] = np.mean([len(set(res.nodes[i]) & set(gt[i])) / 10.0 for i in range(200)])
        rec[name + "_visited"] = res.visitedCount / 200.0
    # the batched build is a different insert order from the sequential one (batches, in-progress window), so its graph is not the
    # oracle's; its own rows are pinned step by step in tests/test_build_steps.py. Here only searchability, with head-room
    assert rec["dev"] >= rec["ref"] - 0.05, rec
    assert rec["dev_visited"] <= 1.35 * rec["ref_visited"], rec
    vec.close()


def test_encoders_from_resident_dataset(jv, oracle):
    # the *_dataset encoders read rows already in HBM (padded row stride when dim % 4 != 0) and must equal the host-row forms
    rng = np.random.default_rng(41)
    for dim, M, nsub in ((100, 7, 3), (768, 96, 2)):
        data = o.random_unit_vectors(rng, 150, dim)
        vec = jv.F32Vectors(data)
        assert np.array_equal(jv.bq_encode_all(vec), jv.bq_encode_all(data))
        cb, sizes, offsets = o.train_pq_numpy(rng, data, M, 256, iters=1)
        assert np.array_equal(jv.pq_encode_all(vec, cb, M, 256), jv.pq_encode_all(data, cb, M, 256))
        mean = data.mean(0).astype(np.float32)
        p1, b1 = jv.nvq_encode_all(vec, mean, nsub, True)
        p2, b2 = jv.nvq_encode_all(data, mean, nsub, True)
        assert np.array_equal(p1, p2) and np.array_equal(b1, b2)
        vec.close()


# ------------------------------------------------------------------------------------------------ rarely taken paths
def test_search_visited_table_overflow_retry(jv, oracle):
    # a RANDOM graph makes the walk wander: the visited set outgrows the first table, the host re-runs those queries with a 4x
    # table (api.cu search_device) and the result must still equal the oracle traversal exactly
    rng = np.random.default_rng(23)
    n, dim, degree = 20000, 32, 32
    data = o.random_unit_vectors(rng, n, dim)
    queries = o.random_unit_vectors(rng, 24, dim)
    adj = rng.integers(0, n, (n, degree)).astype(np.int32)
    adj[adj == np.arange(n)[:, None]] = 0
    g = o.make_graph(adj, 5)
    gi = jv.GraphIndex(adj, 5)
    vec = jv.F32Vectors(data)
    import os
    os.environ["JV_VISITED_CAP"] = "2048"  # first table: 2048 slots, a query is declared overflowed at 1024 visited nodes
    try:
        res = jv.GraphSearcher(gi).search(vec, queries, o.DOT_PRODUCT, 10, 50)
    finally:
        del os.environ["JV_VISITED_CAP"]
    want = _oracle_search(oracle, g, lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q)), queries, 10, 50)
    assert res.retried > 0, "the test is meant to exercise the retry path"
    _assert_same_search(res, want, "visited-table retry")
    # a wide beam (rerankK = 1000: 8 KB key lists, bitonic sort of 1024) on the same graph
    res = jv.GraphSearcher(gi).search(vec, queries[:4], o.DOT_PRODUCT, 100, 1000)
    want = _oracle_search(oracle, g, lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q)), queries[:4], 100, 1000)
    _assert_same_search(res, want, "wide beam")
    vec.close()
    gi.close()


def test_search_visited_set_in_shared_memory_is_exact(jv, oracle):
    # The walk keeps its visited set in shared memory as 16-bit tags inside per-id-range regions (search.cu visited_insert_smem):
    # it must behave exactly like a set. Same traversal as the oracle (i) on the default table, (ii) on the global-memory table,
    # (iii) with a table so small (1024 slots) that every query outgrows it and is re-run on the global table, (iv) on a graph
    # with many nodes (2^21 ids: 64 regions) where ids differ only in their high bits.
    import os
    rng = np.random.default_rng(77)
    n, dim, degree = 30000, 24, 32
    data = o.random_unit_vectors(rng, n, dim)
    queries = o.random_unit_vectors(rng, 32, dim)
    adj = rng.integers(0, n, (n, degree)).astype(np.int32)
    adj[adj == np.arange(n)[:, None]] = 0
    g = o.make_graph(adj, 7)
    gi = jv.GraphIndex(adj, 7)
    vec = jv.F32Vectors(data)
    want = _oracle_search(oracle, g, lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q)), queries, 10, 60)
    for env, must_retry in (({}, False), ({"JV_VISITED": "global"}, False), ({"JV_VISITED": "smem", "JV_VISITED_SMEM_SLOTS": "1024"}, True)):
        os.environ.update(env)
        try:
            res = jv.GraphSearcher(gi).search(vec, queries, o.DOT_PRODUCT, 10, 60)
        finally:
            for k in env:
                del os.environ[k]
        _assert_same_search(res, want, "visited set %r" % (env,))
        assert res.retried > 0 or not must_retry, (env, res.retried)
    vec.close()
    gi.close()
    # (iv) 2^21 nodes, 8 dimensions: neighbours are id +- multiples of 2^15, 2^16 ... so tags collide unless the region bits work
    n2, dim2 = 1 << 21, 8
    data2 = o.random_unit_vectors(rng, n2, dim2)
    strides = np.array([1 << 15, 1 << 16, 1 << 17, 3 << 15, 5 << 15, 1 << 20, 7, 1], np.int64)
    adj2 = ((np.arange(n2, dtype=np.int64)[:, None] + np.concatenate([strides, -strides])[None, :]) % n2).astype(np.int32)
    g2 = o.make_graph(adj2, 11)
    gi2 = jv.GraphIndex(adj2, 11)
    vec2 = jv.F32Vectors(data2)
    q2 = o.random_unit_vectors(rng, 8, dim2)
    res = jv.GraphSearcher(gi2).search(vec2, q2, o.DOT_PRODUCT, 10, 80)
    want = _oracle_search(oracle, g2, lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data2), n2, dim2, fp(q)), q2, 10, 80)
    _assert_same_search(res, want, "visited set, 2^21 ids")
    vec2.close()
    gi2.close()


def test_host_pointer_search_overlaps_the_query_copy(jv, oracle):
    # jv_graph_search_batch with host buffers: batches of >= 1 MB travel in chunks behind an arrival watermark while the kernel
    # already runs (api.cu). Same answers as the plain path (JV_SEARCH_OVERLAP=0) and as the oracle; dim = 100 makes adjacent
    # queries share cache lines, nq is not a multiple of the chunk alignment.
    import os
    rng = np.random.default_rng(99)
    n, dim, nq = 20000, 100, 4099
    data = o.random_unit_vectors(rng, n, dim)
    queries = o.random_unit_vectors(rng, nq, dim)
    vec = jv.F32Vectors(data)
    gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=40).build(vec)
    s = jv.GraphSearcher(gi)
    a = s.search(vec, queries, o.DOT_PRODUCT, 10, 30)
    os.environ["JV_SEARCH_OVERLAP"] = "0"
    try:
        b = s.search(vec, queries, o.DOT_PRODUCT, 10, 30)
    finally:
        del os.environ["JV_SEARCH_OVERLAP"]
    assert np.array_equal(a.nodes, b.nodes) and np.array_equal(a.scores.view(np.int32), b.scores.view(np.int32))
    assert a.visitedCount == b.visitedCount
    for _ in range(3):  # repeated calls reuse the copy stream and the pinned watermark slots
        c = s.search(vec, queries, o.DOT_PRODUCT, 10, 30)
        assert np.array_equal(a.nodes, c.nodes)
    _, adj = gi.level(0)
    info = gi.info()
    if info["levels"] == 1:
        g = o.make_graph(adj, info["entry_node"])
        want = _oracle_search(oracle, g, lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q)), queries[-16:], 10, 30)
        assert np.array_equal(a.nodes[-16:], want[0])
    vec.close()
    gi.close()


def test_topk_multipass_on_adversarial_layout(jv, oracle):
    # n > 16384 takes the sampled-threshold path. Put LOW scores exactly on the strided sample positions and near-equal HIGH
    # scores everywhere else: the sample thresholds are then far too low, the candidate buffer overflows, and the exact
    # result must come out of the tighten-and-rescan passes.
    n, dim, S = 40000, 8, 16384
    rng = np.random.default_rng(3)
    sampled = np.unique((np.arange(S, dtype=np.int64) * n) // S)
    data = np.zeros((n, dim), np.float32)
    data[:, 0] = 0.9 + 1e-4 * rng.random(n, dtype=np.float32)
    data[sampled, 0] = -0.5
    data[:, 1] = 1e-3 * rng.standard_normal(n).astype(np.float32)
    q = np.zeros((3, dim), np.float32)
    q[:, 0] = 1.0
    q[1, 1] = 0.5
    q[2, 1] = -0.5
    vec = jv.F32Vectors(data)
    for k in (10, 100):
        nodes, scores, keys = jv.topk_bruteforce(vec, o.DOT_PRODUCT, q, k)
        for qi in range(3):
            wk = np.empty(k, np.int64)
            oracle.jvo_bruteforce_topk_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q[qi]), k, lp(wk))
            assert np.array_equal(keys[qi], wk), (k, qi)  # 2-term dot products: bit-identical scores, so identical keys
    vec.close()


def test_device_builder_golden_neighbour_lists(jv):
    # tests:graph/TestVectorGraph.java:457-526 testDiversity — the reference's golden neighbour lists (M=4, beamWidth=10, overflow 1.0,
    # alpha 1.0, 7 unit-circle vectors). The device builder's first batches hold ONE node each (batch = max(1, inserted / 2)), i.e. they
    # are sequential inserts, so the states after 3 and after 4 nodes must equal the reference's, list for list.
    ang = np.array([0.5, 0.75, 0.2, 0.9, 0.8, 0.77, 0.6]) * np.pi
    vec = np.ascontiguousarray(np.stack([np.cos(ang), np.sin(ang)], 1), dtype=np.float32)
    expected = {3: {0: [1, 2], 1: [0], 2: [0]}, 4: {0: [1, 2], 1: [0, 3], 2: [0], 3: [1]}}
    for n, want in expected.items():
        v = jv.F32Vectors(vec[:n])
        g = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=4, beamWidth=10, neighborOverflow=1.0, alpha=1.0).build(v)
        _, adj = g.level(0)
        for node, nbrs in want.items():
            assert sorted(int(x) for x in adj[node] if x >= 0) == nbrs, (n, node, adj[node].tolist(), nbrs)
        g.close()
        v.close()
