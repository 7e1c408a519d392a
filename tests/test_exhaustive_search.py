"""Filtered exhaustive top-k (jv_topk_bruteforce_ex) and exhaustive search (jv_exhaustive_search_batch, ExhaustiveSearcher), asserted
EXACTLY against the warp-order oracle (DESIGN §4.2a):

  - keys: for every storage kind and metric, the device's keys equal the oracle's top-k over all rows (jvo_scorer_topk, order 1) with
    the rejected rows and the rows below the threshold removed, padding included. Shared and per-query bitsets at densities all /
    50 % / 1 % / 0.05 % / one row / none, n not a multiple of 32 with every bit past n set, per-query strides longer than a bitset
    (their extra words set), a per-query batch mixing the whole tier (<= 16384 accepted rows) and the sampled tier, k = 1 and k above
    the accepted count, integer rows with duplicates (ties), PQ LUTs in shared and in global memory, NVQ, BQ at 1 / 5 / 40 words;
  - identity: no options, or an all-ones bitset at threshold 0, give jv_topk_bruteforce's keys byte for byte;
  - search: nodes, score bits, visited and reranked equal a host restatement (candidates = the oracle keys above, NodeQueue.rerank's
    take rule at rerankFloor, exact oracle scores, key order);
  - a filter the graph walk refuses (JV_ERR_OVERFLOW) is answered exactly, with recall 1 against numpy;
  - argument errors leave the outputs untouched; two host threads on shared handles give each call's answer made alone."""
import ctypes as C
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import oracle_lib as o
from oracle_lib import bp, fp, ip, lp, wp

pytestmark = pytest.mark.gpu

METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)
KEY_MIN = np.iinfo(np.int64).min
JV_ERR_INVALID, JV_ERR_UNSUPPORTED, JV_ERR_OVERFLOW = -2, -5, -6
DENSITIES = (1.0, 0.5, 0.01, 0.0005, "one", 0.0)


@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


@pytest.fixture(scope="module")
def nat(jv):
    from jvector_b200 import _native
    return _native


def key_scores(keys):
    s = (np.asarray(keys, np.int64) >> 32).astype(np.int32)
    return (s ^ ((s >> 31) & 0x7fffffff)).view(np.float32)


def key_nodes(keys):
    return ((~np.asarray(keys, np.int64)) & 0xffffffff).astype(np.int64)


def mask_for(rng, n, density):
    if density == "one":
        m = np.zeros(n, bool)
        m[rng.integers(n)] = True
        return m
    return np.ones(n, bool) if density == 1.0 else rng.random(n) < density


def bits_with_garbage(jv, mask):
    """mask [n] or [nq][n] -> accept words with every bit past n set; per query, a stride of the bitset's words + 3, the extra words
    all ones (none of it may be read as a row)"""
    bits = jv.pack_accept_bits(mask).copy()
    n = mask.shape[-1]
    if n % 32:
        bits[..., -1] |= np.uint32(0xffffffff ^ ((1 << (n % 32)) - 1))
    if mask.ndim == 2:
        bits = np.ascontiguousarray(np.concatenate([bits, np.full((mask.shape[0], 3), 0xffffffff, np.uint32)], axis=1))
    return bits


def options(nat, bits, threshold=0.0, floor=0.0):
    if bits is None:
        return nat.SearchOptions(None, 0, float(threshold), float(floor))
    return nat.SearchOptions(bits.ctypes.data, bits.shape[1] if bits.ndim == 2 else 0, float(threshold), float(floor))


def topk_ex(nat, vec, metric, queries, k, bits, threshold=0.0):
    lib = nat.load()
    keys = np.empty((len(queries), k), np.int64)
    opts = options(nat, bits, threshold)
    rc = lib.jv_topk_bruteforce_ex(vec._h, metric, fp(queries), len(queries), k, C.byref(opts), lp(keys))
    assert rc == 0, lib.jv_last_error()
    return keys


def oracle_all(oracle, scorer_for, queries, n):
    """every row's warp-order key per query, best first"""
    return [o.scorer_topk(oracle, scorer_for(q), n) for q in queries]


def want_keys(allk, masks, k, threshold=0.0):
    out = np.full((len(allk), k), KEY_MIN, np.int64)
    for i, keys in enumerate(allk):
        ok = masks[i if masks.ndim == 2 else slice(None)][key_nodes(keys)]
        if threshold > 0:
            ok &= key_scores(keys) >= np.float32(threshold)
        kept = keys[ok][:k]
        out[i, :len(kept)] = kept
    return out


def assert_keys(got, want, what):
    bad = np.flatnonzero((got != want).any(axis=1))
    assert len(bad) == 0, (what, "queries differ:", bad[:8].tolist(), "first bad rank", int(np.argmax(got[bad[0]] != want[bad[0]])) if len(bad) else None)


def check_filters(jv, nat, rng, vec, metric, queries, allk, n, what, k=50):
    """every shared density, a mixed per-query batch, a threshold, k = 1"""
    nq = len(queries)
    for d in DENSITIES:
        m = mask_for(rng, n, d)
        assert_keys(topk_ex(nat, vec, metric, queries, k, bits_with_garbage(jv, m)), want_keys(allk, m, k), (what, "shared", d))
    per = np.stack([mask_for(rng, n, DENSITIES[i % len(DENSITIES)]) for i in range(nq)])
    want = want_keys(allk, per, k)
    bits = bits_with_garbage(jv, per)
    assert_keys(topk_ex(nat, vec, metric, queries, k, bits), want, (what, "per query"))
    assert_keys(topk_ex(nat, vec, metric, queries, 1, bits), want[:, :1], (what, "per query, k = 1"))
    thr = float(key_scores(allk[0][min(n - 1, 3000)]))  # about 3000 rows of query 0 pass: some queries keep fewer than k
    if thr <= 0:  # integer rows under DOT_PRODUCT score below 0: a threshold only applies above 0
        return
    half = rng.random(n) < 0.5
    assert_keys(topk_ex(nat, vec, metric, queries, k, bits_with_garbage(jv, half), thr), want_keys(allk, half, k, thr), (what, "threshold"))
    assert_keys(topk_ex(nat, vec, metric, queries, k, None, thr), want_keys(allk, np.ones(n, bool), k, thr), (what, "threshold alone"))


# ------------------------------------------------------------------------------------------------ keys, every kind
def test_f32_keys(jv, nat, oracle):
    rng = np.random.default_rng(11)
    n, dim = 40003, 37  # sampled tier for the dense filters; n % 32 = 3
    data = o.random_unit_vectors(rng, n, dim)
    queries = o.random_unit_vectors(rng, 6, dim)
    queries[0] = data[n - 1]
    vec = jv.F32Vectors(data)
    for metric in METRICS:
        allk = oracle_all(oracle, lambda q: oracle.jvo_scorer_f32(metric, fp(data), n, dim, fp(q)), queries, n)
        check_filters(jv, nat, rng, vec, metric, queries, allk, n, ("f32", metric))
        # k above every accepted count: 20 accepted rows, 2048 keys, the rest INT64_MIN
        m = np.zeros(n, bool)
        m[rng.choice(n, 20, replace=False)] = True
        got = topk_ex(nat, vec, metric, queries, 2048, bits_with_garbage(jv, m))
        assert_keys(got, want_keys(allk, m, 2048), ("f32 pads", metric))
        assert (got[:, 20:] == KEY_MIN).all()
    vec.close()


@pytest.mark.parametrize("n", [5000, 20011])  # whole tier for every filter / sampled for the dense ones
def test_ties_go_to_the_smaller_id(jv, nat, oracle, n):
    rng = np.random.default_rng(n)
    dim = 12
    data = rng.integers(-4, 5, (n, dim)).astype(np.float32)
    data[np.abs(data).sum(1) == 0, 0] = 1.0
    data[n - 64:] = data[:64]
    queries = rng.integers(-4, 5, (4, dim)).astype(np.float32)
    queries[0] = data[5]
    vec = jv.F32Vectors(data)
    for metric in METRICS:
        allk = oracle_all(oracle, lambda q: oracle.jvo_scorer_f32(metric, fp(data), n, dim, fp(q)), queries, n)
        check_filters(jv, nat, rng, vec, metric, queries, allk, n, ("ties", n, metric), k=100)
    vec.close()


@pytest.mark.parametrize("dim,M,n", [(64, 16, 40003), (256, 256, 20011)])  # 16 KB LUT in shared memory / 256 KB LUT read from global memory
def test_pq_keys(jv, nat, oracle, dim, M, n):
    rng = np.random.default_rng(dim + M)
    data = o.random_unit_vectors(rng, n, dim)
    cb, _, _ = o.train_pq_numpy(rng, data[:2000], M, 256, iters=1)
    codes = jv.pq_encode_all(data, cb, M, 256, None)
    queries = o.random_unit_vectors(rng, 4, dim)
    pqv = jv.PQVectors(codes, cb, dim, 256)
    for metric in METRICS:
        allk = oracle_all(oracle, lambda q: oracle.jvo_scorer_pq(metric, fp(cb), M, 256, dim, None, bp(codes), n, fp(q)), queries, n)
        check_filters(jv, nat, rng, pqv, metric, queries, allk, n, ("pq", M, metric), k=40)
    pqv.close()


def test_nvq_keys(jv, nat, oracle):
    rng = np.random.default_rng(5)
    n, dim, nsub = 20011, 64, 2
    data = o.random_unit_vectors(rng, n, dim)
    mean = data.mean(0).astype(np.float32)
    params, bys = jv.nvq_encode_all(data, mean, nsub, True)
    queries = o.random_unit_vectors(rng, 4, dim)
    nv = jv.NVQVectors(bys, params, mean, nsub)
    for metric in METRICS:
        allk = oracle_all(oracle, lambda q: oracle.jvo_scorer_nvq(metric, fp(mean), dim, nsub, fp(params), bp(bys), n, fp(q)), queries, n)
        check_filters(jv, nat, rng, nv, metric, queries, allk, n, ("nvq", metric), k=30)
    nv.close()


@pytest.mark.parametrize("dim", [64, 300, 2560])  # W = 1, 5 (topk_filter_bq_kernel<4 | 8>), 40 (topk_filter_kernel<BQ>)
def test_bq_keys(jv, nat, oracle, dim):
    rng = np.random.default_rng(dim)
    n = 20011
    data = rng.standard_normal((n, dim)).astype(np.float32)
    words = jv.bq_encode_all(data)
    queries = rng.standard_normal((4, dim)).astype(np.float32)
    bqv = jv.BQVectors(words, dim)
    allk = oracle_all(oracle, lambda q: oracle.jvo_scorer_bq(wp(words), n, dim, fp(q)), queries, n)
    check_filters(jv, nat, rng, bqv, o.COSINE, queries, allk, n, ("bq", dim), k=30)
    bqv.close()


# ------------------------------------------------------------------------------------------------ identity with jv_topk_bruteforce
def test_identity_with_topk_bruteforce(jv, nat):
    rng = np.random.default_rng(3)
    n, dim = 20000, 128  # BQ: even word count, n >= 4096: jv_topk_bruteforce takes the tensor-core contraction
    data = o.random_unit_vectors(rng, n, dim)
    queries = o.random_unit_vectors(rng, 5, dim)
    cb, _, _ = o.train_pq_numpy(rng, data[:2000], 16, 256, iters=1)
    sets = [(jv.F32Vectors(data), METRICS), (jv.PQVectors(jv.pq_encode_all(data, cb, 16, 256, None), cb, dim, 256), METRICS),
            (jv.BQVectors(jv.bq_encode_all(data), dim), (o.COSINE,))]
    lib = nat.load()
    for vec, metrics in sets:
        for metric in metrics:
            want = jv.topk_bruteforce(vec, metric, queries, 64)[2]
            got = np.empty_like(want)
            assert lib.jv_topk_bruteforce_ex(vec._h, metric, fp(queries), 5, 64, None, lp(got)) == 0
            assert np.array_equal(got, want)
            ones = np.ones(n, bool)
            assert np.array_equal(topk_ex(nat, vec, metric, queries, 64, jv.pack_accept_bits(ones)), want)
            assert np.array_equal(topk_ex(nat, vec, metric, queries, 64, jv.pack_accept_bits(np.ones((5, n), bool))), want)
            assert np.array_equal(jv.topk_bruteforce(vec, metric, queries, 64, acceptOrds=ones)[2], want)
        vec.close()


# ------------------------------------------------------------------------------------------------ exhaustive search against a model
def model_search(cand, topK, exact_for=None, floor=0.0):
    """one query: candidates (sorted keys, KEY_MIN padded) -> (nodes, scores, reranked) as jv_exhaustive_search_batch defines them"""
    nodes = np.full(topK, -1, np.int32)
    scores = np.zeros(topK, np.float32)
    valid = cand != KEY_MIN
    if exact_for is None:
        c = cand[valid][:topK]
        nodes[:len(c)], scores[:len(c)] = key_nodes(c), key_scores(c)
        return nodes, scores, 0
    take = valid & ((np.arange(len(cand)) == 0) | (key_scores(cand) >= np.float32(floor)))
    tn = key_nodes(cand[take])
    ex = o.keys_of(np.array([exact_for(int(f)) for f in tn], np.float32), tn)
    ex = np.sort(ex)[::-1][:topK]
    nodes[:len(ex)], scores[:len(ex)] = key_nodes(ex), key_scores(ex)
    return nodes, scores, int(take.sum())


def assert_model(res, cand, topK, exact_for, floor, visited, what):
    rr = 0
    for i in range(len(cand)):
        wn, ws, r = model_search(cand[i], topK, None if exact_for is None else (lambda f, i=i: exact_for(i, f)), floor)
        assert np.array_equal(res.nodes[i], wn), (what, i, res.nodes[i][:10], wn[:10])
        assert np.array_equal(res.scores[i].view(np.int32), ws.view(np.int32)), (what, i)
        rr += r
    assert res.visitedCount == visited, (what, res.visitedCount, visited)
    assert res.rerankedCount == rr, (what, res.rerankedCount, rr)
    assert res.expandedCount == 0 and res.expandedCountBaseLayer == 0


def test_search_against_model(jv, nat, oracle):
    rng = np.random.default_rng(17)
    n, dim, nq = 20011, 64, 6
    data = o.random_unit_vectors(rng, n, dim)
    queries = o.random_unit_vectors(rng, nq, dim)
    cb, _, _ = o.train_pq_numpy(rng, data[:2000], 16, 256, iters=1)
    codes = jv.pq_encode_all(data, cb, 16, 256, None)
    mean = data.mean(0).astype(np.float32)
    params, bys = jv.nvq_encode_all(data, mean, 2, True)
    pqv, f32v, nvv = jv.PQVectors(codes, cb, dim, 256), jv.F32Vectors(data), jv.NVQVectors(bys, params, mean, 2)
    searcher = jv.ExhaustiveSearcher()
    per = np.stack([mask_for(rng, n, DENSITIES[i % len(DENSITIES)]) for i in range(nq)])
    shared = rng.random(n) < 0.01
    for metric in METRICS:
        allk = oracle_all(oracle, lambda q: oracle.jvo_scorer_pq(metric, fp(cb), 16, 256, dim, None, bp(codes), n, fp(q)), queries, n)
        rerankers = {"f32": (f32v, lambda q: oracle.jvo_scorer_f32(metric, fp(data), n, dim, fp(q))),
                     "nvq": (nvv, lambda q: oracle.jvo_scorer_nvq(metric, fp(mean), dim, 2, fp(params), bp(bys), n, fp(q)))}
        thr = float(key_scores(allk[0][2000]))
        for name, (rv, mk) in rerankers.items():
            scorers = []
            for q in queries:
                sf = mk(q)
                oracle.jvo_scorer_set_order(sf, 1)
                scorers.append(sf)
            exact_for = lambda i, f: oracle.jvo_scorer_score(scorers[i], f)
            for acc, masks in ((per, per), (shared, shared), (None, np.ones(n, bool))):
                visited = int(masks.sum()) if masks.ndim == 2 else int(masks.sum()) * nq
                for topK, rerankK, floor, t in ((10, 40, 0.0, 0.0), (10, 40, 2.0, 0.0), (10, 40, None, 0.0), (20, 20, 0.0, thr), (5, 30, None, thr)):
                    cand = want_keys(allk, masks, rerankK, t)
                    if floor is None:  # a floor between the candidates' scores: some are taken, some are not
                        floor = float(np.median(key_scores(cand[cand != KEY_MIN]))) if (cand != KEY_MIN).any() else 0.5
                    res = searcher.search(pqv, queries, metric, topK, rerankK, reranker=rv, threshold=t, rerankFloor=floor, acceptOrds=acc)
                    assert_model(res, cand, topK, exact_for, floor, visited, (name, metric, topK, rerankK, floor, t, acc is None))
                    if name == "f32" and floor == 0.0:
                        res = searcher.search(pqv, queries, metric, topK, rerankK, threshold=t, acceptOrds=acc)
                        assert_model(res, cand, topK, None, 0.0, visited, ("no reranker", metric, topK, t))
            for sf in scorers:
                oracle.jvo_scorer_free(sf)
    for v in (pqv, f32v, nvv):
        v.close()


# ------------------------------------------------------------------------------------------------ the case the walk refuses
def test_selective_filter_the_walk_refuses(jv, nat, oracle):
    rng = np.random.default_rng(29)
    n, dim, nq = 20000, 32, 8
    data = o.random_unit_vectors(rng, n, dim)
    queries = o.random_unit_vectors(rng, nq, dim)
    vec = jv.F32Vectors(data)
    gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60).build(vec)
    acc = np.zeros(n, bool)
    acc[rng.choice(n, 10, replace=False)] = True  # 0.05 %: fewer accepted rows than rerankK, so the walk's list fills with rejected ones
    with pytest.raises(jv.JVectorB200Error) as e:
        jv.GraphSearcher(gi).search(vec, queries, o.DOT_PRODUCT, 10, 20, acceptOrds=acc)
    assert e.value.code == JV_ERR_OVERFLOW
    res = jv.ExhaustiveSearcher().search(vec, queries, o.DOT_PRODUCT, 10, 20, acceptOrds=acc)
    allk = oracle_all(oracle, lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q)), queries, n)
    assert_model(res, want_keys(allk, acc, 20), 10, None, 0.0, 10 * nq, "walk refused")
    ids = np.flatnonzero(acc)
    truth = ids[np.argsort(-(queries @ data[ids].T), axis=1, kind="stable")]
    assert all(set(res.nodes[i]) == set(truth[i]) for i in range(nq))  # recall 1.0: all 10 accepted rows, the only ones there are
    gi.close()
    vec.close()


# ------------------------------------------------------------------------------------------------ refusals
def test_errors_leave_outputs_untouched(jv, nat):
    rng = np.random.default_rng(2)
    n, dim, nq = 1000, 16, 3
    data = o.random_unit_vectors(rng, n, dim)
    queries = o.random_unit_vectors(rng, nq, dim)
    vec, small = jv.F32Vectors(data), jv.F32Vectors(data[:999])
    cb = o.train_pq_numpy(rng, data, 4, 16, iters=1)[0]
    pqv = jv.PQVectors(jv.pq_encode_all(data, cb, 4, 16, None), cb, dim, 16)
    wide = jv.F32Vectors(o.random_unit_vectors(rng, n, dim + 1))
    lib = nat.load()
    words = (n + 31) // 32
    bits = np.full((nq, words), 0xffffffff, np.uint32)

    def ex(k=10, opts=None, nq_=nq):
        keys = np.full((nq, max(k, 1)), 7, np.int64)
        rc = lib.jv_topk_bruteforce_ex(vec._h, o.DOT_PRODUCT, fp(queries), nq_, k, C.byref(opts) if opts else None, lp(keys))
        assert (keys == 7).all()
        return rc, lib.jv_last_error()

    def search(topK=5, rerankK=10, reranker=None, opts=None, nq_=nq):
        nodes = np.full((nq, max(topK, 1)), 7, np.int32)
        scores = np.full((nq, max(topK, 1)), 7, np.float32)
        st = nat.SearchStats()
        rc = lib.jv_exhaustive_search_batch(vec._h, reranker._h if reranker else None, o.DOT_PRODUCT, fp(queries), nq_, topK, rerankK,
                                            C.byref(opts) if opts else None, ip(nodes), fp(scores), C.byref(st))
        assert (nodes == 7).all() and (scores == 7).all()
        return rc, lib.jv_last_error()

    short = nat.SearchOptions(bits.ctypes.data, words - 1, 0.0, 0.0)
    assert ex(k=0) == (JV_ERR_INVALID, b"topk_bruteforce_ex: bad arguments")
    assert ex(nq_=0) == (JV_ERR_INVALID, b"topk_bruteforce_ex: bad arguments")
    assert ex(k=2049)[0] == JV_ERR_INVALID
    assert ex(opts=short) == (JV_ERR_INVALID, b"topk_bruteforce_ex: accept_stride_words shorter than one bitset")
    assert ex(opts=nat.SearchOptions(bits.ctypes.data, 0, 0.0, 0.5)) == (JV_ERR_INVALID, b"topk_bruteforce_ex: rerank_floor must be 0 (nothing is reranked)")
    assert ex(opts=nat.SearchOptions(None, 0, -1.0, 0.0))[0] == JV_ERR_INVALID
    assert search(topK=0) == (JV_ERR_INVALID, b"exhaustive_search: need 1 <= topK <= rerankK")
    assert search(topK=10, rerankK=5) == (JV_ERR_INVALID, b"exhaustive_search: need 1 <= topK <= rerankK")
    assert search(nq_=0) == (JV_ERR_INVALID, b"exhaustive_search: bad arguments")
    assert search(opts=short) == (JV_ERR_INVALID, b"exhaustive_search: accept_stride_words shorter than one bitset")
    assert search(reranker=small) == (JV_ERR_INVALID, b"exhaustive_search: reranker shape mismatch")
    assert search(reranker=wide) == (JV_ERR_INVALID, b"exhaustive_search: reranker shape mismatch")
    assert search(reranker=pqv)[0] == JV_ERR_UNSUPPORTED
    for v in (vec, small, pqv, wide):
        v.close()


# ------------------------------------------------------------------------------------------------ host threads
def test_two_threads_on_shared_handles(jv, nat):
    rng = np.random.default_rng(23)
    n, dim, nq = 30000, 48, 40
    data = o.random_unit_vectors(rng, n, dim)
    queries = o.random_unit_vectors(rng, nq, dim)
    cb, _, _ = o.train_pq_numpy(rng, data[:2000], 12, 256, iters=1)
    codes = jv.pq_encode_all(data, cb, 12, 256, None)
    per = rng.random((nq, n)) < np.linspace(0.0005, 0.6, nq)[:, None]
    shared = rng.random(n) < 0.2

    def calls(pqv, f32v):
        s = jv.ExhaustiveSearcher()
        return [lambda: s.search(pqv, queries, o.DOT_PRODUCT, 10, 50, reranker=f32v, acceptOrds=per, rerankFloor=0.5),
                lambda: jv.topk_bruteforce(f32v, o.EUCLIDEAN, queries, 30, acceptOrds=shared, threshold=0.3)[2]]

    def flat(r):
        return (r.nodes, r.scores.view(np.int32), r.visitedCount, r.rerankedCount) if hasattr(r, "nodes") else (r,)

    pqv, f32v = jv.PQVectors(codes, cb, dim, 256), jv.F32Vectors(data)
    want = [flat(c()) for c in calls(pqv, f32v)]
    pqv.close()
    f32v.close()
    pqv, f32v = jv.PQVectors(codes, cb, dim, 256), jv.F32Vectors(data)
    cs = calls(pqv, f32v)
    start = threading.Barrier(4)

    def run(c):
        start.wait(timeout=120)
        return flat(c())

    with ThreadPoolExecutor(max_workers=4) as pool:
        got = [f.result() for f in [pool.submit(run, c) for c in cs + cs]]
    for g, w in zip(got, want + want):
        assert all(np.array_equal(a, b) for a, b in zip(g, w))
    pqv.close()
    f32v.close()
