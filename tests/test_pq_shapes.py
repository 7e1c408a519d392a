"""Every PQ kernel at codebook shapes other than k = 256 with even sub-spaces: k from 1 to 256, M = 1, 2 and 3 (mod 4), one float per
sub-space, and uneven splits whose 8-float sub-spaces sit at offsets that are (or are not) multiples of 4, which decides between
prepare_blob's vector branch and its generic one (scorers.cuh). Each kernel is checked against a reference that does not come from
the device: the oracle's encoder and warp-order scorers, or the host's exact restatement of a kernel's fmaf chains
(oracle_lib.pq_lut_exact, pq_pair_table_exact).

CPU: the host's exact fmaf, LUT and pair table against Fraction arithmetic, float64 and the oracle (its warp-order ADC scores equal
the host LUT's bit for bit); the triangular index for every k; the oracle encoder's ties; the build model's pair scores.
GPU (-m gpu), per shape: encode; LUT; every score entry point under every metric; the pair table and code-vs-code scores, with and
without the table (and for every k from 1 to 256); brute-force top-k on the whole-set and sampled paths; the plain, reranked and
FusedPQ walks with the LUT in shared memory, in L2 and split. At four shapes, the step-wise build, an add and a removal equal the
models row for row over a pair table computed on the host; a shape whose LUT does not fit the prune is refused."""
import functools
from fractions import Fraction

import numpy as np
import pytest

import graph_model as gm
import oracle_lib as o
from oracle_lib import bp, fp, ip

METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)
F32 = np.float32
JV_ERR_UNSUPPORTED = -5

# (id, dim, M, k, centred)
SHAPES = [
    ("d12_m5_k1", 12, 5, 1, False),            # one centroid: one LUT entry and one pair entry per sub-space; M = 1 (mod 4)
    ("d24_m7_k2_cen", 24, 7, 2, True),         # two distinct centroids; M = 3 (mod 4), sub-spaces of 4 and 3
    ("d45_m15_k16_cen", 45, 15, 16, True),     # M = 3 (mod 4), sub-spaces of 3
    ("d50_m11_k40", 50, 11, 40, False),        # M = 3 (mod 4), sub-spaces of 5 and 4
    ("d30_m10_k3_cen", 30, 10, 3, True),       # three centroids, the last a copy of the first; M = 2 (mod 4)
    ("d33_m33_k16", 33, 33, 16, False),        # M = dim: one float per sub-space
    ("d101_m12_k33_cen", 101, 12, 33, True),   # 9 x 5 then 8 x 7 at offsets 45, 53, ... (1 mod 4): the generic branch
    ("d100_m12_k100", 100, 12, 100, False),    # 9 x 4 then 8 x 8 at offsets 36, 44, ... (0 mod 4): the vector branch
    ("d64_m14_k255_cen", 64, 14, 255, True),   # M = 2 (mod 4), sub-spaces of 5 and 4
    ("d768_m96_k256_cen", 768, 96, 256, True),  # the common case
]
SHAPE_IDS = [s[0] for s in SHAPES]
N, NQ = 2000, 32


# ------------------------------------------------------------------------------------------------ worlds
@functools.lru_cache(maxsize=None)
def host_world(name):
    """latent rows and queries, codebooks trained on the rows (with duplicated centroids, so encodes tie), oracle codes"""
    from test_build_steps import latent_rows
    _, dim, M, k, centred = next(s for s in SHAPES if s[0] == name)
    rng = np.random.default_rng(sum(map(ord, name)))
    rows = latent_rows(rng, N + NQ, dim)
    data, queries = np.ascontiguousarray(rows[:N]), np.ascontiguousarray(rows[N:])
    cen = data.mean(0).astype(F32) if centred else None
    cb, sizes, offsets = o.train_pq_numpy(rng, data - cen if centred else data, M, k, iters=2)
    for m in range(M):  # centroid k - 1 repeats centroid 0 and k - 2 repeats 1: ties that only the lower index may win. At k = 2 the
        sz, off = int(sizes[m]), int(offsets[m])  # two centroids stay distinct, or the shape would have one centroid in effect
        book = cb[k * off:k * (off + sz)].reshape(k, sz)
        if k >= 3:
            book[k - 1] = book[0]
        if k >= 4:
            book[k - 2] = book[1]
    codes = o.encode_pq(o.load(), cb, sizes, offsets, M, k, cen, data)
    queries[0] = data[7]  # a query equal to a row
    return dict(dim=dim, M=M, k=k, cen=cen, data=data, queries=queries, cb=cb, sizes=sizes, offsets=offsets, codes=codes)


def warp_adc_raw(lut, k, codes):
    """score_pq_codes' sum (the oracle's warp_pq_score): word j of a code row to lane j mod 8, a tail code m to lane m - 4 (M / 4),
    each lane in increasing m, then the xor butterfly 4, 2, 1. codes [n][M] -> float32 [n]"""
    n, M = codes.shape
    M4 = M >> 2
    lanes = np.zeros((8, n), F32)
    for m in range(M):
        g = ((m >> 2) if m < 4 * M4 else m - 4 * M4) & 7
        lanes[g] = (lanes[g] + lut[m * k + codes[:, m].astype(np.int64)]).astype(F32)
    for sh in (4, 2, 1):
        lanes = (lanes + lanes[np.arange(8) ^ sh]).astype(F32)
    return lanes[0]


def warp_scorer(oracle, w, metric, codes=None):
    codes = w["codes"] if codes is None else codes
    return lambda q: oracle.jvo_scorer_pq(metric, fp(w["cb"]), w["M"], w["k"], w["dim"], fp(w["cen"]), bp(codes), codes.shape[0], fp(q))


def warp_scores(oracle, w, metric, q, ids):
    sf = warp_scorer(oracle, w, metric)(q)
    oracle.jvo_scorer_set_order(sf, 1)
    out = np.array([oracle.jvo_scorer_score(sf, int(i)) for i in ids], F32)
    oracle.jvo_scorer_free(sf)
    return out


def fp32_bound(terms, depth):
    """the error bound of an fp32 sum of `depth` products or squares, in any order: (2 depth + 2) 2^-24 sum |terms|, plus underflow"""
    return (2 * depth + 2) * 2.0 ** -24 * np.abs(terms).sum(-1) + depth * 2.0 ** -149


def bits_equal(got, want, what):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    bad = np.flatnonzero(got.view(np.int32).ravel() != want.view(np.int32).ravel())
    assert len(bad) == 0, (what, "entries differ", len(bad), bad[:5].tolist(), got.ravel()[bad[:3]].tolist(), want.ravel()[bad[:3]].tolist())


# ------------------------------------------------------------------------------------------------ CPU
def test_fma_f32_rounds_once():
    rng = np.random.default_rng(5)
    a = rng.standard_normal(4000).astype(F32)
    b = rng.standard_normal(4000).astype(F32)
    c = rng.standard_normal(4000).astype(F32)
    # 2^30 + 128 + 64 (1 - 2^-46): float64 rounds it to the midpoint 2^30 + 192, whose tie would go to the even 2^30 + 256, but the
    # exact value lies below it; and 1 + 2^-23 + 2^-24, exactly a midpoint (ties to even)
    a[:2] = (8 * (1 + 2.0 ** -23), 1.0)
    b[:2] = (8 * (1 - 2.0 ** -23), 1 + 2.0 ** -23)
    c[:2] = (2.0 ** 30 + 128, 2.0 ** -24)
    got = o.fma_f32(a, b, c)
    assert got[0] == F32(2.0 ** 30 + 128) and got[1] == F32(1 + 2.0 ** -22)
    for i in range(len(a)):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        r = got[i]
        nb = (np.nextafter(r, F32(-np.inf)), np.nextafter(r, F32(np.inf)))
        err = abs(Fraction(float(r)) - exact)
        assert all(err <= abs(Fraction(float(x)) - exact) for x in nb), (i, a[i], b[i], c[i], r)


@pytest.mark.parametrize("shape", SHAPE_IDS)
def test_host_lut_is_the_warp_oracles(oracle, shape):
    # the exact LUT restated on the host gives, through score_pq_codes' order, the warp-order oracle's ADC bits (whose LUT is its own
    # sequential fmaf chain), and stays within the fp32 bound of a float64 LUT
    w = host_world(shape)
    dim, M, k, cen = w["dim"], w["M"], w["k"], w["cen"]
    for q in w["queries"][:3]:
        qc = (q - cen).astype(F32) if cen is not None else q
        for metric in (o.EUCLIDEAN, o.DOT_PRODUCT):
            lut = o.pq_lut_exact(w["cb"], dim, M, k, cen, q, metric)
            for m in range(M):
                sz, off = int(w["sizes"][m]), int(w["offsets"][m])
                book = w["cb"][k * off:k * (off + sz)].reshape(k, sz).astype(np.float64)
                x = qc[off:off + sz].astype(np.float64)
                terms = (book - x) ** 2 if metric == o.EUCLIDEAN else book * x
                assert (np.abs(lut[m * k:(m + 1) * k] - terms.sum(1)) <= fp32_bound(terms, 2 * sz)).all(), (shape, metric, m)
            raw = warp_adc_raw(lut, k, w["codes"][:300])
            want = warp_scores(oracle, w, metric, q, range(300))
            got = (F32(1) / (F32(1) + raw)) if metric == o.EUCLIDEAN else ((F32(1) + raw) / F32(2))
            bits_equal(got.astype(F32), want, (shape, metric))


@pytest.mark.parametrize("shape", SHAPE_IDS)
def test_host_pair_table_against_oracle(oracle, shape):
    # the exact table within the fp32 bound of the oracle's (separate multiply and add) and of float64, entry by entry
    w = host_world(shape)
    dim, M, k = w["dim"], w["M"], w["k"]
    block = k * (k + 1) // 2
    iu, ju = np.triu_indices(k)
    for metric in (o.EUCLIDEAN, o.DOT_PRODUCT):
        got = o.pq_pair_table_exact(w["cb"], dim, M, k, metric)
        want = np.empty(M * block, F32)
        oracle.jvo_pq_pair_table(fp(w["cb"]), ip(w["sizes"]), ip(w["offsets"]), M, k, metric, fp(want))
        for m in range(M):
            sz, off = int(w["sizes"][m]), int(w["offsets"][m])
            book = w["cb"][k * off:k * (off + sz)].reshape(k, sz).astype(np.float64)
            terms = (book[iu] - book[ju]) ** 2 if metric == o.EUCLIDEAN else book[iu] * book[ju]
            bound = fp32_bound(terms, 2 * sz)
            g, t = got[m * block:(m + 1) * block], want[m * block:(m + 1) * block]
            assert (np.abs(g - terms.sum(1)) <= bound).all() and (np.abs(g.astype(np.float64) - t) <= 2 * bound).all(), (shape, metric, m)
            if metric == o.EUCLIDEAN and k >= 3:
                assert g[gm.tri_index(0, k - 1, k)] == 0  # duplicated centroids


def tri_invert(t, k):
    """pq_pair_table_kernel's inversion of a flat index t into (i, j): a float64 square root, then the two fix-up loops"""
    t = np.asarray(t, np.int64)
    i = ((2.0 * k + 1.0 - np.sqrt((2.0 * k + 1.0) * (2.0 * k + 1.0) - 8.0 * t)) / 2.0).astype(np.int64)
    while ((i > 0) & (i * k - i * (i - 1) // 2 > t)).any():
        i = np.where((i > 0) & (i * k - i * (i - 1) // 2 > t), i - 1, i)
    while (((i + 1) * k - (i + 1) * i // 2) <= t).any():
        i = np.where(((i + 1) * k - (i + 1) * i // 2) <= t, i + 1, i)
    return i, i + (t - (i * k - i * (i - 1) // 2))


def test_triangular_index_for_every_k():
    # tri_index (scorers.cuh, graph_model) and the kernel's inversion agree with the row-order upper triangle at every k
    for k in range(1, 257):
        iu, ju = np.triu_indices(k)
        t = np.arange(len(iu))
        assert np.array_equal(gm.tri_index(iu, ju, k), t) and np.array_equal(gm.tri_index(ju, iu, k), t), k
        i, j = tri_invert(t, k)
        assert np.array_equal(i, iu) and np.array_equal(j, ju), k


@pytest.mark.parametrize("shape", SHAPE_IDS)
def test_oracle_encode_ties_and_model_pair_scores(oracle, shape):
    w = host_world(shape)
    dim, M, k, codes = w["dim"], w["M"], w["k"], w["codes"]
    assert (codes < k).all()
    if k >= 3:  # a tie goes to the first minimum: the repeated centroids are never chosen
        assert not (codes == k - 1).any() and (k < 4 or not (codes == k - 2).any())
    # every sub-space uses at least two codes (one at k = 1): the shape's centroids really are distinct where they should be
    assert all(len(np.unique(codes[:, m])) >= min(k, 2) for m in range(M)), shape
    rng = np.random.default_rng(k)
    a, b = rng.integers(0, N, 40), rng.integers(0, N, 40)
    for metric in METRICS:
        table = o.pq_pair_table_exact(w["cb"], dim, M, k, metric)
        got = np.diagonal(gm.pair_scores(metric, table, k, codes[a], codes[b]))
        want = np.array([oracle.jvo_pq_diversity_table(metric, fp(table), M, k, bp(codes[x]), bp(codes[y])) for x, y in zip(a, b)], F32)
        bound = diversity_bound(metric, table, k, codes[a], codes[b])
        assert (np.abs(got.astype(np.float64) - want) <= bound).all(), (shape, metric, np.abs(got - want).max(), bound.min())


def diversity_bound(metric, table, k, ca, cb):
    """how far two summation orders of the same code-vs-code score can be apart, per pair (ca[i], cb[i]): pair_pq_table's (lanes
    then a butterfly, depth <= M + 5) and jvo_pq_diversity_table's (sequential). Each fp32 sum of the M table entries t is within
    (M + 5) 2^-24 sum |t| of the exact sum; the cosine norms (sums of squares) are within (M + 5) 2^-24 relative; the score map,
    the square root and the divide add a few roundings of a score of magnitude <= 1 + |sum|"""
    M = ca.shape[1]
    u = 2.0 ** -24
    T = np.asarray(table, F32).reshape(M, -1).astype(np.float64)

    def entries(x, y):
        return np.stack([T[m][gm.tri_index(x[:, m], y[:, m], k)] for m in range(M)], 1)

    t = entries(ca, cb)
    s, e = t.sum(1), 2 * (M + 5) * u * np.abs(t).sum(1)  # e: the two orders' sums, apart
    if metric == o.EUCLIDEAN:  # 1 / (1 + s), s >= 0: the map shrinks differences
        return e + 8 * u
    if metric == o.DOT_PRODUCT:  # (1 + s) / 2
        return e / 2 + 8 * u * (1 + np.abs(s))
    norms = np.sqrt(entries(ca, ca).sum(1) * entries(cb, cb).sum(1))
    return (e + 2 * (M + 8) * u * np.abs(s)) / norms / 2 + 8 * u


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


@pytest.fixture(scope="module", params=SHAPE_IDS)
def world(request, jv):
    w = dict(host_world(request.param), name=request.param)
    w["pqv"] = jv.PQVectors(w["codes"], w["cb"], w["dim"], w["k"], w["cen"])
    w["f32"] = jv.F32Vectors(w["data"])
    yield w
    w["pqv"].close()
    w["f32"].close()


@pytest.mark.gpu
def test_encode(jv, world):
    w = world
    args = (w["cb"], w["M"], w["k"], w["cen"])
    assert np.array_equal(jv.pq_encode_all(w["data"], *args), w["codes"]), w["name"]
    assert np.array_equal(jv.pq_encode_all(w["f32"], *args), w["codes"]), (w["name"], "resident")


@pytest.mark.gpu
def test_lut_and_score_entry_points(jv, oracle, world):
    w = world
    dim, M, k, cen, pqv = w["dim"], w["M"], w["k"], w["cen"], w["pqv"]
    rng = np.random.default_rng(M * k)
    queries = w["queries"][:4]
    ids = rng.permutation(N)[:500].astype(np.int32)
    offsets = np.array([0, 120, 120, 300, 500], np.int32)  # query 1 scores nothing
    for metric in METRICS:
        want = [warp_scores(oracle, w, metric, q, ids) for q in queries]
        qb = jv.QueryBatch(pqv, queries, metric)
        step = qb.score_step(ids, offsets)
        multi = jv.score_multi(pqv, metric, queries, ids, offsets)
        for i, q in enumerate(queries):
            sf = pqv.score_function_for(q, metric)
            bits_equal(sf.partial_sums(), o.pq_lut_exact(w["cb"], dim, M, k, cen, q, o.EUCLIDEAN if metric == o.EUCLIDEAN else o.DOT_PRODUCT),
                       (w["name"], metric, "LUT", i))
            bits_equal(sf.similarityToBatch(ids), want[i], (w["name"], metric, "similarityToBatch", i))
            sf.close()
            lo, hi = offsets[i], offsets[i + 1]
            bits_equal(step[lo:hi], want[i][lo:hi], (w["name"], metric, "score_step", i))
            bits_equal(multi[lo:hi], want[i][lo:hi], (w["name"], metric, "score_multi", i))
            bits_equal(qb.score_one(i, ids[:64]), want[i][:64], (w["name"], metric, "score_one", i))
        qb.close()


def check_pairs(jv, oracle, pqv, codes, cb, dim, M, k, cen, a, b, what):
    """pair_table(metric) equals the host's exact table; diversity_scores with the table (pair_pq_table) and without it (pair_pq, a
    twin data set with the same global centroid) equal pair_scores over that table bit for bit, and jvo_pq_diversity_table within
    diversity_bound"""
    twin = jv.PQVectors(codes, cb, dim, k, cen)
    for metric in METRICS:
        table = o.pq_pair_table_exact(cb, dim, M, k, metric)
        direct = twin.diversity_scores(a, b, metric)
        pqv.build_pair_table(metric)
        bits_equal(pqv.pair_table(metric), table, what + (metric, "pair table"))
        got = pqv.diversity_scores(a, b, metric)
        want = np.diagonal(gm.pair_scores(metric, table, k, codes[a], codes[b]))
        bits_equal(got, want, what + (metric, "pair_pq_table"))
        bits_equal(direct, want, what + (metric, "pair_pq"))
        seq = np.array([oracle.jvo_pq_diversity_table(metric, fp(table), M, k, bp(codes[x]), bp(codes[y])) for x, y in zip(a, b)], F32)
        assert (np.abs(got.astype(np.float64) - seq) <= diversity_bound(metric, table, k, codes[a], codes[b])).all(), what + (metric,)
    twin.close()


@pytest.mark.gpu
def test_pair_table_and_pair_scores(jv, oracle, world):
    w = world
    rng = np.random.default_rng(w["k"])
    a, b = rng.integers(0, N, 300).astype(np.int32), rng.integers(0, N, 300).astype(np.int32)
    b[:10] = a[:10]
    pqv = jv.PQVectors(w["codes"], w["cb"], w["dim"], w["k"], w["cen"])  # no table yet
    check_pairs(jv, oracle, pqv, w["codes"], w["cb"], w["dim"], w["M"], w["k"], w["cen"], a, b, (w["name"],))
    pqv.close()


@pytest.mark.gpu
def test_pair_table_for_every_k(jv, oracle):
    # the kernel's triangular inversion and tri_index at every k from 1 to 256: 3 sub-spaces of 2, 2 and 1 floats
    rng = np.random.default_rng(256)
    dim, M, n = 5, 3, 96
    for k in range(1, 257):
        cb = rng.standard_normal(k * dim).astype(F32)
        codes = rng.integers(0, k, (n, M)).astype(np.uint8)
        codes[0] = k - 1
        a, b = rng.integers(0, n, 64).astype(np.int32), rng.integers(0, n, 64).astype(np.int32)
        a[0], b[1] = 0, 0
        pqv = jv.PQVectors(codes, cb, dim, k)
        check_pairs(jv, oracle, pqv, codes, cb, dim, M, k, None, a, b, ("k", k))
        pqv.close()


@pytest.mark.gpu
def test_bruteforce_whole_and_sampled(jv, oracle, world):
    # topk_filter_pq_kernel (LUT staged by bulk copies) on the whole-set path (n <= 16384) and the sampled one
    w = world
    rng = np.random.default_rng(w["M"])
    big = np.concatenate([w["codes"], rng.integers(0, w["k"], (18000 - N, w["M"])).astype(np.uint8)])
    sets = ((w["pqv"], w["codes"], "whole"), (jv.PQVectors(big, w["cb"], w["dim"], w["k"], w["cen"]), big, "sampled"))
    queries = w["queries"][:3]
    for vec, codes, path in sets:
        for metric in METRICS:
            want = np.stack([o.scorer_topk(oracle, warp_scorer(oracle, w, metric, codes)(q), 30) for q in queries])
            for kk in (30, 1):
                keys = jv.topk_bruteforce(vec, metric, queries, kk)[2]
                assert np.array_equal(keys, want[:, :kk]), (w["name"], path, metric, kk)
    sets[1][0].close()


@pytest.fixture(scope="module")
def walk_world(jv, oracle, world):
    from test_search_tiers import World
    w = world
    vec = jv.F32Vectors(w["data"])
    gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, addHierarchy=True, seed=1).build(vec)
    vec.close()
    info = gi.info()
    upper = [gi.level(lv) for lv in range(1, info["levels"])] or None
    ww = World(jv, oracle, w["data"], w["queries"], gi.level(0)[1], info["entry_node"], upper, gi)
    ww.sets["pq"] = (w["pqv"], lambda m: warp_scorer(oracle, w, m))
    yield ww
    ww.sets.pop("pq")
    ww.close()


LUT_KNOBS = [{"JV_PQ_LUT": "smem"}, {"JV_PQ_LUT": "l2"}, {"JV_PQ_LUT_SMEM_M": 4}]


@pytest.mark.gpu
def test_walks(walk_world, world, monkeypatch):
    # plain and fp32-reranked PQ walks, the FusedPQ walk, and each LUT placement (the split keeps sub-spaces 0..3 in shared memory)
    from test_search_tiers import knobs
    w = walk_world
    for metric in METRICS:
        w.walk("pq", metric, NQ, rerankK=40, what=(world["name"],))
        w.walk("pq", metric, NQ, rerankK=40, rerank="f32", what=(world["name"],))
        w.walk("pq", metric, NQ, rerankK=40, rerank="f32", fused=True, what=(world["name"], "fused"))
        for env in LUT_KNOBS:
            with knobs(monkeypatch, env):
                w.walk("pq", metric, NQ, rerankK=40, rerank="f32", what=(world["name"], env))
                w.walk("pq", metric, NQ, rerankK=40, rerank="f32", fused=True, what=(world["name"], env, "fused"))


# ------------------------------------------------------------------------------------------------ build, add, remove
# (shape, metric, degree, beam, hierarchy)
MAINTAIN = [
    ("d45_m15_k16_cen", o.COSINE, 16, 60, True),
    ("d64_m14_k255_cen", o.EUCLIDEAN, 16, 60, False),
    ("d33_m33_k16", o.DOT_PRODUCT, 16, 60, True),
    ("d101_m12_k33_cen", o.DOT_PRODUCT, 16, 60, False),
]
NB = 1500


@pytest.mark.gpu
@pytest.mark.parametrize("case", MAINTAIN, ids=[c[0] for c in MAINTAIN])
def test_build_add_remove_equal_the_models(jv, oracle, case):
    import builder_driver as bd
    import delete_model as dm
    from test_graph_build_pq import drive_build_pq, exact_table
    from test_graph_maintain_pq import drive_add_pq
    shape, metric, degree, beam, hier = case
    w = host_world(shape)
    dim, M, k, cen, codes, cb = w["dim"], w["M"], w["k"], w["cen"], w["codes"][:NB], w["cb"]
    world = (codes, cb, cen, dim, k)
    # the build, step by step
    pqv = jv.PQVectors(codes, cb, dim, k, cen)
    drive_build_pq(jv, oracle, pqv, world, metric, degree, beam, -1, 0, hier, shape)
    # an add of 300 rows into a graph built over the first 1200
    n0 = NB - 300
    small = jv.PQVectors(codes[:n0], cb, dim, k, cen)
    b = bd.builder(jv, metric, degree, beam=beam, hier=hier)
    g = b.build(small)
    gi = drive_add_pq(jv, oracle, pqv, world, g, metric, degree, beam, -1, 0, None, shape)
    # a removal of about 10 % of the added graph's nodes
    rng = np.random.default_rng(k)
    levels, entry = bd.levels(gi), gi.info()["entry_node"]
    deleted = rng.random(NB) < 0.1
    got = b.removeDeletedNodes(gi, pqv, deleted)
    pqs = gm.PQScores(oracle, codes, cb, k, dim, cen, exact_table(pqv, cb, dim, k, metric), metric)
    res = dm.remove_deleted(pqs.queries, metric, levels[0][1], entry, levels[1:], deleted, seed=3, prune=pqs.prune)
    hit = bd.assert_removal_matches_model(got, res, shape)
    assert (hit > 0).sum() >= 2, (shape, hit.tolist())
    for h in (g, gi, got, small, pqv):
        h.close()


@pytest.mark.gpu
def test_lut_too_large_for_the_prune_is_refused(jv):
    # M * k = 240 * 255 floats (239 KB) do not fit the prune's shared memory: build, add and removal refuse before any work
    import ctypes as C

    from jvector_b200 import _native as nat
    lib = nat.init()
    rng = np.random.default_rng(240)
    dim, M, k, n = 480, 240, 255, 300
    big = jv.PQVectors(rng.integers(0, k, (n, M)).astype(np.uint8), rng.standard_normal(k * dim).astype(F32), dim, k)
    p = nat.BuildParams(8, 30, 1.2, 1.2, 0, 0, 0, -1)
    out, ms, st = C.c_void_p(), C.c_double(), nat.RemoveStats()
    g = jv.GraphIndex(np.full((200, 8), -1, np.int32), 0)
    full = jv.GraphIndex(np.full((n, 8), -1, np.int32), 0)
    launches = lib.jv_kernel_launch_count()
    assert lib.jv_graph_build_pq(big._h, o.DOT_PRODUCT, C.byref(p), C.byref(out), None) == JV_ERR_UNSUPPORTED
    assert lib.jv_graph_add_nodes_pq(g._h, big._h, o.DOT_PRODUCT, C.byref(p), None, C.byref(out), C.byref(ms)) == JV_ERR_UNSUPPORTED
    none = np.zeros((n + 31) // 32, np.uint32)
    assert lib.jv_graph_remove_deleted_pq(full._h, big._h, o.DOT_PRODUCT, 1.2, 0, none.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(out),
                                          C.byref(st)) == JV_ERR_UNSUPPORTED
    assert lib.jv_kernel_launch_count() == launches and out.value is None
    for h in (big, g, full):
        h.close()
