"""The graph build over PQ codes (jv_graph_build_pq, jv_builder_create_pq: BuildScoreProvider.pqBuildScoreProvider).

CPU: the model's pair scores (pair_pq_table's warp order) agree with the oracle's sequential diversity function; on a lossless world
(integer codebooks, rows that are their own reconstruction, every score exact in fp32) the PQ model and the fp32 model build the
same graph, with and without a global centroid.
GPU (-m gpu): on the lossless world jv_graph_build_pq gives the bytes jv_graph_build gives over the centred reconstruction; on real
PQ the step-wise builder equals the model row for row after every batch, with no near-tie budget; the one-call, step-wise and
sharded builds agree; the graph's recall is close to the fp32 build's; every error code."""
import ctypes as C

import numpy as np
import pytest

import builder_driver as bd
import graph_model as gm
import oracle_lib as o
from oracle_lib import bp, fp

METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)


def lossless_world(rng, n, dim, M, k, centroid):
    """integer codebooks in [0, 15] (products, sums and the 3xTF32 split are exact, DOT scores are positive) and random codes:
    (codes, codebooks, centroid or None, the centred reconstruction = the codebook rows)"""
    codebooks = rng.integers(0, 16, k * dim).astype(np.float32)
    codes = rng.integers(0, k, (n, M)).astype(np.uint8)
    cen = rng.integers(-3, 4, dim).astype(np.float32) if centroid else None
    sizes, offsets = o.pq_layout(dim, M)
    return codes, codebooks, cen, gm.decode(codes, codebooks, sizes, offsets, k, None)


def host_table(codebooks, dim, M, k, metric):
    sizes, offsets = o.pq_layout(dim, M)
    t = np.empty(M * (k * (k + 1) // 2), np.float32)
    o.load().jvo_pq_pair_table(fp(codebooks), sizes.ctypes.data_as(o.i32p), offsets.ctypes.data_as(o.i32p), M, k,
                               o.EUCLIDEAN if metric == o.EUCLIDEAN else o.DOT_PRODUCT, fp(t))
    return t


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("metric", METRICS)
def test_model_pair_scores_match_oracle_diversity(oracle, metric):
    rng = np.random.default_rng(3 + metric)
    dim, M, k = 96, 48, 32  # 48 sub-spaces: lanes 0..15 sum two entries each
    codebooks = rng.random(k * dim).astype(np.float32)  # positive entries: no cancellation, the two orders agree to a few ulps
    codes = rng.integers(0, k, (40, M)).astype(np.uint8)
    table = host_table(codebooks, dim, M, k, metric)
    got = gm.pair_scores(metric, table, k, codes, codes)
    for i in range(len(codes)):
        for j in range(len(codes)):
            want = oracle.jvo_pq_diversity_table(metric, fp(table), M, k, bp(codes[i]), bp(codes[j]))
            assert abs(got[i, j] - want) <= 1e-5 * max(abs(want), 1e-30), (i, j, got[i, j], want)


@pytest.mark.parametrize("metric", (o.EUCLIDEAN, o.DOT_PRODUCT))
@pytest.mark.parametrize("centroid", (False, True), ids=("plain", "centroid"))
def test_lossless_world_pq_model_equals_fp32_model(oracle, metric, centroid):
    rng = np.random.default_rng(11 + metric + 2 * centroid)
    n, dim, M, k = 500, 32, 8, 64
    codes, codebooks, cen, rows = lossless_world(rng, n, dim, M, k, centroid)
    kw = dict(M=8, beam=40, max_batch=0, window=-1)
    pq = gm.BuildModel(gm.PQScores(oracle, codes, codebooks, k, dim, cen, host_table(codebooks, dim, M, k, metric), metric), **kw)
    f32 = gm.BuildModel(gm.F32Scores(oracle, rows, metric), **kw)
    # the two models in lock step, both adopting the PQ model's rows. The fp32 model scores pairs in float64: on integer rows an
    # isDiverse test whose pair distance equals the candidate's own distance is an exact tie, which fp32 (the device, the PQ model)
    # decides one way and float64 may decide the other; the fp32 model flags every such test, and only flagged rows may differ
    differ = flagged = 0

    def step(got, gdeg, want, wdeg, flags):
        nonlocal differ, flagged
        d = (got != want).any(1) | (gdeg != wdeg)
        assert not (d & ~flags).any(), np.flatnonzero(d & ~flags)[:5]
        differ += int(d.sum())
        flagged += int(flags.sum())

    while (nb := pq.next_batch()) is not None:
        assert nb == f32.next_batch()
        got, gdeg, _ = pq.insert_rows(*nb)
        step(got, gdeg, *f32.insert_rows(*nb))
        lst = pq.apply_new(*nb, got, gdeg)
        assert f32.apply_new(*nb, got, gdeg) == lst
        got, gdeg, _ = pq.reprune_rows(lst)
        step(got, gdeg, *f32.reprune_rows(lst))
        pq.apply_repruned(lst, got, gdeg)
        f32.apply_repruned(lst, got, gdeg)
    lst = pq.over_degree()
    assert lst == f32.over_degree()
    got, gdeg, _ = pq.reprune_rows(lst)
    step(got, gdeg, *f32.reprune_rows(lst))
    if metric == o.DOT_PRODUCT:
        assert differ == 0  # (1 + G) / 2 of integer G is exact in both precisions: no tie goes two ways
    assert differ <= 0.05 * n, (differ, flagged)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


# (metric, hierarchy, max_batch, window, centroid): the default schedule and 64-node batches with beam + window = 160
LOSSLESS = [(o.EUCLIDEAN, False, 0, -1, True), (o.DOT_PRODUCT, True, 0, -1, False),
            (o.EUCLIDEAN, True, 64, 60, False), (o.DOT_PRODUCT, False, 64, 60, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", LOSSLESS, ids=["l2_flat_cen", "dot_hier", "l2_hier_b64_w60", "dot_flat_b64_w60_cen"])
def test_lossless_world_byte_equal_to_fp32_build(jv, case):
    from jvector_b200 import _native as nat
    metric, hier, max_batch, window, centroid = case
    rng = np.random.default_rng(7 + metric)
    n, dim, M, k = 20000, 32, 8, 256
    codes, codebooks, cen, rows = lossless_world(rng, n, dim, M, k, centroid)
    params = nat.BuildParams(16, 100, 1.2, 1.2, int(hier), 5, max_batch, window)
    pqv = jv.PQVectors(codes, codebooks, dim, k, cen)
    f32 = jv.F32Vectors(rows)
    g_pq, s_pq = bd.step_build(pqv, metric, params, "_pq")
    g_f32, s_f32 = bd.step_build(f32, metric, params)
    assert s_pq == s_f32 and s_pq[1] == 0, (s_pq, s_f32)
    bd.assert_same_graph(g_pq, g_f32, "lossless")
    g_pq.close(), g_f32.close(), pqv.close(), f32.close()


def real_pq_world(name, n, dim, M, centroid, k=256):
    """latent rows, codebooks trained on them (around their mean when centroid), codes from the oracle encoder"""
    from test_build_steps import latent_rows
    rng = np.random.default_rng(sum(map(ord, name)))
    data = latent_rows(rng, n, dim)
    cen = data.mean(0).astype(np.float32) if centroid else None
    codebooks, sizes, offsets = o.train_pq_numpy(rng, data - cen if centroid else data, M, k, iters=4)
    codes = o.encode_pq(o.load(), codebooks, sizes, offsets, M, k, cen, data)
    return data, codes, codebooks, cen


# (id, dim, PQ M, centroid, metric, degree, beam, window, max_batch, hierarchy, n)
MODEL_CASES = [
    ("l2_m8_cen", 32, 8, True, o.EUCLIDEAN, 16, 60, -1, 0, True, 2000),
    ("dot_m16", 64, 16, False, o.DOT_PRODUCT, 16, 100, -1, 0, False, 2000),
    ("cos_m16_cen", 64, 16, True, o.COSINE, 16, 100, -1, 0, True, 2000),
    ("cos_m8", 32, 8, False, o.COSINE, 8, 60, -1, 0, False, 2000),
    ("l2_m16_b64_w60", 64, 16, False, o.EUCLIDEAN, 16, 100, 60, 64, False, 2000),
    ("dot_m96_d768_cen", 768, 96, True, o.DOT_PRODUCT, 16, 60, -1, 0, False, 1200),
]


def exact_table(pqv, codebooks, dim, k, metric):
    """the centroid-pair table of the metric computed on the host (pq_pair_table_kernel's fmaf chains), asserted equal to the one the
    device holds, bit for bit: the models then score pairs with a table that does not come from the device"""
    table = o.pq_pair_table_exact(codebooks, dim, pqv.M, k, metric)
    got = pqv.pair_table(metric)
    bad = np.flatnonzero(got.view(np.int32) != table.view(np.int32))
    assert len(bad) == 0, ("device pair table differs from the host's", dim, pqv.M, k, metric, len(bad), bad[:5].tolist())
    return table


@pytest.mark.gpu
@pytest.mark.parametrize("case", MODEL_CASES, ids=[c[0] for c in MODEL_CASES])
def test_device_pq_build_equals_model(jv, oracle, case):
    cid, dim, Mq, centroid, metric, M, beam, window, max_batch, hier, n = case
    _, codes, codebooks, cen = real_pq_world(cid, n, dim, Mq, centroid)
    pqv = jv.PQVectors(codes, codebooks, dim, 256, cen)
    drive_build_pq(jv, oracle, pqv, (codes, codebooks, cen, dim, 256), metric, M, beam, window, max_batch, hier, cid)
    pqv.close()


def drive_build_pq(jv, oracle, pqv, world, metric, M, beam, window, max_batch, hier, cid):
    """the build over pqv driven step by step (jv_builder_create_pq + jv_builder_*) against the PQ model over a pair table computed
    on the host: every row equals the model's exactly"""
    from jvector_b200 import _native as nat
    codes, codebooks, cen, dim, k = world
    params = nat.BuildParams(M, beam, 1.2, 1.2, int(hier), 3, max_batch, window)

    def scores():  # the builder made the device's table
        return gm.PQScores(oracle, codes, codebooks, k, dim, cen, exact_table(pqv, codebooks, dim, k, metric), metric)

    bd.drive_build(nat.init(), pqv, metric, params, scores, cid, "_pq")[0].close()


@pytest.mark.gpu
def test_pq_builds_reproduce(jv):
    from jvector_b200 import _native as nat
    from jvector_b200 import parallel
    _, codes, codebooks, cen = real_pq_world("repro", 6000, 64, 16, True)
    pqv = jv.PQVectors(codes, codebooks, 64, 256, cen)
    b = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=80, addHierarchy=True, seed=9)
    one, two = b.build(pqv), b.build(pqv)
    assert b.batches > 0 and b.scored_vectors > 0
    bd.assert_same_graph(one, two, "two calls")
    steps, stats = bd.step_build(pqv, o.DOT_PRODUCT, nat.BuildParams(16, 80, 1.2, 1.2, 1, 9, 0, -1), "_pq")
    assert stats[0] == b.batches and stats[2] == b.dropped_backlinks
    bd.assert_same_graph(one, steps, "one call vs step-wise")
    sharded, _, _ = parallel.sharded_build(None, pqv, o.DOT_PRODUCT, M=16, beamWidth=80, addHierarchy=True, seed=9)
    bd.assert_same_graph(one, sharded, "sharded_build")
    for g in (one, two, steps, sharded):
        g.close()
    pqv.close()


@pytest.mark.gpu
def test_pq_graph_recall_near_fp32_graph(jv):
    from test_build_steps import latent_rows
    rng = np.random.default_rng(21)
    dim, M = 64, 16
    data = latent_rows(rng, 20500, dim)
    base, queries = np.ascontiguousarray(data[:20000]), np.ascontiguousarray(data[20000:])
    codebooks, sizes, offsets = o.train_pq_numpy(rng, base, M, 256, iters=4)
    codes = jv.pq_encode_all(base, codebooks, M)
    f32, pqv = jv.F32Vectors(base), jv.PQVectors(codes, codebooks, dim)
    vsf = o.DOT_PRODUCT
    truth, _, _ = jv.topk_bruteforce(f32, vsf, queries, 10)
    recall = {}
    for name, vec in (("fp32", f32), ("pq", pqv)):
        g = jv.GraphIndexBuilder(vsf, M=16, beamWidth=100, addHierarchy=True).build(vec)
        s = jv.GraphSearcher(g)
        for shape, res in (("f32_walk", s.search(f32, queries, vsf, 10, 100)), ("pq_walk", s.search(pqv, queries, vsf, 10, 100, reranker=f32))):
            recall[(name, shape)] = np.mean([len(set(res.nodes[i]) & set(truth[i])) / 10 for i in range(len(queries))])
        g.close()
    print("recall@10", recall)
    for shape in ("f32_walk", "pq_walk"):
        assert recall[("pq", shape)] >= recall[("fp32", shape)] - 0.03, recall
    f32.close(), pqv.close()


@pytest.mark.gpu
def test_pq_build_errors_and_pair_table(jv):
    from jvector_b200 import _native as nat
    lib = nat.init()
    rng = np.random.default_rng(2)
    _, codes, codebooks, cen = real_pq_world("errors", 600, 32, 8, True)
    pqv = jv.PQVectors(codes, codebooks, 32, 256, cen)
    f32 = jv.F32Vectors(latent_rows_small(rng))
    p = nat.BuildParams(16, 60, 1.2, 1.2, 0, 0, 0, -1)
    g, b, ms = C.c_void_p(), C.c_void_p(), C.c_double()
    assert lib.jv_graph_build_pq(None, 0, C.byref(p), C.byref(g), None) == -2
    assert lib.jv_graph_build_pq(pqv._h, 0, None, C.byref(g), None) == -2
    assert lib.jv_graph_build_pq(pqv._h, 0, C.byref(p), None, None) == -2
    assert lib.jv_graph_build_pq(f32._h, 0, C.byref(p), C.byref(g), None) == -2
    assert lib.jv_graph_build_pq(pqv._h, 7, C.byref(p), C.byref(g), None) == -2
    assert lib.jv_builder_create_pq(f32._h, 0, C.byref(p), None, C.byref(b)) == -2
    assert lib.jv_builder_create_pq(pqv._h, 7, C.byref(p), None, C.byref(b)) == -2
    wide = nat.BuildParams(65, 60, 1.2, 1.2, 0, 0, 0, -1)
    assert lib.jv_graph_build_pq(pqv._h, 0, C.byref(wide), C.byref(g), None) == -5
    assert lib.jv_builder_create_pq(pqv._h, 0, C.byref(wide), None, C.byref(b)) == -5
    # M * k = 256 * 256 entries: a LUT of 256 KB, beyond what the prune holds in shared memory
    big = jv.PQVectors(rng.integers(0, 256, (100, 256)).astype(np.uint8), rng.standard_normal(256 * 512).astype(np.float32), 512)
    assert lib.jv_graph_build_pq(big._h, 0, C.byref(p), C.byref(g), None) == -5
    # the fp32 entry points still refuse PQ data sets
    assert lib.jv_graph_build(pqv._h, 0, C.byref(p), C.byref(g), C.byref(ms)) == -2
    assert lib.jv_builder_create(pqv._h, 0, C.byref(p), None, C.byref(b)) == -2
    # the table the build makes equals the one jv_dataset_pq_pair_table makes on a twin data set
    for metric in METRICS:
        twin = jv.PQVectors(codes, codebooks, 32, 256, cen).build_pair_table(metric)
        one = jv.PQVectors(codes, codebooks, 32, 256, cen)
        jv.GraphIndexBuilder(metric, M=8, beamWidth=30).build(one).close()
        assert np.array_equal(one.pair_table(metric), twin.pair_table(metric)), metric
        one.close(), twin.close()
    big.close(), pqv.close(), f32.close()


def latent_rows_small(rng):
    from test_build_steps import latent_rows
    return latent_rows(rng, 300, 32)
