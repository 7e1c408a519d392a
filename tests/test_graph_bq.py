"""The graph build over BQ codes and its maintenance (jv_graph_build_bq, jv_builder_create_bq, jv_graph_add_nodes_bq,
jv_builder_create_from_graph_bq, jv_graph_remove_deleted_bq: BuildScoreProvider.bqBuildScoreProvider).

CPU: the model's pair scores are jvo_bq_score and 1 - popcount / dim in numpy (dim 100 has padding); on the lossless world (rows
+-1 / sqrt(dim), where DOT_PRODUCT's (1 + dot) / 2 is exactly 1 - hd / dim) the BQ model and the fp32 DOT model build the same graph.
GPU (-m gpu): on the lossless world jv_graph_build_bq gives the bytes of jv_graph_build(DOT_PRODUCT) at every metric, with no
truncated insert search; the step-wise builder equals the model after every batch at dim 100 and 1536; the one-call, step-wise and
sharded builds agree; an add into a one-node graph is the build; adds and removals equal the models row for row, with marked nodes,
holes, and on every removal tier; the metric changes no byte; recall against the fp32 graph; every error code."""
import ctypes as C

import numpy as np
import pytest

import builder_driver as bd
import delete_model as dm
import graph_model as gm
import oracle_lib as o
from oracle_lib import fp

METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)


def lossless_world(rng, n, dim):
    """rows +-1 / sqrt(dim) (dim a power of 4: every product is +-1 / dim, every partial sum exact in fp32 and in 3xTF32) and their
    BQ words. The signs are those of latent rows: near neighbours are then closer than random signs would be, and fewer nodes tie at
    a beam's last score, so that neither walk has to cut a tie tail short"""
    from test_build_steps import latent_rows
    signs = np.where(latent_rows(rng, n, dim, latent=48, noise=0.2) > 0, 1, -1)
    rows = (signs / np.sqrt(dim)).astype(np.float32)
    words = np.zeros((n, (dim + 63) // 64), np.uint64)
    for j in range(dim):
        words[:, j >> 6] |= (signs[:, j] > 0).astype(np.uint64) << np.uint64(j & 63)
    return rows, words


def encode(rows):
    """BinaryQuantization.encode on the host (jvo_bq_encode's rule): bit j of word i = (v[64 i + j] > 0)"""
    n, dim = rows.shape
    words = np.zeros((n, (dim + 63) // 64), np.uint64)
    for j in range(dim):
        words[:, j >> 6] |= (rows[:, j] > 0).astype(np.uint64) << np.uint64(j & 63)
    return words


def latent_world(name, n, dim):
    from test_build_steps import latent_rows
    rows = latent_rows(np.random.default_rng(sum(map(ord, name))), n, dim)
    return rows, encode(rows)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("dim", (64, 100, 1536))
def test_model_pair_scores_are_hamming_scores(oracle, dim):
    rng = np.random.default_rng(dim)
    _, words = latent_world("pairs%d" % dim, 40, dim)
    got = gm.bq_pair_scores(words, dim, np.arange(40), np.arange(40))
    W = words.shape[1]
    hd = np.array([[sum(bin(int(a) ^ int(b)).count("1") for a, b in zip(words[i], words[j])) for j in range(40)] for i in range(40)])
    assert np.array_equal(got, (np.float32(1) - hd.astype(np.float32) / np.float32(dim)).astype(np.float32))
    for i in range(40):
        for j in range(40):
            want = oracle.jvo_bq_score(gm.wp(words[i]), gm.wp(words[j]), W, dim)
            assert np.float32(want).view(np.int32) == got[i, j].view(np.int32), (i, j)
    # the insert query decodes to exactly c_v, padding clear
    back = np.zeros_like(words)
    q = gm.bq_decode(words, dim)
    for v in range(len(words)):
        oracle.jvo_bq_encode(fp(q[v]), dim, gm.wp(back[v]))
    assert np.array_equal(back, words) and set(np.unique(q)) == {-1.0, 1.0}
    del rng


@pytest.mark.parametrize("dim", (64, 256, 1024))
def test_lossless_world_bq_model_equals_fp32_dot_model(oracle, dim):
    rng = np.random.default_rng(dim + 1)
    n = 300
    rows, words = lossless_world(rng, n, dim)
    kw = dict(M=8, beam=40, max_batch=0, window=-1)
    bq = gm.BuildModel(gm.BQScores(oracle, words, dim, o.DOT_PRODUCT), **kw)
    f32 = gm.BuildModel(gm.F32Scores(oracle, rows, o.DOT_PRODUCT), **kw)
    # in lock step, both adopting the BQ model's rows: no row may differ
    while (nb := bq.next_batch()) is not None:
        assert nb == f32.next_batch()
        got, gdeg, _ = bq.insert_rows(*nb)
        want, wdeg, _ = f32.insert_rows(*nb)
        assert np.array_equal(got, want) and np.array_equal(gdeg, wdeg), nb
        lst = bq.apply_new(*nb, got, gdeg)
        assert f32.apply_new(*nb, got, gdeg) == lst
        got, gdeg, _ = bq.reprune_rows(lst)
        want, wdeg, _ = f32.reprune_rows(lst)
        assert np.array_equal(got, want) and np.array_equal(gdeg, wdeg)
        bq.apply_repruned(lst, got, gdeg)
        f32.apply_repruned(lst, got, gdeg)
    lst = bq.over_degree()
    assert lst == f32.over_degree()
    got, gdeg, _ = bq.reprune_rows(lst)
    want, wdeg, _ = f32.reprune_rows(lst)
    assert np.array_equal(got, want) and np.array_equal(gdeg, wdeg)


def test_repair_tiers_of_the_model():
    assert [dm.repair_tier(c) for c in (1, 64, 65, 128, 256, 257, 1024, 1025, 2048, 2049, 4224)] == [0, 0, 1, 1, 2, 3, 3, 4, 4, 5, 5]


def test_bq_graph_entry_points_without_device():
    from jvector_b200 import _native as nat
    lib = nat.load()
    if lib.jv_gpu_device_count() > 0:
        pytest.skip("a GPU is present")
    params = nat.BuildParams(16, 60, 1.2, 1.2, 0, 0, 0, -1)
    out, ms, st = C.c_void_p(1234), C.c_double(7.0), nat.RemoveStats()
    bits = np.zeros(4, np.uint32)
    assert lib.jv_graph_build_bq(None, 1, C.byref(params), C.byref(out), C.byref(ms)) == -1
    assert lib.jv_builder_create_bq(None, 1, C.byref(params), None, C.byref(out)) == -1
    assert lib.jv_graph_add_nodes_bq(None, None, 1, C.byref(params), None, C.byref(out), C.byref(ms)) == -1
    assert lib.jv_builder_create_from_graph_bq(None, None, 1, C.byref(params), None, None, C.byref(out)) == -1
    assert lib.jv_graph_remove_deleted_bq(None, None, 1, 1.2, 0, bits.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(out), C.byref(st)) == -1
    assert out.value == 1234 and ms.value == 7.0


CPP_BQ = r"""
#include <cstdio>
#include <vector>
#include "jvector_b200.hpp"
int main()
{
    try {
        jv::init(0);
    } catch (const jv::Error &e) {
        std::printf("NO_DEVICE_OK\n");
        return 0;
    }
    const int n0 = 200, n = 300, dim = 100, W = 2;
    std::vector<uint64_t> words((size_t)n * W);
    uint64_t s = 88172645463325252ull;
    for (auto &w : words) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; w = s; }
    for (int i = 0; i < n; i++) words[(size_t)i * W + 1] &= (1ull << 36) - 1;  // no bit past dim 100
    jv::BQVectors small(words.data(), n0, dim), all(words.data(), n, dim);
    jv::GraphIndexBuilder b(jv::VectorSimilarityFunction::COSINE, 8, 30, 1.2f, 1.2f, false);
    jv::GraphIndex g = b.build(small);
    jv::GraphIndex grown = b.addGraphNodes(g, all);
    std::vector<uint32_t> del((n + 31) / 32, 0u);
    del[0] = 0x10u;
    jv::GraphIndex r = b.removeDeletedNodes(grown, all, del);
    if (g.size() != n0 || grown.size() != n || r.size() != n || b.removeStats.removed != 1) return 1;
    std::printf("BQ_OK\n");
    return 0;
}
"""


def _cpp_bq(tmp):
    import subprocess

    from jvector_b200 import _native as nat
    src, exe = tmp / "bq_mirror.cpp", tmp / "bq_mirror"
    src.write_text(CPP_BQ)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", str(o.ROOT) + "/include", str(src), "-o", str(exe), nat.SO,
                           "-Wl,-rpath," + __import__("os").path.dirname(nat.SO), "-lpthread", "-ldl"])
    return subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)


def test_cpp_bq_overloads_compile_and_fail_loudly_without_gpu(tmp_path):
    from jvector_b200 import _native as nat
    out = _cpp_bq(tmp_path)
    if nat.load().jv_gpu_device_count() > 0:
        pytest.skip("a GPU is present: covered by the gpu test")
    assert out.returncode == 0 and "NO_DEVICE_OK" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_cpp_bq_overloads_on_gpu(tmp_path):
    out = _cpp_bq(tmp_path)
    assert out.returncode == 0 and "BQ_OK" in out.stdout, out.stdout + out.stderr


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


# (dim, n, degree, beam, hierarchy, max_batch, window). At 64 dimensions there are 65 scores: beam 16 over 1000 rows keeps the nodes
# tied at a beam's last score within the fp32 walk's tie tail (rerankK + 28 entries)
LOSSLESS = [(64, 1000, 8, 16, True, 0, -1), (256, 3000, 16, 60, False, 64, 60), (1024, 4000, 16, 100, True, 0, -1)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", LOSSLESS, ids=("d64_hier", "d256_b64_w60", "d1024_hier"))
def test_lossless_world_byte_equal_to_fp32_dot_build(jv, case):
    from jvector_b200 import _native as nat
    dim, n, M, beam, hier, max_batch, window = case
    rng = np.random.default_rng(7 + dim)
    rows, words = lossless_world(rng, n, dim)
    assert np.array_equal(jv.bq_encode_all(rows), words)
    params = nat.BuildParams(M, beam, 1.2, 1.2, int(hier), 5, max_batch, window)
    bqv, f32 = jv.BQVectors(words, dim), jv.F32Vectors(rows)
    g_f32, s_f32 = bd.step_build(f32, o.DOT_PRODUCT, params)
    assert s_f32[1] == 0, s_f32
    for metric in METRICS:
        g_bq, s_bq = bd.step_build(bqv, metric, params, "_bq")
        assert s_bq == s_f32, (metric, s_bq, s_f32)
        bd.assert_same_graph(g_bq, g_f32, ("lossless step-wise", metric))
        one = bd.builder(jv, metric, M, beam=beam, hier=hier, seed=5, max_batch=max_batch, concurrent_window=window).build(bqv)
        bd.assert_same_graph(one, g_f32, ("lossless one call", metric))
        g_bq.close(), one.close()
    g_f32.close(), bqv.close(), f32.close()


# (id, dim, metric, degree, beam, window, max_batch, hierarchy, n)
MODEL_CASES = [
    ("d100_l2_hier", 100, o.EUCLIDEAN, 16, 60, -1, 0, True, 2000),
    ("d100_dot_b64_w60", 100, o.DOT_PRODUCT, 16, 100, 60, 64, False, 2000),
    ("d1536_cos", 1536, o.COSINE, 16, 60, -1, 0, True, 1200),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", MODEL_CASES, ids=[c[0] for c in MODEL_CASES])
def test_device_bq_build_equals_model(jv, oracle, case):
    from jvector_b200 import _native as nat
    cid, dim, metric, M, beam, window, max_batch, hier, n = case
    _, words = latent_world(cid, n, dim)
    bqv = jv.BQVectors(words, dim)
    params = nat.BuildParams(M, beam, 1.2, 1.2, int(hier), 3, max_batch, window)
    gi = bd.drive_build(nat.init(), bqv, metric, params, lambda: gm.BQScores(oracle, words, dim, metric), cid, "_bq")[0]
    one = bd.builder(jv, metric, M, beam=beam, hier=hier, seed=3, max_batch=max_batch, concurrent_window=window).build(bqv)
    bd.assert_same_graph(one, gi, (cid, "one call vs step-wise"))
    for h in (gi, one, bqv):
        h.close()


@pytest.mark.gpu
def test_bq_builds_reproduce_and_ignore_the_metric(jv):
    from jvector_b200 import _native as nat
    from jvector_b200 import parallel
    _, words = latent_world("repro", 6000, 100)
    bqv = jv.BQVectors(words, 100)
    b = bd.builder(jv, o.DOT_PRODUCT, 16, beam=80, hier=True, seed=9)
    one, two = b.build(bqv), b.build(bqv)
    assert b.batches > 0 and b.scored_vectors > 0
    bd.assert_same_graph(one, two, "two calls")
    steps, stats = bd.step_build(bqv, o.DOT_PRODUCT, nat.BuildParams(16, 80, 1.2, 1.2, 1, 9, 0, -1), "_bq")
    assert stats[0] == b.batches and stats[2] == b.dropped_backlinks
    bd.assert_same_graph(one, steps, "one call vs step-wise")
    sharded, _, _ = parallel.sharded_build(None, bqv, o.DOT_PRODUCT, M=16, beamWidth=80, addHierarchy=True, seed=9)
    bd.assert_same_graph(one, sharded, "sharded_build")
    for metric in (o.EUCLIDEAN, o.COSINE):
        other = bd.builder(jv, metric, 16, beam=80, hier=True, seed=9).build(bqv)
        bd.assert_same_graph(one, other, ("metric", metric))
        other.close()
    for g in (one, two, steps, sharded, bqv):
        g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("hier", (False, True), ids=("flat", "hier"))
def test_add_to_one_node_graph_is_the_bq_build(jv, hier):
    n, dim, M = 3000, 100, 16
    _, words = latent_world("anchor", n, dim)
    bqv = jv.BQVectors(words, dim)
    seed = next(s for s in range(1, 400) if gm.level_draws(n, M, s)[0] >= 1) if hier else 3
    b = bd.builder(jv, o.COSINE, M, hier=hier, seed=seed)
    built = b.build(bqv)
    want = (b.batches, b.dropped_backlinks)
    empty = np.full((1, M), -1, np.int32)
    tops = int(gm.level_draws(n, M, seed)[0]) if hier else 0
    one = jv.GraphIndex(empty, 0, [(np.zeros(1, np.int32), empty)] * tops)
    added = b.addGraphNodes(one, bqv)
    assert (b.batches, b.dropped_backlinks) == want
    bd.assert_same_graph(added, built, ("one-node add", hier))
    assert built.info()["levels"] > 1 or not hier
    for h in (built, one, added, bqv):
        h.close()


# (id, dim, metric, degree, beam, hierarchy, n0, n, origin of the graph)
ADD_CASES = [
    ("d100_l2_hier", 100, o.EUCLIDEAN, 16, 60, True, 1500, 1800, "built"),
    ("d100_dot_marked", 100, o.DOT_PRODUCT, 16, 60, True, 1600, 1800, "marked"),
    ("d1536_cos_removed", 1536, o.COSINE, 16, 60, True, 1000, 1200, "removed"),
    ("d100_l2_all_removed", 100, o.EUCLIDEAN, 16, 60, False, 600, 1000, "all_removed"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ADD_CASES, ids=[c[0] for c in ADD_CASES])
def test_stepwise_bq_add_equals_model(jv, oracle, case):
    from jvector_b200 import _native as nat
    cid, dim, metric, M, beam, hier, n0, n, origin = case
    rng = np.random.default_rng(sum(map(ord, cid)))
    _, words = latent_world(cid, n, dim)
    small, bqv = jv.BQVectors(words[:n0], dim), jv.BQVectors(words, dim)
    b = bd.builder(jv, metric, M, beam=beam, hier=hier)
    g = b.build(small)
    marks = None
    if origin == "marked":
        marks = rng.random(n0) < 0.05
    elif origin == "removed":
        g = b.removeDeletedNodes(g, small, rng.random(n0) < 0.1)
    elif origin == "all_removed":
        g = b.removeDeletedNodes(g, small, np.ones(n0, bool))
        assert g.info()["entry_node"] == -1
    before = bd.levels(g)
    params = nat.BuildParams(M, beam, 1.2, 1.2, 0, 3, 0, -1)
    gi = bd.drive_add(nat.init(), g, bqv, metric, params, marks, lambda: gm.BQScores(oracle, words, dim, metric), cid, "_bq", METRICS)[0]
    if origin == "all_removed":
        assert gi.info()["entry_node"] == n0
    after = bd.levels(g)
    assert len(before) == len(after) and all(np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1]) for a, c in zip(before, after))
    for h in (g, gi, small, bqv):
        h.close()


# (id, dim, metric, degree, hierarchy, n, deleted fraction, entry deleted)
REMOVE_CASES = [
    ("light_d100_dot", 100, o.DOT_PRODUCT, 16, True, 2000, 0.02, False),
    ("heavy_d100_l2", 100, o.EUCLIDEAN, 16, True, 2000, 0.45, True),
    ("heavy_d1536_cos", 1536, o.COSINE, 32, False, 1500, 0.4, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", REMOVE_CASES, ids=[c[0] for c in REMOVE_CASES])
def test_bq_removal_equals_model(jv, oracle, case):
    cid, dim, metric, M, hier, n, frac, kill_entry = case
    rng = np.random.default_rng(sum(map(ord, cid)))
    _, words = latent_world(cid, n, dim)
    bqv = jv.BQVectors(words, dim)
    b = bd.builder(jv, metric, M, hier=hier, seed=17)
    g = b.build(bqv)
    levels, entry = bd.levels(g), g.info()["entry_node"]
    deleted = rng.random(n) < frac
    deleted[entry] = kill_entry
    got = b.removeDeletedNodes(g, bqv, deleted)
    for m in METRICS:  # the same bytes at every metric, and from a second call
        again = bd.builder(jv, m, M, hier=hier, seed=17).removeDeletedNodes(g, bqv, deleted)
        bd.assert_same_graph(got, again, (cid, "metric", m))
        again.close()
    bqs = gm.BQScores(oracle, words, dim, metric)
    res = dm.remove_deleted(bqs.queries, metric, levels[0][1], entry, levels[1:], deleted, seed=17, prune=bqs.prune)
    hit = bd.assert_removal_matches_model(got, res, cid)
    print(cid, "rows per tier", hit.tolist(), got.remove_stats)
    assert got.remove_stats["removed"] == deleted.sum() and (not kill_entry or got.info()["entry_node"] != entry)
    for h in (g, got, bqv):
        h.close()


@pytest.mark.gpu
def test_bq_removal_hits_every_tier_on_a_made_graph(jv, oracle):
    # test_graph_maintain_pq's hand-made degree-64 graph over BQ words: hubs that lose 64, 24, 8 or 3 neighbours naming 64 nodes each
    # gather about 2400, 1200, 450 and 180 candidates (the 8192, 2048, 1024 and 256 tiers), ordinary rows 15 or about 70
    rng = np.random.default_rng(64)
    n, dim, M = 4000, 100, 64
    _, words = latent_world("made", n, dim)
    bqv = jv.BQVectors(words, dim)
    adj = np.full((n, M), -1, np.int32)

    def pick(v, cnt, pool):
        return rng.choice(np.setdiff1d(pool, [v]), cnt, replace=False)

    everyone = np.arange(n)
    for v in range(n):
        adj[v, :8] = pick(v, 8, everyone)
    hubs = {10: 64, 11: 64, 20: 24, 21: 24, 30: 8, 31: 8, 40: 3}
    deleted = np.zeros(n, bool)
    pool = np.arange(100, n)
    for hub, cnt in hubs.items():
        lost = pick(hub, cnt, pool[~deleted[pool]])
        adj[hub] = -1
        adj[hub, :cnt] = lost
        deleted[lost] = True
        for j in lost:
            adj[j] = pick(j, M, pool)
    deleted[rng.choice(np.flatnonzero(~deleted[100:]) + 100, 60, replace=False)] = True
    g = jv.GraphIndex(adj, 0)
    got = bd.builder(jv, o.EUCLIDEAN, M, seed=5).removeDeletedNodes(g, bqv, deleted)
    bqs = gm.BQScores(oracle, words, dim, o.EUCLIDEAN)
    res = dm.remove_deleted(bqs.queries, o.EUCLIDEAN, adj, 0, [], deleted, seed=5, prune=bqs.prune)
    hit = bd.assert_removal_matches_model(got, res, "made graph")
    print("made graph: rows per tier", hit.tolist(), got.remove_stats)
    assert (hit > 0).all() and got.remove_stats["max_candidates"] > 2048, hit.tolist()
    for h in (g, got, bqv):
        h.close()


@pytest.mark.gpu
def test_bq_remove_add_remove_keeps_holes_and_equals_models(jv, oracle):
    rng = np.random.default_rng(21)
    n0, n, dim, M = 1600, 1800, 100, 16
    _, words = latent_world("holes", n, dim)
    small, bqv = jv.BQVectors(words[:n0], dim), jv.BQVectors(words, dim)
    b = bd.builder(jv, o.DOT_PRODUCT, M, hier=True, seed=4)
    g = b.build(small)
    first = rng.random(n0) < 0.1
    rep = b.removeDeletedNodes(g, small, first)
    lv = bd.levels(g)
    bqs = gm.BQScores(oracle, words[:n0], dim, o.DOT_PRODUCT)
    res = dm.remove_deleted(bqs.queries, o.DOT_PRODUCT, lv[0][1], g.info()["entry_node"], lv[1:], first, seed=4, prune=bqs.prune)
    bd.assert_removal_matches_model(rep, res, "first removal")
    grown = b.addGraphNodes(rep, bqv)
    wide = np.concatenate([first, np.zeros(n - n0, bool)])
    assert grown.info()["n"] == n and not np.isin(grown.level(0)[1], np.flatnonzero(first)).any()
    second = (rng.random(n) < 0.05) & ~wide
    again = b.removeDeletedNodes(grown, bqv, second | wide)
    lv = bd.levels(grown)
    bqs = gm.BQScores(oracle, words, dim, o.DOT_PRODUCT)
    res = dm.remove_deleted(bqs.queries, o.DOT_PRODUCT, lv[0][1], grown.info()["entry_node"], lv[1:], second | wide, seed=4, holes=wide,
                            prune=bqs.prune)
    bd.assert_removal_matches_model(again, res, "second removal")
    assert again.remove_stats["removed"] == second.sum(), (again.remove_stats, second.sum())
    assert again.remove_stats["live_nodes"] == n - first.sum() - second.sum()
    for h in (g, rep, grown, again, small, bqv):
        h.close()


def _recall(nodes, truth):
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / truth.shape[1] for i in range(len(nodes))]))


# How far the BQ-built graph's recall@10 may fall below the fp32-built graph's on the same world, under the same walk. Derived on a
# CPU from the host models' flat graphs over this test's world (BQBuildModel against BuildModel(DOT_PRODUCT), the 10 000 x 64 latent
# rows and 1000 queries below, M = 16, beam 100; the oracle's walks; truth by numpy in float64): under the fp32 walk 0.9695 against
# 0.9987, under the BQ walk + fp32 rerank at rerankK 100 0.7395 against 0.7565, a loss of at most 0.029. The device builds add a
# hierarchy, the fp32 one may differ from its model on near-tie rows, and the device's brute force may order near ties differently:
# the margin is that loss plus 0.016.
RECALL_MARGIN = 0.045


@pytest.mark.gpu
def test_bq_graph_recall_near_fp32_graph(jv):
    from test_build_steps import latent_rows
    rng = np.random.default_rng(21)
    dim, n = 64, 10000
    data = latent_rows(rng, n + 1000, dim)
    base, queries = np.ascontiguousarray(data[:n]), np.ascontiguousarray(data[n:])
    f32 = jv.F32Vectors(base)
    bqv = jv.BQVectors(jv.bq_encode_all(base), dim)
    vsf = o.DOT_PRODUCT
    truth, _, _ = jv.topk_bruteforce(f32, vsf, queries, 10)
    recall = {}
    for name, vec in (("fp32", f32), ("bq", bqv)):
        g = bd.builder(jv, vsf, 16, beam=100, hier=True, seed=9).build(vec)
        s = jv.GraphSearcher(g)
        recall[(name, "f32_walk")] = _recall(s.search(f32, queries, vsf, 10, 100).nodes, truth)
        recall[(name, "bq_walk")] = _recall(s.search(bqv, queries, vsf, 10, 100, reranker=f32).nodes, truth)
        g.close()
    print("recall@10", recall)
    for shape in ("f32_walk", "bq_walk"):
        assert recall[("bq", shape)] >= recall[("fp32", shape)] - RECALL_MARGIN, recall
    f32.close(), bqv.close()


@pytest.mark.gpu
def test_bq_graph_errors(jv):
    from jvector_b200 import _native as nat
    lib = nat.init()
    rng = np.random.default_rng(2)
    rows = rng.standard_normal((300, 100)).astype(np.float32)
    words = encode(rows)
    bqv, short, f32 = jv.BQVectors(words, 100), jv.BQVectors(words[:100], 100), jv.F32Vectors(rows)
    padded = words.copy()
    padded[123, 1] |= np.uint64(1) << np.uint64(40)  # bit 104 of a 100-dimensional row
    bad = jv.BQVectors(padded, 100)
    g = jv.GraphIndex(np.full((200, 8), -1, np.int32), 0)
    full = jv.GraphIndex(np.full((300, 8), -1, np.int32), 0)
    params = nat.BuildParams(8, 30, 1.2, 1.2, 0, 0, 0, -1)
    out, ms, st = C.c_void_p(), C.c_double(), nat.RemoveStats()
    none = np.zeros(300, bool)

    def build(ds, metric=1, p=params, o_=C.byref(out)):
        a = lib.jv_graph_build_bq(ds, metric, C.byref(p) if p is not None else None, o_, C.byref(ms))
        c = lib.jv_builder_create_bq(ds, metric, C.byref(p) if p is not None else None, None, o_)
        assert a == c, (a, c)
        return a

    def add(graph, ds, metric=1, p=params, o_=C.byref(out)):
        a = lib.jv_graph_add_nodes_bq(graph, ds, metric, C.byref(p) if p is not None else None, None, o_, C.byref(ms))
        c = lib.jv_builder_create_from_graph_bq(graph, ds, metric, C.byref(p) if p is not None else None, None, None, o_)
        assert a == c, (a, c)
        return a

    def remove(graph, ds, metric=1, alpha=1.2, bits=none, o_=C.byref(out), st_=C.byref(st)):
        return lib.jv_graph_remove_deleted_bq(graph, ds, metric, alpha, 0, bd.bits(bits), o_, st_)

    launches = lib.jv_kernel_launch_count()
    assert build(None) == -2 and build(bqv._h, p=None) == -2 and build(bqv._h, o_=None) == -2
    assert build(f32._h) == -2 and build(bqv._h, metric=7) == -2
    assert build(bqv._h, p=nat.BuildParams(8, 30, 1.2, 0.9, 0, 0, 0, -1)) == -2
    assert build(bqv._h, p=nat.BuildParams(65, 30, 1.2, 1.2, 0, 0, 0, -1)) == -5
    assert add(None, bqv._h) == -2 and add(g._h, None) == -2 and add(g._h, bqv._h, p=None) == -2 and add(g._h, bqv._h, o_=None) == -2
    assert add(g._h, f32._h) == -2  # not BQ
    assert add(g._h, short._h) == -2  # n < n0
    assert add(g._h, bqv._h, metric=7) == -2
    assert add(g._h, bqv._h, p=nat.BuildParams(16, 30, 1.2, 1.2, 0, 0, 0, -1)) == -2  # degree mismatch
    assert remove(None, bqv._h) == -2 and remove(full._h, None) == -2 and remove(full._h, bqv._h, bits=None) == -2
    assert remove(full._h, bqv._h, o_=None) == -2 and remove(full._h, bqv._h, st_=None) == -2
    assert remove(full._h, f32._h) == -2  # not BQ
    assert remove(g._h, bqv._h) == -2  # n != g.n
    assert remove(full._h, bqv._h, metric=7) == -2 and remove(full._h, bqv._h, alpha=0.9) == -2
    wide, wide_full = jv.GraphIndex(np.full((200, 65), -1, np.int32), 0), jv.GraphIndex(np.full((300, 65), -1, np.int32), 0)
    assert add(wide._h, bqv._h, p=nat.BuildParams(65, 30, 1.2, 1.2, 0, 0, 0, -1)) == -5
    assert remove(wide_full._h, bqv._h) == -5
    assert lib.jv_kernel_launch_count() == launches and out.value is None  # refused before any device work
    # a bit past dim: refused after the one padding reduction, before any other device work
    assert build(bad._h) == -2 and add(g._h, bad._h) == -2 and remove(full._h, bad._h) == -2
    assert lib.jv_kernel_launch_count() - launches == 5 and out.value is None  # build and add ran two calls each
    # the fp32 and PQ entry points still refuse a BQ data set
    assert lib.jv_graph_build(bqv._h, 1, C.byref(params), C.byref(out), C.byref(ms)) == -2
    assert lib.jv_builder_create(bqv._h, 1, C.byref(params), None, C.byref(out)) == -2
    assert lib.jv_graph_build_pq(bqv._h, 1, C.byref(params), C.byref(out), C.byref(ms)) == -2
    assert lib.jv_builder_create_pq(bqv._h, 1, C.byref(params), None, C.byref(out)) == -2
    assert lib.jv_graph_add_nodes(g._h, bqv._h, 1, C.byref(params), None, C.byref(out), C.byref(ms)) == -2
    assert lib.jv_builder_create_from_graph(g._h, bqv._h, 1, C.byref(params), None, None, C.byref(out)) == -2
    assert lib.jv_graph_remove_deleted(full._h, bqv._h, 1, 1.2, 0, bd.bits(none), C.byref(out), C.byref(st)) == -2
    assert lib.jv_graph_add_nodes_pq(g._h, bqv._h, 1, C.byref(params), None, C.byref(out), C.byref(ms)) == -2
    assert lib.jv_builder_create_from_graph_pq(g._h, bqv._h, 1, C.byref(params), None, None, C.byref(out)) == -2
    assert lib.jv_graph_remove_deleted_pq(full._h, bqv._h, 1, 1.2, 0, bd.bits(none), C.byref(out), C.byref(st)) == -2
    assert out.value is None
    # the same words without the stray bit build
    assert lib.jv_graph_build_bq(bqv._h, 1, C.byref(params), C.byref(out), C.byref(ms)) == 0
    jv.GraphIndex(_handle=C.c_void_p(out.value)).close()
    for h in (bqv, short, f32, bad, g, full, wide, wide_full):
        h.close()
