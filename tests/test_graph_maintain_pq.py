"""Adds to and removals from a graph over PQ codes (jv_graph_add_nodes_pq, jv_builder_create_from_graph_pq,
jv_graph_remove_deleted_pq: addGraphNode and removeDeletedNodes under BuildScoreProvider.pqBuildScoreProvider).

CPU: on the lossless world of test_graph_build_pq (integer codebooks, rows equal to their reconstruction) the seeded PQ model and
the seeded fp32 model insert the same rows, and the PQ repair model and delete_model repair the same rows, with and without a global
centroid; the entry points report a missing device.
GPU (-m gpu): an add into a one-node graph is jv_graph_build_pq byte for byte; on the lossless world the PQ calls give the bytes of
the fp32 calls; on real PQ the step-wise add equals the model after every batch and the one-call add equals the step-wise add; the
removal equals the model row for row on every prune tier, with the random fallback, a deleted entry and every node deleted; marked
nodes are never picked; holes survive remove -> add -> remove; calls reproduce; recall after an add and after a removal; the fused PQ
walk on a maintained graph equals the oracle; every error code."""
import ctypes as C

import numpy as np
import pytest

import builder_driver as bd
import delete_model as dm
import graph_model as gm
import oracle_lib as o
from oracle_lib import fp, ip
from test_graph_build_pq import exact_table, host_table, lossless_world, real_pq_world

METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)


def warp_keys(oracle, metric, data):
    dim = data.shape[1]
    return lambda v, ids: np.array([oracle.jvo_compare_f32_warp(metric, fp(data[v]), fp(data[i]), dim) for i in ids], np.float32)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("metric", (o.EUCLIDEAN, o.DOT_PRODUCT))
@pytest.mark.parametrize("centroid", (False, True), ids=("plain", "centroid"))
def test_lossless_world_seeded_pq_model_equals_seeded_fp32_model(oracle, metric, centroid):
    rng = np.random.default_rng(31 + metric + 2 * centroid)
    n0, n, dim, M, k = 300, 420, 32, 8, 64
    codes, codebooks, cen, rows = lossless_world(rng, n, dim, M, k, centroid)
    table = host_table(codebooks, dim, M, k, metric)
    kw = dict(M=8, beam=40, max_batch=0, window=-1)
    pqs = gm.PQScores(oracle, codes, codebooks, k, dim, cen, table, metric)
    seed_adj, _ = gm.BuildModel(pqs.subset(np.arange(n0)), **kw).build()
    marks = rng.random(n0) < 0.05
    accept = np.concatenate([~marks, np.ones(n - n0, bool)])
    pq = gm.BuildModel(pqs, rows=seed_adj, entry=7, accept=accept, **kw)
    f32 = gm.BuildModel(gm.F32Scores(oracle, rows, metric), rows=seed_adj, entry=7, accept=accept, **kw)
    assert pq.next_batch() == (n0, n0 // 32)
    # in lock step, both adopting the PQ model's rows; the fp32 model scores pairs in float64 and flags the isDiverse tests that
    # are exact ties on integer rows: only flagged rows may differ (test_graph_build_pq's lossless test)
    differ = 0

    def step(got, gdeg, want, wdeg, flags):
        nonlocal differ
        d = (got != want).any(1) | (gdeg != wdeg)
        assert not (d & ~flags).any(), np.flatnonzero(d & ~flags)[:5]
        differ += int(d.sum())

    while (nb := pq.next_batch()) is not None:
        assert nb == f32.next_batch()
        got, gdeg, _ = pq.insert_rows(*nb)
        assert not marks[got[(got >= 0) & (got < n0)]].any()
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
        assert differ == 0
    assert differ <= 0.05 * n, differ


@pytest.mark.parametrize("metric", (o.EUCLIDEAN, o.DOT_PRODUCT))
@pytest.mark.parametrize("centroid", (False, True), ids=("plain", "centroid"))
def test_lossless_world_pq_repair_model_equals_delete_model(oracle, metric, centroid):
    rng = np.random.default_rng(57 + metric + 2 * centroid)
    n, dim, M, k, degree = 400, 32, 8, 64, 8
    codes, codebooks, cen, rows = lossless_world(rng, n, dim, M, k, centroid)
    table = host_table(codebooks, dim, M, k, metric)
    kw = dict(M=degree, beam=40, max_batch=0, window=-1)
    pqs = gm.PQScores(oracle, codes, codebooks, k, dim, cen, table, metric)
    adj0, _ = gm.BuildModel(pqs, **kw).build()
    ids = np.arange(0, n, 6, dtype=np.int32)
    upper = [(i, a) for i, a, _ in gm.upper_levels(pqs, [ids], **kw)]
    for frac, kill_entry in ((0.05, False), (0.4, True)):
        deleted = rng.random(n) < frac
        deleted[0] = kill_entry
        got = dm.remove_deleted(pqs.queries, metric, adj0, 0, upper, deleted, seed=9, prune=pqs.prune)
        want = dm.remove_deleted(rows, metric, adj0, 0, upper, deleted, seed=9, key_scores=warp_keys(oracle, metric, rows))
        assert (got["entry"], got["levels"]) == (want["entry"], want["levels"])
        differ = repaired = 0
        for (gi, ga), (wi, wa), info in zip([(None, got["adj0"])] + got["upper"], [(None, want["adj0"])] + want["upper"], want["rows"]):
            assert gi is None or np.array_equal(gi, wi)
            node = np.arange(n) if gi is None else gi
            bad = np.flatnonzero((ga != wa).any(1))
            assert all(info[int(node[r])]["flag"] for r in bad), ("an unflagged row differs", node[bad[:5]])
            differ += len(bad)
            repaired += len(info)
        assert repaired > 0 and [set(r) for r in got["rows"]] == [set(r) for r in want["rows"]]
        if metric == o.DOT_PRODUCT:
            assert differ == 0
        assert differ <= 0.05 * repaired, (differ, repaired)


def test_repair_tiers_of_the_model():
    assert [dm.repair_tier(c) for c in (1, 64, 65, 128, 256, 257, 1024, 1025, 2048, 2049, 4224)] == [0, 0, 1, 1, 2, 3, 3, 4, 4, 5, 5]


def test_pq_maintenance_entry_points_without_device():
    from jvector_b200 import _native as nat
    lib = nat.load()
    if lib.jv_gpu_device_count() > 0:
        pytest.skip("a GPU is present")
    params = nat.BuildParams(16, 60, 1.2, 1.2, 0, 0, 0, -1)
    out, ms, st = C.c_void_p(1234), C.c_double(7.0), nat.RemoveStats()
    bits = np.zeros(4, np.uint32)
    assert lib.jv_graph_add_nodes_pq(None, None, 1, C.byref(params), None, C.byref(out), C.byref(ms)) == -1
    assert lib.jv_builder_create_from_graph_pq(None, None, 1, C.byref(params), None, None, C.byref(out)) == -1
    assert lib.jv_graph_remove_deleted_pq(None, None, 1, 1.2, 0, bits.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(out), C.byref(st)) == -1
    assert out.value == 1234 and ms.value == 7.0


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


@pytest.mark.gpu
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("hier", (False, True), ids=("flat", "hier"))
def test_add_to_one_node_graph_is_the_pq_build(jv, metric, hier):
    n, dim, Mq, M = 3000, 64, 16, 16
    _, codes, codebooks, cen = real_pq_world("anchor%d" % metric, n, dim, Mq, metric != o.DOT_PRODUCT)
    pqv = jv.PQVectors(codes, codebooks, dim, 256, cen)
    # a seed whose draw puts node 0 on level 1 or higher: the one-node graph then has the levels an add extends
    seed = next(s for s in range(1, 400) if gm.level_draws(n, M, s)[0] >= 1) if hier else 3
    b = bd.builder(jv, metric, M, hier=hier, seed=seed)
    built = b.build(pqv)
    want = (b.batches, b.dropped_backlinks)
    empty = np.full((1, M), -1, np.int32)
    tops = int(gm.level_draws(n, M, seed)[0]) if hier else 0
    one = jv.GraphIndex(empty, 0, [(np.zeros(1, np.int32), empty)] * tops)
    added = b.addGraphNodes(one, pqv)
    assert (b.batches, b.dropped_backlinks) == want
    bd.assert_same_graph(added, built, ("one-node add", metric, hier))
    assert built.info()["levels"] > 1 or not hier
    for h in (built, one, added, pqv):
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric,centroid", [(o.EUCLIDEAN, True), (o.DOT_PRODUCT, False)], ids=("l2_cen", "dot"))
def test_lossless_world_bytes_equal_the_fp32_calls(jv, metric, centroid):
    rng = np.random.default_rng(17 + metric)
    n0, n, dim, M, k = 7000, 8000, 32, 8, 256
    codes, codebooks, cen, rows = lossless_world(rng, n, dim, M, k, centroid)
    pqv, f32, f32_small = jv.PQVectors(codes, codebooks, dim, k, cen), jv.F32Vectors(rows), jv.F32Vectors(rows[:n0])
    b = bd.builder(jv, metric, 16, beam=100, hier=True, seed=5)
    g = b.build(f32_small)
    marks = rng.random(n0) < 0.03
    a_pq, a_f32 = b.addGraphNodes(g, pqv, marks), b.addGraphNodes(g, f32, marks)
    bd.assert_same_graph(a_pq, a_f32, "lossless add")
    deleted = rng.random(n) < 0.1
    deleted[a_pq.info()["entry_node"]] = True
    r_pq, r_f32 = b.removeDeletedNodes(a_pq, pqv, deleted), b.removeDeletedNodes(a_f32, f32, deleted)
    bd.assert_same_graph(r_pq, r_f32, "lossless removal")
    assert r_pq.remove_stats["repaired_rows"] == r_f32.remove_stats["repaired_rows"] > 0
    assert r_pq.remove_stats["candidates"] == r_f32.remove_stats["candidates"]
    # the holes are the same too: a second removal of nothing counts them as gone in both
    none = np.zeros(n, bool)
    z_pq, z_f32 = b.removeDeletedNodes(r_pq, pqv, none), b.removeDeletedNodes(r_f32, f32, none)
    assert z_pq.remove_stats["live_nodes"] == z_f32.remove_stats["live_nodes"] == n - deleted.sum() and z_pq.remove_stats["removed"] == 0
    for h in (g, a_pq, a_f32, r_pq, r_f32, z_pq, z_f32, pqv, f32, f32_small):
        h.close()


def drive_add_pq(jv, oracle, pqv, world, g, metric, M, beam, window, max_batch, marks, cid):
    """the add of code rows [n0, n) to g driven step by step (jv_builder_create_from_graph_pq + jv_builder_*) against the seeded PQ
    model over a pair table computed on the host: every row equals the model's exactly; then the one-call add gives the same bytes"""
    from jvector_b200 import _native as nat
    codes, codebooks, cen, dim, k = world
    params = nat.BuildParams(M, beam, 1.2, 1.2, 0, 3, max_batch, window)

    def scores():  # the builder made the device's table
        return gm.PQScores(oracle, codes, codebooks, k, dim, cen, exact_table(pqv, codebooks, dim, k, metric), metric)

    gi, _, batches, _, _ = bd.drive_add(nat.init(), g, pqv, metric, params, marks, scores, cid, "_pq")
    assert batches > 0
    return gi


# (id, dim, PQ M, centroid, metric, degree, beam, window, max_batch, hierarchy, n0, n, origin of the graph)
ADD_CASES = [
    ("l2_m8_cen_hier", 32, 8, True, o.EUCLIDEAN, 16, 60, -1, 0, True, 1500, 1800, "built"),
    ("dot_m16_marked", 64, 16, False, o.DOT_PRODUCT, 16, 60, -1, 0, True, 1600, 1800, "marked"),
    ("cos_m16_d50_cen", 50, 16, True, o.COSINE, 16, 60, -1, 0, False, 1000, 1500, "built"),  # sub-spaces of 4 and 3 dimensions
    ("dot_m16_b64_w60_removed", 64, 16, True, o.DOT_PRODUCT, 8, 100, 60, 64, True, 1500, 1800, "removed"),
    ("l2_m16_all_removed", 64, 16, False, o.EUCLIDEAN, 16, 60, -1, 0, True, 600, 1000, "all_removed"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ADD_CASES, ids=[c[0] for c in ADD_CASES])
def test_stepwise_pq_add_equals_model(jv, oracle, case):
    cid, dim, Mq, centroid, metric, M, beam, window, max_batch, hier, n0, n, origin = case
    rng = np.random.default_rng(sum(map(ord, cid)))
    _, codes, codebooks, cen = real_pq_world(cid, n, dim, Mq, centroid)
    small, pqv = jv.PQVectors(codes[:n0], codebooks, dim, 256, cen), jv.PQVectors(codes, codebooks, dim, 256, cen)
    b = bd.builder(jv, metric, M, beam=beam, hier=hier, max_batch=max_batch, concurrent_window=window)
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
    gi = drive_add_pq(jv, oracle, pqv, (codes, codebooks, cen, dim, 256), g, metric, M, beam, window, max_batch, marks, cid)
    if origin == "all_removed":
        assert gi.info()["entry_node"] == n0
    after = bd.levels(g)  # the input graph is untouched
    assert len(before) == len(after) and all(np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1]) for a, c in zip(before, after))
    for h in (g, gi, small, pqv):
        h.close()


@pytest.mark.gpu
def test_zero_new_rows_copies_the_graph(jv):
    _, codes, codebooks, cen = real_pq_world("zero", 1200, 32, 8, True)
    pqv = jv.PQVectors(codes, codebooks, 32, 256, cen)
    b = bd.builder(jv, o.DOT_PRODUCT, 16, hier=True)
    g = b.build(pqv)
    same = b.addGraphNodes(g, pqv)
    bd.assert_same_graph(g, same, "n == n0")
    for h in (g, same, pqv):
        h.close()


# (id, dim, PQ M, centroid, metric, degree, hierarchy, n, deleted fraction, entry deleted, tiers that must be hit)
REMOVE_CASES = [
    ("light_m16_dot", 64, 16, False, o.DOT_PRODUCT, 16, True, 2000, 0.02, False, (0,)),
    ("heavy_m16_l2_cen", 64, 16, True, o.EUCLIDEAN, 16, True, 2000, 0.45, True, (1,)),
    ("heavy_m32_cos_cen", 64, 32, True, o.COSINE, 32, False, 2500, 0.4, True, (2,)),
    ("light_m16_d50_cos", 50, 16, False, o.COSINE, 8, True, 1500, 0.1, False, (0,)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", REMOVE_CASES, ids=[c[0] for c in REMOVE_CASES])
def test_pq_removal_equals_model(jv, oracle, case):
    cid, dim, Mq, centroid, metric, M, hier, n, frac, kill_entry, tiers = case
    rng = np.random.default_rng(sum(map(ord, cid)))
    _, codes, codebooks, cen = real_pq_world(cid, n, dim, Mq, centroid)
    pqv = jv.PQVectors(codes, codebooks, dim, 256, cen)
    b = bd.builder(jv, metric, M, hier=hier, seed=17)
    g = b.build(pqv)
    levels, entry = bd.levels(g), g.info()["entry_node"]
    deleted = rng.random(n) < frac
    deleted[entry] = kill_entry
    got, again = b.removeDeletedNodes(g, pqv, deleted), b.removeDeletedNodes(g, pqv, deleted)
    bd.assert_same_graph(got, again, (cid, "two calls"))
    pqs = gm.PQScores(oracle, codes, codebooks, 256, dim, cen, exact_table(pqv, codebooks, dim, 256, metric), metric)
    res = dm.remove_deleted(pqs.queries, metric, levels[0][1], entry, levels[1:], deleted, seed=17, prune=pqs.prune)
    hit = bd.assert_removal_matches_model(got, res, cid)
    print(cid, "rows per tier", hit.tolist(), got.remove_stats)
    assert all(hit[t] > 0 for t in tiers), (cid, hit.tolist(), tiers)
    assert got.remove_stats["removed"] == deleted.sum() and (not kill_entry or got.info()["entry_node"] != entry)
    after = bd.levels(g)
    assert all(np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1]) for a, c in zip(levels, after))
    for h in (g, got, again, pqv):
        h.close()


@pytest.mark.gpu
def test_pq_removal_hits_every_tier_on_a_made_graph(jv, oracle):
    # degree 64 and a hand-made graph: ordinary nodes name 8 random nodes; seven hubs name 64, 24, 8 or 3 nodes that name 64 nodes
    # each and are all deleted, so the hubs gather about 2400, 1200, 450 and 180 distinct candidates (the 8192, 2048, 1024 and 256
    # tiers); a row that loses an ordinary neighbour gathers 15 (tier 64), one that loses a hub's neighbour about 70 (tier 128)
    rng = np.random.default_rng(64)
    n, dim, Mq, M = 4000, 50, 16, 64
    _, codes, codebooks, cen = real_pq_world("made", n, dim, Mq, True)
    pqv = jv.PQVectors(codes, codebooks, dim, 256, cen)
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
    deleted[rng.choice(np.flatnonzero(~deleted[100:]) + 100, 60, replace=False)] = True  # ordinary nodes
    g = jv.GraphIndex(adj, 0)
    b = bd.builder(jv, o.DOT_PRODUCT, M, seed=5)
    got = b.removeDeletedNodes(g, pqv, deleted)
    pqs = gm.PQScores(oracle, codes, codebooks, 256, dim, cen, exact_table(pqv, codebooks, dim, 256, o.DOT_PRODUCT), o.DOT_PRODUCT)
    res = dm.remove_deleted(pqs.queries, o.DOT_PRODUCT, adj, 0, [], deleted, seed=5, prune=pqs.prune)
    hit = bd.assert_removal_matches_model(got, res, "made graph")
    print("made graph: rows per tier", hit.tolist(), got.remove_stats)
    assert (hit > 0).all() and got.remove_stats["max_candidates"] > 2048, hit.tolist()
    for h in (g, got, pqv):
        h.close()


@pytest.mark.gpu
def test_pq_removal_fallback_and_everything_deleted(jv, oracle):
    rng = np.random.default_rng(31)
    n, dim, Mq, M = 2000, 32, 8, 16
    _, codes, codebooks, cen = real_pq_world("fallback", n, dim, Mq, False)
    pqv = jv.PQVectors(codes, codebooks, dim, 256, cen)
    b = bd.builder(jv, o.EUCLIDEAN, M, beam=40, hier=True, seed=12)
    g = b.build(pqv)
    levels, entry = bd.levels(g), g.info()["entry_node"]
    deleted = np.ones(n, bool)
    deleted[rng.choice(n, 50, replace=False)] = False
    got = b.removeDeletedNodes(g, pqv, deleted)
    pqs = gm.PQScores(oracle, codes, codebooks, 256, dim, cen, exact_table(pqv, codebooks, dim, 256, o.EUCLIDEAN), o.EUCLIDEAN)
    res = dm.remove_deleted(pqs.queries, o.EUCLIDEAN, levels[0][1], entry, levels[1:], deleted, seed=12, prune=pqs.prune)
    bd.assert_removal_matches_model(got, res, "fallback")
    assert got.remove_stats["random_fallbacks"] > 0
    empty = b.removeDeletedNodes(g, pqv, np.ones(n, bool))
    inf = empty.info()
    assert inf["entry_node"] == -1 and inf["levels"] == 1 and empty.remove_stats["live_nodes"] == 0 and (empty.level(0)[1] == -1).all()
    r = jv.GraphSearcher(empty).search(pqv, gm.decode(codes[:4], codebooks, *o.pq_layout(dim, Mq), 256, cen), o.EUCLIDEAN, 5, 10)
    assert (r.nodes == -1).all() and (r.scores == 0).all()
    for h in (g, got, empty, pqv):
        h.close()


@pytest.mark.gpu
def test_pq_remove_add_remove_keeps_holes(jv):
    rng = np.random.default_rng(21)
    n0, n, dim = 3600, 4000, 32
    _, codes, codebooks, cen = real_pq_world("holes", n, dim, 8, True)
    small, pqv = jv.PQVectors(codes[:n0], codebooks, dim, 256, cen), jv.PQVectors(codes, codebooks, dim, 256, cen)
    b = bd.builder(jv, o.DOT_PRODUCT, 16, hier=True, seed=4)
    g = b.build(small)
    first = rng.random(n0) < 0.1
    rep = b.removeDeletedNodes(g, small, first)
    assert rep.remove_stats["removed"] == first.sum()
    grown = b.addGraphNodes(rep, pqv)
    wide = np.concatenate([first, np.zeros(n - n0, bool)])
    assert grown.info()["n"] == n and not np.isin(grown.level(0)[1], np.flatnonzero(first)).any()
    second = (rng.random(n) < 0.05) & ~wide
    again = b.removeDeletedNodes(grown, pqv, second | wide)
    assert again.remove_stats["removed"] == second.sum(), (again.remove_stats, second.sum())
    assert again.remove_stats["live_nodes"] == n - first.sum() - second.sum()
    for h in (g, rep, grown, again, small, pqv):
        h.close()


def _recall(nodes, truth):
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / truth.shape[1] for i in range(len(nodes))]))


@pytest.mark.gpu
def test_maintained_pq_graph_recall(jv):
    # the 20 000 x 64 latent world of test_pq_graph_recall_near_fp32_graph; PQ walk, the fp32 rows only rerank and score the test
    from test_build_steps import latent_rows
    rng = np.random.default_rng(21)
    dim, M, n = 64, 16, 20000
    data = latent_rows(rng, n + 500, dim)
    base, queries = np.ascontiguousarray(data[:n]), np.ascontiguousarray(data[n:])
    codebooks, _, _ = o.train_pq_numpy(rng, base, M, 256, iters=4)
    codes = jv.pq_encode_all(base, codebooks, M)
    vsf = o.DOT_PRODUCT
    f32, pqv = jv.F32Vectors(base), jv.PQVectors(codes, codebooks, dim)
    b = bd.builder(jv, vsf, 16, beam=100, hier=True, seed=9)

    def walk(g, pq_set, rerank, **kw):
        return jv.GraphSearcher(g).search(pq_set, queries, vsf, 10, 100, reranker=rerank, **kw).nodes

    truth, _, _ = jv.topk_bruteforce(f32, vsf, queries, 10)
    fresh = b.build(pqv)
    n0 = int(0.9 * n)
    small = jv.PQVectors(codes[:n0], codebooks, dim)
    part = b.build(small)
    added = b.addGraphNodes(part, pqv)
    r_fresh, r_add = _recall(walk(fresh, pqv, f32), truth), _recall(walk(added, pqv, f32), truth)
    deleted = rng.random(n) < 0.1
    live = np.flatnonzero(~deleted)
    rep = b.removeDeletedNodes(fresh, pqv, deleted)
    sub_f32, sub_pq = jv.F32Vectors(base[live]), jv.PQVectors(codes[live], codebooks, dim)
    survivors = b.build(sub_pq)
    truth_live = live[jv.topk_bruteforce(sub_f32, vsf, queries, 10)[0]]
    r_rep = _recall(walk(rep, pqv, f32), truth_live)
    r_orig = _recall(walk(fresh, pqv, f32, acceptOrds=~deleted), truth_live)
    r_surv = _recall(live[walk(survivors, sub_pq, sub_f32)], truth_live)
    print("recall@10: fresh %.4f, 90%% + 10%% added %.4f; 10%% removed %.4f, original + acceptOrds %.4f, fresh over survivors %.4f"
          % (r_fresh, r_add, r_rep, r_orig, r_surv))
    assert r_add >= r_fresh - 0.02, (r_fresh, r_add)
    assert r_rep >= r_surv - 0.03 and r_rep >= r_orig - 0.02, (r_rep, r_surv, r_orig)
    for h in (fresh, part, added, rep, survivors, small, sub_f32, sub_pq, f32, pqv):
        h.close()


@pytest.mark.gpu
def test_fused_pq_walk_on_maintained_pq_graph(jv, oracle):
    from test_build_steps import latent_rows
    rng = np.random.default_rng(73)
    n0, n, dim, M, k = 2200, 2500, 64, 16, 256
    data = latent_rows(rng, n, dim)
    cb, sizes, offsets = o.train_pq_numpy(rng, data[:1500], M, k, iters=2)
    codes = o.encode_pq(oracle, cb, sizes, offsets, M, k, None, data)
    small, pqv, vec = jv.PQVectors(codes[:n0], cb, dim, k), jv.PQVectors(codes, cb, dim, k), jv.F32Vectors(data)
    b = bd.builder(jv, o.DOT_PRODUCT, 16, beam=40, hier=True, seed=6)
    g = b.build(small)
    grown = b.addGraphNodes(g, pqv)
    rep = b.removeDeletedNodes(grown, pqv, rng.random(n) < 0.1)
    adj = rep.level(0)[1]
    upper = [rep.level(L) for L in range(1, rep.info()["levels"])] or None
    packed = np.empty((n, 16, M), np.uint8)
    oracle.jvo_fused_pq_pack(ip(adj), n, 16, o.bp(codes), M, o.bp(packed))
    rep.fuse_pq(pqv)
    queries = o.random_unit_vectors(rng, 32, dim)
    og = o.make_graph(adj, rep.info()["entry_node"], upper)
    got = jv.GraphSearcher(rep).search(pqv, queries, o.DOT_PRODUCT, 10, 40, reranker=vec)
    for i in range(len(queries)):
        sf = oracle.jvo_scorer_pq(o.DOT_PRODUCT, fp(cb), M, k, dim, None, o.bp(codes), n, fp(queries[i]))
        oracle.jvo_scorer_set_packed_neighbors(sf, o.bp(packed), 16)
        oracle.jvo_scorer_set_order(sf, 1)
        rr = oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(queries[i]))
        oracle.jvo_scorer_set_order(rr, 1)
        nodes = np.full(10, -1, np.int32)
        scores = np.zeros(10, np.float32)
        oracle.jvo_graph_search(C.byref(og), sf, rr, 10, 40, ip(nodes), fp(scores), None)
        oracle.jvo_scorer_free(sf)
        oracle.jvo_scorer_free(rr)
        assert np.array_equal(nodes, got.nodes[i]), i
        assert np.array_equal(scores.view(np.int32), got.scores[i].view(np.int32)), i
    for h in (g, grown, rep, small, pqv, vec):
        h.close()


@pytest.mark.gpu
def test_pq_maintenance_errors(jv):
    from jvector_b200 import _native as nat
    lib = nat.init()
    rng = np.random.default_rng(2)
    _, codes, codebooks, cen = real_pq_world("errors", 300, 32, 8, True)
    pqv, short = jv.PQVectors(codes, codebooks, 32, 256, cen), jv.PQVectors(codes[:100], codebooks, 32, 256, cen)
    f32 = jv.F32Vectors(rng.standard_normal((300, 32)).astype(np.float32))
    g = jv.GraphIndex(np.full((200, 8), -1, np.int32), 0)
    full = jv.GraphIndex(np.full((300, 8), -1, np.int32), 0)
    params = nat.BuildParams(8, 30, 1.2, 1.2, 0, 0, 0, -1)
    out, ms, st = C.c_void_p(), C.c_double(), nat.RemoveStats()
    none = np.zeros(300, bool)

    def add(graph, ds, metric=1, p=params, o_=C.byref(out)):
        a = lib.jv_graph_add_nodes_pq(graph, ds, metric, C.byref(p) if p is not None else None, None, o_, C.byref(ms))
        c = lib.jv_builder_create_from_graph_pq(graph, ds, metric, C.byref(p) if p is not None else None, None, None, o_)
        assert a == c, (a, c)
        return a

    def remove(graph, ds, metric=1, alpha=1.2, bits=none, o_=C.byref(out), st_=C.byref(st)):
        return lib.jv_graph_remove_deleted_pq(graph, ds, metric, alpha, 0, bd.bits(bits), o_, st_)

    assert add(None, pqv._h) == -2 and add(g._h, None) == -2 and add(g._h, pqv._h, p=None) == -2 and add(g._h, pqv._h, o_=None) == -2
    assert add(g._h, f32._h) == -2  # not PQ
    assert add(g._h, short._h) == -2  # n < n0
    assert add(g._h, pqv._h, metric=7) == -2
    assert add(g._h, pqv._h, p=nat.BuildParams(16, 30, 1.2, 1.2, 0, 0, 0, -1)) == -2  # degree mismatch
    assert remove(None, pqv._h) == -2 and remove(full._h, None) == -2 and remove(full._h, pqv._h, bits=None) == -2
    assert remove(full._h, pqv._h, o_=None) == -2 and remove(full._h, pqv._h, st_=None) == -2
    assert remove(full._h, f32._h) == -2  # not PQ
    assert remove(g._h, pqv._h) == -2  # n != g.n
    assert remove(full._h, pqv._h, metric=7) == -2 and remove(full._h, pqv._h, alpha=0.9) == -2
    wide, wide_full = jv.GraphIndex(np.full((200, 65), -1, np.int32), 0), jv.GraphIndex(np.full((300, 65), -1, np.int32), 0)
    assert add(wide._h, pqv._h, p=nat.BuildParams(65, 30, 1.2, 1.2, 0, 0, 0, -1)) == -5
    assert remove(wide_full._h, pqv._h) == -5
    # a LUT too large for the capacity the call needs. Removal at degree 64 needs 8192 slots (106 KB): M * k = 128 * 256 floats do
    # not fit next to them, though they fit next to the 2048 slots of degree 32 and next to the builder's 256
    m128 = jv.PQVectors(rng.integers(0, 256, (300, 128)).astype(np.uint8), rng.standard_normal(256 * 128).astype(np.float32), 128)
    deg64, deg32 = jv.GraphIndex(np.full((300, 64), -1, np.int32), 0), jv.GraphIndex(np.full((300, 32), -1, np.int32), 0)
    launches = lib.jv_kernel_launch_count()
    assert remove(deg64._h, m128._h) == -5
    assert lib.jv_kernel_launch_count() == launches and out.value is None  # refused before any device work
    assert remove(deg32._h, m128._h) == 0
    jv.GraphIndex(_handle=C.c_void_p(out.value)).close()
    out.value = None
    # an add's prune is the builder's: M * k = 256 * 256 floats do not fit at all
    big = jv.PQVectors(rng.integers(0, 256, (300, 256)).astype(np.uint8), rng.standard_normal(256 * 512).astype(np.float32), 512)
    assert add(g._h, big._h) == -5 and out.value is None
    # the fp32 entry points still refuse a PQ data set
    assert lib.jv_graph_add_nodes(g._h, pqv._h, 1, C.byref(params), None, C.byref(out), C.byref(ms)) == -2
    assert lib.jv_builder_create_from_graph(g._h, pqv._h, 1, C.byref(params), None, None, C.byref(out)) == -2
    assert lib.jv_graph_remove_deleted(full._h, pqv._h, 1, 1.2, 0, bd.bits(none), C.byref(out), C.byref(st)) == -2
    assert out.value is None
    for h in (pqv, short, f32, g, full, wide, wide_full, m128, deg64, deg32, big):
        h.close()
