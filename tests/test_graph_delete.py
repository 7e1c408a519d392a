"""Removing deleted nodes from a graph (GraphIndexBuilder.removeDeletedNodes, base:graph/GraphIndexBuilder.java:689-799).

CPU: the host restatement (tests/delete_model.py) against the reference's TestDeletions (jvector-tests/.../graph/TestDeletions.java:74-186)
and the invariants of the repair; the C entry point without a device. GPU (-m gpu): jv_graph_remove_deleted row for row against the
restatement, its other properties, and the recall of repaired graphs."""
import ctypes as C

import numpy as np
import pytest

import delete_model as dm
import oracle_lib as o
from oracle_lib import fp, ip

METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)


# ------------------------------------------------------------------------------------------------ worlds
def oracle_graph(oracle, metric, data, degree, beam=30, alpha=1.2, hier=False, rng=None):
    """a graph built by the oracle's sequential builder; hier: two nested upper levels over sampled ids, the entry on top"""
    n, dim = data.shape
    adj = np.empty((n, degree), np.int32)
    entry = oracle.jvo_graph_build_f32(metric, fp(data), n, dim, degree, beam, 1.2, alpha, ip(adj))
    if not hier:
        return adj, int(entry), []
    upper = []
    ids = np.arange(n, dtype=np.int32)
    for count in (max(4, n // 8), max(2, n // 64)):
        ids = np.sort(rng.choice(ids, count, replace=False)).astype(np.int32)
        a = np.empty((count, degree), np.int32)
        oracle.jvo_graph_build_f32(metric, fp(np.ascontiguousarray(data[ids])), count, dim, degree, beam, 1.2, alpha, ip(a))
        upper.append((ids, np.where(a >= 0, ids[np.clip(a, 0, None)], -1).astype(np.int32)))
    return adj, int(upper[-1][0][0]), upper


def reachable(adj, entry, upper):
    """live nodes a walk can reach: every level's rows from the entry down, then level 0 from everything reached"""
    seen = {entry}
    for ids, a in upper:
        rows = {int(v): r for r, v in enumerate(ids)}
        stack = [v for v in seen if v in rows]
        while stack:
            v = stack.pop()
            for k in a[rows[v]]:
                if k >= 0 and k not in seen:
                    seen.add(int(k))
                    stack.append(int(k))
    stack = list(seen)
    while stack:
        v = stack.pop()
        for k in adj[v]:
            if k >= 0 and k not in seen:
                seen.add(int(k))
                stack.append(int(k))
    return seen


def oracle_search(oracle, metric, data, res, q, k):
    g = o.make_graph(np.ascontiguousarray(res["adj0"]), res["entry"], [(i, np.ascontiguousarray(a)) for i, a in res["upper"]] or None)
    sf = oracle.jvo_scorer_f32(metric, fp(data), data.shape[0], data.shape[1], fp(np.ascontiguousarray(q, np.float32)))
    nodes = np.full(k, -1, np.int32)
    scores = np.zeros(k, np.float32)
    oracle.jvo_graph_search(C.byref(g), sf, None, k, k, ip(nodes), fp(scores), None)
    oracle.jvo_scorer_free(sf)
    return nodes


def check_invariants(res, adj0, upper, deleted, degree):
    dead = res["dead"]
    levels_old = [(np.arange(adj0.shape[0], dtype=np.int32), adj0)] + list(upper)
    new_levels = [(np.arange(adj0.shape[0], dtype=np.int32), res["adj0"])] + list(res["upper"])
    for L, (ids, adj) in enumerate(new_levels):
        old_ids, old_adj = levels_old[L]
        old_row = {int(v): r for r, v in enumerate(old_ids)}
        assert not dead[ids[(adj >= 0).any(1)]].any() if L == 0 else not dead[ids].any()
        for r, v in enumerate(ids):
            if dead[v]:
                assert L == 0 and (adj[r] == -1).all(), ("a removed node keeps a row", L, v)
                continue
            row = adj[r][adj[r] >= 0]
            assert len(row) <= degree and len(set(row.tolist())) == len(row) and v not in row
            assert not dead[row].any(), ("a row names a deleted node", L, v)
            before = old_adj[old_row[int(v)]]
            info = res["rows"][L].get(int(v))
            if info is None:
                assert np.array_equal(adj[r], before), ("a row without a deleted neighbour changed", L, v)
            elif not info["fallback"]:
                assert set(row.tolist()) <= info["cands"]
                two = set()
                for j in before[before >= 0]:
                    if dead[j]:
                        jr = old_row[int(j)]
                        two |= {int(k) for k in old_adj[jr] if k >= 0 and k != v and not dead[k]}
                live = {int(j) for j in before if j >= 0 and not dead[j]}
                assert info["cands"] == live | two


# ------------------------------------------------------------------------------------------------ CPU: the restatement
@pytest.mark.parametrize("hier", [False, True])
def test_cleanup_reconnects_the_isolated_node(oracle, hier):
    # TestDeletions.testCleanup: delete every node that links to a chosen one; it must stay reachable and be its own best match
    rng = np.random.default_rng(11 + hier)
    for trial in range(5):
        data = rng.standard_normal((40, 2)).astype(np.float32)
        adj, entry, upper = oracle_graph(oracle, o.COSINE, data, 4, beam=10, alpha=1.0, hier=hier, rng=rng)
        target = int(rng.integers(40))
        deleted = (adj == target).any(1)
        deleted[target] = False
        if not deleted.any():
            continue
        res = dm.remove_deleted(data, o.COSINE, adj, entry, upper, deleted, alpha=1.0)
        live = (~deleted).sum()
        assert res["entry"] >= 0 and not deleted[res["entry"]]
        assert target in reachable(res["adj0"], res["entry"], res["upper"])
        assert oracle_search(oracle, o.COSINE, data, res, data[target], 10)[0] == target
        assert len(set(range(40)) - set(np.flatnonzero(deleted).tolist())) == live
        check_invariants(res, adj, upper, deleted, 4)


@pytest.mark.parametrize("hier", [False, True])
def test_marking_all_nodes_as_deleted(oracle, hier):
    # TestDeletions.testMarkingAllNodesAsDeleted: nothing is left, and there is no entry node
    rng = np.random.default_rng(3)
    data = rng.standard_normal((10, 2)).astype(np.float32)
    adj, entry, upper = oracle_graph(oracle, o.COSINE, data, 2, beam=10, alpha=1.0, hier=hier, rng=rng)
    res = dm.remove_deleted(data, o.COSINE, adj, entry, upper, np.ones(10, bool), alpha=1.0)
    assert res["entry"] == -1 and res["levels"] == 1 and (res["adj0"] == -1).all()


@pytest.mark.parametrize("hier", [False, True])
def test_no_path_to_live_nodes_two_clusters(oracle, hier):
    # TestDeletions.testNoPathToLiveNodesWhenRemovingDeletedNodes2: the larger of two far-apart clusters is deleted; the entry
    # must be live. Under COSINE (the reference's setting) the 2-d clusters are nearly one direction and the graph is poorly
    # connected to begin with; under EUCLIDEAN the repaired graph must also reach every live node from the entry.
    for metric in (o.COSINE, o.EUCLIDEAN):
        rng = np.random.default_rng(7)
        data = np.concatenate([0.01 + 100 * rng.random((1000, 2)), 10000 + 100 * rng.random((100, 2))]).astype(np.float32)
        adj, entry, upper = oracle_graph(oracle, metric, data, 4, beam=10, alpha=1.0, hier=hier, rng=rng)
        deleted = np.arange(1100) < 1000
        res = dm.remove_deleted(data, metric, adj, entry, upper, deleted, alpha=1.0)
        assert res["entry"] >= 1000
        if metric == o.EUCLIDEAN:
            assert reachable(res["adj0"], res["entry"], res["upper"]) >= set(range(1000, 1100))
        check_invariants(res, adj, upper, deleted, 4)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("hier", [False, True])
def test_restatement_invariants(oracle, metric, hier):
    rng = np.random.default_rng(100 + 3 * metric + hier)
    n, dim, degree = 1500, 16, 12
    data = o.random_unit_vectors(rng, n, dim)
    adj, entry, upper = oracle_graph(oracle, metric, data, degree, hier=hier, rng=rng)
    for frac in (0.01, 0.1, 0.4):
        deleted = rng.random(n) < frac
        deleted[entry] = frac > 0.3  # the entry node goes in one case
        res = dm.remove_deleted(data, metric, adj, entry, upper, deleted, seed=9)
        check_invariants(res, adj, upper, deleted, degree)
        assert res["entry"] >= 0 and not deleted[res["entry"]]
        if hier:
            assert res["entry"] in set(res["upper"][-1][0].tolist())
        # removing again with the result's holes changes nothing
        again = dm.remove_deleted(data, metric, res["adj0"], res["entry"], res["upper"], np.zeros(n, bool), holes=deleted)
        assert np.array_equal(again["adj0"], res["adj0"]) and not any(again["rows"])


def test_random_fallback_draws_live_members(oracle):
    # a row whose deleted neighbours offer no live id takes random live members of its level (GraphIndexBuilder.java:743-759)
    rng = np.random.default_rng(21)
    n, degree = 400, 8
    data = o.random_unit_vectors(rng, n, 8)
    adj, entry, _ = oracle_graph(oracle, o.DOT_PRODUCT, data, degree)
    keep = rng.choice(n, 12, replace=False)
    deleted = np.ones(n, bool)
    deleted[keep] = False
    res = dm.remove_deleted(data, o.DOT_PRODUCT, adj, entry, [], deleted, seed=5)
    fb = [v for v, r in res["rows"][0].items() if r["fallback"]]
    assert fb
    for v in fb:
        row = res["adj0"][v]
        assert set(row[row >= 0].tolist()) <= set(keep.tolist()) - {v}
    assert dm.repair_random(5, 0, 17, 3) == dm.repair_random(5, 0, 17, 3) != dm.repair_random(6, 0, 17, 3)


def test_remove_deleted_without_device():
    from jvector_b200 import _native as nat
    lib = nat.load()
    if lib.jv_gpu_device_count() > 0:
        pytest.skip("a GPU is present")
    st = nat.RemoveStats()
    bits = np.zeros(4, np.uint32)
    out = C.c_void_p()
    assert lib.jv_graph_remove_deleted(None, None, 1, 1.2, 0, bits.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(out), C.byref(st)) == -1


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


def latent_rows(rng, n, dim, latent=16, noise=0.35):
    A = rng.standard_normal((latent, dim)).astype(np.float32) / np.sqrt(latent)
    x = rng.standard_normal((n, latent)).astype(np.float32) @ A + noise * rng.standard_normal((n, dim)).astype(np.float32)
    return np.ascontiguousarray(x / np.linalg.norm(x, axis=1, keepdims=True), dtype=np.float32)


def device_levels(gi):
    inf = gi.info()
    return [gi.level(L) for L in range(inf["levels"])]


def assert_matches_oracle(gi, res, what):
    """entry, levels and memberships equal; every row the restatement did not flag as a near tie equal, id for id"""
    inf = gi.info()
    assert inf["entry_node"] == res["entry"] and inf["levels"] == res["levels"], (what, inf, res["entry"], res["levels"])
    dev = device_levels(gi)
    want = [(np.arange(res["adj0"].shape[0], dtype=np.int32), res["adj0"])] + list(res["upper"])
    repaired = flagged = 0
    for L, ((dids, dadj), (wids, wadj)) in enumerate(zip(dev, want)):
        assert np.array_equal(dids, wids), (what, "members of level", L)
        skip = np.array([bool(res["rows"][L].get(int(v), {}).get("flag")) for v in wids], bool)
        repaired += len(res["rows"][L])
        flagged += int(skip.sum())
        bad = np.flatnonzero(~skip & (dadj != wadj).any(1))
        assert len(bad) == 0, (what, "level", L, "rows differ", bad[:5].tolist(), dadj[bad[:1]].tolist(), wadj[bad[:1]].tolist())
    return repaired, flagged


def warp_keys(oracle, metric, data):
    """the candidates' scores with the device's bits (warp-order oracle scorer): the sort order is then certain"""
    dim = data.shape[1]
    return lambda v, ids: np.array([oracle.jvo_compare_f32_warp(metric, fp(data[v]), fp(data[i]), dim) for i in ids], np.float32)


def _remove(jv, metric, gi, vec, deleted, seed=0, alpha=1.2):
    b = jv.GraphIndexBuilder(metric, M=gi.info()["degree"], alpha=alpha, seed=seed)
    return b.removeDeletedNodes(gi, vec, deleted)


def _upper_of(gi):
    return [gi.level(L) for L in range(1, gi.info()["levels"])]


@pytest.fixture(scope="module")
def latent_world(jv):
    rng = np.random.default_rng(2024)
    data = latent_rows(rng, 20000, 64)
    return data, jv.F32Vectors(data)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("hier", [False, True])
def test_device_equals_restatement(jv, oracle, latent_world, metric, hier):
    data, vec = latent_world
    rng = np.random.default_rng(40 + 2 * metric + hier)
    gi = jv.GraphIndexBuilder(metric, M=16, beamWidth=60, alpha=1.2, addHierarchy=hier, seed=3).build(vec)
    _, adj0 = gi.level(0)
    upper, entry = _upper_of(gi), gi.info()["entry_node"]
    cases = [(0.01, False), (0.1, True)] if metric != o.DOT_PRODUCT else [(0.01, False), (0.1, False), (0.1, True)]
    for frac, kill_entry in cases:
        deleted = rng.random(data.shape[0]) < frac
        deleted[entry] = kill_entry
        got = _remove(jv, metric, gi, vec, deleted, seed=17)
        res = dm.remove_deleted(data, metric, adj0, entry, upper, deleted, seed=17, key_scores=warp_keys(oracle, metric, data))
        repaired, flagged = assert_matches_oracle(got, res, (metric, hier, frac, kill_entry))
        st = got.remove_stats
        assert st["repaired_rows"] == repaired and st["removed"] == deleted.sum() and st["live_nodes"] == (~deleted).sum()
        assert st["candidates"] == sum(len(r["cands"]) for lv in res["rows"] for r in lv.values())
        assert flagged <= 0.01 * repaired, (flagged, repaired)
        got.close()
    gi.close()


@pytest.mark.gpu
def test_device_large_candidate_sets(jv, oracle, latent_world):
    # 40 % deleted at degree 32: candidate sets past 256 take the high-capacity prune kernels, never a clipped set
    data, vec = latent_world
    rng = np.random.default_rng(8)
    for hier in (False, True):
        gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=32, beamWidth=60, alpha=1.2, addHierarchy=hier, seed=4).build(vec)
        _, adj0 = gi.level(0)
        deleted = rng.random(data.shape[0]) < 0.4
        got = _remove(jv, o.DOT_PRODUCT, gi, vec, deleted, seed=1)
        assert got.remove_stats["max_candidates"] > 256
        res = dm.remove_deleted(data, o.DOT_PRODUCT, adj0, gi.info()["entry_node"], _upper_of(gi), deleted, seed=1,
                                key_scores=warp_keys(oracle, o.DOT_PRODUCT, data))
        repaired, flagged = assert_matches_oracle(got, res, ("40%", hier))
        # ~300 candidates per row make ~600 isDiverse tests per row: about 1 % of these rows hold one within 1e-5
        assert flagged <= 0.02 * repaired, (flagged, repaired)
        got.close()
        gi.close()


@pytest.mark.gpu
def test_device_fallback_everything_deleted_and_snapshot(jv, oracle):
    rng = np.random.default_rng(31)
    n = 3000
    data = latent_rows(rng, n, 32)
    vec = jv.F32Vectors(data)
    gi = jv.GraphIndexBuilder(o.EUCLIDEAN, M=16, beamWidth=40, alpha=1.2, addHierarchy=True, seed=2).build(vec)
    before = device_levels(gi)
    _, adj0 = before[0]
    entry, upper = gi.info()["entry_node"], _upper_of(gi)
    # almost everything deleted: rows whose deleted neighbours offer nothing take random live members
    deleted = np.ones(n, bool)
    deleted[rng.choice(n, 60, replace=False)] = False
    got = _remove(jv, o.EUCLIDEAN, gi, vec, deleted, seed=12)
    keys = warp_keys(oracle, o.EUCLIDEAN, data)
    res = dm.remove_deleted(data, o.EUCLIDEAN, adj0, entry, upper, deleted, seed=12, key_scores=keys)
    assert got.remove_stats["random_fallbacks"] == sum(r["fallback"] for lv in res["rows"] for r in lv.values()) > 0
    assert_matches_oracle(got, res, "fallback")
    # two calls give the same bytes; the input graph is untouched
    again = _remove(jv, o.EUCLIDEAN, gi, vec, deleted, seed=12)
    for (a_ids, a_adj), (b_ids, b_adj) in zip(device_levels(got), device_levels(again)):
        assert np.array_equal(a_ids, b_ids) and np.array_equal(a_adj, b_adj)
    for (a_ids, a_adj), (b_ids, b_adj) in zip(before, device_levels(gi)):
        assert np.array_equal(a_ids, b_ids) and np.array_equal(a_adj, b_adj)
    # a second removal on the repaired graph counts the holes as gone and never links one
    more = ~deleted & (rng.random(n) < 0.5)
    second = _remove(jv, o.EUCLIDEAN, got, vec, more, seed=12)
    assert second.remove_stats["live_nodes"] == (~(deleted | more)).sum() and second.remove_stats["removed"] == more.sum()
    res2 = dm.remove_deleted(data, o.EUCLIDEAN, res["adj0"], res["entry"], res["upper"], more, seed=12, holes=deleted, key_scores=keys)
    assert_matches_oracle(second, res2, "second removal")
    _, a2 = second.level(0)
    assert not (deleted | more)[a2[a2 >= 0]].any()
    # everything deleted: no entry, one level, and a search returns padding without launching anything
    empty = _remove(jv, o.EUCLIDEAN, gi, vec, np.ones(n, bool))
    inf = empty.info()
    assert inf["entry_node"] == -1 and inf["levels"] == 1 and empty.remove_stats["live_nodes"] == 0
    assert (empty.level(0)[1] == -1).all()
    from jvector_b200 import _native as nat
    launches = nat.load().jv_kernel_launch_count()
    r = jv.GraphSearcher(empty).search(vec, data[:4], o.EUCLIDEAN, 5, 10)
    assert (r.nodes == -1).all() and (r.scores == 0).all() and nat.load().jv_kernel_launch_count() == launches
    for g in (got, again, second, empty, gi):
        g.close()
    vec.close()


@pytest.mark.gpu
def test_fused_pq_walk_on_repaired_graph(jv, oracle):
    rng = np.random.default_rng(73)
    n, dim, M, k = 2500, 64, 16, 256
    data = latent_rows(rng, n, dim)
    vec = jv.F32Vectors(data)
    gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=40, alpha=1.2, addHierarchy=True, seed=6).build(vec)
    rep = _remove(jv, o.DOT_PRODUCT, gi, vec, rng.random(n) < 0.1, seed=2)
    _, adj = rep.level(0)
    upper = _upper_of(rep) or None
    cb, sizes, offsets = o.train_pq_numpy(rng, data[:1500], M, k, iters=2)
    codes = o.encode_pq(oracle, cb, sizes, offsets, M, k, None, data)
    packed = np.empty((n, 16, M), np.uint8)
    oracle.jvo_fused_pq_pack(ip(adj), n, 16, o.bp(codes), M, o.bp(packed))
    pqv = jv.PQVectors(codes, cb, dim, k)
    rep.fuse_pq(pqv)
    queries = o.random_unit_vectors(rng, 32, dim)
    g = o.make_graph(adj, rep.info()["entry_node"], upper)
    got = jv.GraphSearcher(rep).search(pqv, queries, o.DOT_PRODUCT, 10, 40, reranker=vec)
    for i in range(len(queries)):
        sf = oracle.jvo_scorer_pq(o.DOT_PRODUCT, fp(cb), M, k, dim, None, o.bp(codes), n, fp(queries[i]))
        oracle.jvo_scorer_set_packed_neighbors(sf, o.bp(packed), 16)
        oracle.jvo_scorer_set_order(sf, 1)
        rr = oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(queries[i]))
        oracle.jvo_scorer_set_order(rr, 1)
        nodes = np.full(10, -1, np.int32)
        scores = np.zeros(10, np.float32)
        oracle.jvo_graph_search(C.byref(g), sf, rr, 10, 40, ip(nodes), fp(scores), None)
        oracle.jvo_scorer_free(sf)
        oracle.jvo_scorer_free(rr)
        assert np.array_equal(nodes, got.nodes[i]), i
        assert np.array_equal(scores.view(np.int32), got.scores[i].view(np.int32)), i
    for h in (rep, gi, pqv, vec):
        h.close()


def _recall(nodes, truth):
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / truth.shape[1] for i in range(len(nodes))]))


@pytest.mark.gpu
@pytest.mark.parametrize("world", ["siftsmall", "latent"])
def test_repaired_graph_recall(jv, sift, world):
    rng = np.random.default_rng(55)
    if world == "siftsmall":
        data, queries, _ = sift
        metric = o.EUCLIDEAN
    else:
        data = latent_rows(rng, 20000, 64)
        queries = latent_rows(rng, 200, 64)
        metric = o.DOT_PRODUCT
    n = data.shape[0]
    deleted = rng.random(n) < 0.1
    live = np.flatnonzero(~deleted)
    vec = jv.F32Vectors(data)
    kw = dict(M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=9)
    gi = jv.GraphIndexBuilder(metric, **kw).build(vec)
    rep = jv.GraphIndexBuilder(metric, **kw).removeDeletedNodes(gi, vec, deleted)
    sub = jv.F32Vectors(data[live])
    fresh = jv.GraphIndexBuilder(metric, **kw).build(sub)
    truth_local, _, _ = jv.topk_bruteforce(sub, metric, queries, 10)
    truth = live[truth_local]
    r_orig = _recall(jv.GraphSearcher(gi).search(vec, queries, metric, 10, 100, acceptOrds=~deleted).nodes, truth)
    r_rep = _recall(jv.GraphSearcher(rep).search(vec, queries, metric, 10, 100).nodes, truth)
    r_fresh = _recall(live[jv.GraphSearcher(fresh).search(sub, queries, metric, 10, 100).nodes], truth)
    assert r_rep >= r_orig - 0.02 and r_rep >= r_fresh - 0.03, (world, r_orig, r_rep, r_fresh)
    for h in (gi, rep, fresh, vec, sub):
        h.close()


@pytest.mark.gpu
def test_remove_deleted_errors(jv):
    from jvector_b200 import _native as nat
    rng = np.random.default_rng(1)
    data = latent_rows(rng, 200, 16)
    vec = jv.F32Vectors(data)
    wide = jv.GraphIndex(np.full((200, 65), -1, np.int32), 0)
    with pytest.raises(jv.JVectorB200Error) as e:
        _remove(jv, o.DOT_PRODUCT, wide, vec, np.zeros(200, bool))
    assert e.value.code == -5
    small = jv.GraphIndex(np.full((100, 8), -1, np.int32), 0)
    with pytest.raises(jv.JVectorB200Error) as e:
        _remove(jv, o.DOT_PRODUCT, small, vec, np.zeros(100, bool))
    assert e.value.code == -2
    g = jv.GraphIndex(np.full((200, 8), -1, np.int32), 0)
    with pytest.raises(jv.JVectorB200Error) as e:
        _remove(jv, o.DOT_PRODUCT, g, vec, np.zeros(200, bool), alpha=0.9)
    assert e.value.code == -2
    st = nat.RemoveStats()
    assert nat.load().jv_graph_remove_deleted(g._h, vec._h, 1, 1.2, 0, None, None, C.byref(st)) == -2
    for h in (wide, small, g, vec):
        h.close()
