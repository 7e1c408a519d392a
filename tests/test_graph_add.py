"""addGraphNode for a batch (jv_graph_add_nodes / jv_builder_create_from_graph), checked against the seeded host restatement of the
builder (tests/graph_model.py BuildModel with a graph's rows, extend_levels).

CPU: the seeded model, chained one node per call, reproduces the reference's testDiversity lists; new nodes take the tail of the
build's level draws; both entry points report a missing device.
GPU (-m gpu): an add into a one-node graph is byte-for-byte a build; adds into device builds (50 / 90 / 99 %), repaired graphs,
graphs with marked nodes, hand-made graphs with empty slots mid-row and emptied graphs equal the model batch by batch, row for row,
including the upper levels and the entry; the step-wise and one-call forms agree; n == n0 copies the graph; the result searches
like the oracle over its downloaded levels; the input graph is untouched; errors; holes survive an add; recall of an add against a
fresh build."""
import ctypes as C

import numpy as np
import pytest

import builder_driver as bd
import graph_model as gm
import oracle_lib as o
from oracle_lib import fp, ip
from test_build_steps import CASES, _budget, latent_rows, world

METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)


# ------------------------------------------------------------------------------------------------ CPU
def test_seeded_model_chain_reproduces_golden_diversity_lists(oracle):
    # tests:graph/TestVectorGraph.java:457-525 testDiversity, one node added per call: with overflow 1.0 no row ever exceeds M, so
    # the compacted graph handed to the next call is the builder's own state
    ang = np.array([0.5, 0.75, 0.2, 0.9, 0.8, 0.77, 0.6]) * np.pi
    vec = np.ascontiguousarray(np.stack([np.cos(ang), np.sin(ang)], 1), dtype=np.float32)
    expected = {3: {0: [1, 2], 1: [0], 2: [0]},
                4: {0: [1, 2], 1: [0, 3], 2: [0], 3: [1]},
                5: {0: [1, 2], 1: [0, 3, 4], 2: [0], 3: [1, 4], 4: [1, 3]},
                6: {0: [1, 2], 1: [0, 3, 4, 5], 2: [0], 3: [1, 4], 4: [1, 3, 5], 5: [1, 4]}}
    kw = dict(M=4, beam=10, overflow=1.0, alpha=1.0, window=0)
    adj, flagged = gm.BuildModel(gm.F32Scores(oracle, vec[:3], o.DOT_PRODUCT), **kw).build()
    for n, want in expected.items():
        if n > 3:
            m = gm.BuildModel(gm.F32Scores(oracle, vec[:n], o.DOT_PRODUCT), rows=adj, entry=0, **kw)
            assert m.next_batch() == (n - 1, 1)
            adj, flagged = m.build()
        assert flagged == 0
        for node, nbrs in want.items():
            assert sorted(int(x) for x in adj[node] if x >= 0) == nbrs, (n, node, adj[node].tolist())


def test_seeded_model_squeezes_rows_and_starts_at_the_entry(oracle):
    data = o.random_unit_vectors(np.random.default_rng(3), 40, 8)
    rows = np.array([[-1, 2, -1, 1], [0, -1, -1, -1], [-1, -1, -1, -1]], np.int32)
    scores = gm.F32Scores(oracle, data, o.DOT_PRODUCT)
    m = gm.BuildModel(scores, M=4, beam=10, rows=rows, entry=1)
    assert m.adj[0, :3].tolist() == [2, 1, -1] and m.deg[:3].tolist() == [2, 1, 0]
    assert (m.entry, m.inserted, m.next_batch()) == (1, 3, (3, 1))
    empty = gm.BuildModel(scores, M=4, beam=10, rows=rows, entry=-1)
    assert (empty.entry, empty.inserted) == (3, 4)  # no entry: the first new node is the entry, as node 0 is for a build


def test_new_nodes_take_the_tail_of_the_level_draws():
    n0, n, M, seed = 7000, 20000, 16, 5
    members, _ = gm.assign_levels(n, M, seed)
    fresh = gm.added_levels(n0, n, M, seed)
    assert len(fresh) == len(members) or (len(fresh) < len(members) and all(not (m >= n0).any() for m in members[len(fresh):]))
    for lv, ids in enumerate(fresh):
        assert np.array_equal(ids, members[lv][members[lv] >= n0]), lv
    old, _ = gm.assign_levels(n0, M, seed)  # the build of the first n0 rows drew the same levels for them
    for lv, ids in enumerate(old):
        assert np.array_equal(ids, members[lv][members[lv] < n0]), lv


def test_add_entry_points_without_device():
    from jvector_b200 import _native as nat
    lib = nat.load()
    if lib.jv_gpu_device_count() > 0:
        pytest.skip("a GPU is present")
    params = nat.BuildParams(16, 60, 1.2, 1.2, 0, 0, 0, -1)
    out = C.c_void_p(1234)
    ms = C.c_double(7.0)
    assert lib.jv_graph_add_nodes(None, None, 1, C.byref(params), None, C.byref(out), C.byref(ms)) == -1
    assert out.value == 1234 and ms.value == 7.0
    assert lib.jv_builder_create_from_graph(None, None, 1, C.byref(params), None, None, C.byref(out)) == -1
    assert out.value == 1234


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


def drive_add(jv, oracle, vec, data, g, case, marks=None):
    """the add of rows [n0, n) to g driven step by step against the seeded model (builder_driver.drive_add), on whole batches.
    Returns (graph, tally, batches, dropped, upper levels checked)"""
    from jvector_b200 import _native as nat
    cid, _, metric, M, beam, window, alpha, overflow, max_batch, _ = case
    params = nat.BuildParams(M, beam, overflow, alpha, 0, 3, max_batch, window)
    gi, tally, batches, dropped, (up, _) = bd.drive_add(nat.init(), g, vec, metric, params, marks, lambda: gm.F32Scores(oracle, data, metric),
                                                        cid, slices=1)
    return gi, tally, batches, dropped, up


def check_budgets(case, tally):
    # test_build_steps' budgets; a small add (20 rows at 99 %) may still meet one near tie
    for kind, (rows, flagged, differ) in tally.items():
        assert flagged <= max(1, _budget(case, kind) * rows), (case[0], kind, rows, flagged)
        assert differ <= max(1, 0.01 * rows), (case[0], kind, rows, differ)


def _case(cid, metric, M=16, beam=60, window=-1, max_batch=0):
    # the shape of test_build_steps.CASES: (id, world, metric, M, beam, window, alpha, overflow, max_batch, hierarchy)
    return (cid, "latent:48:2000", metric, M, beam, window, 1.2, 1.2, max_batch, False)


def _build(jv, vec, case, hier):
    _, _, metric, M, beam, window, alpha, overflow, max_batch, _ = case
    return jv.GraphIndexBuilder(metric, M=M, beamWidth=beam, neighborOverflow=overflow, alpha=alpha, addHierarchy=hier, seed=3,
                                max_batch=max_batch, concurrent_window=window).build(vec)


# an add into a graph of one node with an empty row starts exactly where a build starts
ANCHOR_CASES = ("tc64_dot", "k256_l2_d33", "k256_win60_dot_b64", "rowcap16_cos_d768")


@pytest.mark.gpu
@pytest.mark.parametrize("cid", ANCHOR_CASES)
def test_add_to_one_node_graph_is_the_build(jv, cid):
    case = next(c for c in CASES if c[0] == cid)
    _, wname, metric, M, beam, window, alpha, overflow, max_batch, _ = case
    data = world(wname)
    vec = jv.F32Vectors(data)
    b = jv.GraphIndexBuilder(metric, M=M, beamWidth=beam, neighborOverflow=overflow, alpha=alpha, max_batch=max_batch, concurrent_window=window)
    built = b.build(vec)
    want = (b.batches, b.dropped_backlinks)
    one = jv.GraphIndex(np.full((1, M), -1, np.int32), 0)
    added = b.addGraphNodes(one, vec)
    assert (b.batches, b.dropped_backlinks) == want, (cid, b.batches, b.dropped_backlinks, want)
    assert added.info() == built.info()
    assert added.level(0)[1].tobytes() == built.level(0)[1].tobytes(), cid
    for h in (built, one, added, vec):
        h.close()


# (id, metric, fraction of the rows in the graph before the add, hierarchy)
ADD_CASES = [("half_dot", o.DOT_PRODUCT, 0.5, False), ("half_cos_hier", o.COSINE, 0.5, True),
             ("p90_l2", o.EUCLIDEAN, 0.9, False), ("p90_dot_hier", o.DOT_PRODUCT, 0.9, True),
             ("p99_cos", o.COSINE, 0.99, False), ("p99_l2_hier", o.EUCLIDEAN, 0.99, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("cid,metric,frac,hier", ADD_CASES, ids=[c[0] for c in ADD_CASES])
def test_add_to_device_build_equals_model(jv, oracle, cid, metric, frac, hier):
    case = _case(cid, metric)
    data = world(case[1])
    n0 = int(frac * data.shape[0])
    small, vec = jv.F32Vectors(data[:n0]), jv.F32Vectors(data)
    g = _build(jv, small, case, hier)
    before = bd.levels(g)
    gi, tally, batches, dropped, up = drive_add(jv, oracle, vec, data, g, case)
    print("%s: %d batches, dropped %d, insert %s, re-prune %s, upper levels checked %d" % (cid, batches, dropped, tally["insert"], tally["reprune"], up))
    check_budgets(case, tally)
    after = bd.levels(g)  # the input graph is untouched
    assert all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) for a, b in zip(before, after)) and len(before) == len(after)
    for h in (g, gi, small, vec):
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("origin", ["removed", "marked", "mid_row_holes", "all_removed"])
def test_add_to_other_graphs_equals_model(jv, oracle, origin):
    rng = np.random.default_rng(sum(map(ord, origin)))
    metric = {"removed": o.DOT_PRODUCT, "marked": o.EUCLIDEAN, "mid_row_holes": o.COSINE, "all_removed": o.DOT_PRODUCT}[origin]
    case = _case(origin, metric)
    data = world(case[1])
    n = data.shape[0]
    n0 = n // 2 if origin == "all_removed" else int(0.9 * n)
    small, vec = jv.F32Vectors(data[:n0]), jv.F32Vectors(data)
    g = _build(jv, small, case, origin != "mid_row_holes")
    marks = None
    b = jv.GraphIndexBuilder(metric, M=16, seed=3)
    if origin == "removed":
        g = b.removeDeletedNodes(g, small, rng.random(n0) < 0.1)
    elif origin == "all_removed":
        g = b.removeDeletedNodes(g, small, np.ones(n0, bool))
        assert g.info()["entry_node"] == -1
    elif origin == "marked":
        marks = rng.random(n0) < 0.05
    else:
        adj = g.level(0)[1].copy()
        hit = rng.random(n0) < 0.3
        adj[hit, 2] = -1  # an empty slot between two neighbours
        adj[hit & (rng.random(n0) < 0.5), 0] = -1
        g = jv.GraphIndex(adj, g.info()["entry_node"])
    gi, tally, batches, dropped, up = drive_add(jv, oracle, vec, data, g, case, marks)
    print("%s: %d batches, dropped %d, insert %s, re-prune %s, upper levels checked %d" % (origin, batches, dropped, tally["insert"], tally["reprune"], up))
    check_budgets(case, tally)
    if origin == "all_removed":
        assert gi.info()["entry_node"] == n0
    for h in (g, gi, small, vec):
        h.close()


@pytest.mark.gpu
def test_zero_new_nodes_copies_the_graph(jv):
    case = _case("zero", o.DOT_PRODUCT)
    data = world(case[1])
    vec = jv.F32Vectors(data)
    b = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60)
    g = _build(jv, vec, case, True)
    same = b.addGraphNodes(g, vec)
    bd.assert_same_graph(g, same, "n == n0")
    assert g.info()["levels"] > 1
    adj = g.level(0)[1].copy()
    adj[::3, 1] = -1
    holes = jv.GraphIndex(adj, g.info()["entry_node"], [g.level(lv) for lv in range(1, g.info()["levels"])])
    copy = b.addGraphNodes(holes, vec)  # rows with empty slots mid-row come back as they were
    bd.assert_same_graph(holes, copy, "empty slots mid-row")
    for h in (g, same, holes, copy, vec):
        h.close()


@pytest.mark.gpu
def test_search_on_the_added_graph_equals_oracle(jv, oracle):
    metric = o.DOT_PRODUCT
    rng = np.random.default_rng(12)
    data = latent_rows(rng, 6000, 64)
    queries = latent_rows(rng, 64, 64)
    n0 = 5000
    small, vec = jv.F32Vectors(data[:n0]), jv.F32Vectors(data)
    b = jv.GraphIndexBuilder(metric, M=16, beamWidth=60, addHierarchy=True, seed=11)
    g = b.build(small)
    gi = b.addGraphNodes(g, vec)
    res = jv.GraphSearcher(gi).search(vec, queries, metric, 10, 40)
    levels = bd.levels(gi)
    og = o.make_graph(np.ascontiguousarray(levels[0][1]), gi.info()["entry_node"],
                      [(i, np.ascontiguousarray(a)) for i, a in levels[1:]] or None)
    tot = np.zeros(3, np.int64)
    for i in range(len(queries)):
        sf = oracle.jvo_scorer_f32(metric, fp(data), data.shape[0], data.shape[1], fp(queries[i]))
        oracle.jvo_scorer_set_order(sf, 1)
        nodes = np.full(10, -1, np.int32)
        scores = np.zeros(10, np.float32)
        st = o.Stats()
        oracle.jvo_graph_search(C.byref(og), sf, None, 10, 40, ip(nodes), fp(scores), C.byref(st))
        oracle.jvo_scorer_free(sf)
        assert np.array_equal(nodes, res.nodes[i]) and scores.tobytes() == res.scores[i].tobytes(), i
        tot += (st.visited, st.expanded, st.expanded_base)
    assert (res.visitedCount, res.expandedCount, res.expandedCountBaseLayer) == tuple(int(x) for x in tot)
    assert (levels[1][0] >= n0).any(), "no new node reached level 1"
    for h in (g, gi, small, vec):
        h.close()


@pytest.mark.gpu
def test_add_nodes_errors(jv):
    from jvector_b200 import _native as nat
    lib = nat.init()
    data = latent_rows(np.random.default_rng(1), 300, 16)
    vec, short = jv.F32Vectors(data), jv.F32Vectors(data[:100])
    g = jv.GraphIndex(np.full((200, 8), -1, np.int32), 0)
    params = nat.BuildParams(8, 30, 1.2, 1.2, 0, 0, 0, -1)
    out, ms = C.c_void_p(), C.c_double()

    def rc(graph, ds, metric=1, p=params, o_=C.byref(out)):
        a = lib.jv_graph_add_nodes(graph, ds, metric, C.byref(p) if p is not None else None, None, o_, C.byref(ms))
        b = lib.jv_builder_create_from_graph(graph, ds, metric, C.byref(p) if p is not None else None, None, None, o_)
        assert a == b, (a, b)
        return a

    assert rc(None, vec._h) == -2
    assert rc(g._h, None) == -2
    assert rc(g._h, vec._h, p=None) == -2
    assert rc(g._h, vec._h, o_=None) == -2
    assert rc(g._h, short._h) == -2  # n < n0
    assert rc(g._h, vec._h, metric=7) == -2
    assert rc(g._h, vec._h, p=nat.BuildParams(16, 30, 1.2, 1.2, 0, 0, 0, -1)) == -2  # degree mismatch
    bq = jv.BQVectors(jv.bq_encode_all(data), 16)
    assert rc(g._h, bq._h) == -2  # not fp32
    wide = jv.GraphIndex(np.full((200, 65), -1, np.int32), 0)
    assert rc(wide._h, vec._h, p=nat.BuildParams(65, 30, 1.2, 1.2, 0, 0, 0, -1)) == -5
    assert out.value is None
    for h in (vec, short, g, bq, wide):
        h.close()


@pytest.mark.gpu
def test_remove_add_remove_keeps_holes(jv):
    rng = np.random.default_rng(21)
    metric = o.DOT_PRODUCT
    data = latent_rows(rng, 4000, 32)
    n0 = 3600
    small, vec = jv.F32Vectors(data[:n0]), jv.F32Vectors(data)
    b = jv.GraphIndexBuilder(metric, M=16, beamWidth=60, addHierarchy=True, seed=4)
    g = b.build(small)
    first = rng.random(n0) < 0.1
    rep = b.removeDeletedNodes(g, small, first)
    assert rep.remove_stats["removed"] == first.sum()
    grown = b.addGraphNodes(rep, vec)
    assert grown.info()["n"] == 4000 and not (np.isin(grown.level(0)[1], np.flatnonzero(first))).any()
    second = (rng.random(4000) < 0.05) & ~np.concatenate([first, np.zeros(400, bool)])
    again = b.removeDeletedNodes(grown, vec, second | np.concatenate([first, np.zeros(400, bool)]))
    assert again.remove_stats["removed"] == second.sum(), (again.remove_stats, second.sum())
    assert again.remove_stats["live_nodes"] == 4000 - first.sum() - second.sum()
    for h in (g, rep, grown, again, small, vec):
        h.close()


def _recall(nodes, truth):
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / truth.shape[1] for i in range(len(nodes))]))


@pytest.mark.gpu
def test_added_graph_recall(jv):
    rng = np.random.default_rng(77)
    metric = o.DOT_PRODUCT
    data = latent_rows(rng, 20000, 128)
    queries = latent_rows(rng, 200, 128)
    n = data.shape[0]
    n0 = int(0.9 * n)
    small, vec = jv.F32Vectors(data[:n0]), jv.F32Vectors(data)
    b = jv.GraphIndexBuilder(metric, M=32, beamWidth=100, addHierarchy=True, seed=9)
    fresh = b.build(vec)
    added = b.addGraphNodes(b.build(small), vec)
    truth, _, _ = jv.topk_bruteforce(vec, metric, queries, 10)
    r_fresh = _recall(jv.GraphSearcher(fresh).search(vec, queries, metric, 10, 100).nodes, truth)
    r_add = _recall(jv.GraphSearcher(added).search(vec, queries, metric, 10, 100).nodes, truth)
    self_top1 = float(np.mean(jv.GraphSearcher(added).search(vec, data[n0:], metric, 1, 100).nodes[:, 0] == np.arange(n0, n)))
    print("recall@10 fresh %.4f, add %.4f; new nodes found as their own top-1: %.4f" % (r_fresh, r_add, self_top1))
    assert r_add >= r_fresh - 0.01 and self_top1 >= 0.99, (r_fresh, r_add, self_top1)
    for h in (fresh, added, small, vec):
        h.close()
