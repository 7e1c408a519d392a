"""The refine pass on the device (jv_graph_refine: GraphIndexBuilder.cleanup's improveConnections and OnDiskGraphIndexCompactor's
refine pass), against the host restatement tests/refine_model.py.

CPU: the restatement on its own: the union, the exclusion of the node itself, the compactor's beam, the maxLevel > 0 gate.
GPU (-m gpu): the search's exclusion against an accept bitset per query; both forms row for row against the restatement (fp32 on all
metrics with several batches, PQ, BQ, the compactor form after a compaction, flat and hierarchical); the invariants of every output;
copies, holes, repeated calls, refineFinalGraph; recall on siftsmall; every error of the ABI."""
import ctypes as C

import numpy as np
import pytest

import graph_model as gm
import oracle_lib as o
import refine_model as rm
from oracle_lib import fp, ip

METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)


def latent_rows(rng, n, dim, latent=16, noise=0.35):
    A = rng.standard_normal((latent, dim)).astype(np.float32) / np.sqrt(latent)
    x = rng.standard_normal((n, latent)).astype(np.float32) @ A + noise * rng.standard_normal((n, dim)).astype(np.float32)
    return np.ascontiguousarray(x / np.linalg.norm(x, axis=1, keepdims=True), dtype=np.float32)


def oracle_levels(oracle, metric, data, M, rng, upper_counts=(), beam=30):
    """a graph built by the oracle's sequential builder, nested upper levels over sampled ids: ([(ids, adj)], entry)"""
    n, dim = data.shape
    adj = np.empty((n, M), np.int32)
    oracle.jvo_graph_build_f32(metric, fp(data), n, dim, M, beam, 1.2, 1.2, ip(adj))
    levels, ids = [(np.arange(n, dtype=np.int32), adj)], np.arange(n, dtype=np.int32)
    for count in upper_counts:
        ids = np.sort(rng.choice(ids, count, replace=False)).astype(np.int32)
        a = np.empty((count, M), np.int32)
        oracle.jvo_graph_build_f32(metric, fp(np.ascontiguousarray(data[ids])), count, dim, M, beam, 1.2, 1.2, ip(a))
        levels.append((ids, np.where(a >= 0, ids[np.clip(a, 0, None)], -1).astype(np.int32)))
    return levels, int(levels[-1][0][0])


# ------------------------------------------------------------------------------------------------ CPU: the restatement
def test_union_deduplicates():
    # the beam's results are distinct nodes: only the row can repeat one
    assert rm.union([5, -1, 3, 9, -1], [3, 7, 5, 8, -1]) == [5, 3, 9, 7, 8]
    assert rm.union([-1, -1], [4, 2]) == [4, 2] and rm.union([1, 2], []) == [1, 2]


def test_compactor_beam_is_8m():
    for M in (1, 2, 8, 16, 32, 64):
        assert rm.compactor_beam(M) == 8 * M


def test_model_excludes_self(oracle):
    rng = np.random.default_rng(2)
    data = latent_rows(rng, 300, 12)
    levels, entry = oracle_levels(oracle, o.DOT_PRODUCT, data, 8, rng, (40,))
    model = rm.RefineModel(gm.F32Scores(oracle, data, o.DOT_PRODUCT), 8, 30, 1.2, 1.2, 0, levels[0][1], entry, False)
    for u in [entry] + list(range(0, 300, 37)):
        res = model.search_excluding(u)
        assert u not in res and len(res) == 30, u
        c = model.candidates(u)
        assert u not in c and len(set(c)) == len(c)


def test_model_max_level_gate(oracle):
    rng = np.random.default_rng(3)
    data = latent_rows(rng, 200, 10)
    flat, entry = oracle_levels(oracle, o.EUCLIDEAN, data, 6, rng)
    res = rm.refine_graph(gm.F32Scores(oracle, data, o.EUCLIDEAN), flat, entry, np.zeros(200, bool), 6, 20, 1.2, 1.2, 0, rm.BUILDER)
    assert res["stats"]["levels"] == 0 and np.array_equal(res["levels"][0][1], flat[0][1])
    # the compactor form refines a flat graph: every node
    res = rm.refine_graph(gm.F32Scores(oracle, data, o.EUCLIDEAN), flat, entry, np.zeros(200, bool), 6, 20, 1.2, 1.2, 0, rm.COMPACTOR)
    assert res["nodes_refined"] == [200] and res["stats"]["levels"] == 1


def test_model_builder_form_invariants(oracle):
    rng = np.random.default_rng(4)
    data = latent_rows(rng, 400, 12)
    levels, entry = oracle_levels(oracle, o.COSINE, data, 8, rng, (60, 12))
    res = rm.refine_graph(gm.F32Scores(oracle, data, o.COSINE), levels, entry, np.zeros(400, bool), 8, 30, 1.2, 1.2, 16, rm.BUILDER)
    assert res["nodes_refined"] == [60, 60, 12]
    check_levels(res["levels"], levels)


def check_levels(got, given):
    """no row names its own node or a node twice; every row has at most M entries, all members of its level; the members are kept"""
    for lv, ((ids, adj, *_), (ids0, _)) in enumerate(zip(got, given)):
        assert np.array_equal(ids, ids0), lv
        members = set(ids.tolist())
        for v, row in zip(ids, adj):
            r = row[row >= 0].tolist()
            assert int(v) not in r and len(set(r)) == len(r) and set(r) <= members, (lv, int(v), r)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


def graph_levels(g):
    return [g.level(lv) for lv in range(g.info()["levels"])]


def holes_of(g):
    """nodes with an empty level-0 row that no row names"""
    _, adj = g.level(0)
    named = np.zeros(len(adj), bool)
    named[adj[adj >= 0]] = True
    return ~(adj >= 0).any(1) & ~named


def check_output(out, g, M):
    """the invariants of a refined graph against the graph it came from"""
    assert out.info() == g.info()
    check_levels(graph_levels(out), graph_levels(g))
    for lv in range(out.info()["levels"]):
        assert (out.level(lv)[1] >= 0).sum(1).max(initial=0) <= M


def compare(out, want, what):
    """levels the model refined without a near tie equal the device's; returns (levels compared, levels flagged)"""
    compared = flagged = 0
    for lv, (ids, adj, fl) in enumerate(want["levels"]):
        dids, dadj = out.level(lv)
        assert np.array_equal(dids, ids), (what, "members", lv)
        if fl:
            flagged += 1
            continue
        bad = np.flatnonzero((dadj != adj).any(1))
        assert len(bad) == 0, (what, "level", lv, ids[bad[:5]].tolist(), dadj[bad[:1]].tolist(), adj[bad[:1]].tolist())
        compared += 1
    st = out.refine_stats
    assert st["levels"] == want["stats"]["levels"] and st["nodes_refined"][:st["levels"]] == want["nodes_refined"], (what, st)
    if flagged == 0:
        for k, v in want["stats"].items():
            assert st[k] == v, (what, k, st[k], v)
    return compared, flagged


def run_model(scores, g, params, mode, holes=None):
    n = g.info()["n"]
    return rm.refine_graph(scores, graph_levels(g), g.info()["entry_node"], np.zeros(n, bool) if holes is None else holes, params.degree,
                           params.beam_width, params.overflow, params.alpha, params.max_batch, mode)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", METRICS)
def test_exclude_equals_accept_bitset(jv, metric):
    from jvector_b200 import _native as nat
    lib = nat.init()
    rng = np.random.default_rng(30 + metric)
    data = latent_rows(rng, 2000, 24)
    vec = jv.F32Vectors(data)
    g = jv.GraphIndexBuilder(metric, M=12, beamWidth=40, addHierarchy=True, seed=3).build(vec)
    nq, K = 48, 20
    ex = rng.choice(2000, nq, replace=False).astype(np.int32)
    ex[0] = g.info()["entry_node"]  # the entry itself excluded
    ex[1] = -1                      # nothing excluded
    queries = np.ascontiguousarray(data[np.where(ex >= 0, ex, 0)])
    nodes = np.empty((nq, K), np.int32)
    scores = np.empty((nq, K), np.float32)
    cnt = np.empty(4, np.int64)
    nat.check(lib.jv_graph_search_exclude(g._h, vec._h, metric, fp(queries), nq, K, K, ip(ex), ip(nodes), fp(scores), cnt.ctypes.data_as(nat.i64p)))
    accept = np.ones((nq, 2000), bool)
    for q in range(nq):
        if ex[q] >= 0:
            accept[q, ex[q]] = False
    want = jv.GraphSearcher(g).search(vec, queries, metric, K, K, acceptOrds=accept)
    assert np.array_equal(nodes, want.nodes)
    assert np.array_equal(scores.view(np.int32), want.scores.view(np.int32))
    assert cnt.tolist() == [want.visitedCount, want.expandedCount, want.expandedCountBaseLayer, want.rerankedCount]
    assert not any(ex[q] in nodes[q] for q in range(nq) if ex[q] >= 0)
    g.close()
    vec.close()


@pytest.mark.gpu
def test_builder_form_equals_model(jv, oracle):
    """every metric, several batches at level 0. A level whose model made a near-tie prune is skipped (later batches search its rows);
    level 0 and every counter must still be compared for at least one metric"""
    from jvector_b200 import _native as nat
    full = []
    for metric in METRICS:
        rng = np.random.default_rng(40 + metric)
        data = latent_rows(rng, 1500, 24)
        vec = jv.F32Vectors(data)
        b = jv.GraphIndexBuilder(metric, M=12, beamWidth=40, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=7, max_batch=48)
        g = b.build(vec)
        out = b.refine(g, vec)
        check_output(out, g, 12)
        want = run_model(gm.F32Scores(oracle, data, metric), g, b.params, nat.REFINE_BUILDER)
        compared, flagged = compare(out, want, ("builder", metric))
        assert out.refine_stats["nodes_refined"][0] > 48, "several batches at level 0"
        print("metric", metric, "levels compared", compared, "flagged", flagged, out.refine_stats)
        if flagged == 0:  # every level, and (in compare) every counter
            full.append(metric)
        # two calls give identical bytes
        again = b.refine(g, vec)
        for (a0, a1), (b0, b1) in zip(graph_levels(out), graph_levels(again)):
            assert np.array_equal(a0, b0) and np.array_equal(a1, b1)
        for h in (out, again, g, vec):
            h.close()
    assert full, "no metric compared level 0 and the counters"


@pytest.mark.gpu
def test_builder_form_pq_equals_model(jv, oracle):
    from jvector_b200 import _native as nat
    from test_graph_build_pq import exact_table, real_pq_world
    metric, dim, k = o.EUCLIDEAN, 32, 256
    _, codes, codebooks, cen = real_pq_world("refine_pq", 1500, dim, 8, True)
    pqv = jv.PQVectors(codes, codebooks, dim, k, cen)
    b = jv.GraphIndexBuilder(metric, M=12, beamWidth=40, addHierarchy=True, seed=5, max_batch=64)
    g = b.build(pqv)
    out = b.refine(g, pqv)
    check_output(out, g, 12)
    scores = gm.PQScores(oracle, codes, codebooks, k, dim, cen, exact_table(pqv, codebooks, dim, k, metric), metric)
    want = run_model(scores, g, b.params, nat.REFINE_BUILDER)
    assert compare(out, want, "pq") == (len(want["levels"]), 0)
    for h in (out, g, pqv):
        h.close()


@pytest.mark.gpu
def test_builder_form_bq_equals_model(jv, oracle):
    from jvector_b200 import _native as nat
    from test_graph_bq import latent_world
    metric, dim = o.DOT_PRODUCT, 128
    _, words = latent_world("refine_bq", 1500, dim)
    bqv = jv.BQVectors(words, dim)
    b = jv.GraphIndexBuilder(metric, M=12, beamWidth=40, addHierarchy=True, seed=6, max_batch=64)
    g = b.build(bqv)
    out = b.refine(g, bqv)
    check_output(out, g, 12)
    want = run_model(gm.BQScores(oracle, words, dim, metric), g, b.params, nat.REFINE_BUILDER)
    assert compare(out, want, "bq") == (len(want["levels"]), 0)
    for h in (out, g, bqv):
        h.close()


def _sources(jv, metric, rng, hier, sizes=(500, 420, 380), dim=24, M=12):
    srcs, live, datas = [], [], []
    for i, n in enumerate(sizes):
        data = latent_rows(rng, n, dim)
        vec = jv.F32Vectors(data)
        srcs.append((jv.GraphIndexBuilder(metric, M=M, beamWidth=40, addHierarchy=hier, seed=20 + i).build(vec), vec))
        live.append(rng.random(n) >= 0.15)
        datas.append(data)
    merged = np.concatenate([d[m] for d, m in zip(datas, live)])
    return srcs, live, merged


def compare_compactor(out, given, want, what):
    """the compactor form has no cascade (every search reads the given graph): every level-0 row equals the model's except a row whose own
    prune was a near tie, at most 1 % of the refined rows + 1 of them; the upper levels are the given ones; the counters are exact but
    rows_changed, which a flagged row may move. Returns (rows compared, rows flagged)"""
    wids, wadj, _ = want["levels"][0]
    dids, dadj = out.level(0)
    assert np.array_equal(dids, wids), what
    flags = want["row_flags"][0]
    flagged = {v for v, f in flags.items() if f}
    bad = [int(v) for v in np.flatnonzero((dadj != wadj).any(1)) if int(v) not in flagged]
    assert not bad, (what, "rows differ", bad[:5], dadj[bad[:1]].tolist(), wadj[bad[:1]].tolist())
    compared = len(flags) - len(flagged)
    assert compared > 0 and len(flagged) <= 0.01 * len(flags) + 1, (what, compared, len(flagged))
    for lv in range(1, out.info()["levels"]):
        assert all(np.array_equal(a, b) for a, b in zip(out.level(lv), given.level(lv))), (what, "level", lv)
    st = out.refine_stats
    assert st["levels"] == 1 and st["nodes_refined"] == want["nodes_refined"] == [len(flags)], (what, st)
    for k in ("candidates", "max_candidates", "backlinks_added", "backlinks_dropped", "rows_repruned"):
        assert st[k] == want["stats"][k], (what, k, st[k], want["stats"][k])
    assert abs(st["rows_changed"] - want["stats"]["rows_changed"]) <= len(flagged), (what, st, want["stats"])
    return compared, len(flagged)


@pytest.mark.gpu
@pytest.mark.parametrize("hier", [False, True], ids=["flat", "hierarchical"])
def test_compactor_form_equals_model(jv, oracle, hier):
    from jvector_b200 import _native as nat
    metric = o.DOT_PRODUCT
    rng = np.random.default_rng(50 + hier)
    srcs, live, merged = _sources(jv, metric, rng, hier)
    g0, rows0 = jv.GraphIndexCompactor(srcs, live, None, metric).compact()
    c = jv.GraphIndexCompactor(srcs, live, None, metric, refineAfterCompaction=True)
    g1, rows1 = c.compact()
    assert (g1.info()["levels"] > 1) == hier
    check_output(g1, g0, 12)
    params = nat.BuildParams(12, 100, 1.2, 1.2, 0, 0, 0, -1)
    want = run_model(gm.F32Scores(oracle, merged, metric), g0, params, nat.REFINE_COMPACTOR)
    compared, flagged = compare_compactor(g1, g0, want, ("compactor", hier))
    print("compactor", "hierarchical" if hier else "flat", "rows compared", compared, "flagged", flagged, c.refine_stats)
    assert c.refine_stats["max_candidates"] <= 12 + 8 * 12
    # setRefineAfterCompaction(False) gives the compaction's graph
    c.setRefineAfterCompaction(False)
    g2, rows2 = c.compact()
    assert all(np.array_equal(a, b) for lv in range(g0.info()["levels"]) for a, b in zip(g2.level(lv), g0.level(lv)))
    for h in [g0, rows0, g1, rows1, g2, rows2] + [x for s in srcs for x in s]:
        h.close()


@pytest.mark.gpu
def test_edge_cases(jv, oracle):
    metric = o.EUCLIDEAN
    rng = np.random.default_rng(60)
    data = latent_rows(rng, 1200, 24)
    vec = jv.F32Vectors(data)
    # a flat graph in builder form: a copy
    b = jv.GraphIndexBuilder(metric, M=12, beamWidth=40, seed=1)
    flat = b.build(vec)
    copy = b.refine(flat, vec)
    assert np.array_equal(copy.level(0)[1], flat.level(0)[1]) and copy.info() == flat.info()
    assert copy.refine_stats["levels"] == 0 and copy.refine_stats["rows_changed"] == 0
    # holes from removeDeletedNodes stay holes
    bh = jv.GraphIndexBuilder(metric, M=12, beamWidth=40, addHierarchy=True, seed=2, max_batch=64)
    g = bh.build(vec)
    dead = rng.random(1200) < 0.2
    dead[g.info()["entry_node"]] = False
    rep = bh.removeDeletedNodes(g, vec, dead)
    out = bh.refine(rep, vec)
    check_output(out, rep, 12)
    assert holes_of(out)[dead].all()
    want = run_model(gm.F32Scores(oracle, data, metric), rep, bh.params, 0, holes=dead)
    compare(out, want, "holes")
    # refineFinalGraph = build() then refine()
    br = jv.GraphIndexBuilder(metric, M=12, beamWidth=40, addHierarchy=True, seed=2, max_batch=64, refineFinalGraph=True)
    one = br.build(vec)
    two = bh.refine(g, vec)
    for (a0, a1), (b0, b1) in zip(graph_levels(one), graph_levels(two)):
        assert np.array_equal(a0, b0) and np.array_equal(a1, b1)
    assert {k: v for k, v in one.refine_stats.items() if k != "device_ms"} == {k: v for k, v in two.refine_stats.items() if k != "device_ms"}
    for h in (flat, copy, g, rep, out, one, two, vec):
        h.close()


def _recall(nodes, truth):
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / truth.shape[1] for i in range(len(nodes))]))


@pytest.mark.gpu
def test_refined_recall_siftsmall(jv, sift):
    data, queries, _ = sift
    metric = o.EUCLIDEAN
    vec = jv.F32Vectors(data)
    b = jv.GraphIndexBuilder(metric, M=16, beamWidth=100, addHierarchy=True, seed=9)
    g = b.build(vec)
    r = b.refine(g, vec)
    truth, _, _ = jv.topk_bruteforce(vec, metric, queries, 10)
    before = _recall(jv.GraphSearcher(g).search(vec, queries, metric, 10, 50).nodes, truth)
    after = _recall(jv.GraphSearcher(r).search(vec, queries, metric, 10, 50).nodes, truth)
    print("siftsmall recall@10 rerankK 50: before", before, "after", after, r.refine_stats)
    assert after >= before - 0.01, (before, after)
    for h in (g, r, vec):
        h.close()


@pytest.mark.gpu
def test_refine_errors(jv):
    from jvector_b200 import _native as nat
    lib = nat.init()
    rng = np.random.default_rng(70)
    data = latent_rows(rng, 300, 16)
    vec = jv.F32Vectors(data)
    g = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=8, beamWidth=20, addHierarchy=True, seed=1).build(vec)
    ok = nat.BuildParams(8, 20, 1.2, 1.2, 0, 0, 0, -1)

    def call(gh=g._h, ds=vec._h, metric=o.DOT_PRODUCT, params=ok, mode=0, st=True):
        out = C.c_void_p(0x1234)
        s = nat.RefineStats()
        launches = lib.jv_kernel_launch_count()
        rc = lib.jv_graph_refine(gh, ds, metric, C.byref(params) if params is not None else None, mode, C.byref(out), C.byref(s) if st else None)
        assert out.value == 0x1234, "a refused call wrote its output"
        assert lib.jv_kernel_launch_count() == launches, "a refused call did device work"
        return rc

    assert call(ds=None) == -2                                                    # null data set
    assert call(params=None) == -2                                                # null params
    assert call(st=False) == -2                                                   # null stats
    assert call(mode=2) == -2 and call(mode=-1) == -2                             # bad mode
    assert call(metric=7) == -2                                                   # bad metric
    assert call(params=nat.BuildParams(16, 20, 1.2, 1.2, 0, 0, 0, -1)) == -2       # degree differs from the graph's
    assert call(params=nat.BuildParams(8, 0, 1.2, 1.2, 0, 0, 0, -1)) == -2         # bad build parameters
    small = jv.F32Vectors(data[:100])
    assert call(ds=small._h) == -2                                                # size mismatch
    words = np.zeros((300, 1), np.uint64)
    bqv = jv.BQVectors(words, 16)
    assert call(ds=bqv._h, mode=1) == -2                                          # the compactor form is fp32 only
    wide = jv.GraphIndex(np.full((300, 65), -1, np.int32), 0)
    p65 = nat.BuildParams(65, 20, 1.2, 1.2, 0, 0, 0, -1)
    assert call(gh=wide._h, params=p65) == -5                                     # degree above 64
    for h in (g, vec, small, bqv, wide):
        h.close()
