"""Merging graphs (OnDiskGraphIndexCompactor's per-node work, jv_graph_compact).

CPU: the host restatement (tests/compact_model.py) on its own: searchTopK, the entry rule, the level union, the small-source rule
and the one-source case. GPU (-m gpu): jv_graph_compact row for row against the restatement, its edge cases, the recall of merged
graphs against a fresh build, a fused PQ walk of a merged graph, and its errors."""
import ctypes as C

import numpy as np
import pytest

import compact_model as cm
import oracle_lib as o
from oracle_lib import fp, ip

METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)


def latent_rows(rng, n, dim, latent=16, noise=0.35):
    A = rng.standard_normal((latent, dim)).astype(np.float32) / np.sqrt(latent)
    x = rng.standard_normal((n, latent)).astype(np.float32) @ A + noise * rng.standard_normal((n, dim)).astype(np.float32)
    return np.ascontiguousarray(x / np.linalg.norm(x, axis=1, keepdims=True), dtype=np.float32)


def oracle_source(oracle, metric, data, degree, rng, upper_counts=(), beam=30):
    """a source built by the oracle's sequential builder; upper_counts: sizes of nested upper levels over sampled ids"""
    n, dim = data.shape
    adj = np.empty((n, degree), np.int32)
    oracle.jvo_graph_build_f32(metric, fp(data), n, dim, degree, beam, 1.2, 1.2, ip(adj))
    upper, ids = [], np.arange(n, dtype=np.int32)
    for count in upper_counts:
        ids = np.sort(rng.choice(ids, count, replace=False)).astype(np.int32)
        a = np.empty((count, degree), np.int32)
        oracle.jvo_graph_build_f32(metric, fp(np.ascontiguousarray(data[ids])), count, dim, degree, beam, 1.2, 1.2, ip(a))
        upper.append((ids, np.where(a >= 0, ids[np.clip(a, 0, None)], -1).astype(np.int32)))
    entry = int(upper[-1][0][0]) if upper else 0
    return {"data": data, "adj0": adj, "upper": upper, "entry": entry, "live": np.ones(n, bool)}


def assign_maps(sources, rng=None):
    """new ids: the live nodes of all sources, in source order, shuffled when rng is given"""
    total = sum(int(s["live"].sum()) for s in sources)
    perm = rng.permutation(total) if rng is not None else np.arange(total)
    base = 0
    for s in sources:
        m = np.full(len(s["live"]), -1, np.int32)
        k = int(s["live"].sum())
        m[s["live"]] = perm[base:base + k]
        s["map"] = m
        base += k
    return sources


# ------------------------------------------------------------------------------------------------ CPU: the restatement
def test_search_top_k():
    assert cm.search_top_k(16, 3) == 24 and cm.search_top_k(32, 4) == 32 and cm.search_top_k(64, 1) == 256
    assert cm.search_top_k(1, 100) == 4 and cm.search_top_k(16, 16) == 4 and cm.search_top_k(16, 17) == 4


def _world(oracle, metric, seed, uppers, n=(160, 140, 120), dim=12, degree=8, dead=0.15):
    rng = np.random.default_rng(seed)
    sources = []
    for i, cnt in enumerate(n):
        s = oracle_source(oracle, metric, latent_rows(rng, cnt, dim), degree, rng, uppers[i])
        s["live"] = rng.random(cnt) >= dead
        sources.append(s)
    return assign_maps(sources, rng), rng


def test_model_level_union_and_entry(oracle):
    sources, _ = _world(oracle, o.DOT_PRODUCT, 5, [(40, 10), (), (30,)])
    res = cm.compact(oracle, o.DOT_PRODUCT, sources)
    assert len(res["levels"]) == 3 and res["stats"]["levels"] == 3
    for L, (ids, adj) in enumerate(res["levels"]):
        want = sorted(int(s["map"][v]) for s in sources if L < cm.levels_of(s) for v in cm.members(s, L)[0] if s["live"][v])
        assert ids.tolist() == want, L
        assert ((adj >= 0).sum(1) <= adj.shape[1]).all() and not any(v in row for v, row in zip(ids, adj))
        assert set(adj[adj >= 0].tolist()) <= set(ids.tolist())
    # the first source reaches the top level: its entry if live, else the top level's lowest new id
    s0 = sources[0]
    want = int(s0["map"][s0["entry"]]) if s0["live"][s0["entry"]] else int(res["levels"][2][0].min())
    assert res["entry"] == want
    # every entry dead: the lowest new id of the top level
    for s in sources:
        s["live"][s["entry"]] = False
    assign_maps(sources)
    res = cm.compact(oracle, o.DOT_PRODUCT, sources)
    assert res["entry"] == int(res["levels"][-1][0].min())


def test_model_small_source_rule(oracle):
    # the third source keeps K or fewer live members: every query's candidates from it are all of them, and no search runs
    sources, rng = _world(oracle, o.EUCLIDEAN, 7, [(), (), ()], n=(150, 130, 60), degree=8)
    K = cm.search_top_k(8, 3)
    sources[2]["live"][:] = False
    sources[2]["live"][rng.choice(60, K - 3, replace=False)] = True
    assign_maps(sources, rng)
    res = cm.compact(oracle, o.EUCLIDEAN, sources)
    small = set(sources[2]["map"][sources[2]["live"]].tolist())
    for s in (0, 1):
        for v in np.flatnonzero(sources[s]["live"]):
            assert small <= res["cands"][0][int(sources[s]["map"][v])]
    n0, n1, n2 = (int(s["live"].sum()) for s in sources)
    assert res["stats"]["exhaustive"] == n0 + n1
    assert res["stats"]["searches"] == (n1 + n2) + (n0 + n2)  # sources 0 and 1 are searched for the rows of the two others


def test_model_one_source(oracle):
    # one source: each live row re-pruned over its live neighbours only; a row whose neighbours all died is empty
    rng = np.random.default_rng(3)
    s = oracle_source(oracle, o.COSINE, latent_rows(rng, 200, 10), 6, rng, (25,))
    s["live"] = rng.random(200) >= 0.3
    assign_maps([s], rng)
    res = cm.compact(oracle, o.COSINE, [s])
    assert res["stats"]["searches"] == 0 and res["stats"]["exhaustive"] == 0
    ids, adj = res["levels"][0]
    inv = np.full(len(ids), -1)
    inv[s["map"][s["live"]]] = np.flatnonzero(s["live"])
    for nv in ids:
        old = inv[nv]
        live_nb = {int(s["map"][j]) for j in s["adj0"][old] if j >= 0 and s["live"][j]}
        assert res["cands"][0][int(nv)] == live_nb
        assert set(adj[nv][adj[nv] >= 0].tolist()) <= live_nb
        if not live_nb:
            assert (adj[nv] == -1).all()


def test_compact_without_device():
    # the C entry point refuses a null argument before it looks for a device
    from jvector_b200 import _native as nat
    lib = nat.load()
    g, r = C.c_void_p(), C.c_void_p()
    st = nat.CompactStats()
    assert lib.jv_graph_compact(None, 1, 1, 1.2, C.byref(g), C.byref(r), C.byref(st)) == -2
    assert g.value is None and r.value is None


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


def device_source(jv, metric, data, degree, hier, seed, live=None, beam=40):
    vec = jv.F32Vectors(data)
    gi = jv.GraphIndexBuilder(metric, M=degree, beamWidth=beam, alpha=1.2, addHierarchy=hier, seed=seed).build(vec)
    return {"gi": gi, "vec": vec, "data": data, "adj0": gi.level(0)[1], "upper": [gi.level(L) for L in range(1, gi.info()["levels"])],
            "entry": gi.info()["entry_node"], "live": np.ones(len(data), bool) if live is None else live}


def refresh(s):
    s["adj0"] = s["gi"].level(0)[1]
    s["upper"] = [s["gi"].level(L) for L in range(1, s["gi"].info()["levels"])]
    s["entry"] = s["gi"].info()["entry_node"]


def run(jv, metric, sources, alpha=1.2):
    c = jv.GraphIndexCompactor([(s["gi"], s["vec"]) for s in sources], [s["live"] for s in sources], [s["map"] for s in sources], metric, alpha)
    g, rows = c.compact()
    return g, rows, c.stats


def check_against_model(jv, oracle, metric, sources, what, max_flag=0.01):
    g, rows, st = run(jv, metric, sources)
    res = cm.compact(oracle, metric, sources)
    inf = g.info()
    assert inf["entry_node"] == res["entry"] and inf["levels"] == len(res["levels"]), (what, inf, res["entry"])
    assert inf["n"] == res["stats"]["nodes"]
    flagged = total = 0
    for L, (wids, wadj) in enumerate(res["levels"]):
        dids, dadj = g.level(L)
        assert np.array_equal(dids, wids), (what, "members of level", L)
        skip = np.array([res["flags"][L][int(v)] for v in wids], bool)
        flagged += int(skip.sum())
        total += len(wids)
        bad = np.flatnonzero(~skip & (dadj != wadj).any(1))
        assert len(bad) == 0, (what, "level", L, bad[:5].tolist(), dadj[bad[:1]].tolist(), wadj[bad[:1]].tolist())
    for k in ("searches", "exhaustive", "candidates", "max_candidates", "search_top_k", "levels"):
        assert st[k] == res["stats"][k], (what, k, st[k], res["stats"][k])
    assert flagged <= max_flag * total + 1, (what, flagged, total)
    return g, rows, st, res


def same_rows(jv, rows, want, rng):
    """whether a resident data set holds `want`: the scores of random queries against every row equal, bit for bit, those of the
    same kernel over `want` uploaded as it is"""
    n, dim = want.shape
    ref = jv.F32Vectors(want)
    q = rng.standard_normal((4, dim)).astype(np.float32)
    ids = np.tile(np.arange(n, dtype=np.int32), 4)
    offs = np.arange(5, dtype=np.int32) * n
    same = all(np.array_equal(jv.score_multi(rows, m, q, ids, offs).view(np.int32), jv.score_multi(ref, m, q, ids, offs).view(np.int32))
               for m in METRICS)
    ref.close()
    return rows.size() == n and rows.dimension() == dim and same


@pytest.mark.gpu
@pytest.mark.parametrize("metric", METRICS)
def test_device_equals_restatement(jv, oracle, metric):
    rng = np.random.default_rng(100 + metric)
    sources = []
    for i, n in enumerate((420, 360, 300)):
        s = device_source(jv, metric, latent_rows(rng, n, 24), 16, True, seed=10 + i)
        s["live"] = rng.random(n) >= 0.15
        sources.append(s)
    assign_maps(sources, rng)
    g, rows, st, res = check_against_model(jv, oracle, metric, sources, ("row for row", metric))
    assert st["searches"] > 0 and rows.size() == res["rows"].shape[0]
    # rows_out holds the gathered source rows in new-id order
    assert same_rows(jv, rows, res["rows"], rng)
    # two identical calls give identical bytes
    g2, rows2, st2 = run(jv, metric, sources)
    for L in range(g.info()["levels"]):
        a, b = g.level(L), g2.level(L)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert st2["candidates"] == st["candidates"] and st2["visited"] == st["visited"]
    for h in [g, rows, g2, rows2] + [x for s in sources for x in (s["gi"], s["vec"])]:
        h.close()


@pytest.mark.gpu
def test_device_edge_worlds(jv, oracle):
    rng = np.random.default_rng(21)
    m = o.EUCLIDEAN
    a = device_source(jv, m, latent_rows(rng, 500, 24), 16, True, seed=1)
    b = device_source(jv, m, latent_rows(rng, 300, 24), 16, False, seed=2)     # no upper levels, next to one with some
    c = device_source(jv, m, latent_rows(rng, 200, 24), 16, True, seed=3)
    a["live"] = rng.random(500) >= 0.1
    b["live"] = rng.random(300) >= 0.1
    # S = 1
    assign_maps([a], rng)
    check_against_model(jv, oracle, m, [a], "one source")[0].close()
    # a source with every node dead, next to one whose live count is below searchTopK (the small-source rule)
    c["live"] = np.zeros(200, bool)
    small = device_source(jv, m, latent_rows(rng, 100, 24), 16, False, seed=4)
    small["live"] = np.zeros(100, bool)
    small["live"][rng.choice(100, 10, replace=False)] = True
    assign_maps([a, b, c, small], rng)
    g, rows, st, _ = check_against_model(jv, oracle, m, [a, b, c, small], "dead and small sources")
    assert st["exhaustive"] > 0
    g.close()
    rows.close()
    # every source's entry dead
    c["live"] = rng.random(200) >= 0.1
    for s in (a, b, c):
        s["live"][s["entry"]] = False
    assign_maps([a, b, c], rng)
    g, rows, _, res = check_against_model(jv, oracle, m, [a, b, c], "entries dead")
    assert g.info()["entry_node"] == int(res["levels"][-1][0].min())
    g.close()
    rows.close()
    # sources that carry holes from jv_graph_remove_deleted (holes are dead, whatever the live mask says)
    holes = rng.random(500) < 0.2
    holes[a["entry"]] = False
    rep = jv.GraphIndexBuilder(m, M=16, alpha=1.2, seed=5).removeDeletedNodes(a["gi"], a["vec"], holes)
    a2 = dict(a, gi=rep, live=~holes & (rng.random(500) >= 0.05))
    refresh(a2)
    assign_maps([a2, b], rng)
    g, rows, _, _ = check_against_model(jv, oracle, m, [a2, b], "holes")
    g.close()
    rows.close()
    # no live masks and no maps: every node live, the sources one after the other
    g, rows = jv.GraphIndexCompactor([(b["gi"], b["vec"]), (c["gi"], c["vec"])], None, None, m).compact()
    assert g.info()["n"] == 500 and same_rows(jv, rows, np.concatenate([b["data"], c["data"]]), rng)
    g.close()
    rows.close()
    for h in (rep, a["gi"], a["vec"], b["gi"], b["vec"], c["gi"], c["vec"], small["gi"], small["vec"]):
        h.close()


def _recall(nodes, truth):
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / truth.shape[1] for i in range(len(nodes))]))


@pytest.mark.gpu
@pytest.mark.parametrize("world", ["siftsmall", "latent"])
def test_compacted_graph_recall(jv, sift, world):
    rng = np.random.default_rng(56)
    if world == "siftsmall":
        data, queries, _ = sift
        metric = o.EUCLIDEAN
    else:
        data = latent_rows(rng, 20000, 64)
        queries = latent_rows(rng, 200, 64)
        metric = o.DOT_PRODUCT
    n = data.shape[0]
    kw = dict(M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=9)
    parts = np.array_split(np.arange(n), 4)
    srcs, live = [], []
    for p in parts:
        vec = jv.F32Vectors(np.ascontiguousarray(data[p]))
        srcs.append((jv.GraphIndexBuilder(metric, **kw).build(vec), vec))
        live.append(rng.random(len(p)) >= 0.1)
    g, rows = jv.GraphIndexCompactor(srcs, live, None, metric).compact()
    keep = np.concatenate([p[m] for p, m in zip(parts, live)])  # new id i = old row keep[i]
    sub = jv.F32Vectors(np.ascontiguousarray(data[keep]))
    fresh = jv.GraphIndexBuilder(metric, **kw).build(sub)
    truth, _, _ = jv.topk_bruteforce(sub, metric, queries, 10)
    r_merged = _recall(jv.GraphSearcher(g).search(rows, queries, metric, 10, 100).nodes, truth)
    r_fresh = _recall(jv.GraphSearcher(fresh).search(sub, queries, metric, 10, 100).nodes, truth)
    print("recall@10", world, "merged", r_merged, "fresh", r_fresh)
    assert r_merged >= r_fresh - 0.03, (world, r_merged, r_fresh)
    for h in [g, rows, sub, fresh] + [x for s in srcs for x in s]:
        h.close()


@pytest.mark.gpu
def test_fused_pq_walk_on_compacted_graph(jv, oracle):
    rng = np.random.default_rng(74)
    dim, M = 64, 16
    sources = [device_source(jv, o.DOT_PRODUCT, latent_rows(rng, n, dim), 16, True, seed=i) for i, n in enumerate((1200, 900))]
    for s in sources:
        s["live"] = rng.random(len(s["data"])) >= 0.1
    assign_maps(sources, rng)
    g, rows, _ = run(jv, o.DOT_PRODUCT, sources)
    n = rows.size()
    data = np.zeros((n, dim), np.float32)
    for s in sources:
        data[s["map"][s["live"]]] = s["data"][s["live"]]
    pq = jv.ProductQuantization.compute(rows, M, 256, seed=1)
    codes = jv.pq_encode_all(rows, pq.codebooks, M, 256, pq.centroid)
    pqv = jv.PQVectors(codes, pq.codebooks, dim, 256, pq.centroid)
    _, adj = g.level(0)
    upper = [g.level(L) for L in range(1, g.info()["levels"])] or None
    packed = np.empty((n, 16, M), np.uint8)
    oracle.jvo_fused_pq_pack(ip(adj), n, 16, o.bp(codes), M, o.bp(packed))
    g.fuse_pq(pqv)
    queries = o.random_unit_vectors(rng, 32, dim)
    got = jv.GraphSearcher(g).search(pqv, queries, o.DOT_PRODUCT, 10, 40, reranker=rows)
    og = o.make_graph(adj, g.info()["entry_node"], upper)
    cen = pq.centroid
    for i in range(len(queries)):
        sf = oracle.jvo_scorer_pq(o.DOT_PRODUCT, fp(pq.codebooks), M, 256, dim, fp(cen) if cen is not None else None, o.bp(codes), n, fp(queries[i]))
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
    for h in [g, rows, pqv] + [x for s in sources for x in (s["gi"], s["vec"])]:
        h.close()


@pytest.mark.gpu
def test_compact_errors(jv):
    from jvector_b200 import _native as nat
    lib = nat.load()
    rng = np.random.default_rng(1)
    data = latent_rows(rng, 200, 16)
    vec = jv.F32Vectors(data)
    g = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=8, beamWidth=20).build(vec)
    ident = np.arange(200, dtype=np.int32)

    def call(srcs, metric=o.DOT_PRODUCT, alpha=1.2, n=None):
        arr = (nat.CompactSource * max(1, len(srcs)))()
        keep = []
        for i, (gh, vh, bits, m) in enumerate(srcs):
            b = jv.pack_accept_bits(bits) if bits is not None else None
            keep.append(b)
            arr[i] = nat.CompactSource(gh, vh, b.ctypes.data_as(C.POINTER(C.c_uint32)) if b is not None else None, ip(m) if m is not None else None)
        go, ro = C.c_void_p(0x1234), C.c_void_p(0x5678)
        st = nat.CompactStats()
        rc = lib.jv_graph_compact(arr, len(srcs) if n is None else n, metric, alpha, C.byref(go), C.byref(ro), C.byref(st))
        assert go.value == 0x1234 and ro.value == 0x5678, "a refused call wrote its outputs"
        return rc

    assert call([(g._h, vec._h, None, ident)], n=0) == -2                        # no source
    assert call([(None, vec._h, None, ident)]) == -2                             # null graph
    assert call([(g._h, vec._h, None, None)]) == -2                              # null map
    assert call([(g._h, vec._h, None, ident)], metric=7) == -2                   # bad metric
    assert call([(g._h, vec._h, None, ident)], alpha=0.9) == -2                  # alpha < 1
    assert call([(g._h, vec._h, np.zeros(200, bool), ident)]) == -2              # no live node
    bad = ident.copy()
    bad[5] = 7
    assert call([(g._h, vec._h, None, bad)]) == -2                               # a new id used twice
    assert call([(g._h, vec._h, None, ident + 1)]) == -2                         # new ids not [0, live)
    other = jv.F32Vectors(latent_rows(rng, 200, 24))
    g24 = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=8, beamWidth=20).build(other)
    assert call([(g._h, vec._h, None, ident), (g24._h, other._h, None, ident + 200)]) == -2  # unequal dims
    g16 = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=20).build(vec)
    assert call([(g._h, vec._h, None, ident), (g16._h, vec._h, None, ident + 200)]) == -2  # unequal degrees
    small = jv.F32Vectors(data[:100])
    assert call([(g._h, small._h, None, ident)]) == -2                           # rows and graph differ in size
    pqv = jv.PQVectors(np.zeros((200, 4), np.uint8), np.zeros(256 * 16, np.float32), 16)
    assert call([(g._h, pqv._h, None, ident)]) == -2                             # not fp32
    wide = jv.GraphIndex(np.full((200, 65), -1, np.int32), 0)
    assert call([(wide._h, vec._h, None, ident)]) == -5                          # degree above 64
    for h in (g, g24, g16, wide, vec, other, small, pqv):
        h.close()
