"""Merging graphs whose nodes carry PQ codes (jv_graph_compact_pq: OnDiskGraphIndexCompactor's FusedPQ and sidecar compaction, with
PQRetrainer's retraining).

CPU: the retraining sample's quota arithmetic on hand-worked cases, its chunk order, and the PQ forms of the restatement
(tests/compact_pq_model.py) reducing to the fp32 one where they must. GPU (-m gpu): the sidecar form against jv_graph_compact, the
retrained codebooks and the output codes against their host restatements, the fused form row for row against the restatement, its
edge cases, determinism, recall against a fresh build with fresh PQ, and the errors."""
import ctypes as C

import numpy as np
import pytest

import compact_model as cm
import compact_pq_model as cpm
import oracle_lib as o
import pq_train_model as ptm
from oracle_lib import bp, ip
from test_graph_compact import METRICS, assign_maps, device_source, latent_rows, oracle_source, refresh, same_rows


# ------------------------------------------------------------------------------------------------ CPU: the sample
def test_sample_quotas_hand_worked():
    # at most 128 000 live rows: every one of them
    assert cpm.sample_quotas([100000, 28000]) is None
    # proportional shares 42666 each (sum 127998): normalised up round-robin from source 0
    assert cpm.sample_quotas([100000, 100000, 100000]) == [42667, 42667, 42666]
    # a source below MIN = min(1000, 128000 / 3) = 1000 is raised to it: 85191 + 1000 + 42595 = 128786, normalised down by 786
    # round-robin over the sources above MIN (0 and 2), 393 each
    assert cpm.sample_quotas([200000, 500, 100000]) == [85191 - 393, 1000, 42595 - 393]
    # many sources: MIN = 128000 / 200 = 640, and every quota is at least that
    q = cpm.sample_quotas([1000] * 199 + [10 ** 6])
    assert sum(q) == 128000 and min(q) == 640 and q[-1] == 128000 - 199 * 640
    # a dead source still has a quota of MIN, and gives nothing
    assert cpm.sample_quotas([0, 150000]) == [1000, 127000]


def test_retrain_sample_takes_live_nodes_per_chunk():
    rng = np.random.default_rng(3)
    big = {"live": rng.random(200000) >= 0.2}               # about 160k live: above the cap
    short = {"live": np.zeros(3000, bool)}                  # 500 live: fewer than its quota of MIN = 1000
    short["live"][rng.choice(3000, 500, replace=False)] = True
    holes = {"live": rng.random(40000) >= 0.5}              # holes and dead nodes are both "not live"
    srcs = [big, short, holes]
    sample = cpm.retrain_sample(srcs, seed=11)
    quota = cpm.sample_quotas([int(s["live"].sum()) for s in srcs])
    assert len(sample[1]) == 500 and np.array_equal(sample[1], np.flatnonzero(short["live"]))
    assert len(sample[0]) == quota[0] and len(sample[2]) == quota[2]
    assert sum(len(x) for x in sample) < 128000
    for s, x in zip(srcs, sample):
        assert np.all(np.diff(x) > 0) and s["live"][x].all()
    # the chunks are walked in chunk_order: every chunk before the last one touched gives all its live nodes
    order = cpm.chunk_order(11, 0, -(-200000 // 32))
    chunks = set((sample[0] // 32).tolist())
    walked = order[:len(chunks)]
    assert set(walked) == chunks
    for c in walked[:-1]:
        assert np.array_equal(np.flatnonzero(big["live"][c * 32:(c + 1) * 32]) + c * 32, sample[0][sample[0] // 32 == c])
    # at most 128 000 live nodes: every live node
    small = [{"live": rng.random(500) >= 0.5}, {"live": rng.random(700) >= 0.5}]
    assert all(np.array_equal(x, np.flatnonzero(s["live"])) for s, x in zip(small, cpm.retrain_sample(small, 1)))


def test_chunk_order_is_fisher_yates_over_counter_random():
    for seed, s, chunks in ((0, 0, 1), (7, 2, 50), (123456789, 1, 997)):
        order = list(range(chunks))
        for i in range(chunks - 1, 0, -1):
            j = int(ptm.counter_random(seed, 0x7ffffffe, s, i)[0] % np.uint64(i + 1))
            order[i], order[j] = order[j], order[i]
        assert cpm.chunk_order(seed, s, chunks) == order
        assert sorted(order) == list(range(chunks))
    assert cpm.chunk_order(7, 2, 50) != cpm.chunk_order(8, 2, 50) and cpm.chunk_order(7, 2, 50) != cpm.chunk_order(7, 3, 50)


def _host_pq(rng, data, M, k):
    cb, sizes, offsets = o.train_pq_numpy(rng, data, M, k, iters=2)
    return cb, sizes, offsets


def test_model_pq_forms_reduce_to_compact(oracle):
    rng = np.random.default_rng(9)
    dim, M, k = 12, 4, 16
    srcs = []
    for n, up in ((160, (30,)), (140, ())):
        s = oracle_source(oracle, o.EUCLIDEAN, latent_rows(rng, n, dim), 8, rng, up)
        s["live"] = rng.random(n) >= 0.15
        cb, sizes, offsets = _host_pq(rng, s["data"], M, k)
        s["pq"] = {"codes": o.encode_pq(oracle, cb, sizes, offsets, M, k, None, s["data"]), "codebooks": cb, "M": M, "k": k, "centroid": None}
        srcs.append(s)
    assign_maps(srcs, rng)
    # one source: nothing is searched, so the fused form is the fp32 merge
    one = [dict(srcs[0])]
    assign_maps(one, rng)
    a, b = cm.compact(oracle, o.EUCLIDEAN, one), cpm.compact_pq(oracle, o.EUCLIDEAN, one, seed=3)
    assert all(np.array_equal(x[1], y[1]) for x, y in zip(a["levels"], b["levels"])) and a["stats"] == b["stats"]
    # the sidecar form is the fp32 merge, and its sample is every live row in (source, node) order
    a, b = cm.compact(oracle, o.EUCLIDEAN, srcs), cpm.compact_pq(oracle, o.EUCLIDEAN, srcs, seed=3, fused=False)
    assert all(np.array_equal(x[1], y[1]) for x, y in zip(a["levels"], b["levels"])) and a["stats"] == b["stats"]
    assert np.array_equal(b["train_rows"], np.concatenate([s["data"][s["live"]] for s in srcs]))


def test_compact_pq_without_device():
    from jvector_b200 import _native as nat
    lib = nat.load()
    g, r, p = C.c_void_p(), C.c_void_p(), C.c_void_p()
    st = nat.CompactPQStats()
    assert lib.jv_graph_compact_pq(None, None, 1, 1, 1.2, 0, C.byref(g), C.byref(r), C.byref(p), None, None, None, C.byref(st)) == -2
    assert g.value is None and r.value is None and p.value is None


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


def add_pq(jv, s, M, k, centred, seed, fuse):
    """source s gets a PQ of its own (ProductQuantization.compute on its rows), its codes, and (fuse) its graph's FusedPQ records"""
    pq = jv.ProductQuantization.compute(s["vec"], M, k, globallyCenter=centred, seed=seed)
    codes = jv.pq_encode_all(s["vec"], pq.codebooks, M, k, pq.centroid)
    s["pqv"] = jv.PQVectors(codes, pq.codebooks, s["data"].shape[1], k, pq.centroid)
    s["pq"] = {"codes": codes, "codebooks": pq.codebooks, "M": M, "k": k, "centroid": pq.centroid}
    if fuse:
        s["gi"].fuse_pq(s["pqv"])
    return s


def run_pq(jv, metric, sources, seed=5, **kw):
    c = jv.GraphIndexCompactor([(s["gi"], s["vec"], s["pqv"]) for s in sources], [s["live"] for s in sources], [s["map"] for s in sources], metric,
                               seed=seed, **kw)
    g, rows, codes = c.compact()
    return g, rows, codes, c


def check_records(g, codes, M):
    """the merged graph's FusedPQ records equal the oracle's pack of its adjacency with `codes` (FusedPQ.writeInline)"""
    import oracle_lib
    oracle = oracle_lib.load()
    _, adj = g.level(0)
    n, degree = adj.shape
    packed = np.empty((n, degree, M), np.uint8)
    oracle.jvo_fused_pq_pack(ip(np.ascontiguousarray(adj)), n, degree, bp(np.ascontiguousarray(codes)), M, bp(packed))
    rec = g.fused_records()
    cs = (M + 3) & ~3
    assert np.array_equal(rec[:, :4 * degree].copy().view(np.int32), adj)
    got = rec[:, 4 * degree:4 * degree + degree * cs].reshape(n, degree, cs)
    assert np.array_equal(got[:, :, :M], packed) and not got[:, :, M:].any()


def check_retraining(jv, sources, c, codes, rows_host, seed):
    """samples, codebooks and output codes against PQRetrainer restated on the host"""
    sample = cpm.retrain_sample(sources, seed)
    assert c.stats["samples_per_source"] == [len(x) for x in sample]
    assert c.stats["train_rows"] == sum(len(x) for x in sample) == c.stats["train"]["train_rows"]
    p0 = sources[0]["pq"]
    train = np.concatenate([s["data"][x] for s, x in zip(sources, sample)])
    want = ptm.train(train, p0["M"], p0["k"], iters=6, codebooks=p0["codebooks"], centroid=p0["centroid"], seed=seed)
    assert np.array_equal(c.pq.codebooks.view(np.int32), want.codebooks.view(np.int32))
    for key in ("max_lloyd_updates", "changed_last", "empty_reseeds"):
        assert c.stats["train"][key] == want.stats[key], key
    got_codes, got_cb, got_cen = codes.download()
    assert np.array_equal(got_cb.view(np.int32), c.pq.codebooks.view(np.int32))
    if p0["centroid"] is None:
        assert got_cen is None and c.pq.centroid is None
    else:
        assert np.array_equal(got_cen, p0["centroid"]) and np.array_equal(c.pq.centroid, p0["centroid"])
    ref = jv.F32Vectors(rows_host)
    assert np.array_equal(got_codes, jv.pq_encode_all(ref, c.pq.codebooks, p0["M"], p0["k"], p0["centroid"]))
    ref.close()
    return got_codes


def pq_world(jv, metric, rng, sizes, hier, dim=24, degree=16, M=8, k=32, dead=0.15, fuse=True, seed0=10):
    sources = []
    for i, n in enumerate(sizes):
        s = device_source(jv, metric, latent_rows(rng, n, dim), degree, hier[i], seed=seed0 + i)
        s["live"] = rng.random(n) >= dead
        sources.append(add_pq(jv, s, M, k, centred=(i % 2 == 0), seed=seed0 + i, fuse=fuse))
    return assign_maps(sources, rng)


def close_all(handles, sources=()):
    for h in list(handles) + [x for s in sources for x in (s["gi"], s["vec"], s["pqv"])]:
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("metric", METRICS)
def test_sidecar_form_equals_compact(jv, metric):
    rng = np.random.default_rng(200 + metric)
    sources = pq_world(jv, metric, rng, (420, 360, 300), (True, True, False), fuse=False)
    g, rows, codes, c = run_pq(jv, metric, sources, seed=5)
    assert c.stats["fused"] == 0 and c.stats["fuse_ms"] == 0.0
    plain = jv.GraphIndexCompactor([(s["gi"], s["vec"]) for s in sources], [s["live"] for s in sources], [s["map"] for s in sources], metric)
    pg, prows = plain.compact()
    assert g.info() == pg.info()
    for L in range(g.info()["levels"]):
        a, b = g.level(L), pg.level(L)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), L
    for k in ("nodes", "levels", "searches", "exhaustive", "candidates", "max_candidates", "visited", "search_top_k"):
        assert c.stats[k] == plain.stats[k], k
    n = rows.size()
    host = np.zeros((n, 24), np.float32)
    for s in sources:
        host[s["map"][s["live"]]] = s["data"][s["live"]]
    assert same_rows(jv, rows, host, rng)
    check_retraining(jv, sources, c, codes, host, seed=5)
    close_all([g, rows, codes, pg, prows], sources)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", METRICS)
def test_fused_form_equals_restatement(jv, oracle, metric):
    rng = np.random.default_rng(300 + metric)
    sources = pq_world(jv, metric, rng, (420, 360, 300), (True, True, True))
    g, rows, codes, c = run_pq(jv, metric, sources, seed=7)
    assert c.stats["fused"] == 1 and c.stats["searches"] > 0
    res = cpm.compact_pq(oracle, metric, sources, seed=7)
    check_merge(g, c.stats, res, ("fused", metric))
    got_codes = check_retraining(jv, sources, c, codes, res["rows"], seed=7)
    check_records(g, got_codes, 8)
    # two identical calls: identical bytes
    g2, rows2, codes2, c2 = run_pq(jv, metric, sources, seed=7)
    for L in range(g.info()["levels"]):
        assert all(np.array_equal(x, y) for x, y in zip(g.level(L), g2.level(L)))
    assert np.array_equal(g.fused_records(), g2.fused_records())
    assert all(np.array_equal(x, y) for x, y in zip(codes.download()[:2], codes2.download()[:2]))
    assert c2.stats["visited"] == c.stats["visited"]
    close_all([g, rows, codes, g2, rows2, codes2], sources)


def check_merge(g, st, res, what, max_flag=0.01):
    """the merged graph row for row against the restatement, except rows whose prune is a near tie (at most 1 % + 1)"""
    inf = g.info()
    assert inf["entry_node"] == res["entry"] and inf["levels"] == len(res["levels"]), (what, inf, res["entry"])
    flagged = total = 0
    for L, (wids, wadj) in enumerate(res["levels"]):
        dids, dadj = g.level(L)
        assert np.array_equal(dids, wids), (what, "members of level", L)
        skip = np.array([res["flags"][L][int(v)] for v in wids], bool)
        flagged += int(skip.sum())
        total += len(wids)
        bad = np.flatnonzero(~skip & (dadj != wadj).any(1))
        assert len(bad) == 0, (what, "level", L, bad[:5].tolist())
    for k in ("nodes", "searches", "exhaustive", "candidates", "max_candidates", "search_top_k", "levels"):
        assert st[k] == res["stats"][k], (what, k, st[k], res["stats"][k])
    assert flagged <= max_flag * total + 1, (what, flagged, total)


@pytest.mark.gpu
def test_fused_form_edge_worlds(jv, oracle):
    rng = np.random.default_rng(31)
    m = o.EUCLIDEAN
    a, b, c = pq_world(jv, m, rng, (500, 300, 200), (True, False, True), dead=0.1)  # b has no upper levels, next to a and c
    # S = 1
    assign_maps([a], rng)
    g, rows, codes, cp = run_pq(jv, m, [a])
    check_merge(g, cp.stats, cpm.compact_pq(oracle, m, [a], seed=5), "one source")
    check_records(g, codes.download()[0], 8)
    close_all([g, rows, codes])
    # a dead source next to a small one (the small-source rule)
    c["live"] = np.zeros(200, bool)
    small = pq_world(jv, m, rng, (100,), (False,), seed0=40)[0]
    small["live"] = np.zeros(100, bool)
    small["live"][rng.choice(100, 10, replace=False)] = True
    world = [a, b, c, small]
    assign_maps(world, rng)
    g, rows, codes, cp = run_pq(jv, m, world)
    res = cpm.compact_pq(oracle, m, world, seed=5)
    check_merge(g, cp.stats, res, "dead and small sources")
    assert cp.stats["exhaustive"] > 0 and cp.stats["samples_per_source"][2] == 0
    check_retraining(jv, world, cp, codes, res["rows"], seed=5)
    close_all([g, rows, codes])
    # holes from removeDeletedNodes: the repaired graph is fused again with its own codes
    holes = rng.random(500) < 0.2
    holes[a["entry"]] = False
    rep = jv.GraphIndexBuilder(m, M=16, alpha=1.2, seed=5).removeDeletedNodes(a["gi"], a["vec"], holes).fuse_pq(a["pqv"])
    a2 = dict(a, gi=rep, live=~holes & (rng.random(500) >= 0.05))
    refresh(a2)
    assign_maps([a2, b], rng)
    g, rows, codes, cp = run_pq(jv, m, [a2, b])
    res = cpm.compact_pq(oracle, m, [a2, b], seed=5)
    check_merge(g, cp.stats, res, "holes")
    check_retraining(jv, [a2, b], cp, codes, res["rows"], seed=5)
    close_all([g, rows, codes, rep])
    # refineAfterCompaction: the refined graph is jv_graph_refine's on the unfused merge, fused with the new codes
    assign_maps([a, b], rng)
    g, rows, codes, cp = run_pq(jv, m, [a, b])
    from jvector_b200 import _native as nat
    from jvector_b200.api import _refine
    want = _refine(g, rows, m, nat.BuildParams(16, 100, 1.2, 1.2, 0, 5, 0, -1), nat.REFINE_COMPACTOR)
    rg, rrows, rcodes, rc = run_pq(jv, m, [a, b], refineAfterCompaction=True)
    assert rg.info() == want.info()
    for L in range(want.info()["levels"]):
        assert all(np.array_equal(x, y) for x, y in zip(rg.level(L), want.level(L))), L
    assert rc.refine_stats["rows_changed"] == want.refine_stats["rows_changed"]
    check_records(rg, rcodes.download()[0], 8)
    close_all([g, rows, codes, want, rg, rrows, rcodes], [a, b, c, small])


def _recall(nodes, truth):
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / truth.shape[1] for i in range(len(nodes))]))


@pytest.mark.gpu
@pytest.mark.parametrize("world", ["siftsmall", "latent"])
def test_fused_compaction_recall(jv, sift, world):
    rng = np.random.default_rng(57)
    if world == "siftsmall":
        data, queries, _ = sift
        metric, pq_m = o.EUCLIDEAN, 32
    else:
        data = latent_rows(rng, 20000, 64)
        queries = latent_rows(rng, 200, 64)
        metric, pq_m = o.DOT_PRODUCT, 16
    n = data.shape[0]
    kw = dict(M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=True, seed=9)
    parts = np.array_split(np.arange(n), 4)
    srcs, live, keep_alive = [], [], []
    for i, p in enumerate(parts):
        vec = jv.F32Vectors(np.ascontiguousarray(data[p]))
        gi = jv.GraphIndexBuilder(metric, **kw).build(vec)
        pqv = jv.ProductQuantization.compute(vec, pq_m, 256, seed=i).encodeAll(vec)
        srcs.append((gi.fuse_pq(pqv), vec, pqv))
        live.append(rng.random(len(p)) >= 0.1)
    c = jv.GraphIndexCompactor(srcs, live, None, metric, seed=3)
    g, rows, codes = c.compact()
    assert c.stats["fused"] == 1
    keep = np.concatenate([p[m] for p, m in zip(parts, live)])
    sub = jv.F32Vectors(np.ascontiguousarray(data[keep]))
    fresh = jv.GraphIndexBuilder(metric, **kw).build(sub)
    fresh_pq = jv.ProductQuantization.compute(sub, pq_m, 256, seed=0).encodeAll(sub)
    fresh.fuse_pq(fresh_pq)
    truth, _, _ = jv.topk_bruteforce(sub, metric, queries, 10)
    r_merged = _recall(jv.GraphSearcher(g).search(codes, queries, metric, 10, 100, reranker=rows).nodes, truth)
    r_fresh = _recall(jv.GraphSearcher(fresh).search(fresh_pq, queries, metric, 10, 100, reranker=sub).nodes, truth)
    print("recall@10 fused pq", world, "merged", r_merged, "fresh", r_fresh)
    assert r_merged >= r_fresh - 0.03, (world, r_merged, r_fresh)
    for h in [g, rows, codes, sub, fresh, fresh_pq] + [x for s in srcs for x in s]:
        h.close()


@pytest.mark.gpu
def test_resident_encoder_and_download(jv):
    rng = np.random.default_rng(4)
    for dim, M in ((24, 8), (20, 6)):  # M = 6: code rows padded to 8 bytes on the device
        data = latent_rows(rng, 700, dim)
        vec = jv.F32Vectors(data)
        pq = jv.ProductQuantization.compute(vec, M, 64, globallyCenter=True, seed=1)
        res = jv.pq_encode_resident(vec, pq.codebooks, M, 64, pq.centroid)
        codes, cb, cen = res.download()
        assert np.array_equal(codes, jv.pq_encode_all(vec, pq.codebooks, M, 64, pq.centroid))
        assert np.array_equal(cb, pq.codebooks) and np.array_equal(cen, pq.centroid)
        # it scores as the same codes registered from the host
        reg = jv.PQVectors(codes, pq.codebooks, dim, 64, pq.centroid)
        q = rng.standard_normal((3, dim)).astype(np.float32)
        ids = np.tile(np.arange(700, dtype=np.int32), 3)
        offs = np.arange(4, dtype=np.int32) * 700
        for m in METRICS:
            assert np.array_equal(jv.score_multi(res, m, q, ids, offs), jv.score_multi(reg, m, q, ids, offs))
        for h in (vec, res, reg):
            h.close()


@pytest.mark.gpu
def test_compact_pq_errors(jv):
    from jvector_b200 import _native as nat
    lib = nat.load()
    rng = np.random.default_rng(1)
    m = o.DOT_PRODUCT
    a, b = pq_world(jv, m, rng, (300, 260), (False, False), M=4, k=16, dead=0.0)
    other = add_pq(jv, dict(a), 4, 16, centred=False, seed=99, fuse=False)  # a second PQ of a's rows

    def call(pairs, pqs, n=None, centroid=True):
        arr = (nat.CompactSource * len(pairs))()
        for i, (s, bits) in enumerate(pairs):
            arr[i] = nat.CompactSource(s["gi"]._h, s["vec"]._h, bits.ctypes.data_as(C.POINTER(C.c_uint32)) if bits is not None else None, ip(s["map"]))
        hp = (C.c_void_p * len(pqs))(*pqs)
        go, ro, po = C.c_void_p(0x1234), C.c_void_p(0x5678), C.c_void_p(0x9abc)
        cb = np.full(16 * 24, 7.0, np.float32)
        cen = np.full(24, 7.0, np.float32)
        samples = np.full(len(pairs), -9, np.int64)
        st = nat.CompactPQStats()
        rc = lib.jv_graph_compact_pq(arr, hp, len(pairs) if n is None else n, m, 1.2, 0, C.byref(go), C.byref(ro), C.byref(po), o.fp(cb),
                                     o.fp(cen) if centroid else None, samples.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(st))
        assert go.value == 0x1234 and ro.value == 0x5678 and po.value == 0x9abc, "a refused call wrote its outputs"
        assert (cb == 7.0).all() and (cen == 7.0).all() and (samples == -9).all()
        return rc

    both = [(a, None), (b, None)]
    assert call(both, [a["pqv"]._h, b["pqv"]._h], n=0) == -2                          # no source
    assert call(both, [a["pqv"]._h, None]) == -2                                      # null PQ
    assert call(both, [a["pqv"]._h, b["vec"]._h]) == -2                               # not PQ
    assert call(both, [a["pqv"]._h, a["pqv"]._h]) == -2                               # codes of another size
    assert call(both, [other["pqv"]._h, b["pqv"]._h]) == -2                           # a's records were packed from other codes
    plain = dict(b, gi=jv.GraphIndex(b["adj0"], b["entry"]))                          # b without records: a mix of forms
    assert call([(a, None), (plain, None)], [a["pqv"]._h, b["pqv"]._h]) == -2
    cen_src = add_pq(jv, dict(plain), 4, 16, centred=True, seed=3, fuse=False)      # source 0 has a centroid, no centroid_out
    assign_maps([cen_src])
    assert call([(cen_src, None)], [cen_src["pqv"]._h], centroid=False) == -2
    few = np.zeros(300, bool)
    few[:10] = True                                                                    # 10 live rows, k = 16
    a_few = assign_maps([dict(a, live=few)])[0]
    assert call([(a_few, jv.pack_accept_bits(few))], [a["pqv"]._h]) == -2
    bad = dict(a, map=a["map"] + 1)                                                    # what jv_graph_compact refuses, refused alike
    assert call([(bad, None), (b, None)], [a["pqv"]._h, b["pqv"]._h]) == -2
    with pytest.raises(ValueError):
        jv.GraphIndexCompactor([(a["gi"], a["vec"], a["pqv"]), (b["gi"], b["vec"])], None, None, m)
    close_all([plain["gi"], other["pqv"], cen_src["pqv"]], [a, b])
