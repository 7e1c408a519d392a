"""CPU check of the equivalence the device traversal rests on: the kernel's ONE sorted list + shadow result heap (modelled in
tests/search_model.py, structure for structure) against the oracle's literal two-heap restatement of GraphSearcher.search —
on tie-heavy scores (BQ Hamming, duplicated vectors), hierarchies, acceptOrds / threshold / rerankFloor, and with candidate
lists short enough to force the overflow-and-retry path. Identical id lists, scores and visited counts are required."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as o
import search_model as sm
from oracle_lib import fp, ip, wp


def _levels(adj, upper):
    lv = [{i: [int(x) for x in adj[i]] for i in range(adj.shape[0])}]
    for ids, a in (upper or []):
        lv.append({int(ids[i]): [int(x) for x in a[i]] for i in range(len(ids))})
    return lv


def _run_model(levels, entry, L, sf, topK, rerankK, rr, cap, **kw):
    score = lambda node: L.jvo_scorer_score(sf, int(node))
    rfn = (lambda node: L.jvo_scorer_score(rr, int(node))) if rr else None
    retries = 0
    while True:
        try:
            return sm.search(levels, entry, score, topK, rerankK, cap, rfn, **kw) + (retries,)
        except sm.ListOverflow:
            cap *= 4
            retries += 1
            assert cap <= 1 << 16


def _bits(mask):
    n = len(mask)
    words = np.zeros((n + 31) // 32, np.uint32)
    for i in np.flatnonzero(mask):
        words[i >> 5] |= np.uint32(1) << np.uint32(i & 31)
    return words


@pytest.fixture(scope="module")
def world(oracle):
    rng = np.random.default_rng(77)
    n, dim, deg = 1200, 64, 12
    data = o.random_unit_vectors(rng, n, dim)
    data[300:330] = data[100:130]  # duplicated vectors: exact score ties in every scorer, exact AND approximate
    adj = np.empty((n, deg), np.int32)
    entry = oracle.jvo_graph_build_f32(o.DOT_PRODUCT, fp(data), n, dim, deg, 40, 1.2, 1.2, ip(adj))
    ids1 = np.sort(rng.choice(n, 150, replace=False)).astype(np.int32)
    a1 = np.empty((150, deg), np.int32)
    oracle.jvo_graph_build_f32(o.DOT_PRODUCT, fp(np.ascontiguousarray(data[ids1])), 150, dim, deg, 40, 1.2, 1.2, ip(a1))
    a1 = np.where(a1 >= 0, ids1[np.clip(a1, 0, None)], -1).astype(np.int32)
    ids2 = ids1[:12].copy()
    a2 = np.empty((12, deg), np.int32)
    oracle.jvo_graph_build_f32(o.DOT_PRODUCT, fp(np.ascontiguousarray(data[ids2])), 12, dim, deg, 40, 1.2, 1.2, ip(a2))
    a2 = np.where(a2 >= 0, ids2[np.clip(a2, 0, None)], -1).astype(np.int32)
    words = np.zeros((n, 1), np.uint64)
    for i in range(n):
        oracle.jvo_bq_encode(fp(data[i]), dim, wp(words[i]))
    queries = o.random_unit_vectors(rng, 12, dim)
    queries[0] = data[100]
    return dict(n=n, dim=dim, data=data, adj=adj, entry=entry, upper=[(ids1, a1), (ids2, a2)], words=words, queries=queries)


@pytest.mark.parametrize("hier", [False, True])
@pytest.mark.parametrize("kind", ["bq", "f32", "f32x30"])
def test_list_model_equals_two_heap_reference(oracle, world, hier, kind):
    w = world
    upper = w["upper"] if hier else None
    entry = int(w["upper"][1][0][0]) if hier else w["entry"]
    g = o.make_graph(w["adj"], entry, upper)
    levels = _levels(w["adj"], upper)
    n, dim = w["n"], w["dim"]
    rng = np.random.default_rng(5)
    accept = rng.random(n) < 0.35
    total_retries = 0
    cases = [dict(topK=10, rerankK=10), dict(topK=10, rerankK=40), dict(topK=1, rerankK=1), dict(topK=5, rerankK=25, rerank=True),
             dict(topK=10, rerankK=30, rerank=True, rerank_floor=0.55), dict(topK=10, rerankK=30, rerank=True, rerank_floor=2.0),
             dict(topK=10, rerankK=20, accept=accept), dict(topK=10, rerankK=20, accept=accept, threshold=0.52, rerank=True),
             dict(topK=10, rerankK=20, threshold=0.6), dict(topK=10, rerankK=20, accept=np.ones(n, bool))]
    for case in cases:
        topK, rerankK = case["topK"], case["rerankK"]
        thr, floor = case.get("threshold", 0.0), case.get("rerank_floor", 0.0)
        acc = case.get("accept")
        bits = _bits(acc) if acc is not None else None
        # f32x30: queries x 30, so about half the DOT_PRODUCT scores (1 + q.x) / 2 are below 0, which searchOneLayer refuses at
        # threshold 0 on every level, with or without acceptOrds; the last query scores every node of the top level below 0
        qs = w["queries"]
        if kind == "f32x30":
            top = w["data"][w["upper"][1][0]].sum(0)
            qs = np.concatenate([qs * np.float32(30), (-30 * top / np.linalg.norm(top))[None].astype(np.float32)])
        for q in qs:
            mk = (lambda: oracle.jvo_scorer_bq(wp(w["words"]), n, dim, fp(q))) if kind == "bq" else \
                 (lambda: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(w["data"]), n, dim, fp(q)))
            sf = mk()
            rr = oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(w["data"]), n, dim, fp(q)) if case.get("rerank") else None
            wn = np.full(topK, -1, np.int32)
            ws = np.zeros(topK, np.float32)
            st = o.Stats()
            cnt = oracle.jvo_graph_search_ex(C.byref(g), sf, rr, topK, rerankK, thr, floor,
                                             bits.ctypes.data_as(C.POINTER(C.c_uint32)) if bits is not None else None, ip(wn), fp(ws), C.byref(st))
            # the tightest legal list (cap = rerankK) must overflow-and-retry its way to the same answer as a roomy one
            for cap in (rerankK, rerankK + 28):
                nodes, scores, visited, nrr, retries = _run_model(levels, entry, oracle, sf, topK, rerankK, rr, cap, threshold=thr, rerank_floor=floor, accept=acc)
                total_retries += retries
                assert nodes == [int(x) for x in wn[:cnt]], (case.keys(), kind, hier, cap, nodes, wn[:cnt].tolist())
                assert np.array_equal(np.array(scores, np.float32), ws[:cnt])
                assert visited == st.visited and nrr == st.reranked
            oracle.jvo_scorer_free(sf)
            if rr:
                oracle.jvo_scorer_free(rr)
    if kind == "bq":
        assert total_retries > 0, "tie tails were expected to overflow the tight list at least once"


def test_visited_set_in_shared_memory_model_is_an_exact_set():
    # the shared-memory visited set (search.cu visited_insert_smem) must behave exactly like a set of ids: the id -> (region, tag)
    # map is a bijection, so two different ids never look alike; checked at the sizes plan_search picks for 30k, 1M, 2^21 and 10M
    # nodes, with id streams that collide in their low bits, their high bits, and at random
    rng = np.random.default_rng(5)
    for n, cap in ((30_000, 8192), (1_000_000, 16384), (1 << 21, 8192), (10_000_000, 16384)):
        plan = sm.visited_smem_plan(n, cap)
        assert plan is not None, n
        slog, rlog, idmask = plan
        # bijection of id -> x on [0, 2^bits): multiplication by an odd constant modulo a power of two
        probe = np.unique(np.concatenate([rng.integers(0, n, 200_000), np.arange(min(n, 70_000)), n - 1 - np.arange(min(n, 70_000))]))
        x = (probe.astype(np.uint64) * np.uint64(sm.VIS_MUL)) & np.uint64(idmask)
        assert len(np.unique(x)) == len(probe)
        limit = 3 * (1 << slog) // 4
        streams = [rng.integers(0, n, 3000),
                   (rng.integers(0, 8, 3000) << 15) % n,                                  # ids that differ only above bit 15
                   (7 + (np.arange(3000, dtype=np.int64) << 12)) % n,                       # same low 12 bits
                   np.repeat(rng.integers(0, n, 500), 6)]                                  # every id six times
        for ids in streams:
            vs, seen = sm.VisitedSmem(slog, rlog, idmask), set()
            for v in ids[:limit]:
                new = vs.insert(v)
                if vs.failed:
                    break  # a full region: the kernel re-runs the query on the global table, never answers from this one
                assert new == (int(v) not in seen), (n, int(v))
                seen.add(int(v))
    # beyond 2^24 nodes (regions would fall under 32 slots) and for beams whose table would not fit 32 KB the global table stays
    assert sm.visited_smem_plan(1 << 26, 16384) is None
    assert sm.visited_smem_plan(1_000_000, 1 << 17) is None


def test_pq_partial_sums_fold_like_the_butterfly():
    # score_pq_partial / pq_fold8 (one warp per partial sum, one thread folds) must give the bits of the 8-lane xor butterfly
    rng = np.random.default_rng(6)
    for _ in range(2000):
        parts = (rng.standard_normal(8) * 10.0 ** rng.integers(-3, 4)).astype(np.float32)
        lanes = sm.pq_group_sum8(parts)
        want = lanes[0]
        assert all(np.float32(v).view(np.int32) == np.float32(want).view(np.int32) for v in lanes)  # every lane ends with the same bits
        assert sm.pq_fold8(parts).view(np.int32) == np.float32(want).view(np.int32)
