"""Routing of the edge tier of the sketched fp32 DOT_PRODUCT walk (the gather phase of graph_search_kernel, DESIGN §4.1): a new
neighbour that its edge bound does not settle goes straight to its full row, skipping its sketch, when the bound's point estimate
(lowrank_bound's est; point_estimate in row_bound_direct.py) scores enough above the list's last entry.

CPU: the model's point estimate is t fl(u . c) in fp32, within the rounding of that sum of float64 t (u . c). GPU: walks that route
neighbours direct (jv_search_last_direct: routed > 0) and route some wrongly (routed_dropped > 0) equal the warp-order oracle's
traversal: ids, score bits, visited and reranked counters, on flat and hierarchical graphs, with acceptOrds, a threshold and a forced
tie-tail retry. The world gives the queries and a share of the rows opposed components along a direction outside the rows' main
subspace, which the basis does not hold: the point estimate misses (q - B u) . w there and rates those rows too high."""
import os

import numpy as np
import pytest

import oracle_lib as o
import row_bound_direct as rd
import row_bound_lowrank as rl
from oracle_lib import fp


@pytest.mark.parametrize("dim", (8, 130, 768))
def test_point_estimate_is_the_rounded_low_rank_dot(dim):
    rng = np.random.default_rng(300 + dim)
    x = rng.standard_normal((400, dim)).astype(np.float32) * rng.uniform(1e-3, 1e3, (400, 1)).astype(np.float32)
    q = rng.standard_normal(dim).astype(np.float32)
    B = rl.basis(x, rl.LR_K) if dim >= rl.LR_K else rng.standard_normal((dim, rl.LR_K)).astype(np.float32)
    codes, t, _, _, _ = rl.encode_rows(x, B)
    est = rd.point_estimate(q, B, codes, t)
    assert est.dtype == np.float32
    u = rl.prepare_query(q, B)[0][0].astype(np.float64)
    c = codes.astype(np.float64)
    want = t.astype(np.float64) * (c @ u)
    # fp32 sum of 32 products, then one fp32 product: (k + 2) 2^-24 of the sum of the absolute terms
    tol = (rl.LR_K + 2) * 2.0 ** -24 * t.astype(np.float64) * (np.abs(c) @ np.abs(u)) + 1e-37
    assert (np.abs(est.astype(np.float64) - want) <= tol).all()
    # and the same per-row queries give the same estimates as one shared query
    assert np.array_equal(rd.point_estimate(np.repeat(q[None], 400, axis=0), B, codes, t), est)


# ------------------------------------------------------------------------------------------------ GPU
NQ = 3000  # more queries than an H100 keeps resident (132 SMs x 9 CTAs): the batch takes the sketch path


@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


@pytest.fixture(scope="module")
def world(jv):
    rng = np.random.default_rng(91)
    n, dim, latent = 20000, 130, 32
    A = rng.standard_normal((latent, dim)) / np.sqrt(latent)
    # v: a unit direction orthogonal to the latent space; 3 % of the rows carry -0.35 v, every query +0.6 v. Along v the rows vary
    # less than along any latent direction, so the 32-column basis misses it and the point estimate over-rates those rows
    v = rng.standard_normal(dim)
    v -= A.T @ np.linalg.lstsq(A.T, v, rcond=None)[0]
    v /= np.linalg.norm(v)

    def rows(k, off):
        x = rng.standard_normal((k, latent)) @ A + 0.2 * rng.standard_normal((k, dim))
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        return (x + off[:, None] * v).astype(np.float32)

    data = rows(n, np.where(rng.random(n) < 0.03, -0.35, 0.0))
    queries = rows(NQ, np.full(NQ, 0.6))
    vec = jv.F32Vectors(data)
    gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, addHierarchy=True, seed=5).build(vec)
    info = gi.info()
    adj0 = gi.level(0)[1]
    upper = [gi.level(lv) for lv in range(1, info["levels"])]
    yield data, queries, vec, gi, adj0, upper, info["entry_node"]
    gi.close()
    vec.close()


def last_direct(jv):
    import ctypes as C
    routed, dropped = C.c_int64(), C.c_int64()
    jv.load().jv_search_last_direct(C.byref(routed), C.byref(dropped))
    return routed.value, dropped.value


@pytest.mark.gpu
def test_walks_routing_rows_direct_equal_oracle(jv, oracle, world):
    from test_gpu_parity import _assert_same_search, _oracle_search
    data, queries, vec, gi0, adj0, upper, entry = world
    n, dim = data.shape
    mk = lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q))
    rng = np.random.default_rng(17)
    shared = rng.random(n) < 0.4
    for up in (None, upper):
        name = "flat" if up is None else "levels"
        gi = jv.GraphIndex(adj0, entry, up)
        g = o.make_graph(adj0, entry, up)
        s = jv.GraphSearcher(gi)
        for topK, rerankK in ((10, 40), (10, 100)):
            res = s.search(vec, queries, o.DOT_PRODUCT, topK, rerankK)
            _assert_same_search(res, _oracle_search(oracle, g, mk, queries, topK, rerankK), (name, topK, rerankK))
            routed, dropped = last_direct(jv)
            assert 0 < jv.load().jv_search_last_settled(), (name, "the walk was expected to settle neighbours on the records")
            assert 0 < routed <= res.visitedCount - jv.load().jv_search_last_settled(), (name, topK, rerankK, routed)
            assert 0 < dropped < routed, (name, topK, rerankK, routed, dropped)
        res = s.search(vec, queries, o.DOT_PRODUCT, 10, 40, acceptOrds=shared)
        _assert_same_search(res, _oracle_search(oracle, g, mk, queries, 10, 40, accept=shared), (name, "accept"))
        assert last_direct(jv)[0] > 0, (name, "accept")
        res = s.search(vec, queries, o.DOT_PRODUCT, 10, 40, threshold=0.7)
        _assert_same_search(res, _oracle_search(oracle, g, mk, queries, 10, 40, threshold=0.7), (name, "threshold"))
        os.environ["JV_LIST_CAP"] = "40"
        try:
            res = s.search(vec, queries, o.DOT_PRODUCT, 10, 40, acceptOrds=shared)
        finally:
            del os.environ["JV_LIST_CAP"]
        assert res.retried > 0, "the tight list was expected to overflow"
        _assert_same_search(res, _oracle_search(oracle, g, mk, queries, 10, 40, accept=shared), (name, "tie tail retry"))
        gi.close()
