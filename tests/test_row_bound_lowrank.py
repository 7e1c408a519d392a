"""The low-rank edge bound of the sketched fp32 DOT_PRODUCT walk (lowrank_bound, lowrank_rows_kernel, prepare_lowrank, the gather
phase of graph_search_kernel; numpy restatement in row_bound_lowrank.py).

CPU: the bound is >= the kernel's own score (the warp-order oracle, compared as sortable ints) on adversarial rows, for a basis fitted
to the rows, a non-orthonormal basis and a random one. GPU: the low-rank rows the device built equal their definition over the
device's basis, a graph's edge records are the rows of its adjacency, the device's bound (jv_lowrank_bound_pairs) is >= the
warp-order score on the adversarial rows and within a tenth of its eps term of the model's bound, and walks that settle neighbours
on the records (jv_search_last_settled > 0) equal the warp-order oracle's traversal: ids, score bits, visited and reranked counters,
on flat and hierarchical graphs and on graphs produced by removing and adding nodes."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as o
import row_bound_lowrank as rl
import row_bound_model as rb
from oracle_lib import fp
from test_row_bound import adversarial_rows, queries_for

DIMS = (4, 8, 100, 768, 1021)


def bases(rng, rows, dim):
    k = rl.LR_K
    fitted = rl.basis(np.concatenate([rows, o.random_unit_vectors(rng, 64, dim)]), k)
    skew = (fitted.astype(np.float64) * rng.uniform(0.3, 3.0, k) + 0.1 * rng.standard_normal((dim, k))).astype(np.float32)
    return {"fitted": fitted, "non_orthonormal": skew, "random": rng.standard_normal((dim, k)).astype(np.float32)}


@pytest.mark.parametrize("dim", DIMS)
def test_bound_is_at_least_the_warp_order_score(oracle, dim):
    rng = np.random.default_rng(100 + dim)
    stride = (dim + 3) & ~3
    for qi, q in enumerate(queries_for(rng, dim)):
        rows = adversarial_rows(rng, dim, q)
        exact = np.array([oracle.jvo_compare_f32_warp(o.DOT_PRODUCT, fp(q), fp(r), dim) for r in rows], np.float32)
        ids = np.arange(len(rows))
        for name, B in bases(rng, rows[:64], dim).items():
            codes, t, rho, beta, xn = rl.encode_rows(rows, B)
            assert (rho >= 0).all() and (beta >= 0).all()
            ub = rb.dot_score_up(rl.upper_bound_raw(q, B, codes, t, rho, beta, xn, stride))
            ok = np.isnan(exact) | np.isnan(ub) | (rb.sortable(ub) >= rb.sortable(exact))
            assert ok.all(), (dim, qi, name, np.flatnonzero(~ok)[:5], ub[~ok][:5], exact[~ok][:5])
            fin = ~np.isnan(ub)
            assert (rb.topk_key(ub, ids)[fin] >= rb.topk_key(np.where(np.isnan(exact), ub, exact), ids)[fin]).all()


def test_bound_is_tight_on_low_rank_rows():
    # what makes the records worth reading: rows near a 16-dimensional subspace get a bound within a few 1e-2 of their score
    rng = np.random.default_rng(11)
    dim = 256
    A = rng.standard_normal((16, dim)) / 4.0
    x = rng.standard_normal((500, 16)) @ A + 0.1 * rng.standard_normal((500, dim))
    x = (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)
    q = x[0]
    B = rl.basis(x, 32)
    codes, t, rho, beta, xn = rl.encode_rows(x, B)
    ub = rb.dot_score_up(rl.upper_bound_raw(q, B, codes, t, rho, beta, xn, dim)).astype(np.float64)
    exact = (1.0 + x.astype(np.float64) @ q.astype(np.float64)) / 2.0
    assert (ub >= exact).all()
    assert np.median(ub - exact) < 0.02


# ------------------------------------------------------------------------------------------------ GPU
NQ = 3000  # more queries than an H100 keeps resident (132 SMs x 9 CTAs): the batch takes the sketch path


@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


@pytest.fixture(scope="module")
def world(jv):
    rng = np.random.default_rng(77)
    n, dim, latent = 20000, 130, 24  # stride 132: a row of 4 m floats that is not a multiple of 8
    A = rng.standard_normal((latent, dim)) / np.sqrt(latent)

    def rows(k):
        x = rng.standard_normal((k, latent)) @ A + 0.25 * rng.standard_normal((k, dim))
        return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)

    data, queries = rows(n), rows(NQ)
    vec = jv.F32Vectors(data)
    gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, addHierarchy=True, seed=3).build(vec)
    info = gi.info()
    adj0 = gi.level(0)[1]
    upper = [gi.level(lv) for lv in range(1, info["levels"])]
    yield data, queries, vec, gi, adj0, upper, info["entry_node"]
    gi.close()
    vec.close()


def download_lowrank(jv, vec, n, dim):
    lib = jv.load()
    stride = (dim + 3) & ~3
    k = C.c_int()
    basis = np.empty((rl.LR_K, stride), np.float32)
    rows = np.empty((n, 48), np.uint8)
    assert lib.jv_dataset_lowrank_download(vec._h, fp(basis), rows.ctypes.data, C.byref(k)) == 0, lib.jv_last_error()
    assert k.value == rl.LR_K
    return basis, rows


@pytest.mark.gpu
def test_device_lowrank_rows_equal_their_definition(jv, world):
    data, queries, vec, gi, adj0, upper, entry = world
    n, dim = data.shape
    jv.GraphSearcher(gi).search(vec, queries, o.DOT_PRODUCT, 10, 40)  # the first sketched search builds them
    basis, rows = download_lowrank(jv, vec, n, dim)
    assert not basis[:, dim:].any()
    B = basis[:, :dim].T.astype(np.float64)
    cols = np.linalg.norm(B, axis=0)
    assert np.allclose(cols, 1.0, atol=1e-5) and np.allclose(B.T @ B, np.eye(rl.LR_K), atol=1e-4)
    codes = rows[:, :32].view(np.int8).astype(np.float64)
    meta = rows[:, 32:].copy().view(np.float32)
    t, rho, beta, xn = (meta[:, i].astype(np.float64) for i in range(4))
    x = data.astype(np.float64)
    a = x @ B
    assert (t == (np.abs(a).max(axis=1) / 127.0).astype(np.float32)).mean() > 0.999
    assert (np.abs(a / t[:, None] - codes) <= 0.5 + 1e-6).all()
    w = x - t[:, None] * (codes @ B.T)
    for got, want in ((rho, np.linalg.norm(w, axis=1)), (beta, np.linalg.norm(w @ B, axis=1)), (xn, np.linalg.norm(x, axis=1))):
        assert (got >= want * (1 - 1e-12)).all()
        assert (got <= want * (1 + 1e-5) + 1e-6).all()


@pytest.mark.gpu
def test_edge_records_are_the_rows_of_the_adjacency(jv, world):
    data, queries, vec, gi, adj0, upper, entry = world
    n, dim = data.shape
    jv.GraphSearcher(gi).search(vec, queries, o.DOT_PRODUCT, 10, 40)
    _, rows = download_lowrank(jv, vec, n, dim)
    deg = adj0.shape[1]
    rec = np.empty((n, deg, 48), np.uint8)
    assert jv.load().jv_graph_edge_records_download(gi._h, rec.ctypes.data) == 0
    want = np.where((adj0 >= 0)[:, :, None], rows[np.maximum(adj0, 0)], 0)
    assert (rec == want).all()


@pytest.mark.gpu
def test_walks_settled_on_edge_records_equal_oracle(jv, oracle, world):
    import os
    from test_gpu_parity import _assert_same_search, _oracle_search
    data, queries, vec, gi0, adj0, upper, entry = world
    n, dim = data.shape
    mk = lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q))
    rng = np.random.default_rng(12)
    shared = rng.random(n) < 0.4
    for up in (None, upper):
        name = "flat" if up is None else "levels"
        gi = jv.GraphIndex(adj0, entry, up)
        g = o.make_graph(adj0, entry, up)
        s = jv.GraphSearcher(gi)
        for topK, rerankK in ((10, 40), (10, 100)):
            res = s.search(vec, queries, o.DOT_PRODUCT, topK, rerankK)
            _assert_same_search(res, _oracle_search(oracle, g, mk, queries, topK, rerankK), (name, topK, rerankK))
        assert jv.load().jv_graph_edge_records_download(gi._h, None) == 0, "the walk was expected to build edge records"
        assert 0 < jv.load().jv_search_last_settled() <= res.visitedCount, "the walk was expected to settle neighbours on the records"
        res = s.search(vec, queries, o.DOT_PRODUCT, 10, 40, acceptOrds=shared)
        _assert_same_search(res, _oracle_search(oracle, g, mk, queries, 10, 40, accept=shared), (name, "accept"))
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


def _walk_matches_oracle(jv, oracle, gi, vec, data, queries, what):
    from test_gpu_parity import _assert_same_search, _oracle_search
    n, dim = data.shape
    info = gi.info()
    adj0 = gi.level(0)[1]
    g = o.make_graph(adj0, info["entry_node"], [gi.level(lv) for lv in range(1, info["levels"])])
    mk = lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q))
    res = jv.GraphSearcher(gi).search(vec, queries, o.DOT_PRODUCT, 10, 40)
    _assert_same_search(res, _oracle_search(oracle, g, mk, queries, 10, 40), what)
    assert jv.load().jv_search_last_settled() > 0, what
    # the new handle built its own records, from its own adjacency
    _, rows = download_lowrank(jv, vec, n, dim)
    rec = np.empty((n, adj0.shape[1], 48), np.uint8)
    assert jv.load().jv_graph_edge_records_download(gi._h, rec.ctypes.data) == 0, what
    assert (rec == np.where((adj0 >= 0)[:, :, None], rows[np.maximum(adj0, 0)], 0)).all(), what


@pytest.mark.gpu
def test_walks_after_remove_and_add_equal_oracle(jv, oracle, world):
    data, queries, vec, gi, adj0, upper, entry = world
    n, dim = data.shape
    rng = np.random.default_rng(14)
    jv.GraphSearcher(gi).search(vec, queries, o.DOT_PRODUCT, 10, 40)  # gi has records: the derived graphs must not inherit them
    b = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, addHierarchy=True, seed=3)
    removed = b.removeDeletedNodes(gi, vec, rng.random(n) < 0.05)
    _walk_matches_oracle(jv, oracle, removed, vec, data, queries, "after remove")
    removed.close()
    A = data[:2000].astype(np.float64)
    extra = (A[rng.permutation(2000)] + A[rng.permutation(2000)]).astype(np.float32)
    data2 = np.concatenate([data, extra / np.linalg.norm(extra, axis=1, keepdims=True)]).astype(np.float32)
    vec2 = jv.F32Vectors(data2)
    added = b.addGraphNodes(gi, vec2)
    _walk_matches_oracle(jv, oracle, added, vec2, data2, queries, "after add")
    added.close()
    vec2.close()


def _device_bound(jv, B, rows, q):
    n, dim = rows.shape
    out = np.empty(n, np.float32)
    rec = np.empty((n, 48), np.uint8)
    qs = np.ascontiguousarray(np.repeat(q[None, :], n, axis=0).astype(np.float32))
    assert jv.load().jv_lowrank_bound_pairs(fp(np.ascontiguousarray(B)), dim, fp(rows), fp(qs), n, rec.ctypes.data, fp(out)) == 0, jv.load().jv_last_error()
    return out, rec


@pytest.mark.gpu
@pytest.mark.parametrize("dim", DIMS)
def test_device_bound_on_adversarial_rows(jv, oracle, dim):
    # the device's records and bound (lowrank_rows_kernel, prepare_lowrank, lowrank_bound) against the warp-order score on the
    # adversarial rows, and against the model's bound on the unit rows, close enough that losing any of its error terms shows
    rng = np.random.default_rng(200 + dim)
    stride = (dim + 3) & ~3
    for qi, q in enumerate(queries_for(rng, dim)):
        rows = adversarial_rows(rng, dim, q)
        exact = np.array([oracle.jvo_compare_f32_warp(o.DOT_PRODUCT, fp(q), fp(r), dim) for r in rows], np.float32)
        for name, B in bases(rng, rows[:64], dim).items():
            dev, rec = _device_bound(jv, B, rows, q)
            ok = np.isnan(exact) | (rb.sortable(dev) >= rb.sortable(exact))
            assert ok.all(), (dim, qi, name, np.flatnonzero(~ok)[:5], dev[~ok][:5], exact[~ok][:5])
            if qi != 0 or dim < 100:  # (at a few dimensions the two summation orders of u differ by a larger share of eps)
                continue
            unit = slice(0, 64)  # o.random_unit_vectors rows against a unit query
            codes = rec[unit, :32].view(np.int8)
            t, rho, beta, xn = (rec[unit, 32:].copy().view(np.float32)[:, i] for i in range(4))
            raw = rl.upper_bound_raw(q, B, codes, t, rho, beta, xn, stride)
            u, e, sigma, nu = rl.prepare_query(q, B)
            eps_term = t.astype(np.float64) * (np.abs(codes.astype(np.float64)) * e[0]).sum(axis=1)
            dev_raw = 2.0 * dev[unit].astype(np.float64) - 1.0
            # (plus a few fp32 ulps of the score, which is all the device returns: a random basis makes the bound large)
            tol = 0.1 * eps_term + 4 * 2.0 ** -23 * (np.abs(raw) + 1.0)
            assert (np.abs(dev_raw - raw) <= tol).all(), (dim, name, np.abs(dev_raw - raw).max(), eps_term.min())


@pytest.mark.gpu
def test_isotropic_rows_get_no_lowrank_rows(jv):
    rng = np.random.default_rng(13)
    data = o.random_unit_vectors(rng, 20000, 256)
    vec = jv.F32Vectors(data)
    gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=40, addHierarchy=False, seed=3).build(vec)
    jv.GraphSearcher(gi).search(vec, o.random_unit_vectors(rng, NQ, 256), o.DOT_PRODUCT, 10, 40)
    assert jv.load().jv_search_last_settled() == 0
    k = C.c_int()
    assert jv.load().jv_dataset_lowrank_download(vec._h, None, None, C.byref(k)) != 0 and k.value == rl.LR_K
    assert jv.load().jv_graph_edge_records_download(gi._h, None) != 0
    gi.close()
    vec.close()
