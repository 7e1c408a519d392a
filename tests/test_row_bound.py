"""The row-sketch bound of the fp32 DOT_PRODUCT walk (sketch_bound_pair, row_sketch_kernel; numpy restatement in row_bound_model.py).

CPU: the bound is >= the kernel's own score (the warp-order oracle, compared as sortable ints) on adversarial rows, so a row dropped
on its bound would have been dropped on its exact score too. GPU: walks that take the sketch path (DOT_PRODUCT, more queries than
resident CTAs) equal the warp-order oracle's traversal: ids, score bits, visited and reranked counters."""
import os

import numpy as np
import pytest

import oracle_lib as o
import row_bound_model as rb
from oracle_lib import fp

DIMS = (4, 100, 768, 1021)


def adversarial_rows(rng, dim, q):
    rows = [o.random_unit_vectors(rng, 64, dim)]
    sign = rng.choice([-1.0, 1.0], (32, dim))
    rows.append(sign * 10.0 ** rng.uniform(-30, 30, (32, dim)))                         # magnitudes 1e-30 .. 1e30 in one row
    rows.append(sign * 10.0 ** rng.uniform(-30, 30, (32, 1)))                           # whole rows at 1e-30 .. 1e30
    rows.append(sign * rng.uniform(2.0 ** -24, 2.0 ** -14, (32, dim)))                  # fp16 subnormal range
    big = rng.standard_normal((8, dim))
    big[:, 0] = 1e4                                                                     # one large value next to small ones
    rows.append(big)
    rows.append(np.zeros((4, dim)))
    rows.append(np.full((4, dim), 0.37))
    rows.append(np.full((4, dim), -3e-20))
    rows.append(np.repeat(q[None, :], 4, axis=0))                                       # the query itself
    rows.append(-np.repeat(q[None, :], 2, axis=0))
    return np.ascontiguousarray(np.concatenate(rows).astype(np.float32))


def queries_for(rng, dim):
    return [o.random_unit_vectors(rng, 1, dim)[0], rng.standard_normal(dim).astype(np.float32) * 1e3,
            (rng.choice([-1.0, 1.0], dim) * 10.0 ** rng.uniform(-3, 3, dim)).astype(np.float32), np.full(dim, 1e-25, np.float32)]


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("encode", [rb.encode_int8, rb.encode_fp16], ids=["int8", "fp16"])
def test_bound_is_at_least_the_warp_order_score(oracle, dim, encode):
    rng = np.random.default_rng(dim)
    stride = (dim + 3) & ~3
    for qi, q in enumerate(queries_for(rng, dim)):
        rows = adversarial_rows(rng, dim, q)
        y, scale, rad = encode(rows, stride)
        assert (rad >= 0).all() and np.isfinite(rad).all()
        ub = rb.dot_score_up(rb.upper_bound_raw(q, y, scale, rad, stride))
        exact = np.array([oracle.jvo_compare_f32_warp(o.DOT_PRODUCT, fp(q), fp(r), dim) for r in rows], np.float32)
        ok = np.isnan(exact) | (rb.sortable(ub) >= rb.sortable(exact))
        assert ok.all(), (dim, qi, np.flatnonzero(~ok)[:5], ub[~ok][:5], exact[~ok][:5])
        ids = np.arange(len(rows))
        assert (rb.topk_key(ub, ids) >= rb.topk_key(np.where(np.isnan(exact), ub, exact), ids)).all()


@pytest.mark.parametrize("dim", DIMS)
def test_bound_is_tight_on_unit_rows(dim):
    # what makes the sketch worth reading: on unit rows the int8 bound sits within a few 1e-3 of the score
    rng = np.random.default_rng(7 + dim)
    rows = o.random_unit_vectors(rng, 200, dim)
    q = o.random_unit_vectors(rng, 1, dim)[0]
    stride = (dim + 3) & ~3
    y, scale, rad = rb.encode_int8(rows, stride)
    ub = rb.dot_score_up(rb.upper_bound_raw(q, y, scale, rad, stride)).astype(np.float64)
    exact = (1.0 + rows.astype(np.float64) @ q.astype(np.float64)) / 2.0
    assert (ub >= exact).all()
    assert (ub - exact).max() < 0.02


# ------------------------------------------------------------------------------------------------ GPU: the walk with the sketch
NQ = 3000  # more queries than an H100 keeps resident (132 SMs x 9 CTAs): the batch takes the sketch path


@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


@pytest.fixture(scope="module")
def latent_world(jv):
    rng = np.random.default_rng(2024)
    n, dim, latent = 20000, 96, 16
    A = rng.standard_normal((latent, dim)) / np.sqrt(latent)

    def rows(k):
        x = rng.standard_normal((k, latent)) @ A + 0.3 * rng.standard_normal((k, dim))
        return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)

    data, queries = rows(n), rows(NQ)
    vec = jv.F32Vectors(data)
    gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, addHierarchy=True, seed=5).build(vec)
    info = gi.info()
    assert info["levels"] >= 3
    adj0 = gi.level(0)[1]
    upper = [gi.level(lv) for lv in range(1, info["levels"])]
    yield data, queries, vec, adj0, upper, info["entry_node"]
    gi.close()
    vec.close()


def _worlds(jv, latent_world):
    data, queries, vec, adj0, upper, entry = latent_world
    for up in (None, upper):
        yield ("flat" if up is None else "levels"), jv.GraphIndex(adj0, entry, up), o.make_graph(adj0, entry, up)


@pytest.mark.gpu
def test_sketch_walk_equals_oracle(jv, oracle, latent_world):
    from test_gpu_parity import _assert_same_search, _oracle_search
    data, queries, vec, adj0, upper, entry = latent_world
    n, dim = data.shape
    mk = lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q))
    rng = np.random.default_rng(9)
    shared = rng.random(n) < 0.4
    for name, gi, g in _worlds(jv, latent_world):
        s = jv.GraphSearcher(gi)
        for topK, rerankK in ((10, 40), (10, 100)):
            res = s.search(vec, queries, o.DOT_PRODUCT, topK, rerankK)
            _assert_same_search(res, _oracle_search(oracle, g, mk, queries, topK, rerankK), (name, topK, rerankK))
        res = s.search(vec, queries, o.DOT_PRODUCT, 10, 40, acceptOrds=shared)
        _assert_same_search(res, _oracle_search(oracle, g, mk, queries, 10, 40, accept=shared), (name, "accept"))
        res = s.search(vec, queries, o.DOT_PRODUCT, 10, 40, threshold=0.7)
        _assert_same_search(res, _oracle_search(oracle, g, mk, queries, 10, 40, threshold=0.7), (name, "threshold"))
        gi.close()


@pytest.mark.gpu
def test_sketch_walk_per_query_accept_and_tie_tail_retry(jv, oracle, latent_world):
    # JV_LIST_CAP = rerankK leaves the list no room: with acceptOrds every drop leaves fewer than rerankK accepted entries above it,
    # so queries report overflow code 2 and are re-run with a 4x list; the answers still equal the oracle's
    from test_gpu_parity import _assert_same_search, _oracle_search
    data, queries, vec, adj0, upper, entry = latent_world
    n, dim = data.shape
    mk = lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(data), n, dim, fp(q))
    rng = np.random.default_rng(10)
    per_query = rng.random((NQ, n)) < 0.6
    for name, gi, g in _worlds(jv, latent_world):
        s = jv.GraphSearcher(gi)
        res = s.search(vec, queries, o.DOT_PRODUCT, 10, 40, acceptOrds=per_query, threshold=0.6)
        _assert_same_search(res, _oracle_search(oracle, g, mk, queries, 10, 40, accept=per_query, threshold=0.6), (name, "per-query accept + threshold"))
        os.environ["JV_LIST_CAP"] = "40"
        try:
            res = s.search(vec, queries, o.DOT_PRODUCT, 10, 40, acceptOrds=per_query[0])
        finally:
            del os.environ["JV_LIST_CAP"]
        assert res.retried > 0, "the tight list was expected to overflow"
        _assert_same_search(res, _oracle_search(oracle, g, mk, queries, 10, 40, accept=per_query[0]), (name, "tie tail retry"))
        gi.close()
