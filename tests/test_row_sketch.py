"""The int8 row sketch of an fp32 data set as the device computes it (row_sketch_kernel in kernels_batch.cu, read back through
jv_dataset_row_sketch_download), and the sketched fp32 DOT_PRODUCT walk (sketch_bound_pair in scorers.cuh, the `sketched` branch of
graph_search_kernel in search.cu) on the data where its bound is tightest: unnormalised (MIPS) rows, near ties, extreme rows and
strides that end in padding codes.

  - the device sketch equals its definition (row_bound_model.encode_int8): codes and scale bit for bit, padding codes 0, and a
    radius at least the exact radius (integer arithmetic, square roots bracketed) and within 4 ulp of the model's, so that a
    radius that is too small and one that is inflated (which would quietly turn the drops off) both fail; on registered and on
    adopted device rows;
  - the bound computed from the device's own codes, scale and radius is >= the kernel's exact score (the warp-order oracle);
  - sketched walks equal the oracle's walk in ids, score bits and the visited, reranked, expanded and level-0 expanded counters
    (test_search_tiers.assert_walk); a full batch leaves a sketch behind, a 48-query batch on a fresh data set does not.

Each graph is built on the device over the unit-normalised rows and searched over the unnormalised ones: the walk does not need its
topology to come from the searched rows, and the builder's Gram prune never sees 1e30-scale products. The rows and queries are
signed, so many scores fall below 0, which the walk refuses on every level as the reference does."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

import oracle_lib as o
import row_bound_model as rb
from oracle_lib import fp
from test_build_steps import latent_rows
from test_row_bound import adversarial_rows, queries_for
from test_search_tiers import World, _device_search, _same_result, full_sizes, knobs, oracle_walk, assert_walk

pytestmark = pytest.mark.gpu

DOT = o.DOT_PRODUCT
SMALL = 48
# stride 4 / 8 / 100 / 104 / 768 / 1024; sketch strides 8 (dims 1-5), 104 (97-101: 4 padding codes after stride 100), 768, 1024
SKETCH_DIMS = (1, 3, 4, 5, 97, 100, 101, 768, 1021, 1024)


@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


def stride_of(dim):
    return (dim + 3) & ~3


# ------------------------------------------------------------------------------------------------ the device sketch
def sketch_rows(rng, dim, queries):
    """adversarial_rows for every query, fp32-subnormal rows (scale subnormal, and scale 0 with nonzero values), rows whose
    largest value is the last one (in the last, padded float4 when dim % 4 != 0)"""
    rows = [adversarial_rows(rng, dim, q) for q in queries]
    sign = rng.choice([-1.0, 1.0], (24, dim))
    rows.append((sign[:16] * rng.uniform(0.5e-40, 2e-40, (16, dim))).astype(np.float32))          # s = max|x| / 127 subnormal
    rows.append((sign[16:] * rng.integers(1, 60, (8, dim)) * 2.0 ** -149).astype(np.float32))     # max|x| / 127 rounds to s = 0
    last = rng.standard_normal((8, dim)).astype(np.float32)
    last[:, dim - 1] = rng.choice([-50.0, 50.0], 8)
    rows.append(last)
    return np.ascontiguousarray(np.concatenate(rows).astype(np.float32))


def exact_radius_up(x, codes, s, stride):
    """per row an upper bracket of ||x - x_hat|| + gamma (||x|| + ||x_hat||), x_hat = s c, as a Fraction: every fp32 value is an
    integer times 2^-149, so the three sums of squares are exact integers; square roots bracketed to 2^-64 units"""
    K = 64
    g = Fraction(stride + 8, 1 << 23)

    def sqrt_up(N):
        r = math.isqrt(N << (2 * K))
        return r if r * r == N << (2 * K) else r + 1

    out = []
    for xr, cr, sr in zip((x.astype(np.float64) * 2.0 ** 149).tolist(), codes.astype(np.int64).tolist(), (s.astype(np.float64) * 2.0 ** 149).tolist()):
        m = [int(v) for v in xr]
        S = int(sr)
        D = sum((a - c * S) ** 2 for a, c in zip(m, cr))
        X = sum(a * a for a in m)
        H = S * S * sum(c * c for c in cr)
        out.append((sqrt_up(D) + g * (sqrt_up(X) + sqrt_up(H))) / Fraction(1 << (149 + K)))
    return out


def build_sketch(jv, vec, n, dim, rng):
    """one full-size DOT walk over a random graph of the rows: the search that builds the sketch"""
    nq = full_sizes(jv)[0]
    gi = jv.GraphIndex(rng.integers(0, n, (n, 16)).astype(np.int32), 0, None)
    try:
        jv.GraphSearcher(gi).search(vec, o.random_unit_vectors(rng, nq, dim), DOT, 10, 40)
    finally:
        gi.close()


def assert_sketch_is_its_definition(rows, codes, meta, what):
    n, dim = rows.shape
    stride = stride_of(dim)
    assert codes.shape == (n, (stride + 7) & ~7), (what, codes.shape)
    c, s, r = rb.encode_int8(rows, stride)
    assert (codes[:, dim:] == 0).all(), (what, "padding codes")
    bad = np.flatnonzero((codes[:, :dim] != c).any(1))
    assert len(bad) == 0, (what, "codes differ in rows", bad[:5].tolist())
    bad = np.flatnonzero(meta[:, 0].view(np.int32) != s.view(np.int32))
    assert len(bad) == 0, (what, "scale bits differ in rows", bad[:5].tolist(), meta[bad[:5], 0], s[bad[:5]])
    ulps = np.abs(rb.sortable(meta[:, 1]) - rb.sortable(r))
    assert ulps.max() <= 4, (what, "radius more than 4 ulp from the model's", int(np.argmax(ulps)), meta[np.argmax(ulps), 1], r[np.argmax(ulps)])
    exact = exact_radius_up(rows, codes[:, :dim], meta[:, 0], stride)
    low = [i for i in range(n) if Fraction(float(meta[i, 1])) < exact[i]]
    assert not low, (what, "radius below the exact radius in rows", low[:5], [float(exact[i]) for i in low[:5]], meta[low[:5], 1])


@pytest.fixture(scope="module", params=SKETCH_DIMS)
def sketched(request, jv):
    dim = request.param
    rng = np.random.default_rng(1000 + dim)
    queries = queries_for(rng, dim)
    rows = sketch_rows(rng, dim, queries)
    vec = jv.F32Vectors(rows)
    assert vec.row_sketch() is None
    build_sketch(jv, vec, len(rows), dim, rng)
    sk = vec.row_sketch()
    assert sk is not None, "a full DOT batch was expected to build the row sketch"
    vec.close()
    return dim, rows, queries, sk


def test_device_sketch_equals_its_definition(sketched):
    dim, rows, _, (codes, meta) = sketched
    assert_sketch_is_its_definition(rows, codes, meta, ("registered", dim))


def test_adopted_rows_sketch_equals_its_definition(jv, sketched):
    import torch
    dim, rows, _, _ = sketched
    n, stride = len(rows), stride_of(dim)
    t = torch.zeros((n, stride), dtype=torch.float32, device="cuda")
    t[:, :dim] = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    h = C.c_void_p()
    lib = jv.load()
    jv.api.check(lib.jv_dataset_adopt_f32_device(C.c_void_p(t.data_ptr()), n, dim, stride, C.byref(h)))
    adopted = jv.api._Vectors(h, t)
    try:
        assert jv.F32Vectors.row_sketch(adopted) is None
        build_sketch(jv, adopted, n, dim, np.random.default_rng(dim))
        sk = jv.F32Vectors.row_sketch(adopted)
        assert sk is not None
        assert_sketch_is_its_definition(rows, sk[0], sk[1], ("adopted", dim))
    finally:
        adopted.close()


def test_bound_over_the_device_sketch(oracle, sketched):
    # test_row_bound.test_bound_is_at_least_the_warp_order_score on the codes, scale and radius the device computed
    dim, rows, queries, (codes, meta) = sketched
    stride = stride_of(dim)
    for qi, q in enumerate(queries):
        ub = rb.dot_score_up(rb.upper_bound_raw(q, codes[:, :dim], meta[:, 0], meta[:, 1], stride))
        exact = np.array([oracle.jvo_compare_f32_warp(DOT, fp(q), fp(r), dim) for r in rows], np.float32)
        ok = np.isnan(exact) | (rb.sortable(ub) >= rb.sortable(exact))
        assert ok.all(), (dim, qi, np.flatnonzero(~ok)[:5], ub[~ok][:5], exact[~ok][:5])
        ids = np.arange(len(rows))
        assert (rb.topk_key(ub, ids) >= rb.topk_key(np.where(np.isnan(exact), ub, exact), ids)).all()


def test_row_sketch_download_arguments(jv):
    lib = jv.load()
    vec = jv.F32Vectors(o.random_unit_vectors(np.random.default_rng(3), 10, 5))
    ss = C.c_int(0)
    assert lib.jv_dataset_row_sketch_download(vec._h, None, None, C.byref(ss)) == -2 and ss.value == 8
    assert b"no row sketch" in lib.jv_last_error()
    vec.close()
    bq = jv.BQVectors(np.zeros((4, 1), np.uint64), 64)
    ss.value = 0
    assert lib.jv_dataset_row_sketch_download(bq._h, None, None, C.byref(ss)) == -2 and ss.value == 0
    with pytest.raises(jv.JVectorB200Error):
        jv.F32Vectors.row_sketch(bq)
    bq.close()


# ------------------------------------------------------------------------------------------------ sketched walks
def mixed_queries(rng, data, nq, pool=None):
    """unit, x 1e3, x 1e-3, a row of the world and the negation of one, in turn (rows drawn from `pool`, default every row). Over
    signed rows many DOT_PRODUCT scores (1 + q.x) / 2 fall below 0, which searchOneLayer refuses even at threshold 0, on every level:
    an x 1e3 query whose upper-level entry scores below 0 has no entry point for level 0 and returns nothing, on the device as in
    the oracle"""
    n, dim = data.shape
    q = latent_rows(rng, nq, dim)
    pool = np.arange(n) if pool is None else pool
    kind = np.arange(nq) % 5
    q[kind == 1] *= np.float32(1e3)
    q[kind == 2] *= np.float32(1e-3)
    q[kind == 3] = data[rng.choice(pool, int((kind == 3).sum()))]
    q[kind == 4] = -data[rng.choice(pool, int((kind == 4).sum()))]
    return np.ascontiguousarray(q, dtype=np.float32)


def device_graph(jv, unit, M, seed):
    """(adj0, entry, upper) of a device build with DOT over unit rows"""
    v = jv.F32Vectors(unit)
    gi = jv.GraphIndexBuilder(DOT, M=M, beamWidth=100, addHierarchy=True, seed=seed).build(v)
    v.close()
    info = gi.info()
    assert info["levels"] >= 2
    out = gi.level(0)[1], info["entry_node"], [gi.level(lv) for lv in range(1, info["levels"])]
    gi.close()
    return out


def unit_rows(x):
    nrm = np.linalg.norm(x.astype(np.float64), axis=1, keepdims=True)
    return np.ascontiguousarray(x / np.where(nrm > 0, nrm, 1.0), dtype=np.float32)


def log_uniform(rng, n, lo, hi):
    return np.exp(rng.uniform(np.log(lo), np.log(hi), n)).astype(np.float32)


def check_full_and_fresh(w):
    """the full walk (already run) left a sketch on its data set; a 48-query walk on a fresh copy builds none and equals the oracle"""
    assert w.sets["f32"][0].row_sketch() is not None, "a full DOT batch was expected to build the row sketch"
    fresh = w.jv.F32Vectors(w.data)
    try:
        q = w.queries[:SMALL]
        res = w.jv.GraphSearcher(w.gi).search(fresh, q, DOT, 10, 40)
        assert_walk(res, oracle_walk(w.oracle, w.g, w.sets["f32"][1](DOT), q, 10, 40), ("fresh", SMALL))
        assert fresh.row_sketch() is None, "a batch that does not fill the GPU must not build the row sketch"
    finally:
        fresh.close()


def walk_accept(w, acc, topK, rerankK, what, threshold=0.0):
    """the walk of every query with acceptOrds `acc` (one row per query) against the oracle's"""
    q = w.queries
    res = w.jv.GraphSearcher(w.gi).search(w.sets["f32"][0], q, DOT, topK, rerankK, acceptOrds=acc, threshold=threshold)
    assert_walk(res, oracle_walk(w.oracle, w.g, w.sets["f32"][1](DOT), q, topK, rerankK, threshold=threshold, accept=acc), what)
    return res


def walk_filtered(w, what):
    # per-query acceptOrds (60 % of the rows), with an all-true bitset (the same admission rule as no bitset: score >= 0), and with a
    # threshold of 0.5 (q.x >= 0: about half the rows for every query)
    nq = len(w.queries)
    walk_accept(w, w.accept(nq), 10, 40, what + ("accept",))
    walk_accept(w, np.ones((nq, w.n), bool), 10, 40, what + ("accept all",))
    walk_accept(w, w.accept(nq), 10, 40, what + ("accept + threshold",), threshold=0.5)


def every_configuration(w, monkeypatch, sms, what):
    nq = len(w.queries)
    w.walk("f32", DOT, nq, topK=10, rerankK=40, what=what)
    check_full_and_fresh(w)
    for topK, rerankK in ((10, 100), (100, 1000)):
        w.walk("f32", DOT, nq, topK=topK, rerankK=rerankK, what=what)
    walk_filtered(w, what)
    for wide in ("0", "1"):
        with knobs(monkeypatch, {"JV_SEARCH_WIDE": wide}):
            host = w.walk("f32", DOT, nq, topK=10, rerankK=40, what=what + ("JV_SEARCH_WIDE", wide))
    _same_result(_device_search(w.jv, w, "f32", None, DOT, w.queries, 10, 40), host, what + ("device",))
    # the overlapped host batch (>= 1 MB of queries) with a tight list: queries overflow on the tie tail and are re-run with a 4x
    # list. JV_LIST_CAP = rerankK and every query filtered: the first retry is itself a full batch and walks with the sketch.
    # Then the shortest list from 80 up on which the unfiltered batch never overflows, and 64 queries that accept 3 % of the rows:
    # only those 64 can overflow, so every retry re-runs at most 64 queries, fewer than the resident CTAs (>= 1 per SM), and walks
    # without the sketch. Either way the answers equal the oracle's.
    assert w.queries.nbytes >= 1 << 20
    acc = w.accept(nq)
    with knobs(monkeypatch, {"JV_LIST_CAP": 40}):
        res = walk_accept(w, acc, 10, 40, what + ("list cap", "every query filtered"))
        assert res.retried > 16 * sms, ("the first retry was expected to fill the GPU", res.retried)
    few = np.ones_like(acc)
    few[:64] = np.random.default_rng(64).random((64, w.n)) < 0.03
    assert 64 < sms
    for cap in (80, 320, 1280):
        with knobs(monkeypatch, {"JV_LIST_CAP": cap}):
            if w.jv.GraphSearcher(w.gi).search(w.sets["f32"][0], w.queries, DOT, 10, 40).retried == 0:
                res = walk_accept(w, few, 10, 40, what + ("list cap", cap, "64 queries filtered"))
                assert res.retried > 0, ("the filtered queries were expected to overflow", cap)
                break
    else:
        pytest.fail("no list cap up to 1280 keeps the unfiltered batch from overflowing")


@pytest.fixture(scope="module")
def sms(jv):
    return int(jv.load().jv_gpu_sm_count())


@pytest.fixture(scope="module", params=[100, 768])
def mips_graph(request, jv):
    dim = request.param
    rng = np.random.default_rng(dim)
    unit = latent_rows(rng, 20000, dim)
    return dim, unit, device_graph(jv, unit, 32, dim)


@pytest.mark.parametrize("norms", [(0.5, 2.0), (1e-3, 1e3)], ids=["norms-0.5-2", "norms-1e-3-1e3"])
def test_mips_walks(jv, oracle, monkeypatch, sms, mips_graph, norms):
    # maximum inner product search: latent rows with log-uniform norms
    dim, unit, (adj0, entry, upper) = mips_graph
    rng = np.random.default_rng(int(norms[1]) + dim)
    data = np.ascontiguousarray(unit * log_uniform(rng, len(unit), *norms)[:, None], dtype=np.float32)
    w = World(jv, oracle, data, mixed_queries(rng, data, full_sizes(jv)[0]), adj0, entry, upper)
    try:
        every_configuration(w, monkeypatch, sms, ("mips", dim, norms))
    finally:
        w.close()


def test_near_tie_walks(jv, oracle, monkeypatch, sms):
    # clusters x (1 -/+ j 2^-24), j = 0 .. 7 (j = 0 twice: exact duplicates): the list boundary often falls inside a cluster, and
    # rows the walk drops score within a few ulp of the last key
    rng = np.random.default_rng(24)
    dim, bases = 100, 1100
    base = latent_rows(rng, bases, dim).astype(np.float64) * log_uniform(rng, bases, 0.5, 2.0)[:, None]
    j = np.arange(8, dtype=np.float64)
    f = np.concatenate([1.0 - j * 2.0 ** -24, 1.0 + j * 2.0 ** -24])
    cl = (base[:, None, :] * f[None, :, None]).reshape(-1, dim)
    rest = latent_rows(rng, 20000 - len(cl), dim) * log_uniform(rng, 20000 - len(cl), 0.5, 2.0)[:, None]
    data = np.concatenate([cl, rest]).astype(np.float32)
    data = np.ascontiguousarray(data[rng.permutation(len(data))])
    adj0, entry, upper = device_graph(jv, unit_rows(data), 32, 24)
    w = World(jv, oracle, data, mixed_queries(rng, data, full_sizes(jv)[0]), adj0, entry, upper)
    try:
        every_configuration(w, monkeypatch, sms, ("near ties",))
    finally:
        w.close()


def test_extreme_walks(jv, oracle):
    # about 1 % of a latent world replaced by the adversarial families of the sketch tests (zero, constant, 1e-30 .. 1e30, the fp16
    # subnormal range, +/- the query), at level-0-only nodes; the rows that score exactly 0.5 stay far below the list's capacity, and
    # the query rows come from the latent rows only (a zero query would tie every row)
    rng = np.random.default_rng(30)
    dim, n = 100, 20000
    unit = latent_rows(rng, n, dim)
    adj0, entry, upper = device_graph(jv, unit, 32, 30)
    data = unit * log_uniform(rng, n, 0.5, 2.0)[:, None]
    odd = adversarial_rows(rng, dim, o.random_unit_vectors(rng, 1, dim)[0])
    upper_nodes = np.concatenate([ids for ids, _ in upper] + [[entry]])
    where = rng.choice(np.setdiff1d(np.arange(n), upper_nodes), len(odd), replace=False)
    data[where] = odd
    data = np.ascontiguousarray(data, dtype=np.float32)
    w = World(jv, oracle, data, mixed_queries(rng, data, full_sizes(jv)[0], np.setdiff1d(np.arange(n), where)), adj0, entry, upper)
    try:
        nq = len(w.queries)
        for topK, rerankK in ((10, 40), (10, 100)):
            w.walk("f32", DOT, nq, topK=topK, rerankK=rerankK, what=("extreme",))
        check_full_and_fresh(w)
        walk_filtered(w, ("extreme",))
    finally:
        w.close()


@pytest.mark.parametrize("dim", [3, 4, 5])
def test_tiny_stride_walks(jv, oracle, dim):
    # stride 4 (dims 3, 4) or 8 (dim 5), sketch stride 8: one 8-code load per row, and for stride 4 its upper half is padding
    # read against q = 0 (the 8 i + 4 < stride guard is false)
    rng = np.random.default_rng(dim)
    n = 8000
    unit = latent_rows(rng, n, dim)
    adj0, entry, upper = device_graph(jv, unit, 16, dim)
    data = np.ascontiguousarray(unit * log_uniform(rng, n, 0.5, 2.0)[:, None], dtype=np.float32)
    w = World(jv, oracle, data, mixed_queries(rng, data, full_sizes(jv)[0]), adj0, entry, upper)
    try:
        nq = len(w.queries)
        for topK, rerankK in ((10, 40), (10, 100)):
            w.walk("f32", DOT, nq, topK=topK, rerankK=rerankK, what=("tiny", dim))
        check_full_and_fresh(w)
        walk_filtered(w, ("tiny", dim))
        codes, _ = w.sets["f32"][0].row_sketch()
        assert codes.shape == (n, 8) and (codes[:, dim:] == 0).all()
    finally:
        w.close()
