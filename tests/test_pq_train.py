"""PQ training on the device (jv_pq_train / jv_pq_refine: ProductQuantization.compute / refine, UNWEIGHTED).

CPU: the model's -ln against np.log over every 24-bit input; the exponential race picks the second seed with probability D_j / sum D;
the fixed-point mean is the exact mean rounded to fp32 on integer data; Floyd's sample is distinct, sorted, in range, of size
min(n, cap).
GPU (-m gpu): codebooks, centroid and every counter equal tests/pq_train_model.py bit for bit, with no near-tie budget, over the
sub-space layouts, the sampled path, degenerate worlds (fallbacks and reseeds) and a strided adopted data set; reproducibility;
refine; the trained codebooks encode the training rows to the model's final assignment; quality against train_pq_numpy; errors."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as o
import pq_train_model as pt

F32 = np.float32


# ------------------------------------------------------------------------------------------------ CPU
def test_neg_ln_matches_log_on_every_input():
    u = np.arange(1, (1 << 24) + 1, dtype=np.int64).astype(F32) * F32(2.0 ** -24)
    got = pt.neg_ln_unit(u).astype(np.float64)
    want = -np.log(u.astype(np.float64))
    assert got[-1] == 0.0 and pt.neg_ln_unit(np.array([1.0], F32)).view(np.uint32)[0] == 0  # ln(1) is +0, so keys stay non-negative
    rel = np.abs(got[:-1] - want[:-1]) / want[:-1]
    assert rel.max() <= 1.5e-6, rel.max()
    assert (got >= 0).all()


def test_race_picks_second_seed_in_proportion_to_distance():
    from scipy.stats import chisquare
    x = np.array([0.0, 1.0, 1.5, 4.0, 7.0, 7.25], F32)
    T = x[None, :, None]  # one sub-space of size 1
    D = (x[:, None] - x[None, :]) ** 2  # D[j0][j]: squared distance of row j to the first pick j0
    seeds = 20000
    obs = np.zeros(6)
    exp = np.zeros(6)
    for s in range(seeds):
        picks, fb = pt.kmeanspp(T, 2, s)
        assert fb == 0
        obs[picks[1, 0]] += 1
        exp += D[picks[0, 0]] / D[picks[0, 0]].sum()
    assert chisquare(obs, exp).pvalue > 1e-3, (obs, exp)


def test_fixed_mean_is_exact_mean_on_integer_data():
    rng = np.random.default_rng(5)
    for n, dim, lo, hi in ((1, 7, -5, 5), (1000, 33, -1000, 1000), (12345, 16, -(1 << 20), 1 << 20), (77, 4, 0, 1)):
        x = rng.integers(lo, hi + 1, (n, dim)).astype(F32)
        want = (x.astype(np.float64).sum(0) / n).astype(F32)
        assert np.array_equal(pt.fixed_mean(x).view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("n,cap,seed", [(10, 10, 0), (9, 100, 1), (9000, 4000, 7), (200000, 128000, 3), (5, 4, 11)])
def test_floyd_sample(n, cap, seed):
    s = pt.floyd_sample(n, cap, seed)
    assert len(s) == min(n, cap)
    assert (np.diff(s) > 0).all() and s[0] >= 0 and s[-1] < n
    if n > cap:
        assert not np.array_equal(s, pt.floyd_sample(n, cap, seed + 1))


# ------------------------------------------------------------------------------------------------ GPU
def _lib():
    import jvector_b200 as jv  # noqa: F401
    from jvector_b200 import _native as nat
    return nat, nat.init()


def _stats(nat, st):
    return {name: getattr(st, name) for name, _ in nat.PQTrainStats._fields_}


def dev_train(vec, M, k, center=False, iters=6, cap=0, seed=0):
    nat, lib = _lib()
    dim = vec.dimension()
    p = nat.PQTrainParams(M, k, int(center), iters, cap, seed)
    cb = np.empty(k * dim, F32)
    cen = np.empty(dim, F32) if center else None
    st = nat.PQTrainStats()
    nat.check(lib.jv_pq_train(vec._h, C.byref(p), nat.fp(cb), nat.fp(cen), C.byref(st)))
    return cb, cen, _stats(nat, st)


def dev_refine(vec, M, k, codebooks, centroid, iters, cap=0, seed=0):
    nat, lib = _lib()
    p = nat.PQTrainParams(M, k, 0, iters, cap, seed)
    cb = np.empty_like(codebooks)
    st = nat.PQTrainStats()
    nat.check(lib.jv_pq_refine(vec._h, C.byref(p), nat.fp(codebooks), nat.fp(centroid), nat.fp(cb), C.byref(st)))
    return cb, _stats(nat, st)


def assert_same(dev, model):
    cb, cen, st = dev
    assert np.array_equal(cb.view(np.uint32), model.codebooks.view(np.uint32)), np.flatnonzero(cb.view(np.uint32) != model.codebooks.view(np.uint32))[:8]
    if model.centroid is not None:
        assert np.array_equal(cen.view(np.uint32), model.centroid.view(np.uint32))
    for key, want in model.stats.items():
        assert st[key] == want, (key, st[key], want, st)


def rows_for(rng, n, dim, center):
    x = rng.standard_normal((n, dim)).astype(F32)
    return (x + F32(3) * rng.standard_normal(dim).astype(F32)) if center else x


@pytest.mark.gpu
@pytest.mark.parametrize("dim,M,k,n,center", [(64, 8, 256, 6000, False), (100, 7, 33, 3000, True), (33, 33, 16, 1000, False),
                                               (48, 1, 64, 2000, True), (768, 96, 256, 20000, False)])
def test_train_equals_model(dim, M, k, n, center):
    import jvector_b200 as jv
    rng = np.random.default_rng(dim + M + k)
    x = rows_for(rng, n, dim, center)
    vec = jv.F32Vectors(x)
    assert_same(dev_train(vec, M, k, center, seed=5), pt.train(x, M, k, center, seed=5))


@pytest.mark.gpu
@pytest.mark.parametrize("center", (False, True), ids=("plain", "centred"))
def test_train_sampled_equals_model(center):
    import jvector_b200 as jv
    rng = np.random.default_rng(21)
    x = rows_for(rng, 9000, 40, center)
    vec = jv.F32Vectors(x)
    dev = dev_train(vec, 10, 64, center, cap=4000, seed=9)
    model = pt.train(x, 10, 64, center, cap=4000, seed=9)
    assert dev[2]["train_rows"] == 4000
    assert_same(dev, model)


@pytest.mark.gpu
def test_few_distinct_rows_fall_back_and_reseed():
    import jvector_b200 as jv
    rng = np.random.default_rng(4)
    x = rng.standard_normal((20, 16)).astype(F32)[rng.integers(0, 20, 500)]
    vec = jv.F32Vectors(x)
    dev = dev_train(vec, 4, 64, seed=2)
    model = pt.train(x, 4, 64, seed=2)
    assert model.stats["seeding_fallbacks"] > 0 and model.stats["empty_reseeds"] > 0, model.stats
    assert_same(dev, model)


@pytest.mark.gpu
def test_adopted_strided_rows():
    import jvector_b200 as jv
    nat, lib = _lib()
    rng = np.random.default_rng(8)
    n, dim, stride = 3000, 30, 32
    x = rows_for(rng, n, dim, True)
    padded = np.zeros((n, stride), F32)
    padded[:, :dim] = x
    buf = C.c_void_p()
    nat.check(lib.jv_device_malloc(C.byref(buf), padded.nbytes))
    try:
        nat.check(lib.jv_memcpy_h2d(buf, padded.ctypes.data, padded.nbytes))
        h = C.c_void_p()
        nat.check(lib.jv_dataset_adopt_f32_device(buf, n, dim, stride, C.byref(h)))
        vec = jv.api._Vectors(h, None)
        assert_same(dev_train(vec, 6, 50, True, seed=3), pt.train(x, 6, 50, True, seed=3))
        vec.close()
    finally:
        lib.jv_device_free(buf)


@pytest.mark.gpu
def test_seed_reproducible_and_different():
    import jvector_b200 as jv
    x = rows_for(np.random.default_rng(1), 4000, 32, False)
    vec = jv.F32Vectors(x)
    a, _, sa = dev_train(vec, 8, 64, seed=1)
    b, _, sb = dev_train(vec, 8, 64, seed=1)
    c, _, _ = dev_train(vec, 8, 64, seed=2)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert {k: v for k, v in sa.items() if k != "device_ms"} == {k: v for k, v in sb.items() if k != "device_ms"}
    assert not np.array_equal(a, c)


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", (0, 1, 2))
@pytest.mark.parametrize("center", (False, True), ids=("plain", "centroid"))
def test_refine_equals_model(rounds, center):
    import jvector_b200 as jv
    rng = np.random.default_rng(30 + rounds)
    dim, M, k = 50, 5, 40
    x0 = rows_for(rng, 3000, dim, center)
    vec0 = jv.F32Vectors(x0)
    cb0, cen0, _ = dev_train(vec0, M, k, center, iters=2, seed=4)
    x1 = (x0[:2500] + F32(0.1) * rng.standard_normal((2500, dim)).astype(F32)).astype(F32)
    vec1 = jv.F32Vectors(x1)
    got, st = dev_refine(vec1, M, k, cb0, cen0, rounds, seed=6)
    if rounds == 0:
        assert np.array_equal(got.view(np.uint32), cb0.view(np.uint32))
    model = pt.train(x1, M, k, iters=rounds, seed=6, codebooks=cb0, centroid=cen0)
    assert_same((got, None, st), model)
    # the Python surface gives the same bits
    pq = jv.ProductQuantization(cb0, M, k, dim, cen0).refine(vec1, rounds, seed=6)
    assert np.array_equal(pq.codebooks.view(np.uint32), got.view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("center", (False, True), ids=("plain", "centred"))
def test_encode_gives_final_assignment(center):
    import jvector_b200 as jv
    rng = np.random.default_rng(12)
    x = rows_for(rng, 7000, 48, center)
    vec = jv.F32Vectors(x)
    cb, cen, _ = dev_train(vec, 12, 128, center, cap=5000, seed=8)
    model = pt.train(x, 12, 128, center, cap=5000, seed=8)
    codes = jv.pq_encode_all(vec, cb, 12, 128, cen)
    assert np.array_equal(codes[model.ordinals].astype(np.int64), model.assignment)
    pq = jv.ProductQuantization.compute(vec, 12, 128, center, seed=8)  # default cap: all 7000 rows
    enc = pq.encodeAll(vec)
    assert enc.size() == 7000 and pq.stats["train_rows"] == 7000


def latent_rows(rng, n, dim, rank=32):
    f = rng.standard_normal((n, rank)).astype(F32) @ rng.standard_normal((rank, dim)).astype(F32)
    x = f + F32(0.3) * rng.standard_normal((n, dim)).astype(F32)
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(F32)


def quality(x, q, codes, codebooks, M, k):
    """(quantisation MSE, ADC brute-force recall@10 with an fp32 rerank of the best 100)"""
    sizes, offsets = o.pq_layout(x.shape[1], M)
    rec = np.empty_like(x)
    for m in range(M):
        cb = codebooks[k * offsets[m]:k * (offsets[m] + sizes[m])].reshape(k, sizes[m])
        rec[:, offsets[m]:offsets[m] + sizes[m]] = cb[codes[:, m]]
    mse = float(((x - rec) ** 2).sum(1).mean())
    truth = np.argsort(-(q @ x.T), axis=1)[:, :10]
    cand = np.argsort(-(q @ rec.T), axis=1)[:, :100]
    hits = 0
    for i in range(len(q)):
        top = cand[i][np.argsort(-(x[cand[i]] @ q[i]))[:10]]
        hits += len(set(top) & set(truth[i]))
    return mse, hits / (10 * len(q))


@pytest.mark.gpu
def test_quality_not_worse_than_numpy_helper():
    import jvector_b200 as jv
    rng = np.random.default_rng(77)
    n, dim, M, k = 20000, 128, 16, 256
    x = latent_rows(rng, n + 200, dim)
    x, q = x[:n], x[n:]
    vec = jv.F32Vectors(x)
    pq = jv.ProductQuantization.compute(vec, M, k)
    dev = quality(x, q, jv.pq_encode_all(vec, pq.codebooks, M, k), pq.codebooks, M, k)
    cb, _, _ = o.train_pq_numpy(np.random.default_rng(78), x, M, k, iters=6)
    ref = quality(x, q, jv.pq_encode_all(vec, cb, M, k), cb, M, k)
    print("device mse %.6f recall %.4f | numpy mse %.6f recall %.4f" % (dev + ref))
    assert dev[0] <= ref[0], (dev, ref)
    assert dev[1] >= ref[1] - 0.01, (dev, ref)


@pytest.mark.gpu
def test_errors():
    import jvector_b200 as jv
    nat, lib = _lib()
    INVALID, OOM = -2, -4
    x = rows_for(np.random.default_rng(2), 300, 16, False)
    vec = jv.F32Vectors(x)
    cb = np.empty(256 * 16, F32)
    cen = np.empty(16, F32)

    def train(M=4, k=16, center=0, iters=6, cap=0, out=cb, centroid=cen, v=vec, params=True):
        p = nat.PQTrainParams(M, k, center, iters, cap, 0)
        return lib.jv_pq_train(v._h, C.byref(p) if params else None, nat.fp(out), nat.fp(centroid), None)

    assert train() == 0
    assert train(M=0) == INVALID and train(M=17) == INVALID
    assert train(k=0) == INVALID and train(k=257) == INVALID
    assert train(k=256, cap=200) == INVALID and train(k=64, cap=63) == INVALID and train(k=64, cap=64) == 0
    assert train(iters=-1) == INVALID and train(cap=-1) == INVALID
    assert train(params=False) == INVALID and train(out=None) == INVALID
    assert train(center=1, centroid=None) == INVALID
    small = jv.F32Vectors(x[:10])
    assert train(v=small) == INVALID
    codes = np.zeros((300, 4), np.uint8)
    pqv = jv.PQVectors(codes, np.zeros(16 * 16, F32), 16, 16)
    assert train(v=pqv) == INVALID
    p = nat.PQTrainParams(4, 16, 0, 1, 0, 0)
    cb16 = np.zeros(16 * 16, F32)
    assert lib.jv_pq_refine(vec._h, C.byref(p), None, None, nat.fp(cb16), None) == INVALID
    assert lib.jv_pq_refine(vec._h, C.byref(p), nat.fp(cb16), None, None, None) == INVALID
    assert lib.jv_pq_refine(pqv._h, C.byref(p), nat.fp(cb16), None, nat.fp(cb16), None) == INVALID
    p.lloyd_iterations = -1
    assert lib.jv_pq_refine(vec._h, C.byref(p), nat.fp(cb16), None, nat.fp(cb16), None) == INVALID
    # training buffers far beyond HBM: the call allocates before it reads a row, and fails with JV_ERR_OOM
    buf = C.c_void_p()
    nat.check(lib.jv_device_malloc(C.byref(buf), 1 << 20))
    try:
        h = C.c_void_p()
        nat.check(lib.jv_dataset_adopt_f32_device(buf, 0x7fffffff, 64, 64, C.byref(h)))
        huge = jv.api._Vectors(h, None)
        p = nat.PQTrainParams(8, 16, 0, 1, 0x7fffffff, 0)
        out = np.empty(16 * 64, F32)
        assert lib.jv_pq_train(huge._h, C.byref(p), nat.fp(out), None, None) == OOM
        huge.close()
    finally:
        lib.jv_device_free(buf)
    assert train() == 0  # the library is still usable
