"""PQ with an anisotropic threshold (ProductQuantization with anisotropicThreshold > UNWEIGHTED) on the device.

CPU: pcm against its formula; the model's Gauss-Jordan against float64 and against a line-by-line transcription of Matrix.invert
(including an |pivot| tie); with pcm = 1 the anisotropic update is the mean; the model's encode never raises its own objective and
keeps a zero row at its start; the model at T = -1 is pq_train_model.train and the unweighted encode.
GPU (-m gpu): jv_pq_train_anisotropic / jv_pq_refine_anisotropic equal tests/pq_aniso_model.py bit for bit (codebooks, centroid and
every counter) over uneven splits, d_s = 1, M = 1, d_s = 64, k < 256, centring, a sampled cap and T in {0.2, 0.5, 0.9, -0.5};
T and -T agree; reseeds in the anisotropic rounds; both encoders equal the model's codes and counters (zero rows, a partial tile,
M = 96 at k = 256, wide sub-spaces, adopted strided rows); T = -1 gives the unweighted calls' bytes; the reference's
testConvergenceAnisotropic; anisotropic codes build and search; errors leave the outputs untouched."""
import ctypes as C

import numpy as np
import pytest

import pq_aniso_model as pa
import pq_train_model as pt

F32 = np.float32


# ------------------------------------------------------------------------------------------------ CPU
def test_pcm_formula():
    for T in (0.0, 0.2, 0.5, 0.9, -0.5, -0.99):
        for d in (1, 2, 8, 64, 768):
            t = float(F32(T))  # the threshold is a float
            par = t * t
            want = 1.0 if d == 1 else max(1.0, par / ((1 - par) / (d - 1)))
            assert pa.pcm(T, d) == F32(want), (T, d)
            assert pa.pcm(-T, d) == pa.pcm(T, d)
    assert pa.pcm(0.2, 8) == 1.0 and abs(float(pa.pcm(0.5, 8)) - 7 / 3) < 1e-6
    assert abs(float(pa.pcm(0.2, 768)) - 0.04 / (0.96 / 767)) < 1e-4 and abs(float(pa.pcm(0.5, 768)) - 255.667) < 1e-2


def _invert_transcribed(A):
    """Matrix.invert (base:vector/Matrix.java:71-123) line by line in fp32 scalars, every column updated"""
    N = len(A)
    a = [[F32(A[i][j]) for j in range(N)] + [F32(1 if i == j else 0) for j in range(N)] for i in range(N)]
    for i in range(N):
        mr = i
        for k in range(i + 1, N):
            if abs(a[k][i]) > abs(a[mr][i]):
                mr = k
        a[i], a[mr] = a[mr], a[i]
        s = F32(1) / a[i][i]
        a[i] = [v * s for v in a[i]]
        for k in range(N):
            if k != i:
                f = a[k][i]
                a[k] = [a[k][j] + (-f) * a[i][j] for j in range(2 * N)]
    return np.array([row[N:] for row in a], F32)


def test_gauss_jordan_matches_float64_and_the_reference_order():
    rng = np.random.default_rng(3)
    for N in (1, 2, 5, 8, 17):
        B = rng.standard_normal((6, N, N)).astype(F32)
        A = (B @ np.swapaxes(B, 1, 2) / F32(N) + np.eye(N, dtype=F32)).astype(F32)
        got = pa.gauss_jordan_inverse(A)
        want = np.linalg.inv(A.astype(np.float64))
        assert np.allclose(got, want, rtol=2e-4, atol=2e-5), (N, np.abs(got - want).max())
        for s in range(3):
            assert np.array_equal(got[s].view(np.uint32), _invert_transcribed(A[s]).view(np.uint32)), (N, s)
    # an |pivot| tie in column 0: the first row stays the pivot; taking the second gives other bits
    tie = np.array([[3.0, 1.0, 0.5], [-3.0, 7.0, 0.25], [1.0, 0.3, 2.0]], F32)
    got = pa.gauss_jordan_inverse(tie[None])[0]
    assert np.array_equal(got.view(np.uint32), _invert_transcribed(tie).view(np.uint32))
    swapped = _invert_transcribed(tie[[1, 0, 2]])[:, [1, 0, 2]]
    assert not np.array_equal(got.view(np.uint32), swapped.view(np.uint32))
    assert np.allclose(got, np.linalg.inv(tie.astype(np.float64)), rtol=1e-5, atol=1e-6)


def test_pcm_one_update_is_the_mean():
    rng = np.random.default_rng(4)
    N = 8
    assert pa.pcm(0.2, N) == 1.0
    ocm = F32(1) / pa.pcm(0.2, N)
    S = rng.standard_normal((5, N, N)).astype(F32)
    A = S * ((F32(1) - ocm) / F32(37))
    idx = np.arange(N)
    A[:, idx, idx] = A[:, idx, idx] + ocm
    mean = rng.standard_normal((5, N)).astype(F32)
    mean[0, 3] = 0.0
    got = pa.solve_centroids(mean, A)
    assert np.array_equal(got, mean)  # as values: a zero's sign may differ


def latent_rows(rng, n, dim, rank=16, noise=0.3):
    f = rng.standard_normal((n, rank)).astype(F32) @ rng.standard_normal((rank, dim)).astype(F32)
    x = f + F32(noise) * rng.standard_normal((n, dim)).astype(F32)
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(F32)


@pytest.mark.parametrize("T", (0.2, 0.5, 0.9))
def test_model_encode_never_raises_its_objective(T):
    rng = np.random.default_rng(int(T * 10))
    dim, M, k = 32, 8, 16
    x = latent_rows(rng, 700, dim)
    x[5] = 0.0
    cb = pt.train(x, M, k, iters=3, seed=1).codebooks
    start, _ = pa.encode(x, cb, M, k, T, sweeps=0)
    codes, st = pa.encode(x, cb, M, k, T)
    assert st["moves"] > 0 and 1 <= st["max_sweeps"] <= 10
    assert np.array_equal(codes[5], start[5])
    with np.errstate(divide="ignore", invalid="ignore"):
        before, after = pa.objective(x, cb, M, k, T, start), pa.objective(x, cb, M, k, T, codes)
    live = np.arange(len(x)) != 5
    assert (after[live] <= before[live] + 1e-5 * np.abs(before[live]) + 1e-7).all()
    assert after[live].sum() < before[live].sum()


def test_model_unweighted_is_the_existing_model():
    rng = np.random.default_rng(6)
    x = latent_rows(rng, 900, 20)
    a, b = pa.train(x, 5, 32, -1, seed=2), pt.train(x, 5, 32, seed=2)
    assert np.array_equal(a.codebooks.view(np.uint32), b.codebooks.view(np.uint32))
    assert np.array_equal(a.assignment, b.assignment)
    codes, st = pa.encode(x, a.codebooks, 5, 32, -1)
    assert np.array_equal(codes[b.ordinals].astype(np.int64), b.assignment) and st["moves"] == 0


# ------------------------------------------------------------------------------------------------ GPU
def _lib():
    import jvector_b200 as jv  # noqa: F401
    from jvector_b200 import _native as nat
    return nat, nat.init()


def _astats(nat, st):
    out = {name: getattr(st.lloyd, name) for name, _ in nat.PQTrainStats._fields_}
    out.update({name: getattr(st, name) for name, _ in nat.PQAnisotropicStats._fields_[1:]})
    return out


def dev_train(vec, M, k, T, center=False, iters=6, cap=0, seed=0):
    nat, lib = _lib()
    dim = vec.dimension()
    p = nat.PQTrainParams(M, k, int(center), iters, cap, seed)
    cb = np.empty(k * dim, F32)
    cen = np.empty(dim, F32) if center else None
    st = nat.PQAnisotropicStats()
    nat.check(lib.jv_pq_train_anisotropic(vec._h, C.byref(p), T, nat.fp(cb), nat.fp(cen), C.byref(st)))
    return cb, cen, _astats(nat, st)


def dev_refine(vec, M, k, T, codebooks, centroid, rounds, seed=0):
    nat, lib = _lib()
    p = nat.PQTrainParams(M, k, 0, rounds, 0, seed)
    cb = np.empty_like(codebooks)
    st = nat.PQAnisotropicStats()
    nat.check(lib.jv_pq_refine_anisotropic(vec._h, C.byref(p), T, nat.fp(codebooks), nat.fp(centroid), nat.fp(cb), C.byref(st)))
    return cb, _astats(nat, st)


def assert_same(dev, model):
    cb, cen, st = dev
    bad = np.flatnonzero(cb.view(np.uint32) != model.codebooks.view(np.uint32))
    assert len(bad) == 0, (bad[:8], cb[bad[:4]], model.codebooks[bad[:4]])
    if model.centroid is not None:
        assert np.array_equal(cen.view(np.uint32), model.centroid.view(np.uint32))
    for key, want in model.stats.items():
        assert st[key] == want, (key, st[key], want, st)


TRAIN_GRID = [  # dim, M, k, n, center, cap, T
    (100, 7, 64, 3000, True, 0, 0.5),     # uneven split: sizes 15 and 14, two pcms
    (33, 33, 16, 1000, False, 0, 0.9),    # d_s = 1: pcm 1
    (48, 1, 32, 1500, True, 0, 0.2),      # M = 1 at d_s = 48
    (128, 2, 16, 1200, False, 0, 0.5),    # d_s = 64 exactly
    (40, 10, 64, 5000, True, 2000, -0.5),  # sampled cap, negative T
    (64, 8, 256, 4000, False, 0, 0.2),    # k = 256, pcm 1 in training
]


@pytest.mark.gpu
@pytest.mark.parametrize("dim,M,k,n,center,cap,T", TRAIN_GRID)
def test_train_equals_model(dim, M, k, n, center, cap, T):
    import jvector_b200 as jv
    rng = np.random.default_rng(dim + M + k)
    x = latent_rows(rng, n, dim)
    if center:
        x = (x + F32(0.2) * rng.standard_normal(dim).astype(F32)).astype(F32)
    vec = jv.F32Vectors(x)
    dev = dev_train(vec, M, k, T, center, cap=cap, seed=5)
    model = pa.train(x, M, k, T, center, cap=cap, seed=5)
    assert model.stats["max_anisotropic_updates"] > 0
    assert_same(dev, model)
    if cap:
        assert dev[2]["train_rows"] == cap


@pytest.mark.gpu
def test_sign_of_threshold_does_not_matter():
    import jvector_b200 as jv
    x = latent_rows(np.random.default_rng(9), 2000, 24)
    vec = jv.F32Vectors(x)
    a, _, sa = dev_train(vec, 6, 32, 0.7, seed=3)
    b, _, sb = dev_train(vec, 6, 32, -0.7, seed=3)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert {k: v for k, v in sa.items() if k != "device_ms"} == {k: v for k, v in sb.items() if k != "device_ms"}


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", (0, 1, 2))
@pytest.mark.parametrize("center", (False, True), ids=("plain", "centroid"))
def test_refine_equals_model(rounds, center):
    import jvector_b200 as jv
    rng = np.random.default_rng(40 + rounds)
    dim, M, k, T = 50, 5, 40, 0.6
    x0 = latent_rows(rng, 3000, dim)
    vec0 = jv.F32Vectors(x0)
    cb0, cen0, _ = dev_train(vec0, M, k, -1.0, center, iters=2, seed=4)
    x1 = latent_rows(rng, 2500, dim)
    vec1 = jv.F32Vectors(x1)
    got, st = dev_refine(vec1, M, k, T, cb0, cen0, rounds, seed=6)
    if rounds == 0:
        assert np.array_equal(got.view(np.uint32), cb0.view(np.uint32))
    model = pa.train(x1, M, k, T, iters=rounds, seed=6, codebooks=cb0, centroid=cen0)
    assert_same((got, None, st), model)
    assert st["max_lloyd_updates"] == 0 and (st["max_anisotropic_updates"] > 0) == (rounds > 0)
    pq = jv.ProductQuantization(cb0, M, k, dim, cen0).refine(vec1, rounds, seed=6, anisotropicThreshold=T)
    assert np.array_equal(pq.codebooks.view(np.uint32), got.view(np.uint32)) and pq.anisotropicThreshold == T


@pytest.mark.gpu
def test_anisotropic_rounds_reseed():
    import jvector_b200 as jv
    rng = np.random.default_rng(4)
    x = latent_rows(rng, 20, 16)[rng.integers(0, 20, 500)]
    vec = jv.F32Vectors(x)
    dev = dev_train(vec, 4, 64, 0.5, seed=2)
    model = pa.train(x, 4, 64, 0.5, seed=2)
    assert model.stats["anisotropic_reseeds"] > 0, model.stats
    assert_same(dev, model)


def dev_encode(rows, cb, M, k, T, cen=None):
    import jvector_b200 as jv
    codes, st = jv.pq_encode_all_anisotropic(rows, cb, M, k, cen, T)
    return codes, st


def assert_codes(got, want):
    codes, st = got
    wcodes, wst = want
    bad = np.flatnonzero((codes != wcodes).any(1))
    assert len(bad) == 0, (len(bad), bad[:8])
    for key, v in wst.items():
        assert st[key] == v, (key, st[key], v)


ENCODE_GRID = [  # dim, M, k, n, center, T
    (768, 96, 256, 300, False, 0.2),  # the c3 shape
    (64, 16, 256, 1037, True, 0.5),   # a partial tile
    (100, 7, 64, 500, True, 0.9),     # uneven split
    (128, 2, 256, 200, False, 0.5),   # d_s = 64: staged codebook, sub-vector from global memory
    (200, 1, 128, 150, False, 0.3),   # a codebook above the shared-memory budget
    (33, 33, 16, 400, False, -0.5),   # d_s = 1
]


@pytest.mark.gpu
@pytest.mark.parametrize("dim,M,k,n,center,T", ENCODE_GRID)
def test_encoders_equal_model(dim, M, k, n, center, T):
    import jvector_b200 as jv
    rng = np.random.default_rng(dim * 3 + M)
    x = latent_rows(rng, n, dim)
    x[[0, n // 2, n - 1]] = 0.0
    cen = (F32(0.05) * rng.standard_normal(dim)).astype(F32) if center else None
    if center:
        x[n // 3] = cen  # zero after centring
    cb = pt.train(latent_rows(rng, max(2 * k, 600), dim), M, k, iters=1, seed=1).codebooks
    want = pa.encode(x, cb, M, k, T, cen)
    assert want[1]["moves"] > 0 or M == dim  # scalar sub-spaces here never move
    assert_codes(dev_encode(x, cb, M, k, T, cen), want)
    vec = jv.F32Vectors(x)
    assert_codes(dev_encode(vec, cb, M, k, T, cen), want)
    vec.close()


@pytest.mark.gpu
def test_encode_adopted_strided_rows():
    import jvector_b200 as jv
    nat, lib = _lib()
    rng = np.random.default_rng(8)
    n, dim, stride, M, k, T = 700, 30, 32, 6, 64, 0.5
    x = latent_rows(rng, n, dim)
    cb = pt.train(x, M, k, iters=2, seed=3).codebooks
    padded = np.zeros((n, stride), F32)
    padded[:, :dim] = x
    buf = C.c_void_p()
    nat.check(lib.jv_device_malloc(C.byref(buf), padded.nbytes))
    try:
        nat.check(lib.jv_memcpy_h2d(buf, padded.ctypes.data, padded.nbytes))
        h = C.c_void_p()
        nat.check(lib.jv_dataset_adopt_f32_device(buf, n, dim, stride, C.byref(h)))
        vec = jv.api._Vectors(h, None)
        assert_codes(dev_encode(vec, cb, M, k, T), pa.encode(x, cb, M, k, T))
        vec.close()
    finally:
        lib.jv_device_free(buf)


@pytest.mark.gpu
def test_unweighted_threshold_gives_the_existing_bytes():
    import jvector_b200 as jv
    from test_pq_train import dev_refine as refine0
    from test_pq_train import dev_train as train0
    rng = np.random.default_rng(11)
    x = latent_rows(rng, 3000, 40)
    vec = jv.F32Vectors(x)
    a, ca, sa = dev_train(vec, 8, 64, -1.0, True, seed=7)
    b, cb_, sb = train0(vec, 8, 64, True, seed=7)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and np.array_equal(ca.view(np.uint32), cb_.view(np.uint32))
    for key in ("train_rows", "max_lloyd_updates", "changed_last", "empty_reseeds", "seeding_fallbacks"):
        assert sa[key] == sb[key]
    assert sa["max_anisotropic_updates"] == 0 and sa["anisotropic_reseeds"] == 0
    r1, _ = dev_refine(vec, 8, 64, -1.0, a, ca, 2, seed=1)
    r2, _ = refine0(vec, 8, 64, a, ca, 2, seed=1)
    assert np.array_equal(r1.view(np.uint32), r2.view(np.uint32))
    codes, st = dev_encode(vec, a, 8, 64, -1.0, ca)
    assert np.array_equal(codes, jv.pq_encode_all(vec, a, 8, 64, ca)) and st["moves"] == 0 and st["max_sweeps"] == 0
    codes, _ = dev_encode(x, a, 8, 64, -1.0, ca)
    assert np.array_equal(codes, jv.pq_encode_all(x, a, 8, 64, ca))
    pq = jv.ProductQuantization.compute(vec, 8, 64, True, seed=7)
    assert pq.anisotropicThreshold == -1.0 and np.array_equal(pq.codebooks.view(np.uint32), a.view(np.uint32))


def _euclid_loss(x, codes, cb, T):
    """TestProductQuantization.loss: rows with x . x_hat >= T add 1 - 1 / (1 + |x - x_hat|^2)"""
    xh = cb.reshape(-1, x.shape[1])[codes[:, 0].astype(np.int64)]
    keep = (x * xh).sum(1) >= T
    d2 = ((x - xh) ** 2).sum(1)
    return float((1 - 1 / (1 + d2))[keep].sum())


@pytest.mark.gpu
@pytest.mark.parametrize("dim", range(2, 12))
def test_convergence_anisotropic(dim):
    """TestProductQuantization.testConvergenceAnisotropic: clustered rows, M = 1, T = 0.2, anisotropic rounds from the k-means++
    seeding lower the loss of the unweighted encoding"""
    import jvector_b200 as jv
    rng = np.random.default_rng(100 + dim)
    k = 256
    nclusters = k + int(rng.integers(0, 10 * k))
    n = 1000 + int(rng.integers(0, 10000))
    centres = rng.uniform(-1, 1, (nclusters, dim)).astype(F32)
    v = rng.uniform(-1, 1, (n, dim)).astype(F32) * (F32(0.1) + F32(0.9) * rng.random((n, 1)).astype(F32))
    x = (v + centres[rng.integers(0, nclusters, n)]).astype(F32)
    vec = jv.F32Vectors(x)
    seeded, _, _ = dev_train(vec, 1, k, -1.0, iters=0, seed=dim)
    trained, st = dev_refine(vec, 1, k, 0.2, seeded, None, 100, seed=dim)
    assert st["max_anisotropic_updates"] >= 1
    before = _euclid_loss(x, jv.pq_encode_all(vec, seeded, 1, k), seeded, 0.2)
    after = _euclid_loss(x, jv.pq_encode_all(vec, trained, 1, k), trained, 0.2)
    assert after < before, (before, after)


@pytest.mark.gpu
def test_anisotropic_pq_builds_and_searches():
    import jvector_b200 as jv
    rng = np.random.default_rng(21)
    dim, M, k = 64, 16, 256
    data = latent_rows(rng, 8200, dim)
    base, queries = np.ascontiguousarray(data[:8000]), np.ascontiguousarray(data[8000:])
    f32 = jv.F32Vectors(base)
    pq = jv.ProductQuantization.compute(f32, M, k, seed=3, anisotropicThreshold=0.2)
    assert pq.anisotropicThreshold == 0.2 and pq.stats["max_anisotropic_updates"] > 0
    pqv = pq.encodeAll(f32)
    vsf = jv.VectorSimilarityFunction.DOT_PRODUCT
    truth, _, _ = jv.topk_bruteforce(f32, vsf, queries, 10)
    g = jv.GraphIndexBuilder(vsf, M=16, beamWidth=100).build(pqv)
    res = jv.GraphSearcher(g).search(pqv, queries, vsf, 10, 100, reranker=f32)
    recall = np.mean([len(set(res.nodes[i]) & set(truth[i])) / 10 for i in range(len(queries))])
    print("anisotropic PQ graph, PQ walk + fp32 rerank recall@10 %.4f" % recall)
    assert recall >= 0.6, recall
    g.close(), pqv.close(), f32.close()


@pytest.mark.gpu
def test_errors_leave_outputs_untouched():
    import jvector_b200 as jv
    nat, lib = _lib()
    INVALID, UNSUPPORTED = -2, -5
    x = latent_rows(np.random.default_rng(2), 300, 130)
    vec = jv.F32Vectors(x)
    cb = np.full(16 * 130, 7.0, F32)
    cen = np.full(130, 7.0, F32)
    codes = np.full((300, 10), 9, np.uint8)
    st = nat.PQAnisotropicStats()
    est = nat.PQEncodeStats()
    est.moves = 123

    def train(T, M=10, out=cb, centroid=cen, params=True):
        p = nat.PQTrainParams(M, 16, 0, 2, 0, 0)
        return lib.jv_pq_train_anisotropic(vec._h, C.byref(p) if params else None, T, nat.fp(out), nat.fp(centroid), C.byref(st))

    def refine(T, M=10, codebooks=cb, out=cb):
        p = nat.PQTrainParams(M, 16, 0, 2, 0, 0)
        return lib.jv_pq_refine_anisotropic(vec._h, C.byref(p), T, nat.fp(codebooks), None, nat.fp(out), C.byref(st))

    def enc_batch(T, rows=x, out=codes, M=10):
        return lib.jv_pq_encode_batch_anisotropic(nat.fp(rows), 300, 130, M, 16, nat.fp(cb), None, T, nat.bp(out), C.byref(est))

    def enc_set(T, out=codes, M=10):
        return lib.jv_pq_encode_dataset_anisotropic(vec._h, M, 16, nat.fp(cb), None, T, nat.bp(out), C.byref(est))

    for T in (float("nan"), 1.0, -1.5, 1.5):
        assert train(T) == INVALID and refine(T) == INVALID and enc_batch(T) == INVALID and enc_set(T) == INVALID
    assert train(0.5, M=2) == UNSUPPORTED and refine(0.5, M=2) == UNSUPPORTED  # ceil(130 / 2) = 65
    assert train(0.5, M=0) == INVALID and train(0.5, params=False) == INVALID and train(0.5, out=None) == INVALID
    assert refine(0.5, codebooks=None) == INVALID and refine(0.5, out=None) == INVALID
    assert enc_batch(0.5, rows=None) == INVALID and enc_batch(0.5, out=None) == INVALID and enc_set(0.5, out=None) == INVALID
    assert enc_batch(0.5, M=131) == INVALID and enc_set(0.5, M=0) == INVALID
    assert lib.jv_pq_train_anisotropic(None, None, 0.5, nat.fp(cb), None, None) == INVALID
    assert (cb == 7.0).all() and (cen == 7.0).all() and (codes == 9).all()
    assert st.lloyd.train_rows == 0 and st.max_anisotropic_updates == 0 and est.moves == 123
    # encoding has no sub-space limit, and the library is still usable
    assert enc_set(0.5, M=2) == 0 and est.max_sweeps >= 1
    assert train(0.5, M=3) == 0 and st.max_anisotropic_updates > 0
