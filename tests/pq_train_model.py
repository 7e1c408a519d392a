"""PQ training on the device (jv_pq_train / jv_pq_refine, csrc/pq_train.cu) restated on the host with the device's fp32 and int64
operations in the device's order, so codebooks, centroid and every counter compare bit for bit. TEST INFRASTRUCTURE.

  sample      Floyd's algorithm over counter_random(seed, TAG_SAMPLE, j, 0), ordinals sorted
  centre      int64 fixed-point column sums (fixed_exp / to_fixed / from_fixed)
  seeding     k-means++ as an exponential race: argmin E_j / D_j, E_j = neg_ln_unit(u_j), u_j a 24-bit uniform of (seed, m, round, j)
  Lloyd       KMeansPlusPlusClusterer.cluster(iterations, 0) with fixed-point centroid sums and counter_random reseeds

Sub-spaces are held padded to the widest size with zeros: a padded dimension adds (0 - 0)^2 = +0 to a distance after the real ones,
which leaves every fp32 sum bit for bit as it was."""
import numpy as np

MAX_PQ_TRAINING_SET_SIZE = 128000
TAG_RESEED, TAG_SAMPLE = 0x40000000, 0x7fffffff
F32 = np.float32
_U = np.uint64


def _f(bits):
    return np.array([bits], np.uint32).view(np.float32)[0]


SQRT2, LN2 = _f(0x3fb504f3), _f(0x3f317218)
C3, C5, C7, C9 = _f(0x3eaaaaab), _f(0x3e4ccccd), _f(0x3e124925), _f(0x3de38e39)


def mix64(x):
    """common.cuh mix64 on uint64 arrays (wrapping arithmetic)"""
    with np.errstate(over="ignore"):
        x = x + _U(0x9E3779B97F4A7C15)
        x = (x ^ (x >> _U(30))) * _U(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> _U(27))) * _U(0x94D049BB133111EB)
        return x ^ (x >> _U(31))


def _u32(v):
    return np.asarray(v, np.int64).astype(np.uint32).astype(np.uint64)


def counter_random(seed, a, b, c):
    """common.cuh counter_random(seed, a, b, c), broadcast over array arguments"""
    h = mix64(np.atleast_1d(np.asarray(seed, np.uint64)) ^ _u32(a))
    return mix64(mix64(h ^ _u32(b)) ^ _u32(c))


def neg_ln_unit(u):
    """common.cuh neg_ln_unit: -ln(u) for float32 u in (0, 1], the same sequence of round-to-nearest fp32 operations"""
    u = np.asarray(u, F32)
    bits = u.view(np.int32)
    e = ((bits >> 23) & 0xff) - 127
    m = ((bits & 0x7fffff) | 0x3f800000).astype(np.int32).view(F32)
    big = m > SQRT2
    m = np.where(big, m * F32(0.5), m)
    e = e + big
    s = (m - F32(1)) / (m + F32(1))
    z = s * s
    p = C9
    for c in (C7, C5, C3, F32(1)):
        p = (p * z) + c
    ln_m = (F32(2) * s) * p
    ln_u = (e.astype(F32) * LN2) + ln_m
    return F32(0) - ln_u


def uniform24(r):
    """u in (0, 1] from the top 24 bits of a draw"""
    return ((r >> _U(40)) + _U(1)).astype(F32) * F32(2.0 ** -24)


def fixed_exp(colmax, n):
    """exponent of a column's int64 fixed point: 62 - ea - bit_length(n), colmax < 2^ea; 0 for an all-zero column"""
    bits = np.asarray(colmax, F32).view(np.uint32).astype(np.int64)
    E = (bits >> 23) & 0xff
    e = 62 - np.where(E > 0, E - 126, -126) - int(n).bit_length()
    return np.where(bits == 0, 0, e).astype(np.int32)


def to_fixed(x, e):
    return np.rint(np.asarray(x, F32).astype(np.float64) * np.ldexp(1.0, e)).astype(np.int64)


def from_fixed(s, e, count):
    return ((s.astype(np.float64) * np.ldexp(1.0, -e)) / np.asarray(count, np.float64)).astype(F32)


def fixed_mean(x):
    """the device's column mean of rows x [n][dim]"""
    x = np.asarray(x, F32)
    e = fixed_exp(np.abs(x).max(0), len(x))
    return from_fixed(to_fixed(x, e).sum(0), e, len(x))


def floyd_sample(n, cap, seed):
    """the training ordinals: all rows when n <= cap, else Floyd's algorithm (ProductQuantization.extractTrainingVectors), sorted"""
    if n <= cap:
        return np.arange(n, dtype=np.int64)
    js = np.arange(n - cap, n, dtype=np.int64)
    draws = counter_random(seed, TAG_SAMPLE, js, 0) % (js + 1).astype(np.uint64)
    chosen = set()
    for j, t in zip(js.tolist(), draws.tolist()):
        chosen.add(j if t in chosen else t)
    return np.array(sorted(chosen), dtype=np.int64)


def pq_layout(dim, M):
    base, rem = divmod(dim, M)
    sizes = np.array([base + (1 if m < rem else 0) for m in range(M)], np.int64)
    return sizes, np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)


def _split(x, sizes, offsets):
    """rows [n][dim] -> [M][n][szmax], zero padded"""
    out = np.zeros((len(sizes), x.shape[0], int(sizes.max())), x.dtype)
    for m, (sz, off) in enumerate(zip(sizes, offsets)):
        out[m, :, :sz] = x[:, off:off + sz]
    return out


def _sq_dist(P, c):
    """(x - c)^2 accumulated in order over the (padded) sub-vector: P [..][n][sz], c broadcastable"""
    s = np.zeros(P.shape[:-1], F32)
    for t in range(P.shape[-1]):
        df = P[..., t] - c[..., t]
        s = s + df * df
    return s


def _nearest(P, C, chunk=2048):
    """first nearest centroid of every row: P [n][sz], C [k][sz]"""
    out = np.empty(len(P), np.int64)
    for i in range(0, len(P), chunk):
        Q = P[i:i + chunk]
        s = np.zeros((len(Q), len(C)), F32)
        for t in range(P.shape[1]):
            df = Q[:, t, None] - C[None, :, t]
            np.multiply(df, df, out=df)
            np.add(s, df, out=s)
        out[i:i + chunk] = s.argmin(1)
    return out


def kmeanspp(T, k, seed):
    """the k-means++ race over training rows T [M][n][sz]: (picks [k][M], seeding fallbacks). Round r picks the least
    E_j / D_j (round 0: E_j; rows with D_j = 0 never), ties to the lower j; with no finite key it takes the least E_j."""
    M, nt = T.shape[:2]
    marr = np.arange(M)
    j = np.arange(nt, dtype=np.uint64)
    D = None
    picks = np.zeros((k, M), np.int64)
    fallbacks = 0
    for r in range(k):
        h = mix64(mix64(np.asarray(seed, np.uint64) ^ _u32(marr)) ^ _u32(r))  # counter_random(seed, m, r, j) = mix64(h_m ^ j)
        E = neg_ln_unit(uniform24(mix64(h[:, None] ^ j[None, :])))
        if r == 0:
            picks[0] = E.argmin(1)
            continue
        dj = _sq_dist(T, T[marr, picks[r - 1]][:, None, :])
        D = dj if r == 1 else np.where(dj < D, dj, D)
        key = np.where(D > 0, E / np.where(D > 0, D, F32(1)), F32(np.inf))
        best = key.argmin(1)
        fb = ~np.isfinite(key[marr, best])
        fallbacks += int(fb.sum())
        picks[r] = np.where(fb, E.argmin(1), best)
    return picks, fallbacks


class Trained:
    def __init__(self, codebooks, centroid, stats, ordinals, assignment):
        self.codebooks, self.centroid, self.stats = codebooks, centroid, stats
        self.ordinals = ordinals      # training rows, ascending
        self.assignment = assignment  # [n_train][M]: each training row's cluster under the returned codebooks


def train(rows, M, k, globally_center=False, iters=6, cap=0, seed=0, codebooks=None, centroid=None):
    """jv_pq_train (codebooks None) or jv_pq_refine (from codebooks, minus centroid) on host rows [n][dim]"""
    rows = np.asarray(rows, F32)
    n, dim = rows.shape
    ords = floyd_sample(n, cap or MAX_PQ_TRAINING_SET_SIZE, seed)
    nt = len(ords)
    X = rows[ords]
    sizes, offsets = pq_layout(dim, M)
    seeding = codebooks is None
    if seeding:
        centroid = fixed_mean(X) if globally_center else None
    if centroid is not None:
        X = X - np.asarray(centroid, F32)
    T = _split(X, sizes, offsets)
    e_tr = _split(fixed_exp(np.abs(X).max(0), nt)[None, :], sizes, offsets)[:, 0, :]
    marr = np.arange(M)
    fallbacks = 0
    if seeding:
        picks, fallbacks = kmeanspp(T, k, seed)
        C = np.stack([T[marr, picks[c]] for c in range(k)], axis=1)
    else:
        cb = np.asarray(codebooks, F32).reshape(-1)
        C = np.zeros((M, k, T.shape[2]), F32)
        for m, (sz, off) in enumerate(zip(sizes, offsets)):
            C[m, :, :sz] = cb[k * off:k * (off + sz)].reshape(k, sz)
    assign = np.stack([_nearest(T[m], C[m]) for m in range(M)])
    Q = to_fixed(T, e_tr[:, None, :])
    active = np.ones(M, bool)
    updates = np.zeros(M, np.int64)
    last = np.zeros(M, np.int64)
    reseeds = 0
    for it in range(iters):
        if not active.any():
            break
        for m in np.flatnonzero(active):
            cnt = np.bincount(assign[m], minlength=k)
            sums = np.zeros((k, T.shape[2]), np.int64)
            np.add.at(sums, assign[m], Q[m])
            new = from_fixed(sums, e_tr[m][None, :], np.maximum(cnt, 1)[:, None])
            for c in np.flatnonzero(cnt == 0):
                r = int(counter_random(seed, int(m) | TAG_RESEED, it, int(c))[0] % np.uint64(nt))
                new[c] = T[m, r]
                reseeds += 1
            C[m] = new
        for m in np.flatnonzero(active):
            a = _nearest(T[m], C[m])
            changed = int((a != assign[m]).sum())
            assign[m] = a
            updates[m] += 1
            last[m] = changed
            if changed <= 0.01 * nt:
                active[m] = False
    out = np.empty(k * dim, F32)
    for m, (sz, off) in enumerate(zip(sizes, offsets)):
        out[k * off:k * (off + sz)] = C[m, :, :sz].reshape(-1)
    stats = {"train_rows": nt, "max_lloyd_updates": int(updates.max()), "changed_last": int(last.sum()), "empty_reseeds": reseeds,
             "seeding_fallbacks": fallbacks}
    return Trained(out, centroid if seeding else None, stats, ords, assign.T.copy())
