"""PQ with an anisotropic threshold on the device (jv_pq_train_anisotropic / jv_pq_refine_anisotropic, csrc/pq_train.cu step 5;
jv_pq_encode_*_anisotropic, csrc/pq_encode_aniso.cu) restated on the host with the device's fp32 and int64 operations in the
device's order, so codebooks, codes and every counter compare bit for bit. TEST INFRASTRUCTURE.

  pcm          KMeansPlusPlusClusterer.computeParallelCostMultiplier in double, rounded to fp32
  training     pq_train_model.train (sampling, centring, seeding, Lloyd), then per sub-space up to `iters` anisotropic rounds:
               fixed-point means, fixed-point sums of fl(fl(x_a x_b) * fl(1 / |x|^2)), Matrix.invert's Gauss-Jordan, the row-wise
               product with the mean, then the weighted reassignment; the 1 % early stop
  encoding     ProductQuantization.encodeAnisotropic: minimum-residual start, then up to 10 coordinate-descent sweeps

The quirks are the reference's: the training pcm uses the sub-space's size, the encoding pcm the full dimension, and P squares each
sub-space's parallel term before the sum is squared again."""
import numpy as np

import pq_train_model as pt

F32 = np.float32
TAG_ARESEED = 0x20000000
FLT_MAX = F32(3.402823466e+38)
SWEEPS = 10


def pcm(threshold, d):
    """computeParallelCostMultiplier(threshold, d): (float) max(1, T^2 / ((1 - T^2) / (d - 1))) in double, T the fp32 threshold
    (ProductQuantization keeps it as a float)"""
    t = float(F32(threshold))
    par = t * t
    with np.errstate(divide="ignore"):
        perp = np.float64(1 - par) / np.float64(d - 1)
        return F32(max(1.0, float(np.float64(par) / perp)))


def _seq_dot(A, B):
    """sum over the last axis in order, in fp32: fl(s + fl(a_t b_t))"""
    s = np.zeros(np.broadcast_shapes(A.shape[:-1], B.shape[:-1]), F32)
    for t in range(A.shape[-1]):
        s = s + A[..., t] * B[..., t]
    return s


def gauss_jordan_inverse(A):
    """Matrix.invert for a stack of fp32 systems A [..][N][N] as the device runs it: the first largest |pivot| (strictly larger
    wins), the pivot row times fl(1 / pivot), every other row plus fl(-factor * pivot row). Columns left of the pivot are never
    read again and are left as they are."""
    A = np.asarray(A, F32)
    N = A.shape[-1]
    lead = A.shape[:-2]
    a = np.concatenate([A, np.broadcast_to(np.eye(N, dtype=F32), A.shape)], axis=-1).reshape(-1, N, 2 * N).copy()
    sys = np.arange(a.shape[0])
    for i in range(N):
        mr = np.full(a.shape[0], i)
        for r in range(i + 1, N):
            mr = np.where(np.abs(a[:, r, i]) > np.abs(a[sys, mr, i]), r, mr)
        ri, rm = a[:, i].copy(), a[sys, mr].copy()
        a[sys, mr] = ri
        a[:, i] = rm
        rp = F32(1) / a[:, i, i]
        a[:, i, i + 1:] = a[:, i, i + 1:] * rp[:, None]
        fac = a[:, :, i].copy()
        others = np.array([r for r in range(N) if r != i], np.int64)
        if len(others):
            a[:, others, i + 1:] = a[:, others, i + 1:] + (-fac[:, others, None]) * a[:, i, None, i + 1:]
    return a[:, :, N:].reshape(lead + (N, N))


def solve_centroids(mean, A):
    """invert(A) * mean, row-wise dot products accumulated in order: mean [..][N], A [..][N][N]"""
    inv = gauss_jordan_inverse(A)
    return _seq_dot(inv, np.asarray(mean, F32)[..., None, :])


def _outer_sums(X, rinv, assign, k, e, chunk=4096):
    """int64 fixed-point sums per cluster of fl(fl(x_a x_b) * rinv) over rows with rinv != 0: [k][sz][sz]"""
    sz = X.shape[1]
    out = np.zeros((k, sz, sz), np.int64)
    for i in range(0, len(X), chunk):
        x, r, a = X[i:i + chunk], rinv[i:i + chunk], assign[i:i + chunk]
        keep = r != 0
        x, r, a = x[keep], r[keep], a[keep]
        if not len(x):
            continue
        terms = (x[:, :, None] * x[:, None, :]) * r[:, None, None]
        fx = pt.to_fixed(terms, e)
        order = np.argsort(a, kind="stable")
        a_s = a[order]
        starts = np.flatnonzero(np.r_[True, a_s[1:] != a_s[:-1]])
        out[a_s[starts]] += np.add.reduceat(fx[order], starts, axis=0)
    return out


def weighted_assign(X, C, xn, p, old):
    """updateAssignedPointsAnisotropic for one sub-space: X [n][sz], C [k][sz], xn [n], old [n] -> new assignment"""
    cn = _seq_dot(C, C)
    out = old.copy()
    for i in range(0, len(X), 2048):
        x = X[i:i + 2048]
        dot = np.zeros((len(x), len(C)), F32)
        for t in range(X.shape[1]):
            dot = dot + C[None, :, t] * x[:, t, None]
        xx = xn[i:i + 2048, None]
        e = dot - xx
        resid = (cn[None, :] - F32(2) * dot) + xx
        par = e * e
        d = p * par + (resid - par)
        d = np.where(d < FLT_MAX, d, np.inf)
        j = d.argmin(1)
        take = d[np.arange(len(x)), j] < FLT_MAX
        out[i:i + 2048] = np.where(take, j, old[i:i + 2048])
    return out


def train(rows, M, k, threshold, globally_center=False, iters=6, cap=0, seed=0, codebooks=None, centroid=None):
    """jv_pq_train_anisotropic (codebooks None) or jv_pq_refine_anisotropic on host rows [n][dim]. threshold == -1 is
    pq_train_model.train; otherwise compute runs `iters` Lloyd and `iters` anisotropic rounds, refine `iters` anisotropic rounds."""
    rows = np.asarray(rows, F32)
    refine = codebooks is not None
    if threshold == -1:
        base = pt.train(rows, M, k, globally_center, iters, cap, seed, codebooks, centroid)
        base.stats.update(max_anisotropic_updates=0, changed_last_anisotropic=0, anisotropic_reseeds=0)
        return base
    base = pt.train(rows, M, k, globally_center, 0 if refine else iters, cap, seed, codebooks, centroid)
    n, dim = rows.shape
    ords = base.ordinals
    nt = len(ords)
    cen = centroid if refine else base.centroid
    X = rows[ords]
    if cen is not None:
        X = X - np.asarray(cen, F32)
    sizes, offsets = pt.pq_layout(dim, M)
    e_col = pt.fixed_exp(np.abs(X).max(0), nt)
    eo = int(pt.fixed_exp(F32(1.0), nt))
    cb = base.codebooks.copy()
    assign = base.assignment.T.copy()  # [M][nt]
    active = np.ones(M, bool)
    updates = np.zeros(M, np.int64)
    last = np.zeros(M, np.int64)
    reseeds = 0
    Xm = [X[:, off:off + sz] for sz, off in zip(sizes, offsets)]
    xn = [_seq_dot(x, x) for x in Xm]
    rinv = [np.where(v > 0, F32(1) / np.where(v > 0, v, F32(1)), F32(0)).astype(F32) for v in xn]
    Qm = [pt.to_fixed(x, e_col[off:off + sz][None, :]) for x, sz, off in zip(Xm, sizes, offsets)]
    for r in range(iters):
        if not active.any():
            break
        for m in np.flatnonzero(active):
            sz, off = int(sizes[m]), int(offsets[m])
            p = pcm(threshold, sz)
            ocm = F32(1) / p
            a = assign[m]
            cnt = np.bincount(a, minlength=k)
            sums = np.zeros((k, sz), np.int64)
            np.add.at(sums, a, Qm[m])
            mean = pt.from_fixed(sums, e_col[off:off + sz][None, :], np.maximum(cnt, 1)[:, None])
            S = (_outer_sums(Xm[m], rinv[m], a, k, eo).astype(np.float64) * np.ldexp(1.0, -eo)).astype(F32)
            scale = (F32(1) - ocm) / np.maximum(cnt, 1).astype(F32)
            A = S * scale[:, None, None]
            idx = np.arange(sz)
            A[:, idx, idx] = A[:, idx, idx] + ocm
            new = solve_centroids(mean, A)
            for c in np.flatnonzero(cnt == 0):
                j = int(pt.counter_random(seed, int(m) | TAG_ARESEED, r, int(c))[0] % np.uint64(nt))
                new[c] = Xm[m][j]
                reseeds += 1
            cb[k * off:k * (off + sz)] = new.reshape(-1)
        for m in np.flatnonzero(active):
            sz, off = int(sizes[m]), int(offsets[m])
            C = cb[k * off:k * (off + sz)].reshape(k, sz)
            a = weighted_assign(Xm[m], C, xn[m], pcm(threshold, sz), assign[m])
            changed = int((a != assign[m]).sum())
            assign[m] = a
            updates[m] += 1
            last[m] = changed
            if changed <= 0.01 * nt:
                active[m] = False
    stats = dict(base.stats)
    stats.update(max_anisotropic_updates=int(updates.max()), changed_last_anisotropic=int(last.sum()), anisotropic_reseeds=reseeds)
    return pt.Trained(cb, base.centroid, stats, ords, assign.T.copy())


def encode_unweighted(rows, codebooks, M, k, centroid=None):
    """jv_pq_encode: per sub-space the first minimum of (c - x)^2 accumulated in order"""
    rows = np.asarray(rows, F32)
    x = rows - np.asarray(centroid, F32) if centroid is not None else rows
    sizes, offsets = pt.pq_layout(rows.shape[1], M)
    cb = np.asarray(codebooks, F32).reshape(-1)
    return np.stack([pt._nearest(x[:, off:off + sz], cb[k * off:k * (off + sz)].reshape(k, sz)) for sz, off in zip(sizes, offsets)],
                    axis=1).astype(np.uint8)


def residual_tables(x, codebooks, M, k):
    """(R, P) [M][n][k] and inv [n] of centred rows x [n][dim], in the device's operation order"""
    n, dim = x.shape
    sizes, offsets = pt.pq_layout(dim, M)
    cb = np.asarray(codebooks, F32).reshape(-1)
    vn = np.zeros(n, F32)
    for d in range(dim):
        vn = vn + x[:, d] * x[:, d]
    with np.errstate(divide="ignore"):
        inv = (1.0 / np.sqrt(vn.astype(np.float64))).astype(F32)
    R = np.empty((M, n, k), F32)
    P = np.empty((M, n, k), F32)
    for m, (sz, off) in enumerate(zip(sizes, offsets)):
        C = cb[k * off:k * (off + sz)].reshape(k, sz)
        xs = x[:, off:off + sz]
        cn = _seq_dot(C, C)
        xx = _seq_dot(xs, xs)[:, None]
        dot = np.zeros((n, k), F32)
        for t in range(sz):
            dot = dot + C[None, :, t] * xs[:, t, None]
        R[m] = (cn[None, :] - F32(2) * dot) + xx
        e = dot - xx
        with np.errstate(invalid="ignore"):
            P[m] = (e * e) * inv[:, None]
    return R, P, inv


def encode(rows, codebooks, M, k, threshold, centroid=None, sweeps=SWEEPS):
    """jv_pq_encode_*_anisotropic: (codes [n][M] uint8, stats {rows_moved, moves, max_sweeps}); threshold == -1 is jv_pq_encode.
    sweeps = 0 gives the minimum-residual start."""
    rows = np.asarray(rows, F32)
    if threshold == -1:
        return encode_unweighted(rows, codebooks, M, k, centroid), {"rows_moved": 0, "moves": 0, "max_sweeps": 0}
    n, dim = rows.shape
    x = rows - np.asarray(centroid, F32) if centroid is not None else rows
    p = pcm(threshold, dim)
    R, P, _ = residual_tables(x, codebooks, M, k)
    ar = np.arange(n)
    code = np.zeros((n, M), np.int64)
    S = np.zeros(n, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for m in range(M):
            Rv = np.where(R[m] < np.inf, R[m], np.inf)
            j = Rv.argmin(1)
            code[:, m] = np.where(Rv[ar, j] < np.inf, j, 0)
            S = S + P[m][ar, code[:, m]]
        active = np.ones(n, bool)
        moves = np.zeros(n, np.int64)
        swept = np.zeros(n, np.int64)
        cand = np.arange(k)[None, :]
        for _ in range(sweeps):
            if not active.any():
                break
            changed = np.zeros(n, bool)
            for m in range(M):
                old = code[:, m]
                Rold, Pold = R[m][ar, old], P[m][ar, old]
                Sn = (S - Pold)[:, None] + P[m]
                dP = Sn * Sn - (S * S)[:, None]
                cost = p * dP + ((R[m] - Rold[:, None]) - dP)
                ok = ~(dP > 0) & (cand != old[:, None]) & (cost < 0)
                cost = np.where(ok, cost, np.inf)
                j = cost.argmin(1)
                mv = active & (cost[ar, j] < 0)
                code[:, m] = np.where(mv, j, old)
                S = np.where(mv, Sn[ar, j], S)
                moves += mv
                changed |= mv
            swept += active
            active &= changed
    stats = {"rows_moved": int((moves > 0).sum()), "moves": int(moves.sum()), "max_sweeps": int(swept.max()) if n else 0}
    return code.astype(np.uint8), stats


def objective(rows, codebooks, M, k, threshold, codes, centroid=None):
    """(pcm - 1) S^2 + sum R of each row's codes, recomputed in float64"""
    rows = np.asarray(rows, np.float64)
    x = rows - np.asarray(centroid, np.float64) if centroid is not None else rows
    n, dim = x.shape
    sizes, offsets = pt.pq_layout(dim, M)
    cb = np.asarray(codebooks, np.float64).reshape(-1)
    inv = 1.0 / np.sqrt((x * x).sum(1))
    S = np.zeros(n)
    Rsum = np.zeros(n)
    for m, (sz, off) in enumerate(zip(sizes, offsets)):
        c = cb[k * off:k * (off + sz)].reshape(k, sz)[codes[:, m].astype(np.int64)]
        xs = x[:, off:off + sz]
        dot, xx = (c * xs).sum(1), (xs * xs).sum(1)
        Rsum += ((c - xs) ** 2).sum(1)
        S += (dot - xx) ** 2 * inv
    return (float(pcm(threshold, dim)) - 1) * S * S + Rsum
