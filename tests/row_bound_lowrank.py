"""numpy restatement of the low-rank edge bound: an upper bound of an fp32 DOT_PRODUCT score from k int8 codes of the row in a
d x k basis B plus four floats, small enough to store with the adjacency rows (DESIGN §4.1).

B is any fp32 d x k matrix, taken as exact reals; it only decides how tight the bound is. Per row x (build time, float64):

    a = B^T x,  t = max|a_j| / 127 (fp32),  c = round(a / t) (int8),  w = x - t B c (exact real),
    rho >= ||w||,  beta >= ||B^T w||,  xn >= ||x||

Per query q: u = fl(B^T q) (fp32, any order), eps_j >= |(B^T q)_j - u_j|, sigma >= ||q - B u||, nu >= ||u||. Exactly,

    q.x = t (u.c) + t (B^T q - u).c + (q - B u).w + u.(B^T w)
        <= t fl(u.c) + t (sum_j |c_j| (gk |u_j| + eps_j) + kdk) + sigma rho + nu beta

with gk = (k + 8) 2^-23 and kdk = (k + 512) 2^-149 bounding fl(u.c)'s rounding and underflow; the warp-order exact score adds at
most gamma(stride) ||q|| ||x|| + kd (row_bound_model). Float64 sums are bounded by (n + 8) 2^-53 of their absolute terms."""
import numpy as np

import row_bound_model as rb

LR_K = 32  # basis columns of the device's build (scorers.cuh)
TWO_M149 = rb.TWO_M149
PAD = 1.0 + 2.0 ** -40


def g64(n):
    """relative error bound of an n-term float64 sum of products (n multiplications and additions), generous"""
    return (n + 8) * 2.0 ** -53


def gk(k):
    return (k + 8) * 2.0 ** -23


def sample_rows(n, s):
    """the rows the basis is fitted on: min(n, s) rows, step max(1, n // s) apart (api.cu ensure_lowrank)"""
    return np.arange(min(n, s), dtype=np.int64) * max(1, n // s)


def orthonormalise(y):
    """modified Gram-Schmidt over the columns of y [d][k] in float64 (a column that vanishes becomes 0)"""
    v = np.array(y, dtype=np.float64)
    for j in range(v.shape[1]):
        for i in range(j):
            v[:, j] -= (v[:, i] @ v[:, j]) * v[:, i]
        nj = np.linalg.norm(v[:, j])
        v[:, j] = v[:, j] / nj if nj > 0 else 0.0
    return v


def basis(xs, k, iters=4):
    """subspace iteration over the sampled rows xs [s][d]: V <- orth(xs^T (xs V)), started from the first k sampled rows; fp32 d x k"""
    xs = np.asarray(xs, dtype=np.float64)
    v = orthonormalise(xs[:k].T)
    for _ in range(iters):
        v = orthonormalise(xs.T @ (xs @ v))
    return v.astype(np.float32)


def encode_rows(x, B):
    """x [n][d] fp32, B [d][k] fp32 -> (codes [n][k] int8, t, rho, beta, xn [n] fp32)"""
    x64 = np.asarray(x, dtype=np.float32).astype(np.float64)
    B64 = np.asarray(B, dtype=np.float32).astype(np.float64)
    d, k = B64.shape
    a = x64 @ B64
    t = (np.abs(a).max(axis=1) / 127.0).astype(np.float32)
    safe = np.where(t > 0, t, np.float32(1)).astype(np.float64)
    c = np.clip(np.rint(a / safe[:, None]), -127, 127)
    c[t == 0] = 0
    tb = t.astype(np.float64)[:, None]
    w = x64 - tb * (c @ B64.T)
    A = np.abs(x64) + tb * (np.abs(c) @ np.abs(B64).T)  # what each w_i's float64 sum is made of
    rho = rb.round_up_f32((np.linalg.norm(w, axis=1) + g64(k + 2) * np.linalg.norm(A, axis=1)) * PAD)
    # |(B^T w)_j| <= |fl(B^T w~)_j| + g (|B|^T (|w~| + A))_j: the float64 error of w~ and of the product
    bw = np.abs(w @ B64) + g64(d + k + 2) * ((np.abs(w) + A) @ np.abs(B64))
    beta = rb.round_up_f32(np.linalg.norm(bw, axis=1) * PAD)
    xn = rb.round_up_f32(np.linalg.norm(x64, axis=1) * PAD)
    return c.astype(np.int8), t, rho, beta, xn


def prepare_query(q, B):
    """q [d] or [m][d] fp32 -> (u [.., k] fp32, e [.., k] float64 = gk |u| + eps rounded up to fp32, sigma, nu)"""
    q = np.atleast_2d(np.asarray(q, dtype=np.float32))
    B = np.asarray(B, dtype=np.float32)
    d, k = B.shape
    u = np.zeros((q.shape[0], k), dtype=np.float32)
    for i in range(d):  # fp32, sequential: any order is covered by eps
        u = (u + q[:, i:i + 1] * B[i][None, :]).astype(np.float32)
    q64, B64, u64 = q.astype(np.float64), B.astype(np.float64), u.astype(np.float64)
    eps = rb.gamma(d) * (np.abs(q64) @ np.abs(B64)) + (d + 512) * TWO_M149
    e = rb.round_up_f32((gk(k) * np.abs(u64) + eps) * PAD).astype(np.float64)
    r = q64 - u64 @ B64.T
    A = np.abs(q64) + np.abs(u64) @ np.abs(B64).T
    sigma = rb.round_up_f32((np.linalg.norm(r, axis=1) + g64(k + 2) * np.linalg.norm(A, axis=1)) * PAD).astype(np.float64)
    nu = rb.round_up_f32(np.linalg.norm(u64, axis=1) * PAD).astype(np.float64)
    return u, e, sigma, nu


def code_dot_f32(u, c):
    """fl(u . c) summed sequentially in float32 (the bound covers any order). u [k] or [m][k], c [m][k]"""
    u = np.asarray(u, dtype=np.float32)
    c = np.asarray(c).astype(np.float32)
    s = np.zeros(c.shape[0], dtype=np.float32)
    for j in range(c.shape[1]):
        s = (s + u[..., j] * c[:, j]).astype(np.float32)
    return s


def upper_bound_raw(q, B, codes, t, rho, beta, xn, stride):
    """upper bound of the kernel's fp32 dot product q . x for every encoded row, as float64. q: [d] (every row against it) or
    [m][d] (row i against query i)"""
    u, e, sigma, nu = prepare_query(q, B)
    q = np.atleast_2d(np.asarray(q, dtype=np.float32))
    if q.shape[0] == 1:
        u, e, sigma, nu = u[0], e[0], sigma[0], nu[0]
    k = np.asarray(B).shape[1]
    s = code_dot_f32(u, codes).astype(np.float64)
    E = (np.abs(codes.astype(np.float64)) * e).sum(axis=-1) * PAD + (k + 512) * TWO_M149
    tb = t.astype(np.float64)
    qn = rb.query_norm_up(q, stride) if q.shape[0] > 1 else rb.query_norm_up(q[0], stride)
    kd = (stride + 512) * TWO_M149
    rest = tb * E + sigma * rho.astype(np.float64) + nu * beta.astype(np.float64) + rb.gamma(stride) * qn * xn.astype(np.float64) + kd
    return tb * s + rest + (np.abs(tb * s) + rest) * 2.0 ** -40
