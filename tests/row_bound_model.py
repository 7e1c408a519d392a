"""numpy restatement of the row sketch that lets the fp32 DOT_PRODUCT walk drop a hopeless neighbour on an upper bound of its score
instead of reading its full row (row_sketch_kernel in kernels_batch.cu, the bound in graph_search_kernel, DESIGN §4.1).

int8 sketch (the shipped format): per row a scale s = max|x| / 127 and codes round(x / s) (fp32 division, ties to even), x_hat = s c,
and a radius r = ||x - x_hat|| + gamma (||x|| + ||x_hat||), gamma = (stride + 8) 2^-23, rounded up to fp32. For any summation order
of the fp32 dot products fl(q . x) and s_c = fl(q . c):

    fl(q . x) <= s s_c + ||q|| r + kd (1 + s),   kd = (stride + 512) 2^-149 (what underflow can add to either sum)

fp16 sketch (measured by tools/row_bound_stats.py, not shipped): a power of two 2^e with max|x| 2^-e in [2^14, 2^15), the values
x 2^-e rounded to fp16, the same radius and bound with 2^e in place of s."""
import numpy as np

TWO_M149 = 2.0 ** -149


def gamma(stride):
    return (stride + 8) * 2.0 ** -23


def round_up_f32(v):
    """the smallest float32 >= v (v float64)"""
    v = np.asarray(v, dtype=np.float64)
    f = v.astype(np.float32)
    low = f.astype(np.float64) < v
    f[low] = np.nextafter(f[low], np.float32(np.inf))
    return f


def sketch_exponent(x):
    """per row e with max|x| 2^-e in [2^14, 2^15), clamped to [-126, 113] so that 2^e is a normal float32 (0 for a zero row)"""
    m = np.abs(x).max(axis=1).astype(np.float64)
    _, E = np.frexp(m)
    e = np.where(m > 0, E - 15, 0)
    return np.clip(e, -126, 113).astype(np.int32)


def radius(x, xh, stride):
    """||x - x_hat|| + gamma (||x|| + ||x_hat||) in float64, padded by 2^-40 relative for float64's own rounding, rounded up"""
    x = x.astype(np.float64)
    r = np.linalg.norm(x - xh, axis=1) + gamma(stride) * (np.linalg.norm(x, axis=1) + np.linalg.norm(xh, axis=1))
    return round_up_f32(r * (1.0 + 2.0 ** -40))


def encode_fp16(x, stride=None):
    """x: [n][dim] float32 -> (y [n][dim] float16, scale [n] float32 = 2^e, radius [n] float32)"""
    x = np.asarray(x, dtype=np.float32)
    stride = stride or ((x.shape[1] + 3) & ~3)
    e = sketch_exponent(x)
    y = np.ldexp(x.astype(np.float64), -e[:, None]).astype(np.float16)
    xh = np.ldexp(y.astype(np.float64), e[:, None])
    return y, np.ldexp(np.float32(1.0), e).astype(np.float32), radius(x, xh, stride)


def encode_int8(x, stride=None):
    """x: [n][dim] float32 -> (codes [n][dim] int8, scale [n] float32, radius [n] float32)"""
    x = np.asarray(x, dtype=np.float32)
    stride = stride or ((x.shape[1] + 3) & ~3)
    s = (np.abs(x).max(axis=1) / np.float32(127)).astype(np.float32)
    safe = np.where(s > 0, s, np.float32(1))
    with np.errstate(over="ignore"):
        c = np.clip(np.rint(x / safe[:, None]), -127, 127).astype(np.int8)
    c[s == 0] = 0
    xh = c.astype(np.float64) * s.astype(np.float64)[:, None]
    return c, s, radius(x, xh, stride)


def query_norm_up(q, stride):
    """an upper bound of ||q|| from the float64 norm (the kernel bounds its own fp32 sum of squares the same way). q: [dim] or [n][dim]"""
    q = np.asarray(q, dtype=np.float64)
    n2 = (q * q).sum(axis=-1)
    return round_up_f32(np.sqrt((n2 + (stride + 512) * TWO_M149) * (1.0 + 2.0 * gamma(stride))) * (1.0 + 2.0 ** -40)).astype(np.float64)


def sketch_dot_f32(q, y):
    """fl(q . y) summed sequentially in float32 (any order satisfies the bound; this is one of them). y: [n][dim], q: [dim] or [n][dim]"""
    q = np.asarray(q, dtype=np.float32)
    y = np.asarray(y).astype(np.float32)
    s = np.zeros(y.shape[0], dtype=np.float32)
    for i in range(y.shape[1]):
        s = (s + q[..., i] * y[:, i]).astype(np.float32)  # separate multiply and add: two roundings, within the same gamma
    return s


def upper_bound_raw(q, y, scale, rad, stride):
    """upper bound of the kernel's fp32 dot product q . x for every sketched row, as float64 (>= any fp32 rounding of it)"""
    s = sketch_dot_f32(q, y).astype(np.float64)
    sc = scale.astype(np.float64)
    kd = (stride + 512) * TWO_M149
    ub = s * sc + query_norm_up(q, stride) * rad.astype(np.float64) + kd * (1.0 + sc)
    return ub + np.abs(ub) * 2.0 ** -40


def dot_score_up(raw):
    """DOT_PRODUCT score map (1 + raw) / 2 of an upper bound, rounded up to float32"""
    return round_up_f32((1.0 + np.asarray(raw, dtype=np.float64)) / 2.0)


def sortable(f):
    """NumericUtils.floatToSortableInt as int64"""
    b = np.asarray(f, dtype=np.float32).view(np.int32).astype(np.int64)
    return np.where(b < 0, b ^ 0x7fffffff, b)


def topk_key(score, node):
    """(sortable(score) << 32) | ~node as Python ints compared like the device's signed 64-bit keys"""
    return (sortable(score) << 32) | (~np.asarray(node, dtype=np.int64) & 0xffffffff)
