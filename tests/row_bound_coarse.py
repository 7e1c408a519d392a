"""numpy restatement of a coarse tier of the fp32 row sketch, on top of row_bound_model.py's int8 sketch: what
tools/row_bound_stats.py replays to measure how many drops a bound from the codes' high nibbles alone would settle (DESIGN §4.1).

Every int8 code c splits exactly into h = c >> 4 (arithmetic, in [-8, 7]) and l = c & 15, c = 16 h + l. The coarse code of c is
c1 = 16 h + 8 (in [-120, 120], |c - c1| <= 8), x_hat1 = s c1, and the coarse radius is

    r1 = ||x - x_hat1|| + gamma (||x|| + ||x_hat1||)      over all sketch_stride positions,

x zero padded: a padding code is 0, so its coarse code is 8 and it adds (8 s)^2 to both squared norms. The query is 0 there, so that
only makes r1 larger than it needs to be. The argument of the int8 bound only uses that the codes are integers within 127, so the
coarse bound is row_bound_model's with x_hat1 and r1 in place of x_hat and r:

    fl(q . x) <= s fl(q . c1) + ||q|| r1 + kd (1 + s)."""
import numpy as np

import row_bound_model as rb


def sketch_stride(stride):
    return (stride + 7) & ~7


def coarse_codes(c):
    """c1 = 16 (c >> 4) + 8 for int8 codes c (any shape), as int8"""
    return (16 * (np.asarray(c, dtype=np.int16) >> 4) + 8).astype(np.int8)


def pad(a, width):
    """a [n][k] zero padded on the right to [n][width]"""
    a = np.asarray(a)
    out = np.zeros(a.shape[:-1] + (width,), dtype=a.dtype)
    out[..., :a.shape[-1]] = a
    return out


def encode_coarse(x, stride=None):
    """x: [n][dim] float32 -> (c1 [n][sketch_stride] int8, scale [n] float32, r1 [n] float32); scale is encode_int8's"""
    x = np.asarray(x, dtype=np.float32)
    stride = stride or ((x.shape[1] + 3) & ~3)
    ss = sketch_stride(stride)
    c, s, _ = rb.encode_int8(x, stride)
    c1 = coarse_codes(pad(c, ss))
    xh1 = c1.astype(np.float64) * s.astype(np.float64)[:, None]
    return c1, s, rb.radius(pad(x, ss), xh1, stride)


def upper_bound_raw(q, c1, scale, r1, stride):
    """upper bound of the kernel's fp32 dot product q . x from the coarse codes, as float64. q: [dim] or [n][dim]"""
    return rb.upper_bound_raw(pad(np.asarray(q, dtype=np.float32), c1.shape[1]), c1, scale, r1, stride)
