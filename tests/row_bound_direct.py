"""numpy restatement of the point estimate of the low-rank edge bound (row_bound_lowrank.py), on which the edge tier of the
sketched fp32 DOT walk routes a likely list entrant straight to its full row (DESIGN §4.1):

    est = t fl(u . c)  (fp32),  score = fl((1 + est) / 2)

It leaves out every slack term of the bound, so it bounds the score in neither direction: only bytes depend on it, never results."""
import numpy as np

import row_bound_lowrank as rl


def point_estimate(q, B, codes, t):
    """t fl(u . c) of the raw dot product, rounded to fp32 as lowrank_bound rounds it. q: [d] (every row against it) or [m][d]
    (row i against query i), as in row_bound_lowrank.upper_bound_raw"""
    u = rl.prepare_query(q, B)[0]
    if u.shape[0] == 1:
        u = u[0]
    return (np.asarray(t, dtype=np.float32) * rl.code_dot_f32(u, codes)).astype(np.float32)
