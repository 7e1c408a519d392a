"""The coarse tier of the int8 row sketch that tools/row_bound_stats.py measures (numpy restatement in row_bound_coarse.py): the
high nibble of every int8 code, c1 = 16 (c >> 4) + 8, and the coarse radius r1. The split is exact, and the coarse bound is >= the
kernel's own score (the warp-order oracle) on adversarial rows, so the catch rate the tool reports for it is one a device bound of
the same form could reach without changing a result."""
import numpy as np
import pytest

import oracle_lib as o
import row_bound_coarse as rbc
import row_bound_model as rb
from oracle_lib import fp
from test_row_bound import adversarial_rows, queries_for

DOT = o.DOT_PRODUCT
# strides 4, 8, 100 and 1020 end in 4 padding codes (8 m + 4), 768 and 1024 in none
DIMS = (1, 4, 5, 100, 101, 768, 1017, 1024)


def test_codes_split_into_nibbles():
    c = np.arange(-127, 128)
    h, lo = c >> 4, c & 15
    assert (16 * h + lo == c).all() and h.min() == -8 and h.max() == 7
    c1 = rbc.coarse_codes(c.astype(np.int8)).astype(np.int64)
    assert (c1 == 16 * h + 8).all() and np.abs(c - c1).max() <= 8 and np.abs(c1).max() == 120


def subnormal_rows(rng, dim):
    """fp32-subnormal rows: a subnormal scale, and a scale that rounds to 0 with nonzero values"""
    sign = rng.choice([-1.0, 1.0], (24, dim))
    return np.concatenate([sign[:16] * rng.uniform(0.5e-40, 2e-40, (16, dim)), sign[16:] * rng.integers(1, 60, (8, dim)) * 2.0 ** -149]).astype(np.float32)


@pytest.mark.parametrize("dim", DIMS)
def test_coarse_bound_is_at_least_the_warp_order_score(oracle, dim):
    rng = np.random.default_rng(50 + dim)
    stride = (dim + 3) & ~3
    for qi, q in enumerate(queries_for(rng, dim)):
        rows = np.ascontiguousarray(np.concatenate([adversarial_rows(rng, dim, q), subnormal_rows(rng, dim)]))
        c1, scale, r1 = rbc.encode_coarse(rows, stride)
        assert (r1 >= 0).all() and np.isfinite(r1).all()
        assert (c1[:, dim:] == 8).all()
        ub = rb.dot_score_up(rbc.upper_bound_raw(q, c1, scale, r1, stride))
        exact = np.array([oracle.jvo_compare_f32_warp(DOT, fp(q), fp(r), dim) for r in rows], np.float32)
        ok = np.isnan(exact) | (rb.sortable(ub) >= rb.sortable(exact))
        assert ok.all(), (dim, qi, np.flatnonzero(~ok)[:5], ub[~ok][:5], exact[~ok][:5])
        ids = np.arange(len(rows))
        assert (rb.topk_key(ub, ids) >= rb.topk_key(np.where(np.isnan(exact), ub, exact), ids)).all()
