"""Host-side helpers of bench.py (no GPU): deterministic data generation, recall metric, peak lookup."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_gen_unit_rows_deterministic_and_unit_norm():
    import torch

    import bench
    gen = lambda seed, dist, chunk=128: bench.gen_unit_rows_device(torch, seed, 300, 64, dist, chunk=chunk, device="cpu").numpy()
    a, b = gen(123, "latent"), gen(123, "latent")
    assert np.array_equal(a, b) and a.dtype == np.float32 and a.shape == (300, 64)
    np.testing.assert_allclose(np.linalg.norm(a, axis=1), 1.0, rtol=1e-5)
    assert not np.array_equal(a, gen(124, "latent"))
    iid = gen(123, "iid")
    # the latent model has neighbourhood structure: pairwise similarities spread far wider than for i.i.d. rows
    assert (a @ a.T)[np.triu_indices(300, 1)].std() > 1.4 * (iid @ iid.T)[np.triu_indices(300, 1)].std()


def test_recall_at_k_matches_accuracy_metrics_semantics():
    import bench
    # jvector-examples/.../util/AccuracyMetrics.java:38-50: |top-k found ∩ top-k truth| / (queries * k)
    found = np.array([[1, 2, 3, -1], [9, 8, 7, 6]])
    truth = np.array([[3, 2, 5, 6], [6, 7, 8, 9]])
    assert bench.recall_at_k(found, truth, 4) == (2 + 4) / 8.0
    assert bench.recall_at_k(found, truth, 2) == (1 + 0) / 4.0


def test_measured_peaks():
    import bench
    peak, src = bench.measured_peaks()
    assert peak > 1000
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        assert peak == float(json.load(open(p))["hbm_gbs"]) and src.startswith("measured")
    else:
        assert peak == bench.HBM_PEAK_GBS == 3350.0 and "not measured" in src
