"""The device graph build checked batch by batch, row for row, against its host restatement (tests/graph_model.py).

CPU: the restatement reproduces the reference's testDiversity lists; the pair bound of delete_model.pair_bound holds for a numpy
emulation of the Gram product's arithmetic, and the untranslated L2 Gram form breaks it on rows that share a large offset.
GPU (-m gpu): jv_builder_* driven the way parallel.sharded_build drives it; after every batch the inserted rows, the overflow
count and the re-pruned rows equal the model's (except rows the model flags as near ties), then the mirror adopts the device's
rows; at the end the adjacency, the dropped back-links, the truncated searches and the upper levels equal the model's."""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import delete_model as dm
import graph_model as gm
import oracle_lib as o

METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)


# ------------------------------------------------------------------------------------------------ CPU
def test_model_reproduces_golden_diversity_lists(oracle):
    # tests:graph/TestVectorGraph.java:457-525 testDiversity (M = 4, beamWidth 10, overflow 1.0, alpha 1.0, unit-circle vectors):
    # one node per batch and no window are the reference's sequential inserts
    ang = np.array([0.5, 0.75, 0.2, 0.9, 0.8, 0.77, 0.6]) * np.pi
    vec = np.ascontiguousarray(np.stack([np.cos(ang), np.sin(ang)], 1), dtype=np.float32)
    expected = {3: {0: [1, 2], 1: [0], 2: [0]},
                4: {0: [1, 2], 1: [0, 3], 2: [0], 3: [1]},
                5: {0: [1, 2], 1: [0, 3, 4], 2: [0], 3: [1, 4], 4: [1, 3]},
                6: {0: [1, 2], 1: [0, 3, 4, 5], 2: [0], 3: [1, 4], 4: [1, 3, 5], 5: [1, 4]}}
    for n, want in expected.items():
        m = gm.BuildModel(gm.F32Scores(oracle, vec[:n], o.DOT_PRODUCT), 4, 10, overflow=1.0, alpha=1.0, window=0)
        assert m.next_batch() == (1, 1)  # below 32 inserted nodes every batch holds one
        adj, flagged = m.build()
        assert flagged == 0
        for node, nbrs in want.items():
            assert sorted(int(x) for x in adj[node] if x >= 0) == nbrs, (n, node, adj[node].tolist())


def test_window_candidates():
    # prune_candidate: W = 4 around u = 10 in batch [8, 13): 8, 9, 11, 12 (u skipped); clipped at the batch's ends
    assert gm.window_candidates(10, 4, 8, 5) == [8, 9, 11, 12]
    assert gm.window_candidates(8, 4, 8, 5) == [9, 10]
    assert gm.window_candidates(9, 3, 8, 5) == [8, 10, 11]
    assert gm.window_candidates(5, 0, 0, 10) == []
    assert gm.default_window(100) == 28 and gm.default_window(30) == 32 and gm.default_window(200) == 0


def test_assign_levels_distribution():
    members, entry = gm.assign_levels(20000, 16, 7)
    assert len(members) >= 2 and entry in set(members[-1].tolist())
    assert abs(len(members[0]) / 20000 - 1 / 16) < 0.01  # P(level >= 1) = 1 / M
    for a, b in zip(members, members[1:]):
        assert set(b.tolist()) <= set(a.tolist())


def _tf32(x):
    return (np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xffffe000)).view(np.float32)


def gram_emulation(rows):
    """prune_gram_tc_kernel's Gram product in numpy: x = hi + lo (hi = x truncated to tf32, lo exact), the tensor cores read lo
    truncated to tf32 as well; hi hi + hi lo + lo hi accumulated in fp32, one rounding per add, over k in order"""
    X = np.asarray(rows, np.float32)
    hi = _tf32(X)
    lo = _tf32((X - hi).astype(np.float32))
    acc = np.zeros((len(X), len(X)), np.float32)
    for k in range(X.shape[1]):
        for a, b in ((hi, hi), (hi, lo), (lo, hi)):
            acc = (acc + np.outer(a[:, k], b[:, k]).astype(np.float32)).astype(np.float32)
    return acc


def emulated_pair_scores(metric, G):
    d = np.diag(G)
    if metric == o.EUCLIDEAN:
        raw = np.maximum(np.float32(0), (d[:, None] + d[None, :]).astype(np.float32) - np.float32(2) * G).astype(np.float32)
        return (np.float32(1) / (np.float32(1) + raw)).astype(np.float32)
    if metric == o.DOT_PRODUCT:
        return ((np.float32(1) + G) / np.float32(2)).astype(np.float32)
    cos = (G / np.sqrt((d[:, None] * d[None, :]).astype(np.float32))).astype(np.float32)
    return ((np.float32(1) + cos) / np.float32(2)).astype(np.float32)


def _worlds(rng, n=129, dim=128):
    unit = o.random_unit_vectors(rng, n, dim)
    return {"unit": unit,
            "sift": np.floor(rng.random((n, dim)) * 128).astype(np.float32),
            "offset10": (10 + 0.1 * unit).astype(np.float32),
            "offset100": (100 + 0.1 * unit).astype(np.float32)}


@pytest.mark.parametrize("metric", METRICS)
def test_pair_bound_holds_for_gram_emulation(metric):
    # 128 candidates x 128 dims; row 0 is the pruned node. L2 stages x_c - x_v (build.cu gram_row), DOT / COSINE x_c itself.
    rng = np.random.default_rng(5 + metric)
    for name, rows in _worlds(rng).items():
        xv, X = rows[0], rows[1:]
        staged = (X - xv).astype(np.float32) if metric == o.EUCLIDEAN else X
        got = emulated_pair_scores(metric, gram_emulation(staged)).astype(np.float64)
        X64, xv64 = X.astype(np.float64), xv.astype(np.float64)
        exact = dm._pairs(metric, X64, xv64)
        bound = dm.pair_bound(metric, X64, xv64, X.shape[1])
        err = np.abs(got - exact)
        assert (err <= bound).all(), (name, float((err / bound).max()))


def test_untranslated_gram_form_breaks_the_bound_on_offset_rows():
    # G_ii + G_jj - 2 G_ij over the rows themselves: its error scales with |x|^2, not with the neighbourhood. Unit and SIFT rows stay
    # inside the bound; 100 + 0.1 N(0, 1) rows do not, by orders of magnitude (distances of ~0.02 against |x|^2 ~ 1.3e6)
    rng = np.random.default_rng(5)
    worst = {}
    for name, rows in _worlds(rng).items():
        xv, X = rows[0], rows[1:]
        got = emulated_pair_scores(o.EUCLIDEAN, gram_emulation(X)).astype(np.float64)
        X64, xv64 = X.astype(np.float64), xv.astype(np.float64)
        worst[name] = float((np.abs(got - dm._pairs(o.EUCLIDEAN, X64, xv64)) / dm.pair_bound(o.EUCLIDEAN, X64, xv64, X.shape[1])).max())
    assert worst["unit"] <= 1 and worst["sift"] <= 1, worst
    assert worst["offset100"] > 100, worst


def test_builder_stats_without_device():
    from jvector_b200 import _native as nat
    lib = nat.load()
    if lib.jv_gpu_device_count() > 0:
        pytest.skip("a GPU is present")
    n = C.c_int64(7)
    assert lib.jv_builder_stats(None, C.byref(n), None, None) == -1 and n.value == 7


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


def latent_rows(rng, n, dim, latent=16, noise=0.35):
    A = rng.standard_normal((latent, dim)).astype(np.float32) / np.sqrt(latent)
    x = rng.standard_normal((n, latent)).astype(np.float32) @ A + noise * rng.standard_normal((n, dim)).astype(np.float32)
    return np.ascontiguousarray(x / np.linalg.norm(x, axis=1, keepdims=True), dtype=np.float32)


def world(name, sift=None):
    rng = np.random.default_rng(sum(map(ord, name)))
    kind, dim, n = name.split(":")
    dim, n = int(dim), int(n)
    if kind == "sift":
        return np.ascontiguousarray(sift[0][:n])
    if kind == "hubs":  # 8 tight clusters: every batch sends the nodes near a cluster's middle more back-links than a row holds
        c = rng.standard_normal((8, dim)).astype(np.float32)
        return np.ascontiguousarray(c[rng.integers(0, 8, n)] + 0.1 * rng.standard_normal((n, dim)), dtype=np.float32)
    x = latent_rows(rng, n, dim)
    if kind == "dup":  # the last 1 % of the rows repeat earlier ones exactly
        x[n - n // 100:] = x[rng.integers(0, n // 2, n // 100)]
    if kind == "offset":
        x = np.ascontiguousarray(100 + 0.1 * x, dtype=np.float32)
    return x


# (id, world kind:dim:n, metric, M, beam, window, alpha, overflow, max_batch, hierarchy). The prune tiers each case reaches, mode 0
# by beam + window, mode 1 by row_cap = max(2 M, (int)(overflow M) + 1):
CASES = [
    ("tc64_dot", "latent:64:3000", o.DOT_PRODUCT, 16, 30, 0, 1.2, 1.2, 0, False),          # 0: tc<64>       1: 32 tc<64>
    ("tc128_cos_d100", "latent:100:3000", o.COSINE, 16, 100, -1, 1.4, 1.2, 0, True),       # 0: 128 tc<128>  1: 32 tc<64>
    ("k256_l2_d33", "latent:33:2500", o.EUCLIDEAN, 16, 200, -1, 1.0, 1.0, 0, False),       # 0: 200 <256>    1: 32 tc<64>
    ("k256_win60_dot_b64", "latent:64:3000", o.DOT_PRODUCT, 32, 100, 60, 1.2, 1.2, 64, False),  # 0: 160 <256>  1: 64 tc<64>
    ("rowcap128_l2_d7", "latent:7:2000", o.EUCLIDEAN, 64, 100, -1, 1.2, 1.2, 0, False),    # 0: tc<128>      1: 128 tc<128>
    ("rowcap16_cos_d768", "latent:768:2000", o.COSINE, 8, 60, -1, 1.2, 1.0, 0, False),     # 0: 92 tc<128>   1: 16 tc<64>
    ("dup_dot", "dup:64:3000", o.DOT_PRODUCT, 16, 100, -1, 1.2, 1.2, 64, False),
    ("offset_l2", "offset:64:3000", o.EUCLIDEAN, 16, 100, -1, 1.2, 1.2, 0, False),
    ("drops_l2", "hubs:16:4000", o.EUCLIDEAN, 4, 60, -1, 1.2, 1.0, 0, False),              # M = 4, row_cap 8: hubs drop back-links
    ("siftsmall_c1", "sift:128:10000", o.EUCLIDEAN, 16, 100, -1, 1.2, 1.2, 0, True),        # the c1 graph, integer rows and ties
]
# the CUDA-core Gram kernel (JV_PRUNE_GRAM=ffma, read once per process) over the Gram-tier cases that matter most
FFMA_CASES = ("tc64_dot", "tc128_cos_d100", "offset_l2")


def run_case(jv, oracle, sift, case):
    import builder_driver as bd
    from jvector_b200 import _native as nat
    cid, wname, metric, M, beam, window, alpha, overflow, max_batch, hier = case
    data = world(wname, sift)
    vec = jv.F32Vectors(data)
    params = nat.BuildParams(M, beam, overflow, alpha, int(hier), 3, max_batch, window)
    gi, tally, batches, dropped, (upper_checked, upper_flagged) = bd.drive_build(nat.init(), vec, metric, params,
                                                                                 lambda: gm.F32Scores(oracle, data, metric), cid)
    gi.close()
    vec.close()
    return tally, dropped, batches, upper_checked, upper_flagged


def _budget(case, kind):
    """flagged rows allowed: 1 % of the re-pruned rows, 2 % of the inserted ones (a prune over a whole beam makes several hundred
    isDiverse tests), 3 % past the 128-candidate tier. The proven pair bound grows with the depth of the dot product, so at
    stride 768 it is ten times the stride-64 one and flags proportionally more rows"""
    cid, wname, _, _, beam, window, *_ = case
    w = gm.default_window(beam) if window < 0 else window
    frac = (0.03 if beam + w > 128 else 0.02) if kind == "insert" else 0.01
    if wname.startswith("dup"):
        # a node whose exact duplicate d is selected first meets sim(c, d) = score(c) for every other candidate c: an exact tie at
        # alpha 1.0 that fp32 rounding decides, flagged on the rows of the duplicated nodes and their neighbours
        frac = 0.04
    return frac * (8 if int(wname.split(":")[1]) > 256 else 1)


def check_case(jv, oracle, sift, case):
    t0 = time.time()
    tally, dropped, batches, up_ok, up_flag = run_case(jv, oracle, sift, case)
    print("%s: %.1f s, %d batches, dropped back-links %d, insert rows/flagged/differ %s, re-pruned %s, upper levels checked %d "
          "(skipped for a near tie: %d)" % (case[0], time.time() - t0, batches, dropped, tally["insert"], tally["reprune"], up_ok, up_flag))
    for kind, (rows, flagged, differ) in tally.items():
        assert flagged <= _budget(case, kind) * max(rows, 1), (case[0], kind, rows, flagged)
        # the exact ties of duplicated rows do go either way; elsewhere nearly every flagged row comes out equal anyway
        assert differ <= (0.04 if case[1].startswith("dup") else 0.01) * max(rows, 1), (case[0], kind, rows, differ)
    if case[0] == "drops_l2":
        assert dropped > 0, "the hub case drops no back-link"
    return dropped


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_device_build_equals_model(jv, oracle, sift, case):
    check_case(jv, oracle, sift, case)


@pytest.mark.gpu
def test_device_build_equals_model_ffma_gram():
    # the CUDA-core Gram kernel: a child process, since the kernel choice is read once per process
    env = dict(os.environ, JV_PRUNE_GRAM="ffma")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-s", "-p", "no:cacheprovider", "-m", "gpu",
                        "-k", "test_device_build_equals_model and (%s)" % " or ".join(FFMA_CASES)],
                       env=env, capture_output=True, text=True, timeout=230)
    assert r.returncode == 0 and "%d passed" % len(FFMA_CASES) in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


@pytest.mark.gpu
def test_window_past_the_prune_capacity_is_rejected(jv):
    rng = np.random.default_rng(1)
    vec = jv.F32Vectors(latent_rows(rng, 300, 16))
    with pytest.raises(jv.JVectorB200Error) as e:
        jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=200, concurrent_window=57).build(vec)
    assert e.value.code == -2
    g = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=200, concurrent_window=56).build(vec)  # exactly 256 candidates
    g.close()
    vec.close()
