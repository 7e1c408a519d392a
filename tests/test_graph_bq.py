"""The graph build over BQ codes and its maintenance (jv_graph_build_bq, jv_builder_create_bq, jv_graph_add_nodes_bq,
jv_builder_create_from_graph_bq, jv_graph_remove_deleted_bq: BuildScoreProvider.bqBuildScoreProvider).

CPU: the model's pair scores are jvo_bq_score and 1 - popcount / dim in numpy (dim 100 has padding); on the lossless world (rows
+-1 / sqrt(dim), where DOT_PRODUCT's (1 + dot) / 2 is exactly 1 - hd / dim) the BQ model and the fp32 DOT model build the same graph.
GPU (-m gpu): on the lossless world jv_graph_build_bq gives the bytes of jv_graph_build(DOT_PRODUCT) at every metric, with no
truncated insert search; the step-wise builder equals the model after every batch at dim 100 and 1536; the one-call, step-wise and
sharded builds agree; an add into a one-node graph is the build; adds and removals equal the models row for row, with marked nodes,
holes, and on every removal tier; the metric changes no byte; recall against the fp32 graph; every error code."""
import ctypes as C

import numpy as np
import pytest

import add_model as am
import bq_build_model as qm
import build_model as bm
import oracle_lib as o
from oracle_lib import fp

METRICS = (o.EUCLIDEAN, o.DOT_PRODUCT, o.COSINE)


def lossless_world(rng, n, dim):
    """rows +-1 / sqrt(dim) (dim a power of 4: every product is +-1 / dim, every partial sum exact in fp32 and in 3xTF32) and their
    BQ words. The signs are those of latent rows: near neighbours are then closer than random signs would be, and fewer nodes tie at
    a beam's last score, so that neither walk has to cut a tie tail short"""
    from test_build_steps import latent_rows
    signs = np.where(latent_rows(rng, n, dim, latent=48, noise=0.2) > 0, 1, -1)
    rows = (signs / np.sqrt(dim)).astype(np.float32)
    words = np.zeros((n, (dim + 63) // 64), np.uint64)
    for j in range(dim):
        words[:, j >> 6] |= (signs[:, j] > 0).astype(np.uint64) << np.uint64(j & 63)
    return rows, words


def encode(rows):
    """BinaryQuantization.encode on the host (jvo_bq_encode's rule): bit j of word i = (v[64 i + j] > 0)"""
    n, dim = rows.shape
    words = np.zeros((n, (dim + 63) // 64), np.uint64)
    for j in range(dim):
        words[:, j >> 6] |= (rows[:, j] > 0).astype(np.uint64) << np.uint64(j & 63)
    return words


def latent_world(name, n, dim):
    from test_build_steps import latent_rows
    rows = latent_rows(np.random.default_rng(sum(map(ord, name))), n, dim)
    return rows, encode(rows)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("dim", (64, 100, 1536))
def test_model_pair_scores_are_hamming_scores(oracle, dim):
    rng = np.random.default_rng(dim)
    _, words = latent_world("pairs%d" % dim, 40, dim)
    got = qm.pair_scores(words, dim, np.arange(40), np.arange(40))
    W = words.shape[1]
    hd = np.array([[sum(bin(int(a) ^ int(b)).count("1") for a, b in zip(words[i], words[j])) for j in range(40)] for i in range(40)])
    assert np.array_equal(got, (np.float32(1) - hd.astype(np.float32) / np.float32(dim)).astype(np.float32))
    for i in range(40):
        for j in range(40):
            want = oracle.jvo_bq_score(qm.wp(words[i]), qm.wp(words[j]), W, dim)
            assert np.float32(want).view(np.int32) == got[i, j].view(np.int32), (i, j)
    # the insert query decodes to exactly c_v, padding clear
    back = np.zeros_like(words)
    q = qm.decode(words, dim)
    for v in range(len(words)):
        oracle.jvo_bq_encode(fp(q[v]), dim, qm.wp(back[v]))
    assert np.array_equal(back, words) and set(np.unique(q)) == {-1.0, 1.0}
    del rng


@pytest.mark.parametrize("dim", (64, 256, 1024))
def test_lossless_world_bq_model_equals_fp32_dot_model(oracle, dim):
    rng = np.random.default_rng(dim + 1)
    n = 300
    rows, words = lossless_world(rng, n, dim)
    kw = dict(M=8, beam=40, max_batch=0, window=-1)
    bq = qm.BQBuildModel(oracle, words, dim, o.DOT_PRODUCT, **kw)
    f32 = bm.BuildModel(oracle, rows, o.DOT_PRODUCT, **kw)
    # in lock step, both adopting the BQ model's rows: no row may differ
    while (nb := bq.next_batch()) is not None:
        assert nb == f32.next_batch()
        got, gdeg, _ = bq.insert_rows(*nb)
        want, wdeg, _ = f32.insert_rows(*nb)
        assert np.array_equal(got, want) and np.array_equal(gdeg, wdeg), nb
        lst = bq.apply_new(*nb, got, gdeg)
        assert f32.apply_new(*nb, got, gdeg) == lst
        got, gdeg, _ = bq.reprune_rows(lst)
        want, wdeg, _ = f32.reprune_rows(lst)
        assert np.array_equal(got, want) and np.array_equal(gdeg, wdeg)
        bq.apply_repruned(lst, got, gdeg)
        f32.apply_repruned(lst, got, gdeg)
    lst = bq.over_degree()
    assert lst == f32.over_degree()
    got, gdeg, _ = bq.reprune_rows(lst)
    want, wdeg, _ = f32.reprune_rows(lst)
    assert np.array_equal(got, want) and np.array_equal(gdeg, wdeg)


def test_repair_tiers_of_the_model():
    assert [qm.repair_tier(c) for c in (1, 64, 65, 128, 256, 257, 1024, 1025, 2048, 2049, 4224)] == [0, 0, 1, 1, 2, 3, 3, 4, 4, 5, 5]


def test_bq_graph_entry_points_without_device():
    from jvector_b200 import _native as nat
    lib = nat.load()
    if lib.jv_gpu_device_count() > 0:
        pytest.skip("a GPU is present")
    params = nat.BuildParams(16, 60, 1.2, 1.2, 0, 0, 0, -1)
    out, ms, st = C.c_void_p(1234), C.c_double(7.0), nat.RemoveStats()
    bits = np.zeros(4, np.uint32)
    assert lib.jv_graph_build_bq(None, 1, C.byref(params), C.byref(out), C.byref(ms)) == -1
    assert lib.jv_builder_create_bq(None, 1, C.byref(params), None, C.byref(out)) == -1
    assert lib.jv_graph_add_nodes_bq(None, None, 1, C.byref(params), None, C.byref(out), C.byref(ms)) == -1
    assert lib.jv_builder_create_from_graph_bq(None, None, 1, C.byref(params), None, None, C.byref(out)) == -1
    assert lib.jv_graph_remove_deleted_bq(None, None, 1, 1.2, 0, bits.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(out), C.byref(st)) == -1
    assert out.value == 1234 and ms.value == 7.0


CPP_BQ = r"""
#include <cstdio>
#include <vector>
#include "jvector_b200.hpp"
int main()
{
    try {
        jv::init(0);
    } catch (const jv::Error &e) {
        std::printf("NO_DEVICE_OK\n");
        return 0;
    }
    const int n0 = 200, n = 300, dim = 100, W = 2;
    std::vector<uint64_t> words((size_t)n * W);
    uint64_t s = 88172645463325252ull;
    for (auto &w : words) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; w = s; }
    for (int i = 0; i < n; i++) words[(size_t)i * W + 1] &= (1ull << 36) - 1;  // no bit past dim 100
    jv::BQVectors small(words.data(), n0, dim), all(words.data(), n, dim);
    jv::GraphIndexBuilder b(jv::VectorSimilarityFunction::COSINE, 8, 30, 1.2f, 1.2f, false);
    jv::GraphIndex g = b.build(small);
    jv::GraphIndex grown = b.addGraphNodes(g, all);
    std::vector<uint32_t> del((n + 31) / 32, 0u);
    del[0] = 0x10u;
    jv::GraphIndex r = b.removeDeletedNodes(grown, all, del);
    if (g.size() != n0 || grown.size() != n || r.size() != n || b.removeStats.removed != 1) return 1;
    std::printf("BQ_OK\n");
    return 0;
}
"""


def _cpp_bq(tmp):
    import subprocess

    from jvector_b200 import _native as nat
    src, exe = tmp / "bq_mirror.cpp", tmp / "bq_mirror"
    src.write_text(CPP_BQ)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", str(o.ROOT) + "/include", str(src), "-o", str(exe), nat.SO,
                           "-Wl,-rpath," + __import__("os").path.dirname(nat.SO), "-lpthread", "-ldl"])
    return subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)


def test_cpp_bq_overloads_compile_and_fail_loudly_without_gpu(tmp_path):
    from jvector_b200 import _native as nat
    out = _cpp_bq(tmp_path)
    if nat.load().jv_gpu_device_count() > 0:
        pytest.skip("a GPU is present: covered by the gpu test")
    assert out.returncode == 0 and "NO_DEVICE_OK" in out.stdout, out.stdout + out.stderr


@pytest.mark.gpu
def test_cpp_bq_overloads_on_gpu(tmp_path):
    out = _cpp_bq(tmp_path)
    assert out.returncode == 0 and "BQ_OK" in out.stdout, out.stdout + out.stderr


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _bptr(bits):
    return bits.ctypes.data_as(C.POINTER(C.c_uint32)) if bits is not None else None


def _levels(gi):
    return [gi.level(lv) for lv in range(gi.info()["levels"])]


def assert_same_graph(a, b, what):
    ia, ib = a.info(), b.info()
    assert ia == ib, (what, ia, ib)
    for lv, ((ids_a, adj_a), (ids_b, adj_b)) in enumerate(zip(_levels(a), _levels(b))):
        assert np.array_equal(ids_a, ids_b) and np.array_equal(adj_a, adj_b), (what, "level", lv)


def _builder(jv, metric, M, beam=60, hier=False, seed=3, **kw):
    return jv.GraphIndexBuilder(metric, M=M, beamWidth=beam, neighborOverflow=1.2, alpha=1.2, addHierarchy=hier, seed=seed, **kw)


def drive(jv, lib, b, model, cid):
    """a created builder driven batch by batch against `model` (a BQBuildModel or SeededBQBuildModel in the builder's state): every
    batch's inserted rows, overflow list and re-pruned rows equal the model's. Returns (GraphIndex, (batches, truncated, dropped))."""
    import torch

    from jvector_b200 import _native as nat
    deg_, cap_, mb_ = C.c_int(), C.c_int(), C.c_int()
    nat.check(lib.jv_builder_info(b, C.byref(deg_), C.byref(cap_), C.byref(mb_)))
    assert (deg_.value, cap_.value) == (model.degree, model.row_cap)
    rows_t = torch.empty((mb_.value, model.degree), dtype=torch.int32, device="cuda")
    rdeg_t = torch.empty(mb_.value, dtype=torch.int32, device="cuda")

    def reprune_round(L, lst, what):
        assert L == len(lst), (what, "rows to re-prune", L, len(lst))
        if L == 0:
            return
        rp = torch.empty((L, model.row_cap), dtype=torch.int32, device="cuda")
        rpd = torch.empty(L, dtype=torch.int32, device="cuda")
        nat.check(lib.jv_builder_reprune_slice(b, 0, L, _ptr(rp), _ptr(rpd)))
        got, gdeg = rp.cpu().numpy(), rpd.cpu().numpy()
        want, wdeg, _ = model.reprune_rows(lst)
        bad = np.flatnonzero((got != want).any(1) | (gdeg != wdeg))
        assert len(bad) == 0, (what, "re-pruned rows differ", [lst[i] for i in bad[:5]], got[bad[:1]].tolist(), want[bad[:1]].tolist())
        model.apply_repruned(lst, got, gdeg)
        nat.check(lib.jv_builder_apply_repruned(b, L, _ptr(rp), _ptr(rpd)))

    first, count, L = C.c_int32(), C.c_int32(), C.c_int32()
    batches = 0
    try:
        while True:
            nat.check(lib.jv_builder_next_batch(b, C.byref(first), C.byref(count)))
            f, c = first.value, count.value
            if c == 0:
                assert model.next_batch() is None
                break
            assert (f, c) == model.next_batch()
            for lo, hi in ([(0, c // 2), (c // 2, c)] if batches % 2 else [(0, c)]):
                nat.check(lib.jv_builder_insert_slice(b, f, c, lo, hi, _ptr(rows_t), _ptr(rdeg_t)))
            got, gdeg = rows_t[:c].cpu().numpy(), rdeg_t[:c].cpu().numpy()
            want, wdeg, _ = model.insert_rows(f, c)
            bad = np.flatnonzero((got != want).any(1) | (gdeg != wdeg))
            assert len(bad) == 0, (cid, "batch", batches, "rows differ", (f + bad[:5]).tolist(), got[bad[:1]].tolist(), want[bad[:1]].tolist())
            nat.check(lib.jv_builder_apply_new(b, f, c, _ptr(rows_t), _ptr(rdeg_t), C.byref(L)))
            reprune_round(L.value, model.apply_new(f, c, got, gdeg), (cid, "batch", batches))
            batches += 1
        nat.check(lib.jv_builder_collect_over_degree(b, C.byref(L)))
        reprune_round(L.value, model.over_degree(), (cid, "cleanup"))
        s = [C.c_int64() for _ in range(3)]
        nat.check(lib.jv_builder_stats(b, *[C.byref(x) for x in s]))
        h = C.c_void_p()
        nat.check(lib.jv_builder_finish(b, C.byref(h), None))
    finally:
        lib.jv_builder_free(b)
    gi = jv.GraphIndex(_handle=h)
    stats = tuple(x.value for x in s)
    assert stats == (batches, 0, model.dropped), (cid, stats, model.dropped)
    assert np.array_equal(gi.level(0)[1], model.compact()), (cid, "finished adjacency")
    return gi, stats


def step_build(jv, vectors, metric, params, bq):
    """jv_builder_create(_bq) + jv_builder_* the way sharded_build drives them on one GPU: (GraphIndex, (batches, truncated, dropped))"""
    import torch

    from jvector_b200 import _native as nat
    lib = nat.init()
    st = torch.cuda.current_stream().cuda_stream
    b = C.c_void_p()
    nat.check((lib.jv_builder_create_bq if bq else lib.jv_builder_create)(vectors._h, metric, C.byref(params), C.c_void_p(st), C.byref(b)))
    try:
        deg_, cap_, mb_ = C.c_int(), C.c_int(), C.c_int()
        nat.check(lib.jv_builder_info(b, C.byref(deg_), C.byref(cap_), C.byref(mb_)))
        rows = torch.empty((mb_.value, deg_.value), dtype=torch.int32, device="cuda")
        rdeg = torch.empty(mb_.value, dtype=torch.int32, device="cuda")
        first, count, L = C.c_int32(), C.c_int32(), C.c_int32()

        def reprune(L):
            if L:
                rp = torch.empty((L, cap_.value), dtype=torch.int32, device="cuda")
                rpd = torch.empty(L, dtype=torch.int32, device="cuda")
                nat.check(lib.jv_builder_reprune_slice(b, 0, L, _ptr(rp), _ptr(rpd)))
                nat.check(lib.jv_builder_apply_repruned(b, L, _ptr(rp), _ptr(rpd)))

        while True:
            nat.check(lib.jv_builder_next_batch(b, C.byref(first), C.byref(count)))
            if count.value == 0:
                break
            nat.check(lib.jv_builder_insert_slice(b, first.value, count.value, 0, count.value, _ptr(rows), _ptr(rdeg)))
            nat.check(lib.jv_builder_apply_new(b, first.value, count.value, _ptr(rows), _ptr(rdeg), C.byref(L)))
            reprune(L.value)
        nat.check(lib.jv_builder_collect_over_degree(b, C.byref(L)))
        reprune(L.value)
        s = [C.c_int64() for _ in range(3)]
        nat.check(lib.jv_builder_stats(b, *[C.byref(x) for x in s]))
        g = C.c_void_p()
        nat.check(lib.jv_builder_finish(b, C.byref(g), None))
    finally:
        lib.jv_builder_free(b)
    return jv.GraphIndex(_handle=g), tuple(x.value for x in s)


# (dim, n, degree, beam, hierarchy, max_batch, window). At 64 dimensions there are 65 scores: beam 16 over 1000 rows keeps the nodes
# tied at a beam's last score within the fp32 walk's tie tail (rerankK + 28 entries)
LOSSLESS = [(64, 1000, 8, 16, True, 0, -1), (256, 3000, 16, 60, False, 64, 60), (1024, 4000, 16, 100, True, 0, -1)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", LOSSLESS, ids=("d64_hier", "d256_b64_w60", "d1024_hier"))
def test_lossless_world_byte_equal_to_fp32_dot_build(jv, case):
    from jvector_b200 import _native as nat
    dim, n, M, beam, hier, max_batch, window = case
    rng = np.random.default_rng(7 + dim)
    rows, words = lossless_world(rng, n, dim)
    assert np.array_equal(jv.bq_encode_all(rows), words)
    params = nat.BuildParams(M, beam, 1.2, 1.2, int(hier), 5, max_batch, window)
    bqv, f32 = jv.BQVectors(words, dim), jv.F32Vectors(rows)
    g_f32, s_f32 = step_build(jv, f32, o.DOT_PRODUCT, params, False)
    assert s_f32[1] == 0, s_f32
    for metric in METRICS:
        g_bq, s_bq = step_build(jv, bqv, metric, params, True)
        assert s_bq == s_f32, (metric, s_bq, s_f32)
        assert_same_graph(g_bq, g_f32, ("lossless step-wise", metric))
        one = _builder(jv, metric, M, beam=beam, hier=hier, seed=5, max_batch=max_batch, concurrent_window=window).build(bqv)
        assert_same_graph(one, g_f32, ("lossless one call", metric))
        g_bq.close(), one.close()
    g_f32.close(), bqv.close(), f32.close()


# (id, dim, metric, degree, beam, window, max_batch, hierarchy, n)
MODEL_CASES = [
    ("d100_l2_hier", 100, o.EUCLIDEAN, 16, 60, -1, 0, True, 2000),
    ("d100_dot_b64_w60", 100, o.DOT_PRODUCT, 16, 100, 60, 64, False, 2000),
    ("d1536_cos", 1536, o.COSINE, 16, 60, -1, 0, True, 1200),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", MODEL_CASES, ids=[c[0] for c in MODEL_CASES])
def test_device_bq_build_equals_model(jv, oracle, case):
    import torch

    from jvector_b200 import _native as nat
    cid, dim, metric, M, beam, window, max_batch, hier, n = case
    _, words = latent_world(cid, n, dim)
    lib = nat.init()
    bqv = jv.BQVectors(words, dim)
    seed = 3
    params = nat.BuildParams(M, beam, 1.2, 1.2, int(hier), seed, max_batch, window)
    kw = dict(M=M, beam=beam, overflow=1.2, alpha=1.2, max_batch=max_batch, window=window)
    b = C.c_void_p()
    nat.check(lib.jv_builder_create_bq(bqv._h, metric, C.byref(params), C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(b)))
    gi, stats = drive(jv, lib, b, qm.BQBuildModel(oracle, words, dim, metric, **kw), cid)
    assert stats[1] == 0
    if hier:
        members, entry = bm.assign_levels(n, M, seed)
        inf = gi.info()
        assert inf["entry_node"] == entry and inf["levels"] == 1 + len(members), (cid, inf, entry)
        for lv, (ids, want_adj) in enumerate(qm.upper_levels(oracle, words, dim, metric, members, **kw), 1):
            gids, gadj = gi.level(lv)
            assert np.array_equal(gids, ids) and np.array_equal(gadj, want_adj), (cid, "level", lv)
    one = _builder(jv, metric, M, beam=beam, hier=hier, seed=seed, max_batch=max_batch, concurrent_window=window).build(bqv)
    assert_same_graph(one, gi, (cid, "one call vs step-wise"))
    for h in (gi, one, bqv):
        h.close()


@pytest.mark.gpu
def test_bq_builds_reproduce_and_ignore_the_metric(jv):
    from jvector_b200 import _native as nat
    from jvector_b200 import parallel
    _, words = latent_world("repro", 6000, 100)
    bqv = jv.BQVectors(words, 100)
    b = _builder(jv, o.DOT_PRODUCT, 16, beam=80, hier=True, seed=9)
    one, two = b.build(bqv), b.build(bqv)
    assert b.batches > 0 and b.scored_vectors > 0
    assert_same_graph(one, two, "two calls")
    steps, stats = step_build(jv, bqv, o.DOT_PRODUCT, nat.BuildParams(16, 80, 1.2, 1.2, 1, 9, 0, -1), True)
    assert stats[0] == b.batches and stats[2] == b.dropped_backlinks
    assert_same_graph(one, steps, "one call vs step-wise")
    sharded, _, _ = parallel.sharded_build(None, bqv, o.DOT_PRODUCT, M=16, beamWidth=80, addHierarchy=True, seed=9)
    assert_same_graph(one, sharded, "sharded_build")
    for metric in (o.EUCLIDEAN, o.COSINE):
        other = _builder(jv, metric, 16, beam=80, hier=True, seed=9).build(bqv)
        assert_same_graph(one, other, ("metric", metric))
        other.close()
    for g in (one, two, steps, sharded, bqv):
        g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("hier", (False, True), ids=("flat", "hier"))
def test_add_to_one_node_graph_is_the_bq_build(jv, hier):
    n, dim, M = 3000, 100, 16
    _, words = latent_world("anchor", n, dim)
    bqv = jv.BQVectors(words, dim)
    seed = next(s for s in range(1, 400) if am.level_draws(n, M, s)[0] >= 1) if hier else 3
    b = _builder(jv, o.COSINE, M, hier=hier, seed=seed)
    built = b.build(bqv)
    want = (b.batches, b.dropped_backlinks)
    empty = np.full((1, M), -1, np.int32)
    tops = int(am.level_draws(n, M, seed)[0]) if hier else 0
    one = jv.GraphIndex(empty, 0, [(np.zeros(1, np.int32), empty)] * tops)
    added = b.addGraphNodes(one, bqv)
    assert (b.batches, b.dropped_backlinks) == want
    assert_same_graph(added, built, ("one-node add", hier))
    assert built.info()["levels"] > 1 or not hier
    for h in (built, one, added, bqv):
        h.close()


def drive_add(jv, oracle, bqv, words, dim, g, metric, M, beam, marks, cid):
    """the add of word rows [n0, n) to g, step by step against SeededBQBuildModel, then its upper levels and entry; the one-call add
    gives the same bytes, at every metric"""
    import torch

    from jvector_b200 import _native as nat
    seed = 3
    lib = nat.init()
    n, n0 = words.shape[0], g.info()["n"]
    entry0, levels0 = g.info()["entry_node"], _levels(g)
    params = nat.BuildParams(M, beam, 1.2, 1.2, 0, seed, 0, -1)
    from jvector_b200.api import pack_accept_bits
    bits = None if marks is None else pack_accept_bits(marks)
    b = C.c_void_p()
    nat.check(lib.jv_builder_create_from_graph_bq(g._h, bqv._h, metric, C.byref(params), _bptr(bits), C.c_void_p(torch.cuda.current_stream().cuda_stream),
                                                  C.byref(b)))
    kw = dict(M=M, beam=beam, overflow=1.2, alpha=1.2, max_batch=0, window=-1)
    accept = None if marks is None else np.concatenate([~marks, np.ones(n - n0, bool)])
    model = qm.SeededBQBuildModel(oracle, words, dim, metric, levels0[0][1], entry0, accept, **kw)
    gi, _ = drive(jv, lib, b, model, cid)
    inf = gi.info()
    if len(levels0) > 1:
        want_levels, want_entry = qm.extend_levels(oracle, words, dim, metric, levels0[1:], entry0, n0, seed, marks, **kw)
        assert inf["entry_node"] == want_entry and inf["levels"] == 1 + len(want_levels), (cid, inf, want_entry, len(want_levels))
        for lv, (ids, want_adj) in enumerate(want_levels, 1):
            gids, gadj = gi.level(lv)
            assert np.array_equal(gids, ids) and np.array_equal(gadj, want_adj), (cid, "level", lv)
    else:
        assert inf["levels"] == 1 and inf["entry_node"] == model.entry, (cid, inf, model.entry)
    ms = C.c_double()
    for m in METRICS:
        h1 = C.c_void_p()
        nat.check(lib.jv_graph_add_nodes_bq(g._h, bqv._h, m, C.byref(params), _bptr(bits), C.byref(h1), C.byref(ms)))
        one = jv.GraphIndex(_handle=h1)
        assert_same_graph(gi, one, (cid, "step-wise vs one call", m))
        one.close()
    if marks is not None:
        marked = np.concatenate([marks, np.zeros(n - n0, bool)])
        for lv, (ids, ladj) in enumerate(_levels(gi)):
            new_rows = ladj[ids >= n0]
            assert not marked[new_rows[new_rows >= 0]].any(), (cid, "a new row names a marked node on level", lv)
    return gi


# (id, dim, metric, degree, beam, hierarchy, n0, n, origin of the graph)
ADD_CASES = [
    ("d100_l2_hier", 100, o.EUCLIDEAN, 16, 60, True, 1500, 1800, "built"),
    ("d100_dot_marked", 100, o.DOT_PRODUCT, 16, 60, True, 1600, 1800, "marked"),
    ("d1536_cos_removed", 1536, o.COSINE, 16, 60, True, 1000, 1200, "removed"),
    ("d100_l2_all_removed", 100, o.EUCLIDEAN, 16, 60, False, 600, 1000, "all_removed"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ADD_CASES, ids=[c[0] for c in ADD_CASES])
def test_stepwise_bq_add_equals_model(jv, oracle, case):
    cid, dim, metric, M, beam, hier, n0, n, origin = case
    rng = np.random.default_rng(sum(map(ord, cid)))
    _, words = latent_world(cid, n, dim)
    small, bqv = jv.BQVectors(words[:n0], dim), jv.BQVectors(words, dim)
    b = _builder(jv, metric, M, beam=beam, hier=hier)
    g = b.build(small)
    marks = None
    if origin == "marked":
        marks = rng.random(n0) < 0.05
    elif origin == "removed":
        g = b.removeDeletedNodes(g, small, rng.random(n0) < 0.1)
    elif origin == "all_removed":
        g = b.removeDeletedNodes(g, small, np.ones(n0, bool))
        assert g.info()["entry_node"] == -1
    before = _levels(g)
    gi = drive_add(jv, oracle, bqv, words, dim, g, metric, M, beam, marks, cid)
    if origin == "all_removed":
        assert gi.info()["entry_node"] == n0
    after = _levels(g)
    assert len(before) == len(after) and all(np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1]) for a, c in zip(before, after))
    for h in (g, gi, small, bqv):
        h.close()


def assert_removal_matches_model(gi, res, what):
    inf = gi.info()
    assert inf["entry_node"] == res["entry"] and inf["levels"] == res["levels"], (what, inf, res["entry"], res["levels"])
    want = [(np.arange(res["adj0"].shape[0], dtype=np.int32), res["adj0"])] + list(res["upper"])
    for L, ((dids, dadj), (wids, wadj)) in enumerate(zip(_levels(gi), want)):
        assert np.array_equal(dids, wids), (what, "members of level", L)
        bad = np.flatnonzero((dadj != wadj).any(1))
        assert len(bad) == 0, (what, "level", L, "rows differ", wids[bad[:5]].tolist(), dadj[bad[:1]].tolist(), wadj[bad[:1]].tolist())
    cands = [len(r["cands"] - {v}) for lv in res["rows"] for v, r in lv.items()]
    st = gi.remove_stats
    assert st["repaired_rows"] == len(cands) and st["candidates"] == sum(cands) and st["max_candidates"] == max(cands, default=0), (what, st)
    assert st["random_fallbacks"] == sum(r["fallback"] for lv in res["rows"] for r in lv.values()), (what, st)
    assert st["live_nodes"] == (~res["dead"]).sum()
    return np.bincount([qm.repair_tier(c) for c in cands], minlength=len(qm.REPAIR_TIERS))


# (id, dim, metric, degree, hierarchy, n, deleted fraction, entry deleted)
REMOVE_CASES = [
    ("light_d100_dot", 100, o.DOT_PRODUCT, 16, True, 2000, 0.02, False),
    ("heavy_d100_l2", 100, o.EUCLIDEAN, 16, True, 2000, 0.45, True),
    ("heavy_d1536_cos", 1536, o.COSINE, 32, False, 1500, 0.4, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", REMOVE_CASES, ids=[c[0] for c in REMOVE_CASES])
def test_bq_removal_equals_model(jv, oracle, case):
    cid, dim, metric, M, hier, n, frac, kill_entry = case
    rng = np.random.default_rng(sum(map(ord, cid)))
    _, words = latent_world(cid, n, dim)
    bqv = jv.BQVectors(words, dim)
    b = _builder(jv, metric, M, hier=hier, seed=17)
    g = b.build(bqv)
    levels, entry = _levels(g), g.info()["entry_node"]
    deleted = rng.random(n) < frac
    deleted[entry] = kill_entry
    got = b.removeDeletedNodes(g, bqv, deleted)
    for m in METRICS:  # the same bytes at every metric, and from a second call
        again = _builder(jv, m, M, hier=hier, seed=17).removeDeletedNodes(g, bqv, deleted)
        assert_same_graph(got, again, (cid, "metric", m))
        again.close()
    res = qm.BQRepairModel(oracle, words, dim, metric, M).remove_deleted(levels[0][1], entry, levels[1:], deleted, seed=17)
    hit = assert_removal_matches_model(got, res, cid)
    print(cid, "rows per tier", hit.tolist(), got.remove_stats)
    assert got.remove_stats["removed"] == deleted.sum() and (not kill_entry or got.info()["entry_node"] != entry)
    for h in (g, got, bqv):
        h.close()


@pytest.mark.gpu
def test_bq_removal_hits_every_tier_on_a_made_graph(jv, oracle):
    # test_graph_maintain_pq's hand-made degree-64 graph over BQ words: hubs that lose 64, 24, 8 or 3 neighbours naming 64 nodes each
    # gather about 2400, 1200, 450 and 180 candidates (the 8192, 2048, 1024 and 256 tiers), ordinary rows 15 or about 70
    rng = np.random.default_rng(64)
    n, dim, M = 4000, 100, 64
    _, words = latent_world("made", n, dim)
    bqv = jv.BQVectors(words, dim)
    adj = np.full((n, M), -1, np.int32)

    def pick(v, cnt, pool):
        return rng.choice(np.setdiff1d(pool, [v]), cnt, replace=False)

    everyone = np.arange(n)
    for v in range(n):
        adj[v, :8] = pick(v, 8, everyone)
    hubs = {10: 64, 11: 64, 20: 24, 21: 24, 30: 8, 31: 8, 40: 3}
    deleted = np.zeros(n, bool)
    pool = np.arange(100, n)
    for hub, cnt in hubs.items():
        lost = pick(hub, cnt, pool[~deleted[pool]])
        adj[hub] = -1
        adj[hub, :cnt] = lost
        deleted[lost] = True
        for j in lost:
            adj[j] = pick(j, M, pool)
    deleted[rng.choice(np.flatnonzero(~deleted[100:]) + 100, 60, replace=False)] = True
    g = jv.GraphIndex(adj, 0)
    got = _builder(jv, o.EUCLIDEAN, M, seed=5).removeDeletedNodes(g, bqv, deleted)
    res = qm.BQRepairModel(oracle, words, dim, o.EUCLIDEAN, M).remove_deleted(adj, 0, [], deleted, seed=5)
    hit = assert_removal_matches_model(got, res, "made graph")
    print("made graph: rows per tier", hit.tolist(), got.remove_stats)
    assert (hit > 0).all() and got.remove_stats["max_candidates"] > 2048, hit.tolist()
    for h in (g, got, bqv):
        h.close()


@pytest.mark.gpu
def test_bq_remove_add_remove_keeps_holes_and_equals_models(jv, oracle):
    rng = np.random.default_rng(21)
    n0, n, dim, M = 1600, 1800, 100, 16
    _, words = latent_world("holes", n, dim)
    small, bqv = jv.BQVectors(words[:n0], dim), jv.BQVectors(words, dim)
    b = _builder(jv, o.DOT_PRODUCT, M, hier=True, seed=4)
    g = b.build(small)
    first = rng.random(n0) < 0.1
    rep = b.removeDeletedNodes(g, small, first)
    lv = _levels(g)
    res = qm.BQRepairModel(oracle, words[:n0], dim, o.DOT_PRODUCT, M).remove_deleted(lv[0][1], g.info()["entry_node"], lv[1:], first, seed=4)
    assert_removal_matches_model(rep, res, "first removal")
    grown = b.addGraphNodes(rep, bqv)
    wide = np.concatenate([first, np.zeros(n - n0, bool)])
    assert grown.info()["n"] == n and not np.isin(grown.level(0)[1], np.flatnonzero(first)).any()
    second = (rng.random(n) < 0.05) & ~wide
    again = b.removeDeletedNodes(grown, bqv, second | wide)
    lv = _levels(grown)
    res = qm.BQRepairModel(oracle, words, dim, o.DOT_PRODUCT, M).remove_deleted(lv[0][1], grown.info()["entry_node"], lv[1:], second | wide,
                                                                               seed=4, holes=wide)
    assert_removal_matches_model(again, res, "second removal")
    assert again.remove_stats["removed"] == second.sum(), (again.remove_stats, second.sum())
    assert again.remove_stats["live_nodes"] == n - first.sum() - second.sum()
    for h in (g, rep, grown, again, small, bqv):
        h.close()


def _recall(nodes, truth):
    return float(np.mean([len(set(nodes[i].tolist()) & set(truth[i].tolist())) / truth.shape[1] for i in range(len(nodes))]))


# How far the BQ-built graph's recall@10 may fall below the fp32-built graph's on the same world, under the same walk. Derived on a
# CPU from the host models' flat graphs over this test's world (BQBuildModel against BuildModel(DOT_PRODUCT), the 10 000 x 64 latent
# rows and 1000 queries below, M = 16, beam 100; the oracle's walks; truth by numpy in float64): under the fp32 walk 0.9695 against
# 0.9987, under the BQ walk + fp32 rerank at rerankK 100 0.7395 against 0.7565, a loss of at most 0.029. The device builds add a
# hierarchy, the fp32 one may differ from its model on near-tie rows, and the device's brute force may order near ties differently:
# the margin is that loss plus 0.016.
RECALL_MARGIN = 0.045


@pytest.mark.gpu
def test_bq_graph_recall_near_fp32_graph(jv):
    from test_build_steps import latent_rows
    rng = np.random.default_rng(21)
    dim, n = 64, 10000
    data = latent_rows(rng, n + 1000, dim)
    base, queries = np.ascontiguousarray(data[:n]), np.ascontiguousarray(data[n:])
    f32 = jv.F32Vectors(base)
    bqv = jv.BQVectors(jv.bq_encode_all(base), dim)
    vsf = o.DOT_PRODUCT
    truth, _, _ = jv.topk_bruteforce(f32, vsf, queries, 10)
    recall = {}
    for name, vec in (("fp32", f32), ("bq", bqv)):
        g = _builder(jv, vsf, 16, beam=100, hier=True, seed=9).build(vec)
        s = jv.GraphSearcher(g)
        recall[(name, "f32_walk")] = _recall(s.search(f32, queries, vsf, 10, 100).nodes, truth)
        recall[(name, "bq_walk")] = _recall(s.search(bqv, queries, vsf, 10, 100, reranker=f32).nodes, truth)
        g.close()
    print("recall@10", recall)
    for shape in ("f32_walk", "bq_walk"):
        assert recall[("bq", shape)] >= recall[("fp32", shape)] - RECALL_MARGIN, recall
    f32.close(), bqv.close()


@pytest.mark.gpu
def test_bq_graph_errors(jv):
    from jvector_b200 import _native as nat
    lib = nat.init()
    rng = np.random.default_rng(2)
    rows = rng.standard_normal((300, 100)).astype(np.float32)
    words = encode(rows)
    bqv, short, f32 = jv.BQVectors(words, 100), jv.BQVectors(words[:100], 100), jv.F32Vectors(rows)
    padded = words.copy()
    padded[123, 1] |= np.uint64(1) << np.uint64(40)  # bit 104 of a 100-dimensional row
    bad = jv.BQVectors(padded, 100)
    g = jv.GraphIndex(np.full((200, 8), -1, np.int32), 0)
    full = jv.GraphIndex(np.full((300, 8), -1, np.int32), 0)
    params = nat.BuildParams(8, 30, 1.2, 1.2, 0, 0, 0, -1)
    out, ms, st = C.c_void_p(), C.c_double(), nat.RemoveStats()
    none = np.zeros(10, np.uint32)

    def build(ds, metric=1, p=params, o_=C.byref(out)):
        a = lib.jv_graph_build_bq(ds, metric, C.byref(p) if p is not None else None, o_, C.byref(ms))
        c = lib.jv_builder_create_bq(ds, metric, C.byref(p) if p is not None else None, None, o_)
        assert a == c, (a, c)
        return a

    def add(graph, ds, metric=1, p=params, o_=C.byref(out)):
        a = lib.jv_graph_add_nodes_bq(graph, ds, metric, C.byref(p) if p is not None else None, None, o_, C.byref(ms))
        c = lib.jv_builder_create_from_graph_bq(graph, ds, metric, C.byref(p) if p is not None else None, None, None, o_)
        assert a == c, (a, c)
        return a

    def remove(graph, ds, metric=1, alpha=1.2, bits=none, o_=C.byref(out), st_=C.byref(st)):
        return lib.jv_graph_remove_deleted_bq(graph, ds, metric, alpha, 0, _bptr(bits), o_, st_)

    launches = lib.jv_kernel_launch_count()
    assert build(None) == -2 and build(bqv._h, p=None) == -2 and build(bqv._h, o_=None) == -2
    assert build(f32._h) == -2 and build(bqv._h, metric=7) == -2
    assert build(bqv._h, p=nat.BuildParams(8, 30, 1.2, 0.9, 0, 0, 0, -1)) == -2
    assert build(bqv._h, p=nat.BuildParams(65, 30, 1.2, 1.2, 0, 0, 0, -1)) == -5
    assert add(None, bqv._h) == -2 and add(g._h, None) == -2 and add(g._h, bqv._h, p=None) == -2 and add(g._h, bqv._h, o_=None) == -2
    assert add(g._h, f32._h) == -2  # not BQ
    assert add(g._h, short._h) == -2  # n < n0
    assert add(g._h, bqv._h, metric=7) == -2
    assert add(g._h, bqv._h, p=nat.BuildParams(16, 30, 1.2, 1.2, 0, 0, 0, -1)) == -2  # degree mismatch
    assert remove(None, bqv._h) == -2 and remove(full._h, None) == -2 and remove(full._h, bqv._h, bits=None) == -2
    assert remove(full._h, bqv._h, o_=None) == -2 and remove(full._h, bqv._h, st_=None) == -2
    assert remove(full._h, f32._h) == -2  # not BQ
    assert remove(g._h, bqv._h) == -2  # n != g.n
    assert remove(full._h, bqv._h, metric=7) == -2 and remove(full._h, bqv._h, alpha=0.9) == -2
    wide, wide_full = jv.GraphIndex(np.full((200, 65), -1, np.int32), 0), jv.GraphIndex(np.full((300, 65), -1, np.int32), 0)
    assert add(wide._h, bqv._h, p=nat.BuildParams(65, 30, 1.2, 1.2, 0, 0, 0, -1)) == -5
    assert remove(wide_full._h, bqv._h) == -5
    assert lib.jv_kernel_launch_count() == launches and out.value is None  # refused before any device work
    # a bit past dim: refused after the one padding reduction, before any other device work
    assert build(bad._h) == -2 and add(g._h, bad._h) == -2 and remove(full._h, bad._h) == -2
    assert lib.jv_kernel_launch_count() - launches == 5 and out.value is None  # build and add ran two calls each
    # the fp32 and PQ entry points still refuse a BQ data set
    assert lib.jv_graph_build(bqv._h, 1, C.byref(params), C.byref(out), C.byref(ms)) == -2
    assert lib.jv_builder_create(bqv._h, 1, C.byref(params), None, C.byref(out)) == -2
    assert lib.jv_graph_build_pq(bqv._h, 1, C.byref(params), C.byref(out), C.byref(ms)) == -2
    assert lib.jv_builder_create_pq(bqv._h, 1, C.byref(params), None, C.byref(out)) == -2
    assert lib.jv_graph_add_nodes(g._h, bqv._h, 1, C.byref(params), None, C.byref(out), C.byref(ms)) == -2
    assert lib.jv_builder_create_from_graph(g._h, bqv._h, 1, C.byref(params), None, None, C.byref(out)) == -2
    assert lib.jv_graph_remove_deleted(full._h, bqv._h, 1, 1.2, 0, _bptr(none), C.byref(out), C.byref(st)) == -2
    assert lib.jv_graph_add_nodes_pq(g._h, bqv._h, 1, C.byref(params), None, C.byref(out), C.byref(ms)) == -2
    assert lib.jv_builder_create_from_graph_pq(g._h, bqv._h, 1, C.byref(params), None, None, C.byref(out)) == -2
    assert lib.jv_graph_remove_deleted_pq(full._h, bqv._h, 1, 1.2, 0, _bptr(none), C.byref(out), C.byref(st)) == -2
    assert out.value is None
    # the same words without the stray bit build
    assert lib.jv_graph_build_bq(bqv._h, 1, C.byref(params), C.byref(out), C.byref(ms)) == 0
    jv.GraphIndex(_handle=C.c_void_p(out.value)).close()
    for h in (bqv, short, f32, bad, g, full, wide, wide_full):
        h.close()
