"""Several host threads on shared handles (INTEGRATION §3, §3a: data sets and graphs may be shared across threads, each thread has its
own stream and staging buffers), bit for bit against the same calls made alone.

Every scenario computes its expected answers first, on one thread, over handles of its own; then it makes fresh handles from the same
arrays, so that whatever the library builds lazily on them (an fp32 data set's row sketch and low-rank rows, a graph's edge records,
a PQ data set's centroid-pair tables) is built while the threads race for it. The threads start together on one barrier and make
their call once; ctypes releases the GIL, so the calls overlap on the host and on the device. Every call compared here is
deterministic by contract (DESIGN §8), so the comparisons are exact whatever the interleaving. Each scenario runs its threads in a
pool of its own: they exit, and the library's per-thread contexts with them, while the handles live on.

  a. the first sketched fp32 DOT search of a data set and a graph, from every thread at once: results, the per-thread counters of
     the edge tier (jv_search_last_settled, jv_search_last_direct), the sketch, the low-rank rows and the edge records;
  b. one graph searched over two data sets with different rows, threads alternating between them, so that the graph's edge
     records are replaced while other threads' searches still hold the previous ones;
  c. builds, a removal and the diversity scores over one PQ data set whose pair tables do not exist yet (one table per metric
     family, each built once: the data set's device bytes equal those of a data set that built both alone);
  d. an fp32 build, a BQ build, an add, PQ training and the resident PQ encoder over shared rows;
  e. the batch scorers over shared data sets of every kind, the stream-ordered BQ top-k and merge on each thread's own stream;
  f. a refused call among (e)'s: its thread gets its own error message, every other thread succeeds."""
import ctypes as C
import threading
import types
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import builder_driver as bd
import oracle_lib as o
from oracle_lib import fp
from test_build_steps import latent_rows

pytestmark = pytest.mark.gpu

NQ = 3000  # more queries than an H100 keeps resident (132 SMs x 9 CTAs): a search batch takes the sketch path
SEARCHERS = 6
JV_ERR_INVALID = -2


@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


def race(calls):
    """every call once, each on a thread of its own, all released by one barrier; their results in order (a worker's exception
    is raised here)"""
    start = threading.Barrier(len(calls))

    def run(call):
        start.wait(timeout=120)
        return call()

    with ThreadPoolExecutor(max_workers=len(calls)) as pool:
        futures = [pool.submit(run, call) for call in calls]
        return [f.result() for f in futures]


def snapshot(gi):
    """a graph's info and every level on the host; the handle is closed"""
    try:
        return gi.info(), bd.levels(gi)
    finally:
        gi.close()


def assert_same_snapshot(got, want, what):
    assert got[0] == want[0], (what, got[0], want[0])
    for lv, ((ids_a, adj_a), (ids_b, adj_b)) in enumerate(zip(got[1], want[1])):
        assert np.array_equal(ids_a, ids_b) and np.array_equal(adj_a, adj_b), (what, "level", lv)


def build_stats(b):
    return b.scored_vectors, b.batches, b.dropped_backlinks


def without_ms(stats):
    return {k: v for k, v in stats.items() if not k.endswith("_ms")}


# ------------------------------------------------------------------------------------------------ a, b: sketched fp32 searches
@pytest.fixture(scope="module")
def latent(jv):
    """20 000 rows near a rank-32 subspace (their low-rank rows exist), SEARCHERS batches of NQ queries from the same subspace, a
    second set of rows in it that differs from the first everywhere, and a DOT_PRODUCT graph over the first"""
    rng = np.random.default_rng(61)
    n, dim = 20000, 130
    rows = latent_rows(rng, n + SEARCHERS * NQ, dim, latent=32, noise=0.2)
    data, queries = rows[:n], rows[n:]
    other = data.astype(np.float64) + 0.25 * data[rng.permutation(n)]
    other = (other / np.linalg.norm(other, axis=1, keepdims=True)).astype(np.float32)
    vec = jv.F32Vectors(data)
    gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, addHierarchy=True, seed=5).build(vec)
    vec.close()
    info = gi.info()
    adj0 = gi.level(0)[1]
    upper = [gi.level(lv) for lv in range(1, info["levels"])]
    gi.close()
    return types.SimpleNamespace(data=data, other=other, batches=np.split(queries, SEARCHERS), adj0=adj0, upper=upper, entry=info["entry_node"],
                                 graph=lambda: jv.GraphIndex(adj0, info["entry_node"], upper))


def sketched_search(jv, vec, gi, queries):
    """the search and this thread's counters of it: (result, (settled, routed, routed_dropped))"""
    res = jv.GraphSearcher(gi).search(vec, queries, o.DOT_PRODUCT, 10, 40)
    routed, dropped = C.c_int64(), C.c_int64()
    lib = jv.load()
    lib.jv_search_last_direct(C.byref(routed), C.byref(dropped))
    return res, (lib.jv_search_last_settled(), routed.value, dropped.value)


def assert_same_result(got, want, what):
    assert np.array_equal(got.nodes, want.nodes), (what, "ids differ for queries", np.flatnonzero((got.nodes != want.nodes).any(axis=1))[:8].tolist())
    assert np.array_equal(got.scores.view(np.int32), want.scores.view(np.int32)), (what, "score bits differ")
    for name in ("visitedCount", "expandedCount", "expandedCountBaseLayer", "rerankedCount", "retried"):
        assert getattr(got, name) == getattr(want, name), (what, name, getattr(got, name), getattr(want, name))


def lowrank(jv, vec, n, dim):
    stride = (dim + 3) & ~3
    basis, rows, k = np.empty((32, stride), np.float32), np.empty((n, 48), np.uint8), C.c_int()
    assert jv.load().jv_dataset_lowrank_download(vec._h, fp(basis), rows.ctypes.data, C.byref(k)) == 0, jv.load().jv_last_error()
    return basis, rows


def edge_records(jv, gi, n, degree):
    rec = np.empty((n, degree, 48), np.uint8)
    assert jv.load().jv_graph_edge_records_download(gi._h, rec.ctypes.data) == 0, jv.load().jv_last_error()
    return rec


def test_first_sketched_search_raced(jv, oracle, latent):
    from test_gpu_parity import _assert_same_search, _oracle_search
    w = latent
    n, dim = w.data.shape
    vec, gi = jv.F32Vectors(w.data), w.graph()
    want = [sketched_search(jv, vec, gi, q) for q in w.batches]
    assert all(c[0] > 0 for _, c in want), "every batch was expected to settle neighbours on the edge records"
    fresh, fresh_gi = jv.F32Vectors(w.data), w.graph()
    assert fresh.row_sketch() is None
    got = race([lambda q=q: sketched_search(jv, fresh, fresh_gi, q) for q in w.batches])
    for i, ((res, counters), (wres, wcounters)) in enumerate(zip(got, want)):
        assert_same_result(res, wres, ("thread", i))
        assert counters == wcounters, ("thread", i, "settled / routed / routed_dropped", counters, wcounters)
    mk = lambda q: oracle.jvo_scorer_f32(o.DOT_PRODUCT, fp(w.data), n, dim, fp(q))
    _assert_same_search(got[0][0], _oracle_search(oracle, o.make_graph(w.adj0, w.entry, w.upper), mk, w.batches[0], 10, 40), "thread 0 vs oracle")
    for a, b in zip(fresh.row_sketch(), vec.row_sketch()):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "row sketch"
    for a, b in zip(lowrank(jv, fresh, n, dim), lowrank(jv, vec, n, dim)):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "low-rank basis / rows"
    assert np.array_equal(edge_records(jv, fresh_gi, n, w.adj0.shape[1]), edge_records(jv, gi, n, w.adj0.shape[1])), "edge records"
    for h in (vec, gi, fresh, fresh_gi):
        h.close()


def test_edge_records_replaced_under_running_searches(jv, latent):
    # threads 0, 2, 4 search the graph over one data set, threads 1, 3, 5 over the other: each data set's low-rank rows get their
    # own build id, so every change of data set rebuilds the graph's edge records while the other data set's searches still read
    # the records they started with
    w = latent
    datasets = (w.data, w.other)
    vecs, gi = [jv.F32Vectors(d) for d in datasets], w.graph()
    want = [sketched_search(jv, vecs[i % 2], gi, q) for i, q in enumerate(w.batches)]
    fresh, fresh_gi = [jv.F32Vectors(d) for d in datasets], w.graph()
    got = race([lambda i=i, q=q: sketched_search(jv, fresh[i % 2], fresh_gi, q) for i, q in enumerate(w.batches)])
    for i, ((res, counters), (wres, wcounters)) in enumerate(zip(got, want)):
        assert_same_result(res, wres, ("thread", i, "data set", i % 2))
        assert counters[0] > 0, ("thread", i, "the walk was expected to settle neighbours on edge records")
        assert counters == wcounters, ("thread", i, counters, wcounters)
    for h in vecs + fresh + [gi, fresh_gi]:
        h.close()


# ------------------------------------------------------------------------------------------------ c: the PQ pair tables
@pytest.fixture(scope="module")
def pq_world(jv):
    rng = np.random.default_rng(67)
    n, dim, M = 8000, 64, 16
    rows = latent_rows(rng, n, dim)
    f32 = jv.F32Vectors(rows)
    pq = jv.ProductQuantization.compute(f32, M, 256, globallyCenter=True, seed=3)
    codes = jv.pq_encode_all(f32, pq.codebooks, M, 256, pq.centroid)
    base = snapshot(jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, addHierarchy=True, seed=3).build(f32))
    f32.close()
    info, lv = base
    return types.SimpleNamespace(n=n, dim=dim, codes=codes, codebooks=pq.codebooks, centroid=pq.centroid,
                                 graph=lambda: jv.GraphIndex(lv[0][1], info["entry_node"], lv[1:]),
                                 a=rng.integers(0, n, 50000).astype(np.int32), b=rng.integers(0, n, 50000).astype(np.int32),
                                 deleted=rng.random(n) < 0.05)


def pq_calls(jv, w, pqv):
    """the calls of scenario (c) over one PQ data set; each needs the pair table of its metric family"""

    def build(metric):
        b = bd.builder(jv, metric, 16, hier=True, seed=7)
        return snapshot(b.build(pqv)), build_stats(b)

    def scores(metric):
        return pqv.build_pair_table(metric).diversity_scores(w.a, w.b, metric)

    def remove(metric):
        gi = w.graph()
        out = bd.builder(jv, metric, 16, hier=True, seed=7).removeDeletedNodes(gi, pqv, w.deleted)
        gi.close()
        return snapshot(out), without_ms(out.remove_stats)

    return [lambda: build(o.EUCLIDEAN), lambda: build(o.DOT_PRODUCT), lambda: scores(o.EUCLIDEAN), lambda: scores(o.COSINE),
            lambda: scores(o.DOT_PRODUCT), lambda: remove(o.DOT_PRODUCT)]


def test_pq_pair_tables_raced(jv, pq_world):
    w = pq_world
    make = lambda: jv.PQVectors(w.codes, w.codebooks, w.dim, 256, w.centroid)
    serial = make()
    want = [call() for call in pq_calls(jv, w, serial)]
    fresh = make()
    no_tables = fresh.device_bytes()
    got = race(pq_calls(jv, w, fresh))
    for i, (g, x) in enumerate(zip(got, want)):
        if isinstance(x, np.ndarray):
            assert np.array_equal(g.view(np.int32), x.view(np.int32)), ("call", i, "diversity score bits")
        else:
            assert_same_snapshot(g[0], x[0], ("call", i))
            assert g[1] == x[1], ("call", i, "build / removal counters", g[1], x[1])
    # one table per metric family, built once: EUCLIDEAN, and DOT_PRODUCT shared with COSINE
    M, k = w.codes.shape[1], 256
    assert serial.device_bytes() - no_tables == 2 * M * (k * (k + 1) // 2) * 4
    assert fresh.device_bytes() == serial.device_bytes(), (fresh.device_bytes(), serial.device_bytes())
    for metric in (o.EUCLIDEAN, o.DOT_PRODUCT):
        assert np.array_equal(fresh.pair_table(metric).view(np.int32), serial.pair_table(metric).view(np.int32)), metric
    serial.close()
    fresh.close()


# ------------------------------------------------------------------------------------------------ d: builds and training
def test_builds_and_training_on_shared_rows(jv):
    rng = np.random.default_rng(71)
    n, n0, dim, M = 8000, 6000, 64, 16
    rows = latent_rows(rng, n, dim)
    words = jv.bq_encode_all(rows)
    small = jv.F32Vectors(rows[:n0])
    base = snapshot(jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, addHierarchy=True, seed=9).build(small))
    codebooks = jv.ProductQuantization.compute(small, M, 256, seed=2).codebooks
    small.close()

    def calls(f32, bq):
        def build(vectors):
            b = bd.builder(jv, o.DOT_PRODUCT, 16, hier=True, seed=9)
            return snapshot(b.build(vectors)), build_stats(b)

        def add():
            gi = jv.GraphIndex(base[1][0][1], base[0]["entry_node"], base[1][1:])
            b = bd.builder(jv, o.DOT_PRODUCT, 16, hier=True, seed=9)
            out = snapshot(b.addGraphNodes(gi, f32))
            gi.close()
            return out, build_stats(b)

        def train():
            pq = jv.ProductQuantization.compute(f32, M, 256, globallyCenter=True, seed=11)
            return pq.codebooks, pq.centroid, without_ms(pq.stats)

        def encode():
            pqv = jv.pq_encode_resident(f32, codebooks, M, 256)
            try:
                return pqv.download()[0]
            finally:
                pqv.close()

        return [lambda: build(f32), lambda: build(bq), add, train, encode]

    serial = jv.F32Vectors(rows), jv.BQVectors(words, dim)
    want = [call() for call in calls(*serial)]
    fresh = jv.F32Vectors(rows), jv.BQVectors(words, dim)
    got = race(calls(*fresh))
    for what, g, x in zip(("fp32 build", "BQ build", "add"), got, want):
        assert_same_snapshot(g[0], x[0], what)
        assert g[1] == x[1], (what, g[1], x[1])
    for a, b in zip(got[3][:2], want[3][:2]):
        assert np.array_equal(a.view(np.int32), b.view(np.int32)), "trained codebooks / centroid"
    assert got[3][2] == want[3][2], (got[3][2], want[3][2])
    assert np.array_equal(got[4], want[4]), "resident PQ codes"
    for h in serial + fresh:
        h.close()


# ------------------------------------------------------------------------------------------------ e, f: batch scorers
class ScorerWorld:
    """20 000 rows in every storage kind (BQ at dim 256 in two halves as well, each on the tensor-core path of the stream-ordered
    top-k), queries, and the host-driven steps (ids, offsets) the query batch and score_multi score"""

    def __init__(self, jv):
        rng = np.random.default_rng(73)
        n, dim, nq = 20000, 100, 50
        self.n, self.dim, self.nq, self.k = n, dim, nq, 30
        rows = latent_rows(rng, n + nq, dim)
        self.data, self.queries = rows[:n], rows[n:]
        f32 = jv.F32Vectors(self.data)
        pq = jv.ProductQuantization.compute(f32, 10, 256, globallyCenter=True, seed=4)
        f32.close()
        self.pq = (jv.pq_encode_all(self.data, pq.codebooks, 10, 256, pq.centroid), pq.codebooks, pq.centroid)
        self.mean = self.data.mean(0).astype(np.float32)
        self.nvq = jv.nvq_encode_all(self.data, self.mean, 3, True)
        self.bq_dim = 256
        self.bq_queries = rng.standard_normal((nq, self.bq_dim)).astype(np.float32)
        self.words = jv.bq_encode_all(rng.standard_normal((n, self.bq_dim)).astype(np.float32))
        lengths = rng.integers(0, 150, nq)  # up to 64 ids travel in the kernel's parameters, more through mapped memory
        self.offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
        self.ids = rng.integers(0, n, int(self.offsets[-1])).astype(np.int32)

    def handles(self, jv):
        codes, cb, cen = self.pq
        params, bys = self.nvq
        half = self.n // 2
        return types.SimpleNamespace(f32=jv.F32Vectors(self.data), pq=jv.PQVectors(codes, cb, self.dim, 256, cen),
                                     nvq=jv.NVQVectors(bys, params, self.mean, 3), bq=jv.BQVectors(self.words, self.bq_dim),
                                     halves=(jv.BQVectors(self.words[:half], self.bq_dim), jv.BQVectors(self.words[half:], self.bq_dim)))


def close_all(h):
    for v in (h.f32, h.pq, h.nvq, h.bq) + h.halves:
        v.close()


def scorer_calls(jv, w, h):
    lib = jv.load()

    def topk(vec, metric, queries):
        return jv.topk_bruteforce(vec, metric, queries, w.k)[2]

    def query_batch():
        qb = jv.QueryBatch(h.pq, w.queries, o.DOT_PRODUCT)
        try:
            return qb.score_step(w.ids, w.offsets), qb.score_one(3, w.ids[:100])
        finally:
            qb.close()

    def stream_ordered_bq():
        # the local top-k of each half with global ids, then the merge, on this thread's own stream with no host wait in between
        import torch
        from jvector_b200 import _native as nat
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            q = torch.from_numpy(w.bq_queries).cuda()
            parts = torch.empty((2, w.nq, w.k), dtype=torch.int64, device="cuda")
            status = torch.full((2,), -7, dtype=torch.int32, device="cuda")
            merged = torch.empty((w.nq, w.k), dtype=torch.int64, device="cuda")
        for i, half in enumerate(h.halves):
            nat.check(lib.jv_topk_bruteforce_device_async(half._h, o.COSINE, C.c_void_p(q.data_ptr()), w.nq, w.k, i * (w.n // 2),
                                                          C.c_void_p(parts[i].data_ptr()), C.c_void_p(status[i].data_ptr()), C.c_void_p(s.cuda_stream)))
        nat.check(lib.jv_topk_merge_device_async(C.c_void_p(parts.data_ptr()), w.nq, 2, w.k, C.c_void_p(merged.data_ptr()), C.c_void_p(s.cuda_stream)))
        s.synchronize()
        return merged.cpu().numpy(), status.cpu().numpy()

    return [lambda: topk(h.f32, o.DOT_PRODUCT, w.queries), lambda: topk(h.pq, o.EUCLIDEAN, w.queries), lambda: topk(h.nvq, o.COSINE, w.queries),
            lambda: topk(h.bq, o.COSINE, w.bq_queries), query_batch, lambda: jv.score_multi(h.nvq, o.EUCLIDEAN, w.queries, w.ids, w.offsets),
            stream_ordered_bq]


def assert_same_scores(got, want, what):
    for a, b in zip(got if isinstance(got, tuple) else (got,), want if isinstance(want, tuple) else (want,)):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), what


@pytest.fixture(scope="module")
def scorers(jv):
    """(world, expected answers of scorer_calls, each made alone)"""
    w = ScorerWorld(jv)
    h = w.handles(jv)
    want = [call() for call in scorer_calls(jv, w, h)]
    close_all(h)
    merged, status = want[-1]
    assert (status == 0).all() and np.array_equal(merged, want[3]), "the merged halves were expected to equal the whole BQ top-k"
    return w, want


def test_batch_scorers_raced(jv, scorers):
    w, want = scorers
    h = w.handles(jv)
    got = race(scorer_calls(jv, w, h))
    for i, (g, x) in enumerate(zip(got, want)):
        assert_same_scores(g, x, ("call", i))
    close_all(h)


def test_error_message_stays_with_its_thread(jv, scorers):
    # one thread's search is refused before any device work (rerankK < topK) while the others run (e); after every call has
    # returned, the refused thread still reads its own message and no other thread reads it
    w, want = scorers
    h = w.handles(jv)
    lib = jv.load()
    n = w.n
    chain = np.full((n, 4), -1, np.int32)
    chain[:, 0] = (np.arange(n) + 1) % n
    gi = jv.GraphIndex(chain, 0)
    done = threading.Barrier(len(want) + 1)

    def then_message(call):
        def run():
            try:
                out = call()
            except Exception as e:  # noqa: BLE001 (handed back to the main thread, which checks it)
                out = e
            done.wait(timeout=120)
            return out, lib.jv_last_error().decode()
        return run

    refused = lambda: jv.GraphSearcher(gi).search(h.f32, w.queries, o.DOT_PRODUCT, 10, 5)
    got = race([then_message(c) for c in scorer_calls(jv, w, h)] + [then_message(refused)])
    (err, message) = got[-1]
    assert isinstance(err, jv.JVectorB200Error) and err.code == JV_ERR_INVALID, err
    assert "rerankK" in str(err) and "rerankK" in message, (str(err), message)
    for i, ((g, msg), x) in enumerate(zip(got[:-1], want)):
        if isinstance(g, Exception):
            raise g
        assert_same_scores(g, x, ("call", i))
        assert "rerankK" not in msg, ("call", i, "read another thread's error message", msg)
    gi.close()
    close_all(h)
