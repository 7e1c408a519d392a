"""Multi-segment search (jv_segments_search_batch, SegmentSearcher): every segment answers exactly what its own call answers
(jv_graph_search_batch_ex, or jv_exhaustive_search_batch for a segment without graph), and the answers are merged stably:

  - CPU: merge_model, the host restatement of the merge rule (padding dropped; score descending as the top-k key's sortable score,
    so -0.0 below +0.0; equal scores in segment order, then in list order; padded with -1 / -1 / 0), on synthetic lists;
  - GPU: segments, ids and score bits equal merge_model over the single calls, and every segment's counters equal its single call's,
    for every walk the planner picks (fp32 DOT sketched with edge records, L2, cosine; PQ with FusedPQ records and an fp32 rerank;
    PQ with an NVQ rerank; BQ with an fp32 rerank; no reranker) over 1, 3 and 16 segments of unequal sizes (a one-node segment, flat
    and hierarchical graphs, holes left by removeDeletedNodes, a segment with every node removed) at 1, 7 and a GPU-filling batch;
  - one segment gives jv_graph_search_batch_ex's bytes; per-segment filters, a threshold, a rerank floor and segments without graph;
    the same rows registered twice tie lower segment first; overflowing walks are re-run with the same answers; 16 segments prepared
    alike take the launches 2 take; every refusal leaves the outputs untouched; two host threads on shared handles; siftsmall recall."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_lib as o
from oracle_lib import fp, ip

JV_ERR_INVALID, JV_ERR_UNSUPPORTED = -2, -5
BIG = 2500  # queries per call that fill the GPU on their own (more than the fp32 walk's resident CTAs on 132 SMs)


def sortable(scores):
    s = np.ascontiguousarray(scores, np.float32).view(np.int32)
    return s ^ ((s >> 31) & 0x7fffffff)


def merge_model(lists, topK):
    """lists: per segment (nodes [nq][k], scores [nq][k]) -> segments, nodes, scores [nq][topK] of the stable merge"""
    nq = lists[0][0].shape[0]
    seg = np.full((nq, topK), -1, np.int32)
    nodes = np.full((nq, topK), -1, np.int32)
    scores = np.zeros((nq, topK), np.float32)
    for q in range(nq):
        ents = []
        for s, (nd, sc) in enumerate(lists):
            key = sortable(sc[q])
            ents += [(-int(key[j]), s, j) for j in range(nd.shape[1]) if nd[q, j] >= 0]
        ents.sort()
        for r, (_, s, j) in enumerate(ents[:topK]):
            seg[q, r], nodes[q, r], scores[q, r] = s, lists[s][0][q, j], lists[s][1][q, j]
    return seg, nodes, scores


# ------------------------------------------------------------------------------------------------ CPU: the merge rule


def test_merge_model_ties_across_and_within_segments():
    a = (np.array([[3, 1, 2]], np.int32), np.array([[0.9, 0.5, 0.5]], np.float32))
    b = (np.array([[7, 8, -1]], np.int32), np.array([[0.9, 0.5, 0.0]], np.float32))
    seg, nodes, scores = merge_model([a, b], 5)
    assert seg.tolist() == [[0, 1, 0, 0, 1]]
    assert nodes.tolist() == [[3, 7, 1, 2, 8]]  # within a segment the list's own order stays, whatever the ids
    assert scores.tolist() == [[np.float32(0.9), np.float32(0.9), 0.5, 0.5, 0.5]]


def test_merge_model_negative_zero_below_positive_zero():
    a = (np.array([[4]], np.int32), np.array([[-0.0]], np.float32))
    b = (np.array([[5]], np.int32), np.array([[0.0]], np.float32))
    seg, nodes, scores = merge_model([a, b], 2)
    assert seg.tolist() == [[1, 0]] and nodes.tolist() == [[5, 4]]
    assert scores.view(np.int32).tolist() == [[0, np.float32(-0.0).view(np.int32)]]


def test_merge_model_all_padding_and_short_lists():
    pad = (np.full((2, 3), -1, np.int32), np.zeros((2, 3), np.float32))
    one = (np.array([[1, -1, -1], [-1, -1, -1]], np.int32), np.array([[0.25, 0, 0], [0, 0, 0]], np.float32))
    seg, nodes, scores = merge_model([pad, one, pad], 8)
    assert seg.tolist() == [[1] + [-1] * 7, [-1] * 8]
    assert nodes.tolist() == [[1] + [-1] * 7, [-1] * 8]
    assert scores.tolist() == [[0.25] + [0.0] * 7, [0.0] * 8]


# ------------------------------------------------------------------------------------------------ GPU


@pytest.fixture(scope="module")
def jv():
    import jvector_b200
    jvector_b200.init()
    return jvector_b200


@pytest.fixture(scope="module")
def nat(jv):
    from jvector_b200 import _native
    return _native


SIZES = (1500, 1, 2500, 37, 800, 300, 2000, 120, 640, 999, 64, 1200, 450, 33, 700, 260)
HOLES, EMPTY = 4, 9  # the segment with holes, the segment with every node removed


@pytest.fixture(scope="module")
def world(jv):
    """16 segments of rows near a 32-dimensional subspace (so the fp32 DOT walk gets low-rank rows and edge records), each with its
    own graph, and the same rows as PQ (one codebook), NVQ and BQ data sets"""
    rng = np.random.default_rng(17)
    dim, latent = 130, 32
    A = rng.standard_normal((latent, dim)) / np.sqrt(latent)

    def rows(k):
        x = rng.standard_normal((k, latent)) @ A + 0.2 * rng.standard_normal((k, dim))
        return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)

    data = [rows(n) for n in SIZES]
    queries = rows(BIG)
    allrows = np.concatenate(data)
    M, k = 13, 64
    cb, _, _ = o.train_pq_numpy(rng, allrows[:4000], M, k, iters=2)
    segs = []
    for s, x in enumerate(data):
        f32 = jv.F32Vectors(x)
        gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, addHierarchy=(s % 2 == 0), seed=s).build(f32)
        if s == HOLES:
            gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, seed=s).removeDeletedNodes(gi, f32, rng.random(len(x)) < 0.2)
        if s == EMPTY:
            gi = jv.GraphIndexBuilder(o.DOT_PRODUCT, M=16, beamWidth=60, seed=s).removeDeletedNodes(gi, f32, np.ones(len(x), bool))
        codes = jv.pq_encode_all(f32, cb, M, k, None)
        pq = jv.PQVectors(codes, cb, dim, k, None)
        mean = allrows.mean(0).astype(np.float32)
        params, bys = jv.nvq_encode_all(f32, mean, 2, True)
        nvq = jv.NVQVectors(bys, params, mean, 2)
        bq = jv.BQVectors(jv.bq_encode_all(f32), dim)
        info = gi.info()
        upper = [gi.level(lv) for lv in range(1, info["levels"])]
        fused = jv.GraphIndex(gi.level(0)[1], info["entry_node"], upper).fuse_pq(pq) if info["entry_node"] >= 0 else gi
        segs.append(dict(n=len(x), x=x, f32=f32, pq=pq, nvq=nvq, bq=bq, gi=gi, fused=fused, keep=(codes, params, bys, mean)))
    return dict(segs=segs, queries=queries, cb=cb)


# walk name -> (approx kind, reranker kind, metric, fused graph)
WALKS = {
    "f32_dot": ("f32", None, o.DOT_PRODUCT, False),
    "f32_l2": ("f32", None, o.EUCLIDEAN, False),
    "f32_cos": ("f32", None, o.COSINE, False),
    "pq_fused_f32": ("pq", "f32", o.DOT_PRODUCT, True),
    "pq_nvq": ("pq", "nvq", o.EUCLIDEAN, False),
    "bq_f32": ("bq", "f32", o.COSINE, False),
}
SEGMENT_SETS = {1: (0,), 3: (1, HOLES, 2), 16: tuple(range(16))}


def segments_of(world, walk, which, graphs=True, accept=None):
    kind, rr, _, fused = WALKS[walk]
    out = []
    for j, s in enumerate(which):
        d = world["segs"][s]
        g = (d["fused"] if fused else d["gi"]) if graphs is True or (graphs and j in graphs) else None
        out.append((g, d[kind], d[rr] if rr else None, None if accept is None else accept[j]))
    return out


def single(nat, seg, metric, queries, topK, rerankK, threshold=0.0, floor=0.0):
    lib = nat.load()
    g, approx, rr, accept = seg
    bits = None if accept is None else __import__("jvector_b200").pack_accept_bits(accept)
    opts = nat.SearchOptions(bits.ctypes.data if bits is not None else None, 0, float(threshold), float(floor))
    nq = len(queries)
    nodes = np.empty((nq, topK), np.int32)
    scores = np.empty((nq, topK), np.float32)
    st = nat.SearchStats()
    rrh = rr._h if rr is not None else None
    if g is not None:
        rc = lib.jv_graph_search_batch_ex(g._h, approx._h, rrh, metric, fp(queries), nq, topK, rerankK, C.byref(opts), ip(nodes), fp(scores), C.byref(st))
    else:
        rc = lib.jv_exhaustive_search_batch(approx._h, rrh, metric, fp(queries), nq, topK, rerankK, C.byref(opts), ip(nodes), fp(scores), C.byref(st))
    assert rc == 0, lib.jv_last_error()
    return nodes, scores, st


COUNTERS = ("visitedCount", "expandedCount", "expandedCountBaseLayer", "rerankedCount")


def check_against_singles(jv, nat, segs, metric, queries, topK, rerankK, threshold=0.0, floor=0.0, what=()):
    res = jv.SegmentSearcher(segs).search(queries, metric, topK, rerankK, threshold, floor)
    singles = [single(nat, s, metric, queries, topK, rerankK, threshold, floor) for s in segs]
    seg, nodes, scores = merge_model([(nd, sc) for nd, sc, _ in singles], topK)
    assert np.array_equal(res.segments, seg), what
    assert np.array_equal(res.nodes, nodes), what
    assert np.array_equal(res.scores.view(np.int32), scores.view(np.int32)), what
    for s, (_, _, st) in enumerate(singles):
        mine = res.segment_stats[s]
        want = (st.visited, st.expanded, st.expanded_base, st.reranked)
        assert tuple(getattr(mine, c) for c in COUNTERS) == want, (what, "segment", s)
    assert res.stats.visitedCount == sum(st.visited for _, _, st in singles)
    assert res.stats.rerankedCount == sum(st.reranked for _, _, st in singles)
    return res, singles


@pytest.mark.gpu
@pytest.mark.parametrize("S", sorted(SEGMENT_SETS))
@pytest.mark.parametrize("walk", sorted(WALKS))
def test_against_single_calls(jv, nat, world, walk, S):
    _, rr, metric, _ = WALKS[walk]
    segs = segments_of(world, walk, SEGMENT_SETS[S])
    for nq in (1, 7, BIG):
        q = world["queries"][:nq]
        check_against_singles(jv, nat, segs, metric, q, 10, 40 if rr else 10, what=(walk, S, nq))
        if walk == "f32_dot" and nq == BIG and S > 1:
            assert nat.load().jv_search_last_settled() > 0, "the sketched walk was expected to settle neighbours on edge records"


@pytest.mark.gpu
def test_one_segment_is_the_single_call_byte_for_byte(jv, nat, world):
    segs = segments_of(world, "pq_fused_f32", (2,))
    q = world["queries"][:300]
    res = jv.SegmentSearcher(segs).search(q, o.DOT_PRODUCT, 10, 50)
    nodes, scores, _ = single(nat, segs[0], o.DOT_PRODUCT, q, 10, 50)
    assert res.nodes.tobytes() == nodes.tobytes() and res.scores.tobytes() == scores.tobytes()
    assert (res.segments[nodes >= 0] == 0).all() and (res.segments[nodes < 0] == -1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("walk", ("f32_dot", "pq_fused_f32"))
def test_filters_and_segments_without_graph(jv, nat, world, walk):
    rng = np.random.default_rng(5)
    which = (2, 0, 6, 4, 11)
    sizes = [world["segs"][s]["n"] for s in which]
    accept = [np.ones(sizes[0], bool), rng.random(sizes[1]) < 0.01, np.zeros(sizes[2], bool), rng.random(sizes[3]) < 0.5, None]
    q = world["queries"][:64]
    for graphs in (True, (0, 1, 3)):  # every segment walked; segments 2 and 4 without graph
        segs = segments_of(world, walk, which, graphs=graphs, accept=accept)
        check_against_singles(jv, nat, segs, WALKS[walk][2], q, 10, 60, what=(walk, graphs))
        check_against_singles(jv, nat, segs, WALKS[walk][2], q, 10, 60, threshold=0.55, floor=0.6, what=(walk, graphs, "threshold, floor"))


@pytest.mark.gpu
def test_same_rows_twice_tie_lower_segment_first(jv, nat, world):
    d = world["segs"][2]
    segs = [(d["gi"], d["f32"], None, None), (d["gi"], jv.F32Vectors(d["x"]), None, None)]
    q = world["queries"][:50]
    res, _ = check_against_singles(jv, nat, segs, o.DOT_PRODUCT, q, 20, 20)
    # every answer comes twice, segment 0 first, then segment 1, with the same node and score bits
    assert (res.segments[:, 0::2] == 0).all() and (res.segments[:, 1::2] == 1).all()
    assert np.array_equal(res.nodes[:, 0::2], res.nodes[:, 1::2])
    assert np.array_equal(res.scores[:, 0::2].view(np.int32), res.scores[:, 1::2].view(np.int32))


@pytest.mark.gpu
def test_overflowing_walks_are_rerun(jv, nat, world, monkeypatch):
    # a small visited table overflows (code 1); a list without slack overflows on the rejected entries of a 30 % filter (code 2)
    rng = np.random.default_rng(8)
    which = (0, 2, 6)
    q = world["queries"][:40]
    for env in ({"JV_VISITED_CAP": "2048"}, {"JV_LIST_CAP": "1"}):
        accept = [rng.random(world["segs"][s]["n"]) < 0.3 for s in which] if "JV_LIST_CAP" in env else None
        segs = segments_of(world, "f32_l2", which, accept=accept)
        want = jv.SegmentSearcher(segs).search(q, o.EUCLIDEAN, 10, 200)
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            got = jv.SegmentSearcher(segs).search(q, o.EUCLIDEAN, 10, 200)
        assert got.stats.retried > 0, env
        assert np.array_equal(got.segments, want.segments) and np.array_equal(got.nodes, want.nodes), env
        assert np.array_equal(got.scores.view(np.int32), want.scores.view(np.int32)), env
        for a, b in zip(got.segment_stats, want.segment_stats):
            assert tuple(getattr(a, c) for c in COUNTERS) == tuple(getattr(b, c) for c in COUNTERS), env


@pytest.mark.gpu
def test_segments_prepared_alike_take_one_walk_launch(jv, nat, world):
    lib = nat.load()
    q = world["queries"][:7]
    many = jv.SegmentSearcher(segments_of(world, "f32_l2", [s for s in range(16) if s != EMPTY] + [0]))
    two = jv.SegmentSearcher(segments_of(world, "f32_l2", (0, 2)))
    counts = []
    for searcher in (many, two, many):
        l0 = lib.jv_kernel_launch_count()
        searcher.search(q, o.EUCLIDEAN, 10, 10)
        counts.append(lib.jv_kernel_launch_count() - l0)
    assert counts[0] == counts[1] == counts[2] == 2, counts  # one walk, one merge


@pytest.mark.gpu
def test_refusals_leave_outputs_untouched(jv, nat, world):
    lib = nat.load()
    q = world["queries"][:4]
    nq = len(q)
    d = world["segs"]

    def seg(s, kind="f32", rr=None, graph=True, bits=None):
        x = d[s]
        return nat.SearchSegment(x["gi"]._h if graph else None, x[kind]._h, x[rr]._h if rr else None, bits)

    def call(segs, topK=5, rerankK=10, metric=o.DOT_PRODUCT, threshold=0.0, floor=0.0, n=None, queries=q, nq_=nq):
        arr = (nat.SearchSegment * max(1, len(segs)))(*segs)
        out = [np.full((nq, 64), 7, np.int32), np.full((nq, 64), 7, np.int32), np.full((nq, 64), 7.0, np.float32)]
        rc = lib.jv_segments_search_batch(arr if segs else None, len(segs) if n is None else n, metric, fp(queries) if queries is not None else None,
                                          nq_, topK, rerankK, threshold, floor, ip(out[0]), ip(out[1]), fp(out[2]), None, None)
        assert (out[0] == 7).all() and (out[1] == 7).all() and (out[2] == 7.0).all(), "a refused call wrote its outputs"
        return rc

    ok = [seg(0), seg(2)]
    cases = [
        (dict(segs=[]), JV_ERR_INVALID),
        (dict(segs=ok, queries=None), JV_ERR_INVALID),
        (dict(segs=ok, n=0), JV_ERR_INVALID),
        (dict(segs=ok, nq_=0), JV_ERR_INVALID),
        (dict(segs=ok, topK=0), JV_ERR_INVALID),
        (dict(segs=ok, topK=11, rerankK=10), JV_ERR_INVALID),
        (dict(segs=[seg(0), nat.SearchSegment(d[2]["gi"]._h, d[3]["f32"]._h, None, None)]), JV_ERR_INVALID),  # graph and data set sizes
        (dict(segs=[seg(0), seg(2, "pq")]), JV_ERR_INVALID),  # kinds differ
        (dict(segs=[seg(0, "pq", "f32"), seg(2, "pq")]), JV_ERR_INVALID),  # rerankers mixed
        (dict(segs=[seg(0, "pq", "f32"), seg(2, "pq", "nvq")]), JV_ERR_INVALID),  # rerankers of different kinds
        (dict(segs=ok, metric=7), JV_ERR_INVALID),
        (dict(segs=ok, threshold=-0.5), JV_ERR_INVALID),
        (dict(segs=ok, floor=-0.5), JV_ERR_INVALID),
        (dict(segs=[seg(0)] * 1025, topK=1, rerankK=1), JV_ERR_UNSUPPORTED),
        (dict(segs=[seg(0)] * 17, topK=1000, rerankK=1000), JV_ERR_UNSUPPORTED),
        (dict(segs=ok, topK=5, rerankK=4097), JV_ERR_UNSUPPORTED),
        (dict(segs=[seg(0), seg(2, graph=False)], topK=5, rerankK=2049), JV_ERR_UNSUPPORTED),
    ]
    for kw, code in cases:
        rc = call(**kw)
        assert rc == code, (kw, rc, lib.jv_last_error())
    # a PQ data set whose M differs
    rng = np.random.default_rng(3)
    cb, _, _ = o.train_pq_numpy(rng, d[2]["x"], 10, 16, iters=1)
    codes = jv.pq_encode_all(d[2]["f32"], cb, 10, 16, None)
    pq10 = jv.PQVectors(codes, cb, 130, 16, None)
    assert call([seg(0, "pq"), nat.SearchSegment(d[2]["gi"]._h, pq10._h, None, None)]) == JV_ERR_INVALID
    # an NVQ reranker of other sub-vectors
    mean = d[0]["keep"][3]
    params, bys = jv.nvq_encode_all(d[2]["f32"], mean, 5, True)
    nvq5 = jv.NVQVectors(bys, params, mean, 5)
    assert call([seg(0, "pq", "nvq"), nat.SearchSegment(d[2]["gi"]._h, d[2]["pq"]._h, nvq5._h, None)]) == JV_ERR_INVALID


@pytest.mark.gpu
def test_two_threads_on_shared_handles(jv, nat, world):
    q = world["queries"][:BIG]
    jobs = [(segments_of(world, "f32_dot", range(16)), o.DOT_PRODUCT, q, 40), (segments_of(world, "pq_fused_f32", (0, 1, 2, 3)), o.DOT_PRODUCT, q[:300], 60)]
    alone = [jv.SegmentSearcher(s).search(qq, m, 10, r) for s, m, qq, r in jobs]
    barrier = threading.Barrier(len(jobs))
    got = [None] * len(jobs)

    def run(i):
        s, m, qq, r = jobs[i]
        barrier.wait()
        got[i] = jv.SegmentSearcher(s).search(qq, m, 10, r)

    ts = [threading.Thread(target=run, args=(i,)) for i in range(len(jobs))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for a, b in zip(alone, got):
        assert np.array_equal(a.segments, b.segments) and np.array_equal(a.nodes, b.nodes)
        assert np.array_equal(a.scores.view(np.int32), b.scores.view(np.int32))


# recall@10 of siftsmall split into 4 segments, each built alone: 1.0 measured on an H100 80GB HBM3 (700 W power limit)
SIFT_RECALL_BOUND = 0.99


@pytest.mark.gpu
def test_siftsmall_recall_over_four_segments(jv, sift):
    base, queries, gt = sift
    bounds = np.linspace(0, len(base), 5).astype(int)
    parts = []
    for i in range(4):
        v = jv.F32Vectors(base[bounds[i]:bounds[i + 1]])
        g = jv.GraphIndexBuilder(o.EUCLIDEAN, M=16, beamWidth=100, addHierarchy=True, seed=i).build(v)
        parts.append((g, v))
    res = jv.SegmentSearcher(parts).search(queries, o.EUCLIDEAN, 10, 50)
    ids = np.where(res.nodes >= 0, res.nodes + bounds[np.maximum(res.segments, 0)], -1)
    recall = np.mean([len(set(ids[i]) & set(gt[i, :10])) / 10.0 for i in range(len(queries))])
    assert recall >= SIFT_RECALL_BOUND, recall
