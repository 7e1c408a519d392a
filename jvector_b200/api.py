"""Host-side mirror of the reference's scoring interface over the C ABI (see package docstring)."""
import ctypes as C
import enum

import numpy as np

from . import _native as nat
from ._native import bp, c32, check, fp, ip, lp, wp


class VectorSimilarityFunction(enum.IntEnum):
    """base:vector/VectorSimilarityFunction.java:34-80 (ordinals are the C ABI's metric codes)"""
    EUCLIDEAN = 0
    DOT_PRODUCT = 1
    COSINE = 2


class _Vectors:
    """A data set resident in HBM."""

    def __init__(self, handle, keep):
        self._h = handle
        self._keep = keep

    def size(self):
        return int(nat.load().jv_dataset_size(self._h))

    def dimension(self):
        return int(nat.load().jv_dataset_dim(self._h))

    def device_bytes(self):
        return int(nat.load().jv_dataset_device_bytes(self._h))

    def close(self):
        if self._h:
            nat.load().jv_dataset_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def score_function_for(self, query, vsf):
        """CompressedVectors.precomputedScoreFunctionFor / DefaultSearchScoreProvider.exact"""
        return ScoreFunction(self, query, vsf)

    # the reference's names
    precomputedScoreFunctionFor = score_function_for
    scoreFunctionFor = score_function_for

    def diversity_scores(self, a, b, vsf):
        """BuildScoreProvider.diversityProviderFor: score(a[i], b[i]) for every pair, one launch."""
        lib = nat.init()
        a = np.ascontiguousarray(a, dtype=np.int32)
        b = np.ascontiguousarray(b, dtype=np.int32)
        out = np.empty(len(a), dtype=np.float32)
        check(lib.jv_score_pairs(self._h, int(vsf), ip(a), ip(b), len(a), fp(out)))
        return out


class F32Vectors(_Vectors):
    def __init__(self, rows):
        lib = nat.init()
        rows = c32(rows)
        h = C.c_void_p()
        check(lib.jv_dataset_register_f32(fp(rows), rows.shape[0], rows.shape[1], C.byref(h)))
        super().__init__(h, None)


class PQVectors(_Vectors):
    """base:quantization/PQVectors.java — codes [n][M] + codebooks (concatenated, codebook m = [k][size_m])."""

    def __init__(self, codes, codebooks, dim, k=256, centroid=None):
        lib = nat.init()
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        codebooks = c32(codebooks).reshape(-1)
        cen = c32(centroid) if centroid is not None else None
        assert codebooks.size == k * dim
        self.M, self.k = codes.shape[1], k
        h = C.c_void_p()
        check(lib.jv_dataset_register_pq(bp(codes), codes.shape[0], dim, codes.shape[1], k, fp(codebooks), fp(cen), C.byref(h)))
        super().__init__(h, None)


    def build_pair_table(self, vsf):
        """ImmutablePQVectors: the triangular centroid-vs-centroid table in HBM; diversity_scores then sums table entries"""
        check(nat.load().jv_dataset_pq_pair_table(self._h, int(vsf)))
        return self

    def pair_table(self, vsf):
        out = np.empty(self.M * (self.k * (self.k + 1) // 2), dtype=np.float32)
        check(nat.load().jv_dataset_pq_pair_table_download(self._h, int(vsf), fp(out)))
        return out


def kmeans_assign(points, centroids):
    """KMeansPlusPlusClusterer.getNearestCluster for a batch of points (the Lloyd assignment step), one launch."""
    lib = nat.init()
    points, centroids = c32(points), c32(centroids)
    out = np.empty(points.shape[0], dtype=np.int32)
    check(lib.jv_kmeans_assign_batch(fp(points), points.shape[0], points.shape[1], fp(centroids), centroids.shape[0], ip(out)))
    return out


class BQVectors(_Vectors):
    """base:quantization/BQVectors.java — words [n][ceil(dim/64)] uint64."""

    def __init__(self, words, dim):
        lib = nat.init()
        words = np.ascontiguousarray(words, dtype=np.uint64)
        h = C.c_void_p()
        check(lib.jv_dataset_register_bq(wp(words), words.shape[0], dim, C.byref(h)))
        super().__init__(h, None)


class NVQVectors(_Vectors):
    """base:quantization/NVQVectors.java — bytes [n][dim], params [n][nsub][4] = {min, max, growthRate, midpoint}."""

    def __init__(self, bytes_, params, mean, nsub):
        lib = nat.init()
        bytes_ = np.ascontiguousarray(bytes_, dtype=np.uint8)
        params = c32(params)
        mean = c32(mean)
        h = C.c_void_p()
        check(lib.jv_dataset_register_nvq(bp(bytes_), fp(params), bytes_.shape[0], bytes_.shape[1], nsub, fp(mean), C.byref(h)))
        super().__init__(h, None)


class ScoreFunction:
    """base:graph/similarity/ScoreFunction.java:30-80 for one query against one data set.
    similarityTo(node) is the n = 1 case of similarityToBatch(ids) (one kernel launch per call)."""

    def __init__(self, vectors, query, vsf):
        lib = nat.init()
        self._vectors = vectors
        q = c32(query)
        self._h = C.c_void_p()
        check(lib.jv_query_begin(vectors._h, fp(q), int(vsf), C.byref(self._h)))

    def similarityToBatch(self, ids):
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        out = np.empty(len(ids), dtype=np.float32)
        check(nat.load().jv_score_batch(self._h, ip(ids), len(ids), fp(out)))
        return out

    def similarityTo(self, node):
        return float(self.similarityToBatch(np.array([node], dtype=np.int32))[0])

    def partial_sums(self):
        """PQ only: the query's LUT (PQDecoder.java:41-54)."""
        v = self._vectors
        out = np.empty(v.M * v.k, dtype=np.float32)
        check(nat.load().jv_query_get_lut(self._h, fp(out)))
        return out

    def close(self):
        if self._h:
            nat.load().jv_query_end(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class QueryBatch:
    """A batch of searches driven hop by hop from the host: prepared queries persist in HBM (jv_query_batch_*)."""

    def __init__(self, vectors, queries, vsf):
        lib = nat.init()
        queries = c32(queries)
        self._vectors = vectors
        self.nq = queries.shape[0]
        self._h = C.c_void_p()
        check(lib.jv_query_batch_begin(vectors._h, int(vsf), fp(queries), self.nq, C.byref(self._h)))

    def score_step(self, ids, offsets, return_ms=False, out=None):
        """one step of all searches: query i scores ids[offsets[i]:offsets[i+1]] (one launch). `ids` / `out` that were pinned with
        jv_host_register are used in place (no staging copy)."""
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        if out is None:
            out = np.empty(len(ids), dtype=np.float32)
        ms = C.c_double()
        check(nat.load().jv_query_batch_score(self._h, ip(ids), ip(offsets), fp(out), C.byref(ms)))
        return (out, ms.value) if return_ms else out

    def score_one(self, qi, ids):
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        out = np.empty(len(ids), dtype=np.float32)
        check(nat.load().jv_query_batch_score_one(self._h, int(qi), ip(ids), len(ids), fp(out)))
        return out

    def single(self, qi):
        return (self, qi)

    def close(self):
        if self._h:
            nat.load().jv_query_batch_end(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def score_multi(vectors, vsf, queries, ids, offsets):
    """One step of many searches: query i scores ids[offsets[i]:offsets[i+1]] (one launch for the whole step)."""
    lib = nat.init()
    queries = c32(queries)
    ids = np.ascontiguousarray(ids, dtype=np.int32)
    offsets = np.ascontiguousarray(offsets, dtype=np.int32)
    out = np.empty(len(ids), dtype=np.float32)
    check(lib.jv_score_multi(vectors._h, int(vsf), fp(queries), queries.shape[0], ip(ids), ip(offsets), fp(out)))
    return out


def topk_bruteforce(vectors, vsf, queries, k):
    """Exhaustive first pass with the reference's ordering key; returns (nodes [nq][k], scores [nq][k], keys)."""
    lib = nat.init()
    queries = c32(queries)
    keys = np.empty((queries.shape[0], k), dtype=np.int64)
    check(lib.jv_topk_bruteforce(vectors._h, int(vsf), fp(queries), queries.shape[0], k, lp(keys)))
    nodes = (~(keys & 0xffffffff)).astype(np.int64) & 0xffffffff
    nodes = nodes.astype(np.int64)
    s = (keys >> 32).astype(np.int32)
    bits = s ^ ((s >> 31) & 0x7fffffff)
    scores = bits.astype(np.int32).view(np.float32)
    nodes = np.where(keys == np.iinfo(np.int64).min, -1, nodes).astype(np.int32)
    return nodes, scores, keys


def bq_encode_all(rows):
    """BinaryQuantization.encodeAll. rows: a host array, or F32Vectors already resident in HBM (no upload)."""
    lib = nat.init()
    if isinstance(rows, _Vectors):
        out = np.empty((rows.size(), (rows.dimension() + 63) // 64), dtype=np.uint64)
        check(lib.jv_bq_encode_dataset(rows._h, wp(out)))
        return out
    rows = c32(rows)
    out = np.empty((rows.shape[0], (rows.shape[1] + 63) // 64), dtype=np.uint64)
    check(lib.jv_bq_encode_batch(fp(rows), rows.shape[0], rows.shape[1], wp(out)))
    return out


def pq_encode_all(rows, codebooks, M, k=256, centroid=None):
    """ProductQuantization.encodeAll. rows: a host array, or F32Vectors already resident in HBM (no upload)."""
    lib = nat.init()
    codebooks = c32(codebooks).reshape(-1)
    cen = c32(centroid) if centroid is not None else None
    if isinstance(rows, _Vectors):
        out = np.empty((rows.size(), M), dtype=np.uint8)
        check(lib.jv_pq_encode_dataset(rows._h, M, k, fp(codebooks), fp(cen), bp(out)))
        return out
    rows = c32(rows)
    out = np.empty((rows.shape[0], M), dtype=np.uint8)
    check(lib.jv_pq_encode_batch(fp(rows), rows.shape[0], rows.shape[1], M, k, fp(codebooks), fp(cen), bp(out)))
    return out


def nvq_encode_all(rows, mean, nsub, learn=True):
    """NVQuantization.encodeAll. rows: a host array, or F32Vectors already resident in HBM (no upload)."""
    lib = nat.init()
    mean = c32(mean)
    if isinstance(rows, _Vectors):
        params = np.empty((rows.size(), nsub, 4), dtype=np.float32)
        out = np.empty((rows.size(), rows.dimension()), dtype=np.uint8)
        check(lib.jv_nvq_encode_dataset(rows._h, nsub, fp(mean), 1 if learn else 0, fp(params), bp(out)))
        return params, out
    rows = c32(rows)
    params = np.empty((rows.shape[0], nsub, 4), dtype=np.float32)
    out = np.empty(rows.shape, dtype=np.uint8)
    check(lib.jv_nvq_encode_batch(fp(rows), rows.shape[0], rows.shape[1], nsub, fp(mean), 1 if learn else 0, fp(params), bp(out)))
    return params, out


def nvq_encode_resident(f32_vectors, mean, nsub, learn=True):
    """NVQuantization.encodeAll of rows already in HBM into a new resident NVQVectors (no host round trip)."""
    lib = nat.init()
    mean = c32(mean)
    h = C.c_void_p()
    check(lib.jv_nvq_encode_dataset_resident(f32_vectors._h, nsub, fp(mean), 1 if learn else 0, C.byref(h)))
    return _Vectors(h, None)


class GraphIndex:
    """ImmutableGraphIndex adjacency in HBM. adj0: [n][degree] int32 (-1 padded); upper: list of (node_ids, adj)."""

    def __init__(self, adj0=None, entry_node=0, upper=None, _handle=None):
        lib = nat.init()
        if _handle is not None:
            self._h = _handle
            return
        adj0 = np.ascontiguousarray(adj0, dtype=np.int32)
        self._h = C.c_void_p()
        check(lib.jv_graph_create(adj0.shape[0], adj0.shape[1], ip(adj0), entry_node, C.byref(self._h)))
        for ids, adj in (upper or []):
            ids = np.ascontiguousarray(ids, dtype=np.int32)
            adj = np.ascontiguousarray(adj, dtype=np.int32)
            check(lib.jv_graph_add_level(self._h, len(ids), ip(ids), ip(adj)))

    def info(self):
        n, e = C.c_int32(), C.c_int32()
        d, l = C.c_int(), C.c_int()
        check(nat.load().jv_graph_info(self._h, C.byref(n), C.byref(d), C.byref(l), C.byref(e)))
        return {"n": n.value, "degree": d.value, "levels": l.value, "entry_node": e.value}

    def level(self, level):
        """(node_ids, adjacency) of a level, copied back to the host."""
        inf = self.info()
        cnt = C.c_int32()
        check(nat.load().jv_graph_download(self._h, level, None, None, C.byref(cnt)))
        ids = np.empty(cnt.value, dtype=np.int32)
        adj = np.empty((cnt.value, inf["degree"]), dtype=np.int32)
        check(nat.load().jv_graph_download(self._h, level, ip(ids), ip(adj), C.byref(cnt)))
        return ids, adj

    def fuse_pq(self, pq_vectors):
        """FusedPQ feature: pack every node's neighbour codes next to its adjacency row (jv_graph_fuse_pq)."""
        check(nat.load().jv_graph_fuse_pq(self._h, pq_vectors._h))
        return self

    def fused_records(self):
        rb = C.c_int()
        check(nat.load().jv_graph_fused_download(self._h, None, C.byref(rb)))
        out = np.empty((self.info()["n"], rb.value), dtype=np.uint8)
        check(nat.load().jv_graph_fused_download(self._h, bp(out), C.byref(rb)))
        return out

    def close(self):
        if self._h:
            nat.load().jv_graph_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SearchResult:
    """base:graph/SearchResult.java for a batch: nodes/scores [nq][topK] best first (-1 padded) + the counters."""

    def __init__(self, nodes, scores, stats):
        self.nodes, self.scores = nodes, scores
        self.visitedCount = int(stats.visited)
        self.expandedCount = int(stats.expanded)
        self.expandedCountBaseLayer = int(stats.expanded_base)
        self.rerankedCount = int(stats.reranked)
        self.retried = int(stats.retried)
        self.device_ms = float(stats.device_ms)


class GraphSearcher:
    """base:graph/GraphSearcher.java: search(scoreProvider, topK, rerankK, ...) for a whole batch of queries, traversal
    on the device. `approx` walks the graph, `reranker` (fp32 or NVQ vectors, optional) rescoring the rerankK survivors."""

    def __init__(self, graph):
        self.graph = graph

    def search(self, approx, queries, vsf, topK, rerankK=None, reranker=None, threshold=0.0, rerankFloor=0.0, acceptOrds=None):
        """acceptOrds: None (Bits.ALL), a bool array [n] shared by the batch, or [nq][n] one per query
        (GraphSearcher.search(sp, topK, rerankK, threshold, rerankFloor, acceptOrds))."""
        lib = nat.init()
        queries = c32(queries)
        if queries.shape[1] != approx.dimension():
            raise ValueError("query dimension %d != data set dimension %d" % (queries.shape[1], approx.dimension()))
        rerankK = rerankK or topK
        nq = queries.shape[0]
        nodes = np.empty((nq, topK), dtype=np.int32)
        scores = np.empty((nq, topK), dtype=np.float32)
        st = nat.SearchStats()
        opts = None
        if acceptOrds is not None or threshold > 0 or rerankFloor > 0:
            opts = nat.SearchOptions(None, 0, float(threshold), float(rerankFloor))
            if acceptOrds is not None:
                bits = pack_accept_bits(acceptOrds)
                opts.accept_bits = bits.ctypes.data
                opts.accept_stride_words = bits.shape[1] if bits.ndim == 2 else 0
        check(lib.jv_graph_search_batch_ex(self.graph._h, approx._h, reranker._h if reranker is not None else None, int(vsf), fp(queries), nq,
                                           topK, rerankK, C.byref(opts) if opts is not None else None, ip(nodes), fp(scores), C.byref(st)))
        return SearchResult(nodes, scores, st)


def pack_accept_bits(mask):
    """bool [n] or [nq][n] -> uint32 words, bit (node & 31) of word (node >> 5) (the layout jv_search_options.accept_bits takes)"""
    m = np.asarray(mask, dtype=bool)
    n = m.shape[-1]
    pad = (-n) % 32
    if pad:
        m = np.concatenate([m, np.zeros(m.shape[:-1] + (pad,), bool)], axis=-1)
    return np.ascontiguousarray(np.packbits(m, axis=-1, bitorder="little").view(np.uint32))


class GraphIndexBuilder:
    """base:graph/GraphIndexBuilder.java: (M, beamWidth, neighborOverflow, alpha, addHierarchy) over exact fp32 scores."""

    def __init__(self, vsf, M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=False, seed=0, max_batch=0, concurrent_window=-1):
        self.vsf = vsf
        self.params = nat.BuildParams(M, beamWidth, neighborOverflow, alpha, 1 if addHierarchy else 0, seed, max_batch, concurrent_window)
        self.device_ms = 0.0

    def build(self, vectors):
        lib = nat.init()
        h = C.c_void_p()
        ms = C.c_double()
        check(lib.jv_graph_build(vectors._h, int(self.vsf), C.byref(self.params), C.byref(h), C.byref(ms)))
        self.device_ms = ms.value
        s, b, d = C.c_int64(), C.c_int64(), C.c_int64()
        lib.jv_graph_build_stats(C.byref(s), C.byref(b), C.byref(d))
        self.scored_vectors, self.batches, self.dropped_backlinks = s.value, b.value, d.value
        return GraphIndex(_handle=h)

    def removeDeletedNodes(self, graph, vectors, deleted):
        """GraphIndexBuilder.markNodeDeleted + cleanup's removeDeletedNodes (GraphIndexBuilder.java:689-799) on the device.

        deleted: bool mask [n] or an array of node ids. Returns a NEW GraphIndex (`graph` is left as it is) in which those nodes are
        holes — no row names them, their own rows are empty, they belong to no upper level — and every live row that named one
        was re-pruned with this builder's similarity function and alpha over its live neighbours and its deleted neighbours' live
        neighbours (random live members of its level, seeded by this builder's seed, when those offer none). The result carries
        `.remove_stats` (jv_remove_stats as a dict) and no FusedPQ records: call fuse_pq on it again if needed.

        Until this is called, a graph with marked nodes is searched with GraphSearcher.search(..., acceptOrds=~deleted): the marked
        nodes stay on the search paths but are never returned."""
        lib = nat.init()
        n = graph.info()["n"]
        d = np.asarray(deleted)
        if d.dtype == bool:
            if d.shape != (n,):
                raise ValueError("deleted mask has shape %s, the graph has %d nodes" % (d.shape, n))
            mask = d
        else:
            ids = d.astype(np.int64).ravel()
            if ids.size and (ids.min() < 0 or ids.max() >= n):
                raise ValueError("deleted ids outside [0, %d)" % n)
            mask = np.zeros(n, bool)
            mask[ids] = True
        bits = pack_accept_bits(mask)
        st = nat.RemoveStats()
        h = C.c_void_p()
        check(lib.jv_graph_remove_deleted(graph._h, vectors._h, int(self.vsf), float(self.params.alpha), int(self.params.seed),
                                          bits.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(h), C.byref(st)))
        out = GraphIndex(_handle=h)
        out.remove_stats = {name: getattr(st, name) for name, _ in nat.RemoveStats._fields_}
        return out
