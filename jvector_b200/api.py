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

    def row_sketch(self):
        """the int8 row sketch a DOT_PRODUCT graph search of a batch that fills the GPU builds (never built here):
        (codes [n][sketch_stride] int8, meta [n][2] float32 = {scale, radius}), or None while no search has built it"""
        lib = nat.load()
        ss = C.c_int(0)
        rc = lib.jv_dataset_row_sketch_download(self._h, None, None, C.byref(ss))
        if rc != 0 and ss.value > 0:  # the stride is set for every fp32 data set: this one has no sketch yet
            return None
        check(rc)
        n = self.size()
        codes = np.empty((n, ss.value), np.int8)
        meta = np.empty((n, 2), np.float32)
        check(lib.jv_dataset_row_sketch_download(self._h, codes.ctypes.data, fp(meta), None))
        return codes, meta


class PQVectors(_Vectors):
    """base:quantization/PQVectors.java — codes [n][M] + codebooks (concatenated, codebook m = [k][size_m])."""

    def __init__(self, codes, codebooks, dim, k=256, centroid=None):
        lib = nat.init()
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        codebooks = c32(codebooks).reshape(-1)
        cen = c32(centroid) if centroid is not None else None
        assert codebooks.size == k * dim
        self.M, self.k, self.has_centroid = codes.shape[1], k, cen is not None
        h = C.c_void_p()
        check(lib.jv_dataset_register_pq(bp(codes), codes.shape[0], dim, codes.shape[1], k, fp(codebooks), fp(cen), C.byref(h)))
        super().__init__(h, None)

    @classmethod
    def _adopt(cls, handle, M, k, has_centroid):
        """a resident PQ data set the library made (jv_pq_encode_dataset_resident, jv_graph_compact_pq)"""
        v = cls.__new__(cls)
        v.M, v.k, v.has_centroid = M, k, has_centroid
        _Vectors.__init__(v, handle, None)
        return v

    def download(self):
        """(codes uint8 [n][M], codebooks float32 [k * dim], centroid float32 [dim] or None), copied back from HBM"""
        codes = np.empty((self.size(), self.M), np.uint8)
        codebooks = np.empty(self.k * self.dimension(), np.float32)
        centroid = np.empty(self.dimension(), np.float32) if self.has_centroid else None
        check(nat.load().jv_dataset_pq_download(self._h, bp(codes), fp(codebooks), fp(centroid)))
        return codes, codebooks, centroid

    def build_pair_table(self, vsf):
        """ImmutablePQVectors: the triangular centroid-vs-centroid table in HBM; diversity_scores then sums table entries"""
        check(nat.load().jv_dataset_pq_pair_table(self._h, int(vsf)))
        return self

    def pair_table(self, vsf):
        out = np.empty(self.M * (self.k * (self.k + 1) // 2), dtype=np.float32)
        check(nat.load().jv_dataset_pq_pair_table_download(self._h, int(vsf), fp(out)))
        return out


class ProductQuantization:
    """base:quantization/ProductQuantization.java, trained on the device (jv_pq_train / jv_pq_refine, or their _anisotropic forms
    when anisotropicThreshold > UNWEIGHTED). codebooks: float32 [k * dim] (codebook m = [k][size_m] at k * offset_m); centroid: the
    global centroid or None; anisotropicThreshold: the T the codebooks were trained or refined with, which encodeAll also uses."""

    K_MEANS_ITERATIONS = 6
    UNWEIGHTED = -1.0

    def __init__(self, codebooks, M, k, dim, centroid=None, stats=None, anisotropicThreshold=UNWEIGHTED):
        self.codebooks, self.M, self.k, self.dim, self.centroid, self.stats = codebooks, M, k, dim, centroid, stats
        self.anisotropicThreshold = float(anisotropicThreshold)

    @staticmethod
    def _stats(st):
        return {name: getattr(st, name) for name, _ in nat.PQTrainStats._fields_}

    @classmethod
    def _astats(cls, st):
        out = cls._stats(st.lloyd)
        out.update({name: getattr(st, name) for name, _ in nat.PQAnisotropicStats._fields_[1:]})
        return out

    @classmethod
    def compute(cls, vectors, M, clusterCount=256, globallyCenter=False, seed=0, anisotropicThreshold=UNWEIGHTED):
        """ProductQuantization.compute over F32Vectors resident in HBM: at most 128 000 sampled training rows, k-means++ seeding,
        K_MEANS_ITERATIONS Lloyd iterations with the reference's early stop, then (anisotropicThreshold > UNWEIGHTED) as many
        anisotropic rounds. The result is a pure function of the rows, the seed and the threshold."""
        lib = nat.init()
        dim = vectors.dimension()
        p = nat.PQTrainParams(M, clusterCount, 1 if globallyCenter else 0, cls.K_MEANS_ITERATIONS, 0, seed)
        cb = np.empty(clusterCount * dim, np.float32)
        cen = np.empty(dim, np.float32) if globallyCenter else None
        if anisotropicThreshold == cls.UNWEIGHTED:
            st = nat.PQTrainStats()
            check(lib.jv_pq_train(vectors._h, C.byref(p), fp(cb), fp(cen), C.byref(st)))
            return cls(cb, M, clusterCount, dim, cen, cls._stats(st))
        st = nat.PQAnisotropicStats()
        check(lib.jv_pq_train_anisotropic(vectors._h, C.byref(p), anisotropicThreshold, fp(cb), fp(cen), C.byref(st)))
        return cls(cb, M, clusterCount, dim, cen, cls._astats(st), anisotropicThreshold)

    def refine(self, vectors, lloydsRounds=1, seed=0, anisotropicThreshold=UNWEIGHTED):
        """ProductQuantization.refine: lloydsRounds Lloyd iterations (anisotropic rounds when anisotropicThreshold > UNWEIGHTED)
        from these codebooks over `vectors` (minus the centroid); returns a new ProductQuantization with the same centroid and
        the threshold it was refined with."""
        lib = nat.init()
        p = nat.PQTrainParams(self.M, self.k, 0, lloydsRounds, 0, seed)
        cb = np.empty_like(self.codebooks)
        if anisotropicThreshold == self.UNWEIGHTED:
            st = nat.PQTrainStats()
            check(lib.jv_pq_refine(vectors._h, C.byref(p), fp(self.codebooks), fp(self.centroid), fp(cb), C.byref(st)))
            return ProductQuantization(cb, self.M, self.k, self.dim, self.centroid, self._stats(st))
        st = nat.PQAnisotropicStats()
        check(lib.jv_pq_refine_anisotropic(vectors._h, C.byref(p), anisotropicThreshold, fp(self.codebooks), fp(self.centroid), fp(cb),
                                           C.byref(st)))
        return ProductQuantization(cb, self.M, self.k, self.dim, self.centroid, self._astats(st), anisotropicThreshold)

    def encodeAll(self, vectors):
        """ProductQuantization.encodeAll of resident F32Vectors into resident PQVectors (the anisotropic encoder when the
        threshold is above UNWEIGHTED)"""
        if self.anisotropicThreshold > self.UNWEIGHTED:
            codes = pq_encode_all_anisotropic(vectors, self.codebooks, self.M, self.k, self.centroid, self.anisotropicThreshold)[0]
        else:
            codes = pq_encode_all(vectors, self.codebooks, self.M, self.k, self.centroid)
        return PQVectors(codes, self.codebooks, self.dim, self.k, self.centroid)


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


def _search_options(threshold, rerankFloor, acceptOrds):
    """jv_search_options for GraphSearcher.search's filter arguments (None when there is no filter), and the packed bitsets it
    points at (keep them alive for the call)"""
    if acceptOrds is None and threshold == 0 and rerankFloor == 0:
        return None, None
    opts = nat.SearchOptions(None, 0, float(threshold), float(rerankFloor))
    bits = None
    if acceptOrds is not None:
        bits = pack_accept_bits(acceptOrds)
        opts.accept_bits = bits.ctypes.data
        opts.accept_stride_words = bits.shape[1] if bits.ndim == 2 else 0
    return opts, bits


def topk_bruteforce(vectors, vsf, queries, k, acceptOrds=None, threshold=0.0):
    """Exhaustive first pass with the reference's ordering key; returns (nodes [nq][k], scores [nq][k], keys).
    acceptOrds (a bool array [n] shared by the batch, or [nq][n] one per query) and threshold restrict it to the accepted rows
    scoring >= threshold (jv_topk_bruteforce_ex)."""
    lib = nat.init()
    queries = c32(queries)
    keys = np.empty((queries.shape[0], k), dtype=np.int64)
    if acceptOrds is None and threshold == 0:
        check(lib.jv_topk_bruteforce(vectors._h, int(vsf), fp(queries), queries.shape[0], k, lp(keys)))
    else:
        opts, bits = _search_options(threshold, 0.0, acceptOrds)
        check(lib.jv_topk_bruteforce_ex(vectors._h, int(vsf), fp(queries), queries.shape[0], k, C.byref(opts) if opts is not None else None, lp(keys)))
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


def pq_encode_all_anisotropic(rows, codebooks, M, k, centroid, anisotropicThreshold):
    """ProductQuantization.encodeAll with an anisotropic threshold (encodeAnisotropic for T > -1). rows: a host array, or
    F32Vectors resident in HBM. Returns (codes [n][M] uint8, stats dict: rows_moved, moves, max_sweeps, device_ms)."""
    lib = nat.init()
    codebooks = c32(codebooks).reshape(-1)
    cen = c32(centroid) if centroid is not None else None
    st = nat.PQEncodeStats()
    if isinstance(rows, _Vectors):
        out = np.empty((rows.size(), M), dtype=np.uint8)
        check(lib.jv_pq_encode_dataset_anisotropic(rows._h, M, k, fp(codebooks), fp(cen), anisotropicThreshold, bp(out), C.byref(st)))
    else:
        rows = c32(rows)
        out = np.empty((rows.shape[0], M), dtype=np.uint8)
        check(lib.jv_pq_encode_batch_anisotropic(fp(rows), rows.shape[0], rows.shape[1], M, k, fp(codebooks), fp(cen), anisotropicThreshold,
                                                 bp(out), C.byref(st)))
    return out, {name: getattr(st, name) for name, _ in nat.PQEncodeStats._fields_}


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


def pq_encode_resident(f32_vectors, codebooks, M, k=256, centroid=None):
    """ProductQuantization.encodeAll of rows already in HBM into new resident PQVectors (no host round trip)."""
    lib = nat.init()
    codebooks = c32(codebooks).reshape(-1)
    cen = c32(centroid) if centroid is not None else None
    h = C.c_void_p()
    check(lib.jv_pq_encode_dataset_resident(f32_vectors._h, M, k, fp(codebooks), fp(cen), C.byref(h)))
    return PQVectors._adopt(h, M, k, cen is not None)


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


class ExhaustiveSearcher:
    """GraphSearcher.search without a graph: every row acceptOrds accepts is scored exactly by `approx` (jv_exhaustive_search_batch),
    at about what the accepted rows cost. For filters too selective for the graph walk; same arguments and SearchResult, so a caller
    can pick the searcher per batch on the filter's density."""

    def search(self, approx, queries, vsf, topK, rerankK=None, reranker=None, threshold=0.0, rerankFloor=0.0, acceptOrds=None):
        lib = nat.init()
        queries = c32(queries)
        if queries.shape[1] != approx.dimension():
            raise ValueError("query dimension %d != data set dimension %d" % (queries.shape[1], approx.dimension()))
        rerankK = rerankK or topK
        nq = queries.shape[0]
        nodes = np.empty((nq, topK), dtype=np.int32)
        scores = np.empty((nq, topK), dtype=np.float32)
        st = nat.SearchStats()
        opts, bits = _search_options(threshold, rerankFloor, acceptOrds)
        check(lib.jv_exhaustive_search_batch(approx._h, reranker._h if reranker is not None else None, int(vsf), fp(queries), nq, topK, rerankK,
                                             C.byref(opts) if opts is not None else None, ip(nodes), fp(scores), C.byref(st)))
        return SearchResult(nodes, scores, st)


class SegmentSearchResult:
    """SegmentSearcher.search's answer: segments / nodes / scores [nq][topK] best first (segment -1, node -1, score 0 padded), the
    call's counters (`stats`, a SearchResult's counters without its arrays) and each segment's (`segment_stats`, a list)."""

    def __init__(self, segments, nodes, scores, stats, segment_stats):
        self.segments, self.nodes, self.scores = segments, nodes, scores
        self.stats = SearchResult(None, None, stats)
        self.segment_stats = [SearchResult(None, None, st) for st in segment_stats]


class SegmentSearcher:
    """One index split into segments, each searched as GraphSearcher.search (or, without a graph, ExhaustiveSearcher.search) searches
    it, and the answers merged per query on the device (jv_segments_search_batch): score descending, equal scores in segment order,
    then in each segment's own order. segments: a list of (graph or None, approx, reranker=None, acceptOrds=None), acceptOrds a bool
    array over the segment's rows shared by every query (its live rows)."""

    def __init__(self, segments):
        self.segments = [tuple(s) + (None,) * (4 - len(s)) for s in segments]
        if not self.segments:
            raise ValueError("SegmentSearcher needs at least one segment")

    def search(self, queries, vsf, topK, rerankK=None, threshold=0.0, rerankFloor=0.0):
        lib = nat.init()
        queries = c32(queries)
        dim = self.segments[0][1].dimension()
        if queries.shape[1] != dim:
            raise ValueError("query dimension %d != data set dimension %d" % (queries.shape[1], dim))
        rerankK = rerankK or topK
        nq, S = queries.shape[0], len(self.segments)
        arr = (nat.SearchSegment * S)()
        keep = []  # the packed bitsets live until the call returns
        for i, (graph, approx, reranker, accept) in enumerate(self.segments):
            bits = None
            if accept is not None:
                bits = pack_accept_bits(accept)
                if bits.ndim != 1:
                    raise ValueError("segment %d: acceptOrds is one bool array over the segment's rows" % i)
                keep.append(bits)
            arr[i] = nat.SearchSegment(graph._h if graph is not None else None, approx._h, reranker._h if reranker is not None else None,
                                       bits.ctypes.data if bits is not None else None)
        segs = np.empty((nq, topK), dtype=np.int32)
        nodes = np.empty((nq, topK), dtype=np.int32)
        scores = np.empty((nq, topK), dtype=np.float32)
        st = nat.SearchStats()
        sst = (nat.SearchStats * S)()
        check(lib.jv_segments_search_batch(arr, S, int(vsf), fp(queries), nq, topK, rerankK, float(threshold), float(rerankFloor), ip(segs), ip(nodes),
                                           fp(scores), C.byref(st), sst))
        return SegmentSearchResult(segs, nodes, scores, st, list(sst))


def pack_accept_bits(mask):
    """bool [n] or [nq][n] -> uint32 words, bit (node & 31) of word (node >> 5) (the layout jv_search_options.accept_bits takes)"""
    m = np.asarray(mask, dtype=bool)
    n = m.shape[-1]
    pad = (-n) % 32
    if pad:
        m = np.concatenate([m, np.zeros(m.shape[:-1] + (pad,), bool)], axis=-1)
    return np.ascontiguousarray(np.packbits(m, axis=-1, bitorder="little").view(np.uint32))


def _by_kind(vectors, f32, pq, bq):
    """the entry point of the kind of `vectors`: fp32 rows, PQ codes or BQ codes"""
    return pq if isinstance(vectors, PQVectors) else bq if isinstance(vectors, BQVectors) else f32


class GraphIndexBuilder:
    """base:graph/GraphIndexBuilder.java: (M, beamWidth, neighborOverflow, alpha, addHierarchy) over exact fp32 scores, over PQ
    codes (BuildScoreProvider.pqBuildScoreProvider) when build(), addGraphNodes() or removeDeletedNodes() is given PQVectors, or over
    BQ codes (BuildScoreProvider.bqBuildScoreProvider) when they are given BQVectors."""

    def __init__(self, vsf, M=32, beamWidth=100, neighborOverflow=1.2, alpha=1.2, addHierarchy=False, seed=0, max_batch=0, concurrent_window=-1,
                 refineFinalGraph=False):
        """refineFinalGraph: build() ends with refine() of its graph, as the reference's cleanup() does. The reference's default is true;
        here it is False, so that a build gives the graph it always gave unless the refine is asked for."""
        self.vsf = vsf
        self.params = nat.BuildParams(M, beamWidth, neighborOverflow, alpha, 1 if addHierarchy else 0, seed, max_batch, concurrent_window)
        self.refineFinalGraph = bool(refineFinalGraph)
        self.device_ms = 0.0

    def build(self, vectors):
        """F32Vectors: exact scores (jv_graph_build). PQVectors: the inserts walk the codes with decode(c_v) as the query and the
        prune compares codes through the centroid-pair table (jv_graph_build_pq), which it builds on the data set if needed.
        BQVectors: the inserts walk the codes with c_v as the query and every score is 1 - hamming / dim (jv_graph_build_bq), whatever
        the similarity function."""
        lib = nat.init()
        h = C.c_void_p()
        ms = C.c_double()
        fn = _by_kind(vectors, lib.jv_graph_build, lib.jv_graph_build_pq, lib.jv_graph_build_bq)
        check(fn(vectors._h, int(self.vsf), C.byref(self.params), C.byref(h), C.byref(ms)))
        self.device_ms = ms.value
        s, b, d = C.c_int64(), C.c_int64(), C.c_int64()
        lib.jv_graph_build_stats(C.byref(s), C.byref(b), C.byref(d))
        self.scored_vectors, self.batches, self.dropped_backlinks = s.value, b.value, d.value
        g = GraphIndex(_handle=h)
        if not self.refineFinalGraph:
            return g
        try:
            return self.refine(g, vectors)
        finally:
            g.close()

    def refine(self, graph, vectors):
        """GraphIndexBuilder.cleanup's improveConnections on the device (jv_graph_refine, JV_REFINE_BUILDER): the step a caller runs
        after addGraphNodes or removeDeletedNodes. Every member of level 1 is refined at level 0 and every member of a level L >= 1 at L:
        a search of the level excluding the node, its row merged with the results, the robust prune at alpha, back-links, and the
        re-prune of rows past neighborOverflow * M; at the end every row is cut to M. A graph without upper levels comes back as a copy.
        vectors: the graph's F32Vectors, PQVectors or BQVectors, scored as build() scores them. Returns a NEW GraphIndex (`graph` is left
        as it is, its holes, entry and levels are kept) carrying `.refine_stats` (jv_refine_stats as a dict) and no FusedPQ records."""
        return _refine(graph, vectors, self.vsf, self.params, nat.REFINE_BUILDER)

    def removeDeletedNodes(self, graph, vectors, deleted):
        """GraphIndexBuilder.markNodeDeleted + cleanup's removeDeletedNodes (GraphIndexBuilder.java:689-799) on the device.

        deleted: bool mask [n] or an array of node ids. Returns a NEW GraphIndex (`graph` is left as it is) in which those nodes are
        holes — no row names them, their own rows are empty, they belong to no upper level — and every live row that named one
        was re-pruned with this builder's similarity function and alpha over its live neighbours and its deleted neighbours' live
        neighbours (random live members of its level, seeded by this builder's seed, when those offer none). The result carries
        `.remove_stats` (jv_remove_stats as a dict) and no FusedPQ records: call fuse_pq on it again if needed.

        vectors: the graph's F32Vectors (exact scores, jv_graph_remove_deleted) or its PQVectors (jv_graph_remove_deleted_pq): the
        repair of node v then scores with decode(c_v)'s ADC and the centroid-pair table, as build() over PQVectors does. Or its
        BQVectors (jv_graph_remove_deleted_bq): Hamming scores, as build() over BQVectors uses.

        Until this is called, a graph with marked nodes is searched with GraphSearcher.search(..., acceptOrds=~deleted): the marked
        nodes stay on the search paths but are never returned."""
        lib = nat.init()
        bits = _deleted_bits(deleted, graph.info()["n"])
        st = nat.RemoveStats()
        h = C.c_void_p()
        fn = _by_kind(vectors, lib.jv_graph_remove_deleted, lib.jv_graph_remove_deleted_pq, lib.jv_graph_remove_deleted_bq)
        check(fn(graph._h, vectors._h, int(self.vsf), float(self.params.alpha), int(self.params.seed),
                 bits.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(h), C.byref(st)))
        out = GraphIndex(_handle=h)
        out.remove_stats = {name: getattr(st, name) for name, _ in nat.RemoveStats._fields_}
        return out

    def addGraphNodes(self, graph, vectors, deleted=None):
        """GraphIndexBuilder.addGraphNode for every node graph.size() .. vectors.size() - 1, on the device (jv_graph_add_nodes, or
        jv_graph_add_nodes_pq for PQVectors, jv_graph_add_nodes_bq for BQVectors).

        vectors: F32Vectors, PQVectors or BQVectors whose first rows are the graph's own nodes, followed by the new ones. A PQ data set
        grows by encoding the new rows with the same codebooks (ProductQuantization.encodeAll) and wrapping the longer code array in new
        PQVectors; the insert of node v then uses decode(c_v) as its query, as build() over PQVectors does. A BQ data set grows by
        encoding the new rows (bq_encode_all) and wrapping the longer word array in new BQVectors. Returns a NEW GraphIndex (`graph`
        is left as it is), built from the graph's rows with this builder's parameters (M must equal the graph's degree); its holes
        stay holes, the hierarchy follows the graph's (addHierarchy is ignored) and it has no FusedPQ records. deleted: nodes marked
        deleted but not removed yet (a bool mask over the graph's nodes or an array of their ids): the new nodes never pick them as
        neighbours. Sets scored_vectors / batches / dropped_backlinks / device_ms as build() does."""
        lib = nat.init()
        bits = _deleted_bits(deleted, graph.info()["n"]) if deleted is not None else None
        h = C.c_void_p()
        ms = C.c_double()
        fn = _by_kind(vectors, lib.jv_graph_add_nodes, lib.jv_graph_add_nodes_pq, lib.jv_graph_add_nodes_bq)
        check(fn(graph._h, vectors._h, int(self.vsf), C.byref(self.params),
                 bits.ctypes.data_as(C.POINTER(C.c_uint32)) if bits is not None else None, C.byref(h), C.byref(ms)))
        self.device_ms = ms.value
        s, b, d = C.c_int64(), C.c_int64(), C.c_int64()
        lib.jv_graph_build_stats(C.byref(s), C.byref(b), C.byref(d))
        self.scored_vectors, self.batches, self.dropped_backlinks = s.value, b.value, d.value
        return GraphIndex(_handle=h)


class GraphIndexCompactor:
    """graph/disk/OnDiskGraphIndexCompactor.java's merge on the device (jv_graph_compact): several graphs over fp32 rows become one
    graph over their live nodes, with the compactor's candidates (each node's live neighbours in its own source, the searchTopK best
    live members of every other source) and the builder's robust prune at alpha.

    sources: a list of (GraphIndex, F32Vectors), all with one dimension and degree. liveNodes: per source a bool mask over its nodes,
    or None; None (the whole list or an entry) means every node but the source's holes. remappers: per source an int array mapping
    old ids to new ids (read for live nodes, which must map onto exactly [0, live nodes)), or None: the sources in order, each one's
    live nodes in id order (a source with holes from removeDeletedNodes then needs a live mask that leaves them out). compact() returns (GraphIndex, F32Vectors): the merged graph and its rows in new-id order. The sources
    are left as they are; `.stats` holds jv_compact_stats as a dict after compact().

    With sources of (GraphIndex, F32Vectors, PQVectors) the merge carries PQ (jv_graph_compact_pq): when every graph is fused with its
    PQVectors, the other sources are searched over their FusedPQ records with an exact rerank and the merged graph comes back fused;
    when none is fused, the merge is the fp32 one above. Either way PQ is retrained on a balanced sample of the live rows, warm-started
    from source 0's codebooks (PQRetrainer), and compact() returns (GraphIndex, F32Vectors, PQVectors) with the merged rows' codes; `.pq`
    holds the retrained ProductQuantization. seed: the sample's chunk order and the retraining's draws."""

    def __init__(self, sources, liveNodes, remappers, vsf, alpha=1.2, refineAfterCompaction=False, seed=0):
        self.sources, self.vsf, self.alpha = list(sources), vsf, float(alpha)
        self.refineAfterCompaction = bool(refineAfterCompaction)
        self.seed = int(seed)
        arity = {len(s) for s in self.sources}
        if not self.sources or len(arity) != 1 or arity.pop() not in (2, 3):
            raise ValueError("sources: all (GraphIndex, F32Vectors) or all (GraphIndex, F32Vectors, PQVectors)")
        self.with_pq = len(self.sources[0]) == 3
        self.pq = None
        sizes = [s[0].info()["n"] for s in self.sources]
        live = liveNodes if liveNodes is not None else [None] * len(sizes)
        if len(live) != len(sizes):
            raise ValueError("one live mask per source")
        self.live = [None if m is None else np.asarray(m, bool) for m in live]
        for m, n in zip(self.live, sizes):
            if m is not None and m.shape != (n,):
                raise ValueError("live mask has shape %s, its graph has %d nodes" % (m.shape, n))
        if remappers is None:
            remappers, base = [], 0
            for m, n in zip(self.live, sizes):
                alive = np.ones(n, bool) if m is None else m
                r = np.full(n, -1, np.int32)
                r[alive] = base + np.arange(int(alive.sum()), dtype=np.int32)
                remappers.append(r)
                base += int(alive.sum())
        if len(remappers) != len(sizes):
            raise ValueError("one remapper per source")
        self.remappers = [np.ascontiguousarray(r, dtype=np.int32) for r in remappers]
        for r, n in zip(self.remappers, sizes):
            if r.shape != (n,):
                raise ValueError("remapper has shape %s, its graph has %d nodes" % (r.shape, n))
        self.stats = None
        self.refine_stats = None

    def setRefineAfterCompaction(self, refine):
        """whether compact() ends with the compactor's refine pass (jv_graph_refine, JV_REFINE_COMPACTOR) over the merged graph: each
        member of level 1, or each node when the merged graph is flat, gets its level-0 row re-pruned at alpha over its row and a beam
        of 8 M from a search of the merged graph that excludes it; all rows are replaced at the end, without back-links"""
        self.refineAfterCompaction = bool(refine)

    def compact(self):
        lib = nat.init()
        bits = [None if m is None else pack_accept_bits(m) for m in self.live]
        src = (nat.CompactSource * len(self.sources))()
        for i, (s, b, r) in enumerate(zip(self.sources, bits, self.remappers)):
            src[i] = nat.CompactSource(s[0]._h, s[1]._h, b.ctypes.data_as(C.POINTER(C.c_uint32)) if b is not None else None, ip(r))
        gh, rh = C.c_void_p(), C.c_void_p()
        codes = None
        if self.with_pq:
            pq0, dim = self.sources[0][2], self.sources[0][1].dimension()
            pqs = (C.c_void_p * len(self.sources))(*[s[2]._h for s in self.sources])
            cb = np.empty(pq0.k * dim, np.float32)
            cen = np.empty(dim, np.float32) if pq0.has_centroid else None
            samples = np.zeros(len(self.sources), np.int64)
            st = nat.CompactPQStats()
            ph = C.c_void_p()
            check(lib.jv_graph_compact_pq(src, pqs, len(self.sources), int(self.vsf), self.alpha, self.seed, C.byref(gh), C.byref(rh), C.byref(ph),
                                          fp(cb), fp(cen), lp(samples), C.byref(st)))
            self.stats = {name: getattr(st.graph, name) for name, _ in nat.CompactStats._fields_}
            self.stats.update({"fused": st.fused, "train_rows": st.train_rows, "retrain_ms": st.retrain_ms, "encode_ms": st.encode_ms,
                               "fuse_ms": st.fuse_ms, "samples_per_source": samples.tolist(), "train": ProductQuantization._stats(st.train)})
            codes = PQVectors._adopt(ph, pq0.M, pq0.k, cen is not None)
            self.pq = ProductQuantization(cb, pq0.M, pq0.k, dim, cen, self.stats["train"])
        else:
            st = nat.CompactStats()
            check(lib.jv_graph_compact(src, len(self.sources), int(self.vsf), self.alpha, C.byref(gh), C.byref(rh), C.byref(st)))
            self.stats = {name: getattr(st, name) for name, _ in nat.CompactStats._fields_}
        rows = F32Vectors.__new__(F32Vectors)
        _Vectors.__init__(rows, rh, None)
        g = GraphIndex(_handle=gh)
        if self.refineAfterCompaction:
            # the refine walks the merged fp32 rows exactly; a fused merge is fused again with the new codes afterwards
            params = nat.BuildParams(g.info()["degree"], 100, 1.2, self.alpha, 0, self.seed, 0, -1)
            try:
                refined = _refine(g, rows, self.vsf, params, nat.REFINE_COMPACTOR)
                if self.with_pq and self.stats["fused"]:
                    refined.fuse_pq(codes)
            except BaseException:
                rows.close()
                if codes is not None:
                    codes.close()
                raise
            finally:
                g.close()
            self.refine_stats, g = refined.refine_stats, refined
        return (g, rows, codes) if self.with_pq else (g, rows)


def _refine(graph, vectors, vsf, params, mode):
    """jv_graph_refine: a new GraphIndex carrying .refine_stats"""
    lib = nat.init()
    st = nat.RefineStats()
    h = C.c_void_p()
    check(lib.jv_graph_refine(graph._h, vectors._h, int(vsf), C.byref(params), mode, C.byref(h), C.byref(st)))
    out = GraphIndex(_handle=h)
    out.refine_stats = {name: getattr(st, name) for name, _ in nat.RefineStats._fields_}
    out.refine_stats["nodes_refined"] = list(st.nodes_refined)[:max(st.levels, 1)]
    return out


def _deleted_bits(deleted, n):
    """a bool mask [n] or an array of node ids -> the accept_bits layout over n nodes, set = deleted"""
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
    return pack_accept_bits(mask)
