// jvector_b200.hpp — header-only C++ host mirror of the reference's scoring interface over the C ABI (jvector_b200.h).
//
// The reference host is Java; no JDK exists in this image, so the host-side mirror the tests can COMPILE is C++ (and the
// ctypes layer in jvector_b200/api.py). Names and argument meaning follow the reference:
//   VectorSimilarityFunction                       base:vector/VectorSimilarityFunction.java:34-80
//   ScoreFunction::similarityTo / similarityToBatch base:graph/similarity/ScoreFunction.java:30-80 (+ the batch form)
//   F32Vectors / PQVectors / BQVectors / NVQVectors  RandomAccessVectorValues / CompressedVectors, resident in HBM
//   GraphSearcher::search(topK, rerankK)            base:graph/GraphSearcher.java:222-243, for a batch of queries
//   GraphIndexBuilder(M, beamWidth, neighborOverflow, alpha, addHierarchy)::build   base:graph/GraphIndexBuilder.java:436-448
// Errors: the reference throws (UnsupportedOperationException at provider load, IllegalArgumentException on bad arguments);
// here every non-zero status becomes a jv::Error carrying jv_last_error(). No CPU fallback.
#ifndef JVECTOR_B200_HPP
#define JVECTOR_B200_HPP

#include <cstdint>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "jvector_b200.h"

namespace jv {

enum class VectorSimilarityFunction : int { EUCLIDEAN = JV_EUCLIDEAN, DOT_PRODUCT = JV_DOT_PRODUCT, COSINE = JV_COSINE };

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string &m) : std::runtime_error("jvector_b200 error " + std::to_string(c) + ": " + m), code(c) {}
};
inline void check(int rc)
{
    if (rc != JV_OK) throw Error(rc, jv_last_error());
}
/// NativeVectorizationProvider's constructor: throws when no sm_90 device can be bound (caller falls back to Panama)
inline void init(int device = 0) { check(jv_gpu_init(device)); }

class Vectors {
public:
    Vectors(const Vectors &) = delete;
    Vectors &operator=(const Vectors &) = delete;
    Vectors(Vectors &&o) noexcept : h_(o.h_) { o.h_ = nullptr; }
    ~Vectors() { if (h_) jv_dataset_free(h_); }
    int64_t size() const { return jv_dataset_size(h_); }
    int dimension() const { return jv_dataset_dim(h_); }
    jv_dataset handle() const { return h_; }
    /// BuildScoreProvider.diversityProviderFor: score(a[i], b[i]) for every pair, one launch
    std::vector<float> diversityScores(const std::vector<int32_t> &a, const std::vector<int32_t> &b, VectorSimilarityFunction vsf) const
    {
        std::vector<float> out(a.size());
        check(jv_score_pairs(h_, (int)vsf, a.data(), b.data(), (int)a.size(), out.data()));
        return out;
    }

protected:
    Vectors() = default;
    jv_dataset h_ = nullptr;
};

struct F32Vectors : Vectors {
    F32Vectors(const float *rows, int64_t n, int dim) { check(jv_dataset_register_f32(rows, n, dim, &h_)); }
    explicit F32Vectors(jv_dataset h) { h_ = h; }
};
struct PQVectors : Vectors {
    PQVectors(const uint8_t *codes, int64_t n, int dim, int M, int k, const float *codebooks, const float *centroid = nullptr)
        : M(M), k(k), hasCentroid(centroid != nullptr)
    {
        check(jv_dataset_register_pq(codes, n, dim, M, k, codebooks, centroid, &h_));
    }
    PQVectors(jv_dataset h, int M, int k, bool hasCentroid) : M(M), k(k), hasCentroid(hasCentroid) { h_ = h; }
    /// the codes [n][M], codebooks [k * dim] and centroid ([dim], empty when there is none) copied back from HBM
    void download(std::vector<uint8_t> &codes, std::vector<float> &codebooks, std::vector<float> &centroid) const
    {
        codes.resize((size_t)size() * M);
        codebooks.resize((size_t)k * dimension());
        centroid.resize(hasCentroid ? dimension() : 0);
        check(jv_dataset_pq_download(h_, codes.data(), codebooks.data(), hasCentroid ? centroid.data() : nullptr));
    }
    int M = 0, k = 0;
    bool hasCentroid = false;
};
struct BQVectors : Vectors {
    BQVectors(const uint64_t *words, int64_t n, int dim) { check(jv_dataset_register_bq(words, n, dim, &h_)); }
};
struct NVQVectors : Vectors {
    NVQVectors(const uint8_t *bytes, const float *params, int64_t n, int dim, int nsub, const float *mean)
    {
        check(jv_dataset_register_nvq(bytes, params, n, dim, nsub, mean, &h_));
    }
};

/// ScoreFunction for one query (CompressedVectors.precomputedScoreFunctionFor / DefaultSearchScoreProvider.exact)
class ScoreFunction {
public:
    ScoreFunction(const Vectors &v, const float *query, VectorSimilarityFunction vsf) { check(jv_query_begin(v.handle(), query, (int)vsf, &q_)); }
    ScoreFunction(const ScoreFunction &) = delete;
    ScoreFunction &operator=(const ScoreFunction &) = delete;
    ~ScoreFunction() { if (q_) jv_query_end(q_); }
    /// the neighbour loop of one processNeighbors call / one rerank list: ONE kernel launch
    void similarityToBatch(const int32_t *ids, int n, float *out) const { check(jv_score_batch(q_, ids, n, out)); }
    std::vector<float> similarityToBatch(const std::vector<int32_t> &ids) const
    {
        std::vector<float> out(ids.size());
        similarityToBatch(ids.data(), (int)ids.size(), out.data());
        return out;
    }
    float similarityTo(int32_t node2) const
    {
        float s;
        similarityToBatch(&node2, 1, &s);
        return s;
    }

private:
    jv_query q_ = nullptr;
};

class GraphIndex {
public:
    GraphIndex(int32_t n, int degree, const int32_t *adj0, int32_t entryNode) { check(jv_graph_create(n, degree, adj0, entryNode, &g_)); }
    explicit GraphIndex(jv_graph g) : g_(g) {}
    GraphIndex(const GraphIndex &) = delete;
    GraphIndex &operator=(const GraphIndex &) = delete;
    GraphIndex(GraphIndex &&o) noexcept : g_(o.g_) { o.g_ = nullptr; }
    ~GraphIndex() { if (g_) jv_graph_free(g_); }
    void addLevel(const std::vector<int32_t> &nodeIds, const std::vector<int32_t> &adj) { check(jv_graph_add_level(g_, (int32_t)nodeIds.size(), nodeIds.data(), adj.data())); }
    jv_graph handle() const { return g_; }
    int32_t size() const { int32_t n = 0; check(jv_graph_info(g_, &n, nullptr, nullptr, nullptr)); return n; }
    int maxDegree() const { int d = 0; check(jv_graph_info(g_, nullptr, &d, nullptr, nullptr)); return d; }
    std::vector<int32_t> adjacency(int level = 0) const
    {
        int32_t cnt = 0;
        check(jv_graph_download(g_, level, nullptr, nullptr, &cnt));
        std::vector<int32_t> adj((size_t)cnt * maxDegree());
        check(jv_graph_download(g_, level, nullptr, adj.data(), &cnt));
        return adj;
    }

private:
    jv_graph g_ = nullptr;
};

/// SearchResult (base:graph/SearchResult.java) for a batch: nodes/scores [nq][topK] best first, -1 padded
struct SearchResult {
    std::vector<int32_t> nodes;
    std::vector<float> scores;
    int topK = 0;
    int64_t visitedCount = 0, expandedCount = 0, expandedCountBaseLayer = 0, rerankedCount = 0;
    double deviceMs = 0;
};

class GraphSearcher {
public:
    explicit GraphSearcher(const GraphIndex &g) : g_(g) {}
    SearchResult search(const Vectors &approx, const float *queries, int nq, VectorSimilarityFunction vsf, int topK, int rerankK, const Vectors *reranker = nullptr) const
    {
        SearchResult r;
        r.topK = topK;
        r.nodes.resize((size_t)nq * topK);
        r.scores.resize((size_t)nq * topK);
        jv_search_stats st;
        check(jv_graph_search_batch(g_.handle(), approx.handle(), reranker ? reranker->handle() : nullptr, (int)vsf, queries, nq, topK, rerankK, r.nodes.data(),
                                    r.scores.data(), &st));
        r.visitedCount = st.visited; r.expandedCount = st.expanded; r.expandedCountBaseLayer = st.expanded_base; r.rerankedCount = st.reranked; r.deviceMs = st.device_ms;
        return r;
    }

private:
    const GraphIndex &g_;
};

/// GraphSearcher::search without a graph: every row the options accept is scored (jv_exhaustive_search_batch), for filters too
/// selective for the walk. opts: acceptOrds bitsets, threshold, rerankFloor (nullptr: none)
class ExhaustiveSearcher {
public:
    SearchResult search(const Vectors &approx, const float *queries, int nq, VectorSimilarityFunction vsf, int topK, int rerankK, const Vectors *reranker = nullptr,
                        const jv_search_options *opts = nullptr) const
    {
        SearchResult r;
        r.topK = topK;
        r.nodes.resize((size_t)nq * topK);
        r.scores.resize((size_t)nq * topK);
        jv_search_stats st;
        check(jv_exhaustive_search_batch(approx.handle(), reranker ? reranker->handle() : nullptr, (int)vsf, queries, nq, topK, rerankK, opts, r.nodes.data(),
                                         r.scores.data(), &st));
        r.visitedCount = st.visited; r.expandedCount = st.expanded; r.expandedCountBaseLayer = st.expanded_base; r.rerankedCount = st.reranked; r.deviceMs = st.device_ms;
        return r;
    }
};

/// SegmentSearcher::search's answer: segments / nodes / scores [nq][topK] best first (-1, -1, 0 padded), the call's counters and each
/// segment's (jv_segments_search_batch)
struct SegmentSearchResult {
    std::vector<int32_t> segments, nodes;
    std::vector<float> scores;
    int topK = 0;
    jv_search_stats stats{};
    std::vector<jv_search_stats> segmentStats;
};

/// GraphSearcher::search over several segment graphs (a segment without graph: ExhaustiveSearcher::search), the answers merged per
/// query on the device: score descending, equal scores in segment order, then in the segment's own order
class SegmentSearcher {
public:
    struct Segment {
        const GraphIndex *graph;         // nullptr: every accepted row is scored
        const Vectors *approx;
        const Vectors *reranker;         // nullptr: none
        const uint32_t *acceptBits;      // one bitset over the segment's rows, shared by every query (its live rows); nullptr: all
    };
    explicit SegmentSearcher(std::vector<Segment> segments) : segs_(std::move(segments)) {}
    SegmentSearchResult search(const float *queries, int nq, VectorSimilarityFunction vsf, int topK, int rerankK, float threshold = 0.f,
                               float rerankFloor = 0.f) const
    {
        std::vector<jv_search_segment> s;
        for (const Segment &g : segs_)
            s.push_back({g.graph ? g.graph->handle() : nullptr, g.approx ? g.approx->handle() : nullptr, g.reranker ? g.reranker->handle() : nullptr, g.acceptBits});
        SegmentSearchResult r;
        r.topK = topK;
        r.segments.resize((size_t)nq * topK);
        r.nodes.resize((size_t)nq * topK);
        r.scores.resize((size_t)nq * topK);
        r.segmentStats.resize(s.size());
        check(jv_segments_search_batch(s.data(), (int)s.size(), (int)vsf, queries, nq, topK, rerankK, threshold, rerankFloor, r.segments.data(), r.nodes.data(),
                                       r.scores.data(), &r.stats, r.segmentStats.data()));
        return r;
    }

private:
    std::vector<Segment> segs_;
};

/// exhaustive top-k keys [nq][k] over the rows the options accept (jv_topk_bruteforce_ex; opts nullptr: every row)
inline std::vector<int64_t> topkBruteforce(const Vectors &v, const float *queries, int nq, VectorSimilarityFunction vsf, int k, const jv_search_options *opts = nullptr)
{
    std::vector<int64_t> keys((size_t)nq * k);
    check(jv_topk_bruteforce_ex(v.handle(), (int)vsf, queries, nq, k, opts, keys.data()));
    return keys;
}

class GraphIndexBuilder {
public:
    GraphIndexBuilder(VectorSimilarityFunction vsf, int M, int beamWidth, float neighborOverflow, float alpha, bool addHierarchy, uint64_t seed = 0)
        : vsf_(vsf), p_{M, beamWidth, neighborOverflow, alpha, addHierarchy ? 1 : 0, seed, 0, -1} {}
    GraphIndex build(const F32Vectors &v)
    {
        jv_graph g = nullptr;
        check(jv_graph_build(v.handle(), (int)vsf_, &p_, &g, &deviceMs));
        return GraphIndex(g);
    }
    /// the build over PQ codes (BuildScoreProvider.pqBuildScoreProvider): ADC scores of decode(c_v) for the inserts, the
    /// centroid-pair table for the diversity test (built on v when it has none)
    GraphIndex build(const PQVectors &v)
    {
        jv_graph g = nullptr;
        check(jv_graph_build_pq(v.handle(), (int)vsf_, &p_, &g, &deviceMs));
        return GraphIndex(g);
    }
    /// the build over BQ codes (BuildScoreProvider.bqBuildScoreProvider): every score is 1 - hamming / dim, whatever vsf is
    GraphIndex build(const BQVectors &v)
    {
        jv_graph g = nullptr;
        check(jv_graph_build_bq(v.handle(), (int)vsf_, &p_, &g, &deviceMs));
        return GraphIndex(g);
    }
    /// markNodeDeleted + removeDeletedNodes (GraphIndexBuilder.java:678-799): a NEW graph without the nodes whose bit is set in
    /// deletedBits (bit node & 31 of word node >> 5), their neighbours' lists repaired on the device; `graph` is left as it is.
    /// Until then, search the marked graph with acceptOrds excluding them. Counters go to removeStats.
    GraphIndex removeDeletedNodes(const GraphIndex &graph, const F32Vectors &v, const std::vector<uint32_t> &deletedBits)
    {
        if ((int64_t)deletedBits.size() * 32 < (int64_t)graph.size()) throw Error(JV_ERR_INVALID, "removeDeletedNodes: deletedBits shorter than the graph");
        jv_graph g = nullptr;
        check(jv_graph_remove_deleted(graph.handle(), v.handle(), (int)vsf_, p_.alpha, p_.seed, deletedBits.data(), &g, &removeStats));
        return GraphIndex(g);
    }
    /// removeDeletedNodes over the graph's PQ codes (jv_graph_remove_deleted_pq): the scores of build(const PQVectors &)
    GraphIndex removeDeletedNodes(const GraphIndex &graph, const PQVectors &v, const std::vector<uint32_t> &deletedBits)
    {
        if ((int64_t)deletedBits.size() * 32 < (int64_t)graph.size()) throw Error(JV_ERR_INVALID, "removeDeletedNodes: deletedBits shorter than the graph");
        jv_graph g = nullptr;
        check(jv_graph_remove_deleted_pq(graph.handle(), v.handle(), (int)vsf_, p_.alpha, p_.seed, deletedBits.data(), &g, &removeStats));
        return GraphIndex(g);
    }
    /// removeDeletedNodes over the graph's BQ codes (jv_graph_remove_deleted_bq): the scores of build(const BQVectors &)
    GraphIndex removeDeletedNodes(const GraphIndex &graph, const BQVectors &v, const std::vector<uint32_t> &deletedBits)
    {
        if ((int64_t)deletedBits.size() * 32 < (int64_t)graph.size()) throw Error(JV_ERR_INVALID, "removeDeletedNodes: deletedBits shorter than the graph");
        jv_graph g = nullptr;
        check(jv_graph_remove_deleted_bq(graph.handle(), v.handle(), (int)vsf_, p_.alpha, p_.seed, deletedBits.data(), &g, &removeStats));
        return GraphIndex(g);
    }
    /// addGraphNode (GraphIndexBuilder.java:588-659) for nodes graph.size() .. v.size() - 1: a NEW graph (`graph` is left as it
    /// is); v's first rows must be graph's own nodes. deletedBits (optional, bit node & 31 of word node >> 5): marked nodes the new
    /// ones never pick as neighbours. The hierarchy follows graph's.
    GraphIndex addGraphNodes(const GraphIndex &graph, const F32Vectors &v, const std::vector<uint32_t> &deletedBits = {})
    {
        if (!deletedBits.empty() && (int64_t)deletedBits.size() * 32 < (int64_t)graph.size()) throw Error(JV_ERR_INVALID, "addGraphNodes: deletedBits shorter than the graph");
        jv_graph g = nullptr;
        check(jv_graph_add_nodes(graph.handle(), v.handle(), (int)vsf_, &p_, deletedBits.empty() ? nullptr : deletedBits.data(), &g, &deviceMs));
        return GraphIndex(g);
    }
    /// addGraphNodes over PQ codes (jv_graph_add_nodes_pq): v holds graph's nodes first, then the new rows' codes (same codebooks)
    GraphIndex addGraphNodes(const GraphIndex &graph, const PQVectors &v, const std::vector<uint32_t> &deletedBits = {})
    {
        if (!deletedBits.empty() && (int64_t)deletedBits.size() * 32 < (int64_t)graph.size()) throw Error(JV_ERR_INVALID, "addGraphNodes: deletedBits shorter than the graph");
        jv_graph g = nullptr;
        check(jv_graph_add_nodes_pq(graph.handle(), v.handle(), (int)vsf_, &p_, deletedBits.empty() ? nullptr : deletedBits.data(), &g, &deviceMs));
        return GraphIndex(g);
    }
    /// addGraphNodes over BQ codes (jv_graph_add_nodes_bq): v holds graph's nodes first, then the new rows' words
    GraphIndex addGraphNodes(const GraphIndex &graph, const BQVectors &v, const std::vector<uint32_t> &deletedBits = {})
    {
        if (!deletedBits.empty() && (int64_t)deletedBits.size() * 32 < (int64_t)graph.size()) throw Error(JV_ERR_INVALID, "addGraphNodes: deletedBits shorter than the graph");
        jv_graph g = nullptr;
        check(jv_graph_add_nodes_bq(graph.handle(), v.handle(), (int)vsf_, &p_, deletedBits.empty() ? nullptr : deletedBits.data(), &g, &deviceMs));
        return GraphIndex(g);
    }
    /// cleanup()'s improveConnections (jv_graph_refine, JV_REFINE_BUILDER): a NEW graph; the counters go to refineStats
    template <typename V>
    GraphIndex refine(const GraphIndex &graph, const V &v)
    {
        jv_graph g = nullptr;
        check(jv_graph_refine(graph.handle(), v.handle(), (int)vsf_, &p_, JV_REFINE_BUILDER, &g, &refineStats));
        return GraphIndex(g);
    }
    double deviceMs = 0;
    jv_remove_stats removeStats = {};
    jv_refine_stats refineStats = {};

private:
    VectorSimilarityFunction vsf_;
    jv_build_params p_;
};

/// OnDiskGraphIndexCompactor's merge (jv_graph_compact): sources[i] is graph i with its rows, liveBits[i] its live nodes (bit
/// node & 31 of word node >> 5; empty = every node but holes) and remappers[i] its old id -> new id map. compact() returns the
/// merged graph and its rows in new-id order; the counters go to stats.
/// Over (graph, rows, PQ codes) triples, compactPQ() merges with PQ (jv_graph_compact_pq: FusedPQ sources walked by their records,
/// or sidecar codes) and returns the merged graph, its rows and their codes under the retrained codebooks (in codebooks / centroid);
/// the counters go to pqStats and samplesPerSource.
class GraphIndexCompactor {
public:
    GraphIndexCompactor(std::vector<std::pair<const GraphIndex *, const F32Vectors *>> sources, std::vector<std::vector<uint32_t>> liveBits,
                        std::vector<std::vector<int32_t>> remappers, VectorSimilarityFunction vsf, float alpha = 1.2f)
        : sources_(std::move(sources)), live_(std::move(liveBits)), maps_(std::move(remappers)), vsf_(vsf), alpha_(alpha) {}
    GraphIndexCompactor(const std::vector<std::tuple<const GraphIndex *, const F32Vectors *, const PQVectors *>> &sources,
                        std::vector<std::vector<uint32_t>> liveBits, std::vector<std::vector<int32_t>> remappers, VectorSimilarityFunction vsf,
                        float alpha = 1.2f, uint64_t seed = 0)
        : live_(std::move(liveBits)), maps_(std::move(remappers)), vsf_(vsf), alpha_(alpha), seed_(seed)
    {
        for (const auto &t : sources) {
            sources_.emplace_back(std::get<0>(t), std::get<1>(t));
            pq_.push_back(std::get<2>(t));
        }
    }
    std::pair<GraphIndex, F32Vectors> compact()
    {
        const std::vector<jv_compact_source> src = sources();
        jv_graph g = nullptr;
        jv_dataset rows = nullptr;
        check(jv_graph_compact(src.data(), (int)src.size(), (int)vsf_, alpha_, &g, &rows, &stats));
        GraphIndex merged(g);
        F32Vectors merged_rows(rows);
        if (!refine_) return {std::move(merged), std::move(merged_rows)};
        return {refine(merged, merged_rows), std::move(merged_rows)};
    }
    std::tuple<GraphIndex, F32Vectors, PQVectors> compactPQ()
    {
        const std::vector<jv_compact_source> src = sources();
        if (pq_.size() != src.size() || pq_.empty()) throw Error(JV_ERR_INVALID, "compactPQ: one PQ data set per source");
        std::vector<jv_dataset> pqs;
        for (const PQVectors *p : pq_) pqs.push_back(p->handle());
        const PQVectors &p0 = *pq_[0];
        codebooks.assign((size_t)p0.k * sources_[0].second->dimension(), 0.f);
        centroid.assign(p0.hasCentroid ? sources_[0].second->dimension() : 0, 0.f);
        samplesPerSource.assign(src.size(), 0);
        jv_graph g = nullptr;
        jv_dataset rows = nullptr, codes = nullptr;
        check(jv_graph_compact_pq(src.data(), pqs.data(), (int)src.size(), (int)vsf_, alpha_, seed_, &g, &rows, &codes, codebooks.data(),
                                  p0.hasCentroid ? centroid.data() : nullptr, samplesPerSource.data(), &pqStats));
        stats = pqStats.graph;
        GraphIndex merged(g);
        F32Vectors merged_rows(rows);
        PQVectors merged_codes(codes, p0.M, p0.k, p0.hasCentroid);
        if (!refine_) return {std::move(merged), std::move(merged_rows), std::move(merged_codes)};
        GraphIndex refined = refine(merged, merged_rows);
        if (pqStats.fused) check(jv_graph_fuse_pq(refined.handle(), merged_codes.handle()));
        return {std::move(refined), std::move(merged_rows), std::move(merged_codes)};
    }
    void setRefineAfterCompaction(bool refine) { refine_ = refine; }
    jv_compact_stats stats = {};
    jv_refine_stats refineStats = {};
    jv_compact_pq_stats pqStats = {};
    std::vector<float> codebooks, centroid;
    std::vector<int64_t> samplesPerSource;

private:
    std::vector<jv_compact_source> sources() const
    {
        if (live_.size() != sources_.size() || maps_.size() != sources_.size()) throw Error(JV_ERR_INVALID, "compact: one live set and one map per source");
        std::vector<jv_compact_source> src(sources_.size());
        for (size_t i = 0; i < sources_.size(); i++) {
            const int32_t n = sources_[i].first->size();
            if ((int64_t)maps_[i].size() < n || (!live_[i].empty() && (int64_t)live_[i].size() * 32 < n))
                throw Error(JV_ERR_INVALID, "compact: a live set or a map shorter than its graph");
            src[i] = {sources_[i].first->handle(), sources_[i].second->handle(), live_[i].empty() ? nullptr : live_[i].data(), maps_[i].data()};
        }
        return src;
    }
    // the compactor's refine pass (jv_graph_refine, JV_REFINE_COMPACTOR) at alpha; beam, overflow and batch are only validated
    GraphIndex refine(const GraphIndex &merged, const F32Vectors &rows)
    {
        jv_build_params p = {merged.maxDegree(), 100, 1.2f, alpha_, 0, seed_, 0, -1};
        jv_graph r = nullptr;
        check(jv_graph_refine(merged.handle(), rows.handle(), (int)vsf_, &p, JV_REFINE_COMPACTOR, &r, &refineStats));
        return GraphIndex(r);
    }
    std::vector<std::pair<const GraphIndex *, const F32Vectors *>> sources_;
    std::vector<std::vector<uint32_t>> live_;
    std::vector<std::vector<int32_t>> maps_;
    VectorSimilarityFunction vsf_;
    float alpha_;
    bool refine_ = false;
    uint64_t seed_ = 0;
    std::vector<const PQVectors *> pq_;
};

}  // namespace jv
#endif
