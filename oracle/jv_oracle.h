/*
 * jv_oracle.h — TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement (plain C, scalar, sequential summation) of the JVector scoring hot path, written from the
 * reference's Java/C++ sources. Every function cites the reference file:line it follows (paths relative to
 * /root/reference; `base:` = jvector-base/src/main/java/io/github/jbellis/jvector/, `native-c:` =
 * jvector-native/src/main/native/).
 *
 * Who may use this: tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs, and
 * only as the CHECKER or the CPU baseline. The product (jvector_b200/, libjvector_b200.so) never links, loads
 * or calls anything in oracle/.
 *
 * Pinning: tests/test_oracle_*.py check this restatement against (a) the reference's own compiled kernels
 * (oracle/_ref/libjvector.so, built by oracle/build_ref.sh from /root/reference), (b) the siftsmall ground
 * truth shipped with the reference, (c) the known answers / tolerances of the reference's unit tests
 * (SURVEY.md §8c).
 */
#ifndef JV_ORACLE_H
#define JV_ORACLE_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

enum { JVO_EUCLIDEAN = 0, JVO_DOT_PRODUCT = 1, JVO_COSINE = 2 }; /* base:vector/VectorSimilarityFunction.java:34-69 */

/* ---- float32 similarities ---- */
float jvo_dot_f32(const float *a, const float *b, int n);
float jvo_l2_f32(const float *a, const float *b, int n);
float jvo_cosine_f32(const float *a, const float *b, int n);        /* Java form: divide in double */
float jvo_cosine_native_f32(const float *a, const float *b, int n); /* native form: sqrtf + fp32 divide */
float jvo_score_from_raw(int metric, float raw);
float jvo_compare_f32(int metric, const float *a, const float *b, int n);

/* ---- top-k key ---- */
int32_t jvo_float_to_sortable_int(float f);
int64_t jvo_topk_key(float score, int32_t node);
float jvo_key_score(int64_t key);
int32_t jvo_key_node(int64_t key);
void jvo_bruteforce_topk_f32(int metric, const float *base, int64_t n, int dim, const float *q, int k, int64_t *keys_out);

/* ---- PQ ---- */
void jvo_pq_layout(int dim, int M, int *sizes, int *offsets);
void jvo_pq_encode(const float *codebooks, const int *sizes, const int *offsets, int M, int k,
                   const float *centroid, const float *v, int dim, uint8_t *codes);
void jvo_pq_lut(const float *codebooks, const int *sizes, const int *offsets, int M, int k,
                const float *centroid, const float *q, int dim, int metric, float *lut);
void jvo_pq_self_magnitudes(const float *codebooks, const int *sizes, const int *offsets, int M, int k, float *mag);
float jvo_pq_adc(const float *lut, int k, const uint8_t *codes, int M);
float jvo_pq_decoded_cosine(const uint8_t *codes, int M, int k, const float *lut, const float *mag, float bMag);
float jvo_pq_score_lut(int metric, const float *lut, const float *mag, float bMag, int k, const uint8_t *codes, int M);
float jvo_pq_score_direct(const float *codebooks, const int *sizes, const int *offsets, int M, int k,
                          const float *centroid, const float *q, int dim, int metric, const uint8_t *codes);
float jvo_pq_diversity_direct(const float *codebooks, const int *sizes, const int *offsets, int M, int k,
                              int metric, const uint8_t *c1, const uint8_t *c2);
void jvo_pq_pair_table(const float *codebooks, const int *sizes, const int *offsets, int M, int k, int metric, float *table);
float jvo_pq_pair_sum(const float *table, int M, int k, const uint8_t *c1, const uint8_t *c2);

/* ---- BQ ---- */
void jvo_bq_encode(const float *v, int dim, uint64_t *words);
int jvo_hamming(const uint64_t *a, const uint64_t *b, int words);
float jvo_bq_score(const uint64_t *a, const uint64_t *b, int words, int dim);

/* ---- NVQ (8-bit) ---- */
float jvo_nvq_logistic(float v, float alpha, float x0);
float jvo_nvq_logit(float v, float inverseAlpha, float x0);
float jvo_nvq_dequant(uint8_t b, float alpha, float x0, float minv, float maxv);
void jvo_nvq_quantize_8bit(const float *v, int n, float alpha, float x0, float minv, float maxv, uint8_t *dst);
float jvo_nvq_loss(const float *v, int n, float alpha, float x0, float minv, float maxv, int nbits);
float jvo_nvq_uniform_loss(const float *v, int n, float minv, float maxv, int nbits);
float jvo_nvq_dot_8bit(const float *q, const uint8_t *b, int n, float alpha, float x0, float minv, float maxv);
float jvo_nvq_l2_8bit(const float *q, const uint8_t *b, int n, float alpha, float x0, float minv, float maxv);
void jvo_nvq_cosine_8bit(const float *q, const uint8_t *b, int n, float alpha, float x0, float minv, float maxv,
                         const float *centroid, float *out2);
/* encode one sub-vector: params_out = {min, max, growthRate, midpoint} */
void jvo_nvq_encode_subvector(const float *v, int n, int learn, float *params_out, uint8_t *bytes_out);
/* encode a whole vector: subtract mean, split into nsub sub-vectors (layout as jvo_pq_layout) */
void jvo_nvq_encode(const float *v, const float *mean, int dim, int nsub, int learn, float *params_out, uint8_t *bytes_out);
float jvo_pq_diversity_table(int metric, const float *table, int M, int k, const uint8_t *c1, const uint8_t *c2);
void jvo_kmeans_assign(const float *points, int64_t n, int dim, const float *centroids, int k, int32_t *assign);
/* the same sums and parameter search under an explicit summation order (see jv_oracle.c): lanes = 1 sequential,
 * lanes = 32 strided accumulators + xor butterfly (a GPU warp's order) */
float jvo_nvq_loss_lanes(const float *v, int n, float alpha, float x0, float minv, float maxv, int nbits, int lanes);
float jvo_nvq_uniform_loss_lanes(const float *v, int n, float minv, float maxv, int nbits, int lanes);
void jvo_nvq_encode_subvector_lanes(const float *v, int n, int learn, int lanes, float *params_out, uint8_t *bytes_out);
void jvo_nvq_encode_lanes(const float *v, const float *mean, int dim, int nsub, int learn, int lanes, float *params_out, uint8_t *bytes_out);
float jvo_nvq_score(int metric, const float *q, const float *mean, int dim, int nsub,
                    const float *params, const uint8_t *bytes);

/* ---- optional: route the inner kernels through the reference's own compiled library ---- */
int jvo_use_ref(const char *path_to_libjvector_so); /* 0 ok; after this, jvo_ctx_* scorers call the reference kernels */
const char *jvo_ref_isa(void);

/* ---- score contexts (one query against a registered data set) ---- */
typedef struct jvo_scorer jvo_scorer;
jvo_scorer *jvo_scorer_f32(int metric, const float *base, int64_t n, int dim, const float *q);
jvo_scorer *jvo_scorer_pq(int metric, const float *codebooks, int M, int k, int dim, const float *centroid,
                          const uint8_t *codes, int64_t n, const float *q);
jvo_scorer *jvo_scorer_bq(const uint64_t *words, int64_t n, int dim, const float *q);
jvo_scorer *jvo_scorer_nvq(int metric, const float *mean, int dim, int nsub, const float *params,
                           const uint8_t *bytes, int64_t n, const float *q);
float jvo_scorer_score(jvo_scorer *s, int32_t node);
void jvo_scorer_free(jvo_scorer *s);

/* ---- graph (host restatement of GraphSearcher / GraphIndexBuilder) ---- */
typedef struct {
    int32_t n;            /* nodes */
    int32_t levels;       /* number of levels (>=1) */
    int32_t degree;       /* max degree, identical on all levels */
    int32_t entry_node;
    int32_t entry_level;
    const int32_t *adj0;      /* [n][degree], -1 padded */
    const int32_t *upper_row; /* [(levels-1)][n]: row index into upper_adj of that level, or -1 */
    const int32_t *upper_adj; /* concatenated per level: rows [count_l][degree] */
    const int64_t *upper_off; /* [(levels-1)] offset (in rows) of each level's block inside upper_adj */
} jvo_graph;

typedef struct {
    int32_t visited;
    int32_t expanded;
    int32_t expanded_base;
    int32_t reranked;
} jvo_search_stats;

/* order 0 (default): sequential sums, or the reference's kernels after jvo_use_ref; order 1: the summation order of the
 * sm_90a kernels (32 / 8 lane accumulators + xor butterfly, see "WARP-ORDER restatements" in jv_oracle.c), which makes a
 * traversal reproducible id for id. Same formulas either way. */
void jvo_scorer_set_order(jvo_scorer *s, int order);
float jvo_compare_f32_warp(int metric, const float *q, const float *row, int dim);

/* FusedPQ feature: packed neighbour codes (FusedPQ.java:122-141) and the decoder's similarityToNeighbor (FusedPQDecoder.java:84-114);
 * a PQ scorer with packed neighbours makes jvo_graph_search take OnDiskGraphIndex.processNeighbors' edge-loading branch on level 0 */
void jvo_fused_pq_pack(const int32_t *adj0, int32_t n, int degree, const uint8_t *codes, int M, uint8_t *packed_out);
void jvo_scorer_set_packed_neighbors(jvo_scorer *s, const uint8_t *packed, int degree);
float jvo_scorer_score_neighbor(jvo_scorer *s, int32_t origin, int neighborIndex);

/* one query; approx scorer walks the graph, optional reranker re-scores the rerankK survivors.
 * Writes up to topK (node, score) pairs ordered best first; returns the count. */
int jvo_graph_search(const jvo_graph *g, jvo_scorer *approx, jvo_scorer *reranker, int topK, int rerankK,
                     int32_t *nodes_out, float *scores_out, jvo_search_stats *stats);

/* GraphSearcher.search(scoreProvider, topK, rerankK, threshold, rerankFloor, acceptOrds) (GraphSearcher.java:166-181):
 * accept_bits: bit (node & 31) of word (node >> 5), NULL = Bits.ALL. threshold: admission rule of :427-431 only (the
 * TwoPhaseTracker early stop is not restated, see jv_oracle.c). */
int jvo_graph_search_ex(const jvo_graph *g, jvo_scorer *approx, jvo_scorer *reranker, int topK, int rerankK, float threshold,
                        float rerankFloor, const uint32_t *accept_bits, int32_t *nodes_out, float *scores_out, jvo_search_stats *stats);

/* batched, multi-threaded driver over f32 / pq(+f32 rerank) data for the CPU baseline.
 * kind: 0 = exact f32 only, 1 = PQ first pass + f32 rerank */
typedef struct {
    int kind, metric, dim;
    const float *base; int64_t n;
    const float *codebooks; int M, k; const float *centroid; const uint8_t *codes;
    int order; /* 0: sequential / reference kernels; 1: warp order (jvo_scorer_set_order) */
} jvo_dataset;
double jvo_graph_search_batch(const jvo_graph *g, const jvo_dataset *ds, const float *queries, int nq,
                              int topK, int rerankK, int threads, int32_t *nodes_out, float *scores_out,
                              int64_t *scored_total);

/* host buffers with pages interleaved over the NUMA nodes (CPU baseline only) */
int jvo_numa_nodes(void);
void *jvo_alloc_interleaved(size_t bytes);
void jvo_free_interleaved(void *p, size_t bytes);

/* multi-threaded NVQ encode (reference kernels when jvo_use_ref was called); returns seconds */
double jvo_nvq_encode_batch(const float *rows, int64_t n, int dim, int nsub, const float *mean, int learn, int threads, float *params_out, uint8_t *bytes_out);

/* multi-threaded BQ brute force, keys_out [nq][k] best first; returns seconds */
double jvo_bq_bruteforce_batch(const uint64_t *words, int64_t n, int dim, const uint64_t *qwords, int nq, int k, int threads, int64_t *keys_out);

/* single-threaded Vamana build (no hierarchy when levels_out==1) following GraphIndexBuilder.addGraphNode;
 * exact f32 scoring. adj_out: [n][degree] -1 padded. Returns entry node. */
int32_t jvo_graph_build_f32(int metric, const float *base, int32_t n, int dim, int degree, int beam,
                            float overflow, float alpha, int32_t *adj_out);
/* Vamana robust prune restated from VamanaDiversityProvider.retainDiverse: candidates sorted by score desc.
 * pair_score(i,j) supplied as a dense matrix [nc][nc] of mapped scores. selected_out[nc] 0/1. returns count */
int jvo_retain_diverse(const float *cand_scores, const int32_t *cand_nodes, int nc, const float *pair_scores,
                       int maxDegree, float alpha, uint8_t *selected_out);

#ifdef __cplusplus
}
#endif
#endif
