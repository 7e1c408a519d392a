/*
 * jvector_b200.h — C ABI of libjvector_b200.so, the H100 (sm_90a) replacement for JVector's libjvector.so.
 *
 * Two groups of entry points:
 *
 *  (1) The 24 symbols of the reference's native library, with identical C signatures, so the library can be
 *      installed as `libjvector.so` under jvector-native unchanged. They replace
 *      /root/reference/jvector-native/src/main/native/src/jvector_simd_kernel_list.h:35-61 and
 *      src/jvector_simd.h:47,53. The reference binds them with Linker.Option.critical(true) on on-heap segments
 *      (jvector-native/src/main/java/.../cnative/NativeSimdOps.java:1164,1226,...), i.e. they must be short,
 *      synchronous, host-memory functions; they are the n = 1 case and stay on the host by contract.
 *
 *  (2) The batched GPU entry points (prefix jv_) that the GPU-backed VectorizationProvider / ScoreFunction
 *      implementations bind with ordinary (non-critical) downcall handles: data sets are registered once and
 *      live in HBM; each hop / rerank list / multi-query step / whole search batch is ONE call.
 *      They replace the per-candidate call sites
 *        base:graph/OnHeapGraphIndex.java:475-483, base:graph/disk/OnDiskGraphIndex.java:639-661 (neighbour loop),
 *        base:graph/NodeQueue.java:168-188 (rerank loop), base:quantization/PQDecoder.java:48-53 (LUT build),
 *        base:graph/GraphIndexBuilder.java:830-835, base:graph/diversity/VamanaDiversityProvider.java:56-95,
 *        base:graph/GraphSearcher.java:263-282,406-457 (whole traversal, device resident).
 *      (`base:` = jvector-base/src/main/java/io/github/jbellis/jvector/)
 *
 * Conventions for group (2): every function returns an int status (0 = JV_OK, negative = error) and never throws
 * or aborts across the ABI; jv_last_error() returns a thread-local message. All pointer arguments are HOST
 * pointers borrowed for the duration of the call unless the name ends in _device. Scores are the reference's
 * similarity scores (base:vector/VectorSimilarityFunction.java:37-69), higher = closer. Top-k keys are the
 * reference's 64-bit ordering key (base:graph/NodeQueue.java:125-137). No CPU fallback exists: without an
 * sm_90 device jv_gpu_init() fails and every other jv_ call returns JV_ERR_NO_DEVICE.
 */
#ifndef JVECTOR_B200_H
#define JVECTOR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define JV_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------------
 * (1) legacy libjvector.so ABI — jvector_simd_kernel_list.h:35-61
 * ---------------------------------------------------------------------------------------------- */
JV_API float cosine_f32(const float *a, size_t aoffset, const float *b, size_t boffset, size_t length);
JV_API float dot_product_f32(const float *a, size_t aoffset, const float *b, size_t boffset, size_t length);
JV_API float euclidean_f32(const float *a, size_t aoffset, const float *b, size_t boffset, size_t length);
JV_API void add_in_place_f32(float *v1, const float *v2, size_t length);
JV_API void add_scalar_in_place_f32(float *v1, float value, size_t length);
JV_API void sub_in_place_f32(float *v1, const float *v2, size_t length);
JV_API void sub_scalar_in_place_f32(float *v1, float value, size_t length);
JV_API float max_f32(const float *v, size_t length);
JV_API void min_in_place_f32(float *v1, const float *v2, size_t length);
JV_API float assemble_and_sum_f32(const float *data, int dataBase, const unsigned char *baseOffsets, int baseOffsetsOffset, size_t baseOffsetsLength);
JV_API float assemble_and_sum_pq_f32(const float *data, size_t subspaceCount, const unsigned char *baseOffsets1, int baseOffsetsOffset1, const unsigned char *baseOffsets2, int baseOffsetsOffset2, int clusterCount);
JV_API float pq_decoded_cosine_similarity_f32(const unsigned char *baseOffsets, int baseOffsetsOffset, size_t baseOffsetsLength, int clusterCount, const float *partialSums, const float *aMagnitude, float bMagnitude);
JV_API void calculate_partial_sums_dot_f32(const float *codebook, int codebookIndex, size_t size, int clusterCount, const float *query, int queryOffset, float *partialSums);
JV_API void calculate_partial_sums_euclidean_f32(const float *codebook, int codebookIndex, size_t size, int clusterCount, const float *query, int queryOffset, float *partialSums);
JV_API void calculate_partial_sums_self_magnitude_f32(const float *codebook, int codebookIndex, size_t size, int clusterCount, float *partialSums);
JV_API void nvq_quantize_8bit(const float *vector, size_t length, float alpha, float x0, float minValue, float maxValue, unsigned char *destination);
JV_API float nvq_loss(const float *vector, size_t length, float alpha, float x0, float minValue, float maxValue, int nBits);
JV_API float nvq_uniform_loss(const float *vector, size_t length, float minValue, float maxValue, int nBits);
JV_API float nvq_square_l2_distance_8bit(const float *vector, const unsigned char *quantized, size_t length, float alpha, float x0, float minValue, float maxValue);
JV_API float nvq_dot_product_8bit(const float *vector, const unsigned char *quantized, size_t length, float alpha, float x0, float minValue, float maxValue);
JV_API int64_t nvq_cosine_8bit_packed(const float *vector, const unsigned char *quantized, size_t length, float alpha, float x0, float minValue, float maxValue, const float *centroid);
/* no-op here: this library reads NVQ bytes in natural order (as base:vector/DefaultVectorUtilSupport.java:454) */
JV_API void nvq_shuffle_query_in_place_8bit(float *vector, size_t length);
/* jvector_simd.h:47,53 — reflected on by base:vector/VectorizationProvider.java:132-136 */
JV_API const char *jvector_simd_get_active_isa(void);
JV_API const char *jvector_simd_get_max_isa_env(void);

/* ------------------------------------------------------------------------------------------------
 * (2) batched GPU ABI
 * ---------------------------------------------------------------------------------------------- */
enum { JV_EUCLIDEAN = 0, JV_DOT_PRODUCT = 1, JV_COSINE = 2 }; /* VectorSimilarityFunction ordinal order */

enum {
    JV_OK = 0,
    JV_ERR_NO_DEVICE = -1,   /* no CUDA device / not sm_90 / jv_gpu_init not called */
    JV_ERR_INVALID = -2,     /* bad argument */
    JV_ERR_CUDA = -3,        /* CUDA runtime error, see jv_last_error() */
    JV_ERR_OOM = -4,
    JV_ERR_UNSUPPORTED = -5, /* combination not implemented (e.g. metric for BQ other than Hamming score) */
    JV_ERR_OVERFLOW = -6     /* device scratch (visited table, candidate list) too small even after retry */
};

typedef struct jv_dataset_s *jv_dataset; /* vectors / codes resident in HBM */
typedef struct jv_query_s *jv_query;     /* one query prepared against one data set (LUT / bits / shifted copy) */
typedef struct jv_graph_s *jv_graph;     /* adjacency resident in HBM */

/* Bind CUDA device `device` and make it the device on which the CALLING THREAD creates data sets and graphs. Idempotent. Every
 * handle remembers its device, so binding another device later never invalidates existing handles. */
JV_API int jv_gpu_init(int device);
/* One process driving several GPUs (the reference host is one JVM: base:vector/VectorizationProvider.java:79-177): bind every
 * device of the mask (bit d = CUDA device d) and enable peer access between them (NVLink / NVSwitch). SURVEY §8(b). */
JV_API int jv_gpu_init_mask(uint32_t device_mask);
JV_API uint32_t jv_gpu_bound_mask(void);
/* the device on which the calling thread's next register / create calls place their data (a bound device) */
JV_API int jv_gpu_set_device(int device);
JV_API int jv_gpu_device_count(void);
JV_API const char *jv_last_error(void);
JV_API const char *jv_version(void);
JV_API int jv_gpu_sm_count(void);

/* ---- data sets (the RandomAccessVectorValues / CompressedVectors a ScoreFunction reads) ---- */
/* Data sets and graphs may be shared across threads: any thread may search, build from, score or train on them concurrently. Their
 * rows, codes and adjacency do not change after creation. What is built lazily on them — an fp32 data set's row sketch and low-rank
 * rows, a graph's edge records, a PQ data set's centroid-pair tables — is built once, under a lock of the handle, by whichever call
 * needs it first. The one exception is jv_graph_fuse_pq (below), which rewrites its graph. */
/* rows: [n][dim] fp32 row-major (base:graph/RandomAccessVectorValues.java) */
JV_API int jv_dataset_register_f32(const float *rows, int64_t n, int dim, jv_dataset *out);
/* PQVectors: codes [n][M] u8 (base:quantization/PQVectors.java:377-395), codebooks concatenated in sub-space order,
 * codebook m = k * size_m floats [k][size_m] (ProductQuantization.java:66), sub-vector sizes per
 * ProductQuantization.java:535-550, centroid = globalCentroid or NULL */
JV_API int jv_dataset_register_pq(const uint8_t *codes, int64_t n, int dim, int M, int k, const float *codebooks,
                                  const float *centroid, jv_dataset *out);
/* BQVectors: words [n][ceil(dim/64)] u64, bit j of word i = (v[64 i + j] > 0) (BinaryQuantization.java:96-109) */
JV_API int jv_dataset_register_bq(const uint64_t *words, int64_t n, int dim, jv_dataset *out);
/* NVQVectors, 8 bit: bytes [n][dim] u8 (sub-vectors concatenated), params [n][nsub][4] = {min,max,growthRate,midpoint}
 * (NVQuantization.java:489-498), mean = globalMean */
JV_API int jv_dataset_register_nvq(const uint8_t *bytes, const float *params, int64_t n, int dim, int nsub,
                                   const float *mean, jv_dataset *out);
/* rows already in HBM on the calling thread's device (e.g. produced by another kernel): BORROWED, not copied — the caller keeps
 * them alive and UNCHANGED until jv_dataset_free. 16-byte aligned, row_stride = dim rounded up to 4 floats, padding floats zero.
 * (A graph searched over them assumes unchanged rows already; so does the row sketch that the first DOT_PRODUCT graph search of a
 * batch larger than the GPU's resident CTAs derives from them: int8 codes + 8 bytes per row, built once, freed with the handle.) */
JV_API int jv_dataset_adopt_f32_device(const float *rows_device, int64_t n, int dim, int row_stride, jv_dataset *out);
/* the row sketch of an fp32 data set, as that search built it: codes_out [n][sketch_stride] int8 (sketch_stride = row stride
 * rounded up to 8, padding codes 0), meta_out [n][2] = {scale, radius} per row. Builds nothing: JV_ERR_INVALID ("no row sketch")
 * while no search has built one. codes_out / meta_out may be NULL (only *sketch_stride_out, and whether the sketch exists). */
JV_API int jv_dataset_row_sketch_download(jv_dataset f32, int8_t *codes_out, float *meta_out, int *sketch_stride_out);
/* The low-rank rows of an fp32 data set, built with its row sketch when the rows lie close to a rank-32 subspace: basis [rank][stride]
   fp32, rows [n][48] bytes = rank int8 codes then float {t, rho, beta, ||x||} (DESIGN §4.1). JV_ERR_INVALID when there are none;
   rank_out is set either way. Either output may be NULL. */
JV_API int jv_dataset_lowrank_download(jv_dataset f32, float *basis_out, uint8_t *rows_out, int *rank_out);
/* A graph's edge records for the low-rank bound: [n][degree][48] bytes, slot t of node v = the low-rank row of its t-th level-0
   neighbour (zeros for an empty slot). Built by the first sketched search; JV_ERR_INVALID when there are none. */
JV_API int jv_graph_edge_records_download(jv_graph g, uint8_t *out);
/* New neighbours the calling thread's last graph search settled on edge records (they are part of jv_search_stats.visited). */
JV_API int64_t jv_search_last_settled(void);
/* Of those that the calling thread's last graph search did not settle on edge records: how many it sent straight to their full row,
   skipping the row sketch, on the records' point estimate (*routed), and how many of these the candidate list then refused
   (*routed_dropped). Either pointer may be NULL. */
JV_API void jv_search_last_direct(int64_t *routed, int64_t *routed_dropped);
/* The low-rank bound as a DOT_PRODUCT score of rows[i] against queries[i] (both [n][dim]) for basis [dim][32] (column j = basis
   vector j), computed by the device functions the search uses; records_out (may be NULL): the rows' [n][48]-byte records. */
JV_API int jv_lowrank_bound_pairs(const float *basis, int dim, const float *rows, const float *queries, int64_t n, uint8_t *records_out, float *bounds_out);
/* The graph search with the refine pass's exclusion (host pointers): query q walks through node exclude_ids[q] (-1: none) but never
   returns it, as acceptOrds without that one node would. No reranker, no threshold. counters_out (may be NULL): visited, expanded,
   expanded_base, reranked. */
JV_API int jv_graph_search_exclude(jv_graph g, jv_dataset approx, int metric, const float *queries, int nq, int topK, int rerankK,
                                   const int32_t *exclude_ids, int32_t *nodes_out, float *scores_out, int64_t *counters_out);
JV_API int jv_dataset_device(jv_dataset ds);
/* ImmutablePQVectors' code-vs-code scoring (base:quantization/ImmutablePQVectors.java:63-105): build the triangular
 * centroid-vs-centroid table of ProductQuantization.createCodebookPartialSums (ProductQuantization.java:609-628; 12.6 MB at M = 96,
 * k = 256) in HBM; jv_score_pairs on this data set then sums table entries — assembleAndSumPQ, native-c:
 * src/jvector_simd_kernels.cpp:729-815 — instead of recomputing centroid distances. EUCLIDEAN and DOT_PRODUCT have their own
 * tables, COSINE uses the dot-product one. Each table is built once per data set, by this call or by the first build, add,
 * removal or refine over the codes that needs it (threads that race for it wait for one build), and freed with the data set. */
JV_API int jv_dataset_pq_pair_table(jv_dataset pq, int metric);
JV_API int jv_dataset_pq_pair_table_download(jv_dataset pq, int metric, float *table_out /* [M][k (k + 1) / 2] */);
JV_API int jv_dataset_free(jv_dataset ds);
JV_API int64_t jv_dataset_size(jv_dataset ds);
JV_API int jv_dataset_dim(jv_dataset ds);
JV_API int64_t jv_dataset_device_bytes(jv_dataset ds);

/* ---- ScoreFunction for one query: CompressedVectors.precomputedScoreFunctionFor / DefaultSearchScoreProvider.exact ---- */
JV_API int jv_query_begin(jv_dataset ds, const float *q, int metric, jv_query *out);
/* the neighbour loop of one processNeighbors call / one rerank list: ids[n] -> scores[n], ONE kernel launch */
JV_API int jv_score_batch(jv_query q, const int32_t *ids, int n, float *scores_out);
JV_API int jv_query_end(jv_query q);
/* PQ only: copy the query's partial-sums table (PQDecoder.java:41-54) back, lut_out[M*k] */
JV_API int jv_query_get_lut(jv_query q, float *lut_out);

/* ---- query batches: the host-driven seam with persistent state ----
 * A batch of searches that the HOST drives hop by hop (GraphSearcher on the JVM, base:graph/GraphSearcher.java:406-457): the
 * prepared queries (LUTs / bit packs / shifted copies) are built once and stay in HBM until jv_query_batch_end; a step uploads
 * only ids + offsets through pinned staging owned by the batch and brings the scores back. */
typedef struct jv_query_batch_s *jv_query_batch;
JV_API int jv_query_batch_begin(jv_dataset ds, int metric, const float *queries, int nq, jv_query_batch *out);
/* one step of all nq searches: query i scores ids[offsets[i] .. offsets[i+1]) -> scores_out in the same order; ONE launch.
 * device_ms (optional): CUDA-event time of the scoring kernel alone */
JV_API int jv_query_batch_score(jv_query_batch b, const int32_t *ids, const int32_t *offsets, float *scores_out, double *device_ms);
/* one hop of search `query_index`: ids[n] -> scores_out[n]; the kernel reads / writes mapped pinned memory (no separate copies) */
JV_API int jv_query_batch_score_one(jv_query_batch b, int query_index, const int32_t *ids, int n, float *scores_out);
JV_API int jv_query_batch_end(jv_query_batch b);

/* one step of many searches: query qi scores ids[offsets[qi] .. offsets[qi+1]) ; one launch for the whole step */
JV_API int jv_score_multi(jv_dataset ds, int metric, const float *queries, int nq, const int32_t *ids,
                          const int32_t *offsets, float *scores_out);
/* diversity scoring (BuildScoreProvider.diversityProviderFor): score(a[i], b[i]) for n pairs, one launch.
 * f32: exact; PQ: codebook-vs-codebook (PQVectors.java:284-350); BQ: BQVectors.java:98-105 */
JV_API int jv_score_pairs(jv_dataset ds, int metric, const int32_t *a, const int32_t *b, int n, float *scores_out);
/* exhaustive scoring of every row for nq queries with a fused device-side top-k; keys_out[nq][k] best first,
 * padded with INT64_MIN */
JV_API int jv_topk_bruteforce(jv_dataset ds, int metric, const float *queries, int nq, int k, int64_t *keys_out);
/* multi-GPU form (SURVEY §8e): the base is range-sharded, this rank holds rows [id_base, id_base + n); queries and keys stay in
 * HBM so the keys can be the NCCL send buffer. Node ids inside the keys are global (local id + id_base). */
JV_API int jv_topk_bruteforce_device(jv_dataset ds, int metric, const float *queries_device, int nq, int k, int64_t id_base,
                                     int64_t *keys_out_device);
/* the merge after the all-gather: keys_in [nq][parts * k] (any order) -> keys_out [nq][k] best first */
JV_API int jv_topk_merge_device(const int64_t *keys_in_device, int nq, int parts, int k, int64_t *keys_out_device);

/* Stream-ordered forms for callers that own a CUDA stream (the multi-process bench puts the local top-k, the NCCL all-gather and
 * the merge on ONE stream with no host synchronisation in between). BQ data sets only (the tensor-core contraction of
 * csrc/bq_imma.cu); *status_device receives the number of queries left unresolved (0 normally; non-zero = call the synchronous
 * form, which falls back to the key-threshold kernels). cuda_stream: a cudaStream_t. The device scratch of the async top-k
 * belongs to the calling thread's context for that device, so async calls from one thread must be ordered on one stream. */
JV_API int jv_topk_bruteforce_device_async(jv_dataset ds, int metric, const float *queries_device, int nq, int k, int64_t id_base,
                                           int64_t *keys_out_device, int32_t *status_device, void *cuda_stream);
/* keys_in: SHARD-MAJOR [parts][nq][k], exactly what an all-gather of the per-rank [nq][k] arrays produces */
JV_API int jv_topk_merge_device_async(const int64_t *keys_in_device, int nq, int parts, int k, int64_t *keys_out_device, void *cuda_stream);

/* ---- several GPUs driven by ONE process (SURVEY §8b last row, §8e) ----
 * jv_multi: a base RANGE-SHARDED by contiguous node id over the devices bound by jv_gpu_init_mask (shard i holds rows
 * [first_row_i, first_row_i + rows_i)). jv_multi_topk_bruteforce: every shard scores all queries on its own stream (one worker
 * thread per device inside the call), the per-shard top-k keys (global node ids) go to the first device by NVLink peer copies
 * and are merged there by the reference key — the same exchange the multi-process path does with an NCCL all-gather. */
typedef struct jv_multi_s *jv_multi;
JV_API int jv_multi_register_bq(const uint64_t *words, int64_t n, int dim, jv_multi *out);
JV_API int jv_multi_register_f32(const float *rows, int64_t n, int dim, jv_multi *out);
JV_API int jv_multi_free(jv_multi m);
JV_API int jv_multi_shard_count(jv_multi m);
JV_API int jv_multi_shard_info(jv_multi m, int shard, int *device, int64_t *first_row, int64_t *rows);
JV_API int jv_multi_topk_bruteforce(jv_multi m, int metric, const float *queries, int nq, int k, int64_t *keys_out);

/* ---- bulk encoders (next to the scoring path: ProductQuantization.encodeAll, BinaryQuantization.encodeAll,
 *      NVQuantization.encodeAll) ---- */
JV_API int jv_bq_encode_batch(const float *rows, int64_t n, int dim, uint64_t *words_out);
JV_API int jv_pq_encode_batch(const float *rows, int64_t n, int dim, int M, int k, const float *codebooks,
                              const float *centroid, uint8_t *codes_out);
JV_API int jv_nvq_encode_batch(const float *rows, int64_t n, int dim, int nsub, const float *mean, int learn,
                               float *params_out, uint8_t *bytes_out);
/* the assignment step of k-means (KMeansPlusPlusClusterer.getNearestCluster, base:quantization/KMeansPlusPlusClusterer.java:329-342)
 * for a batch of points [n][dim] against centroids [k][dim]: index of the nearest centroid, first minimum wins */
JV_API int jv_kmeans_assign_batch(const float *points, int64_t n, int dim, const float *centroids, int k, int32_t *assignments_out);
/* the same encoders over rows that are already resident in HBM (a registered fp32 data set): no host->device copy */
JV_API int jv_bq_encode_dataset(jv_dataset f32, uint64_t *words_out);
JV_API int jv_pq_encode_dataset(jv_dataset f32, int M, int k, const float *codebooks, const float *centroid, uint8_t *codes_out);
JV_API int jv_nvq_encode_dataset(jv_dataset f32, int nsub, const float *mean, int learn, float *params_out, uint8_t *bytes_out);

/* NVQ inline vectors without a host round trip: encode the resident fp32 rows into a NEW resident NVQ data set */
JV_API int jv_nvq_encode_dataset_resident(jv_dataset f32, int nsub, const float *mean, int learn, jv_dataset *out);
/* the same for PQ (ProductQuantization.encodeAll, unweighted): the resident fp32 rows encoded with codebooks [k * dim] (host) and an
 * optional centroid [dim] (host) into a NEW resident PQ data set, as jv_dataset_register_pq would hold the same codes */
JV_API int jv_pq_encode_dataset_resident(jv_dataset f32, int M, int k, const float *codebooks, const float *centroid, jv_dataset *out);
/* a resident PQ data set read back: codes [n][M], codebooks [k * dim], centroid [dim]; any pointer may be NULL. JV_ERR_INVALID for a
 * data set that is not PQ, or a centroid_out when it has no centroid */
JV_API int jv_dataset_pq_download(jv_dataset pq, uint8_t *codes_out, float *codebooks_out, float *centroid_out);

/* ---- PQ training: ProductQuantization.compute / refine with isotropic (UNWEIGHTED) loss, on the device ----
 * The training rows are the resident rows of `f32` (an out-of-core index registers a sample), all of them, or, above the cap, a
 * sample of `cap` rows drawn with Floyd's algorithm from `seed` and sorted. compute: optional global centring (the mean is an int64
 * fixed-point sum, independent of thread order), k-means++ seeding (as an exponential race: the same distribution as the
 * reference's inverse-CDF scan), then Lloyd as KMeansPlusPlusClusterer.cluster(lloyd_iterations, 0): each sub-space stops once at
 * most 1 % of its rows change cluster; an empty cluster is reseeded to a random training row. refine: Lloyd only, from the given
 * codebooks, on the rows minus `centroid`; 0 rounds returns the codebooks bit for bit. The result is a pure function of the rows
 * and the parameters. Errors: JV_ERR_INVALID for a data set that is not fp32, M outside 1..dim, k outside 1..256, fewer training
 * rows than k, a negative iteration count or cap, a null required pointer, globally_center with a NULL centroid_out;
 * JV_ERR_OOM when the training buffers (about n_train * dim * 4 + n_train * M * 8 bytes) do not fit. */
typedef struct {
    int M;                  /* sub-spaces; sizes and offsets as ProductQuantization.getSubvectorSizesAndOffsets */
    int k;                  /* clusterCount, 1..256 */
    int globally_center;    /* compute only: subtract the training rows' mean first (the centroid is written to centroid_out) */
    int lloyd_iterations;   /* K_MEANS_ITERATIONS (6) for compute, lloydsRounds for refine; >= 0 */
    int64_t max_train_rows; /* 0 = MAX_PQ_TRAINING_SET_SIZE (128 000) */
    uint64_t seed;
} jv_pq_train_params;
typedef struct {
    int64_t train_rows;        /* rows trained on */
    int32_t max_lloyd_updates; /* centroid updates of the sub-space that ran longest */
    int64_t changed_last;      /* summed over sub-spaces: rows that changed cluster in the sub-space's last reassignment */
    int64_t empty_reseeds;     /* empty clusters reseeded to a random training row */
    int64_t seeding_fallbacks; /* seeding rounds in which every row already coincided with a chosen centroid */
    double device_ms;
} jv_pq_train_stats;
JV_API int jv_pq_train(jv_dataset f32, const jv_pq_train_params *p, float *codebooks_out /* [k * dim], the jv_dataset_register_pq layout */,
                       float *centroid_out /* [dim] or NULL */, jv_pq_train_stats *stats /* may be NULL */);
JV_API int jv_pq_refine(jv_dataset f32, const jv_pq_train_params *p, const float *codebooks, const float *centroid /* or NULL */,
                        float *codebooks_out, jv_pq_train_stats *stats /* may be NULL */);

/* ---- PQ with an anisotropic threshold T (ProductQuantization with anisotropicThreshold > UNWEIGHTED = -1), on the device ----
 * Training: jv_pq_train's steps, then KMeansPlusPlusClusterer's anisotropic rounds per sub-space: centroids from a per-cluster
 * d_s x d_s Gauss-Jordan solve in the reference's order (the outer-product sums are int64 fixed point, independent of thread order),
 * rows reassigned by the weighted parallel / perpendicular loss, the same 1 % early stop, pcm from T and the sub-space's size.
 * compute runs lloyd_iterations Lloyd rounds and then lloyd_iterations anisotropic rounds; refine runs lloyd_iterations anisotropic
 * rounds only, from the unweighted nearest-centroid assignment. Encoding: the reference's coordinate descent over sub-spaces
 * (at most 10 sweeps, pcm from T and dim), one row at a time, for every row ever encoded with such a PQ.
 * T == -1 gives exactly the bytes and counters of jv_pq_train / jv_pq_refine / jv_pq_encode_*. Errors, all before any device work,
 * leaving the outputs untouched: JV_ERR_INVALID for T NaN, below -1 or at least 1, and whatever the unweighted call rejects;
 * JV_ERR_UNSUPPORTED from the training calls when T > -1 and a sub-space is wider than 64 floats (ceil(dim / M) > 64).
 * Anisotropic codebooks and codes register with jv_dataset_register_pq like any others: search, build, add and remove are unchanged. */
typedef struct {
    jv_pq_train_stats lloyd;          /* the unweighted phase, as jv_pq_train reports it; lloyd.device_ms covers the whole call */
    int32_t max_anisotropic_updates;  /* anisotropic rounds of the sub-space that ran longest */
    int64_t changed_last_anisotropic; /* summed over sub-spaces: rows moved by each one's last anisotropic reassignment */
    int64_t anisotropic_reseeds;      /* empty clusters reseeded to a random training row in the anisotropic rounds */
} jv_pq_anisotropic_stats;
JV_API int jv_pq_train_anisotropic(jv_dataset f32, const jv_pq_train_params *p, float anisotropic_threshold,
                                   float *codebooks_out, float *centroid_out, jv_pq_anisotropic_stats *stats /* may be NULL */);
JV_API int jv_pq_refine_anisotropic(jv_dataset f32, const jv_pq_train_params *p, float anisotropic_threshold, const float *codebooks,
                                    const float *centroid /* or NULL */, float *codebooks_out, jv_pq_anisotropic_stats *stats /* may be NULL */);
typedef struct {
    int64_t rows_moved; /* rows whose code left its minimum-residual start */
    int64_t moves;      /* coordinate-descent moves in all */
    int32_t max_sweeps; /* sweeps of the row that ran longest (0 when T == -1) */
    double device_ms;   /* the call's work on the device stream, copies included */
} jv_pq_encode_stats;
JV_API int jv_pq_encode_batch_anisotropic(const float *rows, int64_t n, int dim, int M, int k, const float *codebooks, const float *centroid,
                                          float anisotropic_threshold, uint8_t *codes_out, jv_pq_encode_stats *stats /* may be NULL */);
JV_API int jv_pq_encode_dataset_anisotropic(jv_dataset f32, int M, int k, const float *codebooks, const float *centroid,
                                            float anisotropic_threshold, uint8_t *codes_out, jv_pq_encode_stats *stats /* may be NULL */);

/* ---- graph: ImmutableGraphIndex adjacency in HBM + GraphSearcher traversal on the device ---- */
/* adj0: [n][degree] int32, -1 padded (level 0). */
JV_API int jv_graph_create(int32_t n, int degree, const int32_t *adj0, int32_t entry_node, jv_graph *out);
/* add level 1, 2, ... in order; node_ids[count] are the members, adj [count][degree] their lists at that level.
 * The entry node must be a member of the last level added. */
JV_API int jv_graph_add_level(jv_graph g, int32_t count, const int32_t *node_ids, const int32_t *adj);
/* FusedPQ feature (base:graph/disk/feature/FusedPQ.java:99-101,122-141,215-241): pack, for every node, its level-0 neighbour ids
 * and the neighbours' PQ codes into ONE record [degree int32 ids][degree code rows, zero padded] (built on the device from the
 * resident adjacency and codes). A later search whose `approx` is this PQ data set then scores neighbours from the expanded
 * node's record — FusedPQDecoder.similarityToNeighbor (base:quantization/FusedPQDecoder.java:84-114), the
 * "useEdgeLoading && level == 0" branch of OnDiskGraphIndex.java:639-651 — one contiguous read per hop; upper levels and the
 * entry node use the plain code rows (the hierarchy's cached source features, FusedPQDecoder.java:96-105). Scores are those of
 * the plain PQ walk. JV_FUSED_PQ=0 in the environment ignores the records (A/B timing). This call rewrites the graph and frees its
 * previous records: it must not run while another thread searches, fuses or otherwise uses g. */
JV_API int jv_graph_fuse_pq(jv_graph g, jv_dataset pq);
/* records_out [n][*record_bytes] (query the size with records_out = NULL first) */
JV_API int jv_graph_fused_download(jv_graph g, uint8_t *records_out, int *record_bytes);
JV_API int jv_graph_free(jv_graph g);
JV_API int jv_graph_info(jv_graph g, int32_t *n, int *degree, int *levels, int32_t *entry_node);
JV_API int jv_graph_download(jv_graph g, int level, int32_t *node_ids_out, int32_t *adj_out, int32_t *count_out);

typedef struct {
    int64_t visited;       /* sum over queries of SearchResult.visitedCount (GraphSearcher.java:445-449) */
    int64_t expanded;      /* expandedCount */
    int64_t expanded_base; /* expandedCountBaseLayer */
    int64_t reranked;      /* reranked */
    int64_t retried;       /* queries re-run with a larger visited table */
    double device_ms;      /* CUDA-event time of the device work of this call */
} jv_search_stats;

/* GraphSearcher.search for nq queries at once: traversal scored by `approx`, optional exact rerank by `reranker`
 * (NULL = none, then rerankK survivors are cut to topK by approximate score as GraphSearcher.java:478-486).
 * nodes_out/scores_out [nq][topK], best first, padded with -1 / 0.
 * Host buffers: a batch of >= 1 MB of queries is copied in chunks on a second stream while the search kernel already runs (each
 * query is read only after its chunk has arrived), so with pinned (jv_host_register / cudaHostRegister) buffers the H2D copy is
 * hidden behind the first wave of queries; pageable buffers work and simply copy first. device_ms then includes that overlap. */
JV_API int jv_graph_search_batch(jv_graph g, jv_dataset approx, jv_dataset reranker, int metric,
                                 const float *queries, int nq, int topK, int rerankK,
                                 int32_t *nodes_out, float *scores_out, jv_search_stats *stats);
/* GraphSearcher.search(scoreProvider, topK, rerankK, threshold, rerankFloor, acceptOrds) — base:graph/GraphSearcher.java:166-181.
 * accept_bits: bit (node & 31) of 32-bit word (node >> 5) set = the node may be a RESULT (it is still traversed), applied on
 * level 0 only as searchOneLayer does (:427-431); accept_stride_words = 0 shares one bitset between all queries of the batch,
 * otherwise query i uses accept_bits + i * accept_stride_words. threshold: minimum approximate score of a result (the
 * TwoPhaseTracker early-termination heuristic of ScoreTracker.java is NOT run: a threshold search here visits at least what
 * the reference visits). rerank_floor: NodeQueue.rerank's rerankFloor (NodeQueue.java:168-230). NULL = {NULL, 0, 0, 0}.
 * A filter that rejects most nodes needs a long candidate list; beyond 8192 live candidates the call fails with JV_ERR_OVERFLOW.
 * For filters that selective (roughly under rerankK / 8192 of the rows accepted), jv_exhaustive_search_batch scores the accepted
 * rows instead, at about what they cost, with the same options and outputs. */
typedef struct {
    const uint32_t *accept_bits;
    int64_t accept_stride_words;
    float threshold;
    float rerank_floor;
} jv_search_options;
JV_API int jv_graph_search_batch_ex(jv_graph g, jv_dataset approx, jv_dataset reranker, int metric,
                                    const float *queries, int nq, int topK, int rerankK, const jv_search_options *opts,
                                    int32_t *nodes_out, float *scores_out, jv_search_stats *stats);
/* same with queries / outputs already in HBM (no host copies in the call) */
JV_API int jv_graph_search_batch_device(jv_graph g, jv_dataset approx, jv_dataset reranker, int metric,
                                        const float *queries_device, int nq, int topK, int rerankK,
                                        int32_t *nodes_out_device, float *scores_out_device, jv_search_stats *stats);

/* _ex form with everything in HBM; opts->accept_bits is a DEVICE pointer here */
JV_API int jv_graph_search_batch_device_ex(jv_graph g, jv_dataset approx, jv_dataset reranker, int metric,
                                           const float *queries_device, int nq, int topK, int rerankK,
                                           const jv_search_options *opts_device_bits, int32_t *nodes_out_device,
                                           float *scores_out_device, jv_search_stats *stats);

/* jv_topk_bruteforce restricted to the rows each query accepts (opts->accept_bits, host memory, the layout and stride above; bits
 * at positions >= n are ignored) and, when opts->threshold > 0, to the rows scoring >= it. Same keys: best first, ties to the
 * smaller id, padded with INT64_MIN. opts == NULL, or accept_bits == NULL at threshold 0, is jv_topk_bruteforce byte for byte.
 * rerank_floor must be 0. Every storage kind; BQ takes the popcount kernels (DESIGN §4.2a). */
JV_API int jv_topk_bruteforce_ex(jv_dataset ds, int metric, const float *queries, int nq, int k, const jv_search_options *opts,
                                 int64_t *keys_out);
/* jv_graph_search_batch_ex without a graph: the candidates are the jv_topk_bruteforce_ex keys at k = rerankK (rerankK <= 2048).
 * No reranker: the first topK. With one (fp32 or NVQ): NodeQueue.rerank's take rule at opts->rerank_floor (the candidates whose
 * approximate score is >= it, or the best one when none is), rescored exactly and returned in key order (equal exact scores: the
 * smaller id first). nodes_out / scores_out [nq][topK], -1 / 0 padded. stats: visited = accepted rows scored (summed over queries),
 * reranked = candidates rescored, expanded = expanded_base = retried = 0, device_ms = CUDA-event time of the call. */
JV_API int jv_exhaustive_search_batch(jv_dataset approx, jv_dataset reranker, int metric, const float *queries, int nq, int topK,
                                      int rerankK, const jv_search_options *opts, int32_t *nodes_out, float *scores_out,
                                      jv_search_stats *stats);

/* Segments: one index split into segment graphs, each over its own rows (data arrives as small segment indexes that are compacted
 * from time to time, jv_graph_compact), searched in one call. Segment s answers what
 *   jv_graph_search_batch_ex(graph, approx, reranker, metric, queries, nq, topK, rerankK, {accept_bits, 0, threshold, rerank_floor})
 * answers, or, with graph == NULL, what jv_exhaustive_search_batch answers with the same arguments; a graph whose every node was
 * removed answers nothing. Each query's output is the first topK entries of the stable merge of those lists: padding dropped, score
 * descending (compared as the top-k key's sortable score), equal scores in segment order, then in list order; padded with segment -1,
 * node -1, score 0. With one segment, nodes_out and scores_out are jv_graph_search_batch_ex's bytes.
 * Every walked (segment, query) pair runs in one launch per kind of walk (segments with and without edge records, DESIGN §4.1); the
 * merge runs on the device. Segments keep their own codebooks; they must share the device, the storage kind and dim (PQ: M and k,
 * NVQ: sub-vectors) and the reranker kind (all NULL or all of one kind). stats sums the segments' visited, expanded, expanded_base
 * and reranked; retried counts the (segment, query) pairs re-run; device_ms is the CUDA-event time of the call. segment_stats
 * (NULL or [nsegments]): each segment's counters as its own call reports them, with this call's retried and device_ms.
 * JV_ERR_UNSUPPORTED: nsegments > 1024, nsegments * topK > 16384, rerankK > 4096 (2048 with a segment without graph), or what the
 * segment's own call refuses as unsupported. All checks precede any device work: a refused call writes no output. */
typedef struct {
    jv_graph graph;              /* NULL: the segment is searched as jv_exhaustive_search_batch searches it */
    jv_dataset approx;           /* walked (or scanned) scores; its n is the graph's n */
    jv_dataset reranker;         /* NULL, or fp32 / NVQ, as for jv_graph_search_batch_ex */
    const uint32_t *accept_bits; /* host; one bitset over the segment's n, shared by every query (the segment's live rows); NULL = all */
} jv_search_segment;
JV_API int jv_segments_search_batch(const jv_search_segment *segments, int nsegments, int metric, const float *queries, int nq, int topK,
                                    int rerankK, float threshold, float rerank_floor, int32_t *segments_out, int32_t *nodes_out,
                                    float *scores_out, jv_search_stats *stats, jv_search_stats *segment_stats);

/* Replicas: graph + data sets registered once per device (jv_gpu_set_device(d), then the ordinary create / register calls); the
 * batch is split into contiguous slices, one per replica, searched concurrently (no data-path exchange). stats sums the counters,
 * device_ms is the slowest replica. */
JV_API int jv_multi_graph_search_batch(int replicas, const jv_graph *graphs, const jv_dataset *approx, const jv_dataset *rerankers,
                                       int metric, const float *queries, int nq, int topK, int rerankK, const jv_search_options *opts,
                                       int32_t *nodes_out, float *scores_out, jv_search_stats *stats);

/* GraphIndexBuilder.build over an f32 data set with exact scoring (BuildScoreProvider.randomAccessScoreProvider):
 * batched inserts, device-side beam search + Vamana robust prune + back-links. */
typedef struct {
    int degree;        /* M */
    int beam_width;    /* efConstruction */
    float overflow;    /* neighborOverflow, e.g. 1.2 */
    float alpha;       /* 1.2 */
    int add_hierarchy; /* HNSW-style upper levels (GraphIndexBuilder.java:562-575) */
    uint64_t seed;
    int max_batch;     /* 0 = default (16384): nodes inserted per round; they play the reference's concurrently inserting threads */
    int concurrent_window; /* in-progress peers each insert sees besides its beam (getConcurrentCandidates,
                              GraphIndexBuilder.java:823-837): -1 = default (what fits the 128-candidate prune tile, <= 32), 0 = none;
                              beam_width + concurrent_window <= 256 (the prune's candidate capacity), else JV_ERR_INVALID */
} jv_build_params;
JV_API int jv_graph_build(jv_dataset f32, int metric, const jv_build_params *params, jv_graph *out, double *device_ms);
/* The same build over PQ codes (BuildScoreProvider.pqBuildScoreProvider, for indexes whose fp32 rows do not fit in memory): the
 * insert of node v searches with the query decode(c_v) over the codes (no rerank, topK = rerankK = beam_width), the prune's keys are
 * the ADC scores under decode(c_v)'s LUT, and its pair similarities sum the centroid-pair table of the metric (ImmutablePQVectors'
 * diversity; built and kept on the data set when it has none, as jv_dataset_pq_pair_table does). Everything else is jv_graph_build's.
 * Errors: JV_ERR_INVALID for a null argument, a data set that is not PQ or a bad metric; JV_ERR_UNSUPPORTED for a degree above 64
 * or a LUT the prune cannot hold in shared memory (M * k above ~56 K entries, e.g. M > 216 at k = 256). jv_graph_build_stats then
 * reports this build. */
JV_API int jv_graph_build_pq(jv_dataset pq, int metric, const jv_build_params *params, jv_graph *out, double *device_ms);
/* The same build advanced batch by batch, for a build SHARDED over several GPUs (BASELINE config 5): every participant holds a
 * replica of the rows and of the adjacency; per batch each one searches + prunes ITS slice (jv_builder_insert_slice), the caller
 * all-gathers the slices (NCCL; jvector_b200/parallel.py sharded_build), every participant applies the whole batch — back-links in
 * sorted order, so all replicas stay bit-identical — and the rows that passed overflow * M are re-pruned slice-wise and exchanged
 * the same way. All *_device pointers are device buffers of the caller (the collective's send / receive buffers); work is
 * enqueued on `cuda_stream`. Slices are positions [lo, hi) of the batch (insert) or of the sorted overflow list (re-prune). */
typedef struct jv_builder_s *jv_builder;
JV_API int jv_builder_create(jv_dataset f32, int metric, const jv_build_params *params, void *cuda_stream, jv_builder *out);
/* the step-wise form of jv_graph_build_pq (same checks and errors); every other jv_builder_* call works on either kind */
JV_API int jv_builder_create_pq(jv_dataset pq, int metric, const jv_build_params *params, void *cuda_stream, jv_builder *out);
JV_API int jv_builder_info(jv_builder b, int *degree, int *row_cap, int *max_batch);
JV_API int jv_builder_next_batch(jv_builder b, int32_t *first, int32_t *count); /* count = 0: every node is inserted */
JV_API int jv_builder_insert_slice(jv_builder b, int32_t first, int32_t count, int32_t lo, int32_t hi,
                                   int32_t *rows_out_device /* [count][degree], rows lo..hi-1 written */, int32_t *deg_out_device /* [count] */);
/* rows of the WHOLE batch; overflow_rows (optional, forces a stream sync): length of the sorted list of rows to re-prune */
JV_API int jv_builder_apply_new(jv_builder b, int32_t first, int32_t count, const int32_t *rows_device, const int32_t *deg_device, int32_t *overflow_rows);
JV_API int jv_builder_reprune_slice(jv_builder b, int32_t lo, int32_t hi, int32_t *rows_out_device /* [.][row_cap] */, int32_t *deg_out_device);
JV_API int jv_builder_apply_repruned(jv_builder b, int32_t count, const int32_t *rows_device, const int32_t *deg_device);
/* cleanup(): the sorted list of rows longer than M (enforceDegree), to be re-pruned with the two calls above */
JV_API int jv_builder_collect_over_degree(jv_builder b, int32_t *rows);
JV_API int jv_builder_finish(jv_builder b, jv_graph *out, double *device_ms);
/* counters so far (synchronises the builder's stream; valid before and after jv_builder_finish): batches applied, insert searches
 * cut short by a full visited table or an oversized tie tail (0 = every insert search was exact), back-links dropped because the
 * target's row was full */
JV_API int jv_builder_stats(jv_builder b, int64_t *batches, int64_t *truncated_searches, int64_t *dropped_backlinks);
JV_API int jv_builder_free(jv_builder b);
/* counters of this thread's last jv_graph_build (level 0): vectors scored by the insert searches, batches, back-links dropped */
JV_API int jv_graph_build_stats(int64_t *scored_vectors, int64_t *batches, int64_t *dropped_backlinks);

/* GraphIndexBuilder.removeDeletedNodes (base:graph/GraphIndexBuilder.java:689-799) on the device: the nodes set in deleted_bits
 * are taken out of every level, and every live row that named one of them is re-pruned (retainDiverse at `alpha`, exact fp32
 * scores over `f32`, which must be the graph's own rows) over its live neighbours and the live neighbours of its deleted ones.
 * A row whose deleted neighbours offer no live candidate tries 2 * degree random live members of its level instead; the
 * generator is a fixed function of (seed, level, node, attempt), so the result is reproducible. Rows that named no deleted node
 * are copied unchanged.
 * The result is a NEW graph (`g` is not modified; searches holding it keep a consistent snapshot) without FusedPQ records.
 * Removed ids stay as holes: their level-0 rows are -1, they belong to no upper level, no row names them, and the new graph
 * remembers them (a later removal counts them as gone). If the entry node is deleted, the new entry is the lowest live id of the
 * highest level that keeps a live member, and emptied levels above it are dropped. With every node deleted the graph has entry
 * -1 and one level; searching it returns -1 / 0 padded results. Degrees above 64 are JV_ERR_UNSUPPORTED. */
typedef struct {
    int32_t live_nodes;       /* level-0 nodes left (graph.size(0) after the call) */
    int32_t removed;          /* nodes removed by this call */
    int64_t repaired_rows;    /* rows (all levels) that lost a neighbour and were re-pruned */
    int64_t candidates;       /* distinct candidates scored, summed over the repaired rows */
    int32_t max_candidates;   /* largest candidate set of one row */
    int64_t random_fallbacks; /* rows whose deleted neighbours offered no live candidate */
    double device_ms;
} jv_remove_stats;
JV_API int jv_graph_remove_deleted(jv_graph g, jv_dataset f32, int metric, float alpha, uint64_t seed,
                                   const uint32_t *deleted_bits /* host, bit (node & 31) of word (node >> 5) */,
                                   jv_graph *out, jv_remove_stats *stats);

/* GraphIndexBuilder.addGraphNode (base:graph/GraphIndexBuilder.java:588-659) for a batch, on the device: nodes n0 .. n-1 of `f32`
 * (n rows, n >= n0 = g's size) are inserted into g in id order, as a build inserts them: batches of inserted / 32 nodes, at most
 * max_batch; beam search of the graph as it stands, robust prune of the beam and the in-progress window, sorted back-links,
 * re-prune of overflowing rows, and the final over-degree cleanup over all n rows. Rows [0, n0) of `f32` must be g's own nodes
 * (the call cannot check it): grow the data set by registering a longer one, or adopt a longer prefix of the same device buffer
 * with jv_dataset_adopt_f32_device, which copies nothing.
 * The result is a NEW graph of n nodes (`g` is not modified) without FusedPQ records. g's holes (jv_graph_remove_deleted) stay
 * holes: the new graph remembers them, widened to n, so a later removal still counts them as gone.
 * Level 0: g's rows seed the builder, each with its -1 slots squeezed out (entries keep their order); the insert searches walk
 * level 0 from g's entry node (not down through the hierarchy). If g has no entry (every node removed), node n0 becomes the
 * entry with an empty row.
 * Upper levels (only when g has them): new node i takes draw i of the build's level draws for n nodes and `params->seed`, so a
 * node's level does not depend on when it was added. A level of g that gains members is extended the same way (its old members'
 * rows seed the builder, the inserts start at the entry); levels above g's top are built over their new members, and the lowest
 * id of the new top level becomes the entry. params->add_hierarchy is ignored: the hierarchy follows g.
 * params: degree must equal g's; beam_width, overflow, alpha, max_batch, concurrent_window and seed mean what they mean for a build.
 * deleted_bits (optional, host, ceil(n0 / 32) words, the accept_bits layout): nodes marked deleted but not yet removed. The
 * insert searches walk through them but never pick one as a neighbour of a new node (the liveNodes() filter of :630-632).
 * n == n0 returns a copy of g. Errors: JV_ERR_INVALID for a null argument, a data set that is not fp32, n < n0, a device
 * mismatch, a degree mismatch or a bad metric; JV_ERR_UNSUPPORTED for a degree above 64. jv_graph_build_stats then reports the
 * level-0 insert; device_ms covers the whole call. */
JV_API int jv_graph_add_nodes(jv_graph g, jv_dataset f32, int metric, const jv_build_params *params, const uint32_t *deleted_bits,
                              jv_graph *out, double *device_ms);
/* The same add, step by step: a builder seeded from g exactly as jv_graph_add_nodes seeds it, driven by the jv_builder_* calls
 * above (jv_builder_next_batch starts at node n0); jv_builder_finish extends the upper levels as jv_graph_add_nodes does. g is no
 * longer read once this returns. */
JV_API int jv_builder_create_from_graph(jv_graph g, jv_dataset f32, int metric, const jv_build_params *params, const uint32_t *deleted_bits,
                                        void *cuda_stream, jv_builder *out);

/* ---- maintaining a graph over PQ codes (addGraphNode / removeDeletedNodes under BuildScoreProvider.pqBuildScoreProvider) ----
 * The three calls below are jv_graph_add_nodes, jv_builder_create_from_graph and jv_graph_remove_deleted over a PQ data set, for
 * an index whose fp32 rows do not fit in memory. Everything their contracts say that does not mention scores holds unchanged: the
 * result is a NEW graph without FusedPQ records and the input is not modified; holes are carried (and widened by an add); the
 * deleted_bits layout; n == n0 returns a copy; an add with no entry makes node n0 the entry; the level draws of new nodes and the
 * extension of upper levels; how a removal picks its new entry, drops emptied levels, and answers searches when every node is gone;
 * what jv_graph_build_stats and jv_remove_stats report.
 * The scores are those of jv_graph_build_pq: the insert or repair of node v uses the query decode(c_v); keys are the ADC scores of
 * the PQ walk under that query's LUT; pair similarities sum the metric's centroid-pair table (built and kept on the data set when
 * it has none). An add into a one-node graph therefore gives the bytes of jv_graph_build_pq, and a node's row does not depend on
 * whether the caller still held its fp32 vector when it was added.
 * Rows [0, n0) of `pq` must be the graph's own nodes, encoded with the same codebooks (the calls cannot check it). A PQ data set
 * does not grow in place: encode the new rows with jv_pq_encode_batch (nothing new is needed for that) and register the longer
 * code array with jv_dataset_register_pq.
 * The removal's prune runs at the smallest of 64 / 128 / 256 / 1024 / 2048 / 8192 candidate slots that holds a row's distinct
 * candidates, and keeps the whole LUT of M * k floats in shared memory next to them (13 bytes per slot). A row gathers at most
 * degree * (degree + 2) candidates, so a call needs the smallest capacity at or above that: 2048 slots up to degree 44, 8192
 * above. When the LUT and that capacity do not fit in 226 KB together (e.g. degree 64 with M above ~118 at k = 256) the call is
 * refused; no candidate set is ever clipped.
 * Errors: JV_ERR_INVALID for a null argument, a data set that is not PQ, n < n0 (add) or n != g's size (remove), a device
 * mismatch, a degree mismatch, a bad metric or alpha < 1; JV_ERR_UNSUPPORTED for a degree above 64, or a LUT the prune cannot hold
 * at the capacity the call may need (add: the builder's 256 slots, as jv_graph_build_pq). Every check precedes the device work:
 * a refused call has done none of it and leaves *out untouched. jv_graph_add_nodes, jv_builder_create_from_graph and
 * jv_graph_remove_deleted keep answering JV_ERR_INVALID for a PQ data set. */
JV_API int jv_graph_add_nodes_pq(jv_graph g, jv_dataset pq, int metric, const jv_build_params *params, const uint32_t *deleted_bits,
                                 jv_graph *out, double *device_ms);
/* the step-wise form, driven by the jv_builder_* calls like jv_builder_create_from_graph's builder */
JV_API int jv_builder_create_from_graph_pq(jv_graph g, jv_dataset pq, int metric, const jv_build_params *params, const uint32_t *deleted_bits,
                                           void *cuda_stream, jv_builder *out);
JV_API int jv_graph_remove_deleted_pq(jv_graph g, jv_dataset pq, int metric, float alpha, uint64_t seed,
                                      const uint32_t *deleted_bits /* host, bit (node & 31) of word (node >> 5) */,
                                      jv_graph *out, jv_remove_stats *stats);

/* ---- building and maintaining a graph over BQ codes (BuildScoreProvider.bqBuildScoreProvider) ----
 * jv_graph_build, jv_builder_create, jv_graph_add_nodes, jv_builder_create_from_graph and jv_graph_remove_deleted over a BQ data
 * set, for an index that keeps only its binary codes (ceil(dim / 64) * 8 bytes per node: 192 B at 1536 dims, against 6 144 B of fp32
 * rows). Everything their contracts say that does not mention scores holds unchanged, as for the PQ calls above: batches, window,
 * back-links, re-prunes and cleanup; the level draws and upper levels; the add's seeding, entry rule and deleted_bits; the removal's
 * candidate gathering, random fallback, entry rule and holes; what jv_graph_build_stats and jv_remove_stats report.
 * The scores are BQVectors': the insert or repair of node v searches with its own code c_v as the query (the BQ walk, no rerank,
 * topK = rerankK = beam_width), the prune's keys are 1 - hd(c_v, c_u) / dim — the walk's own scores — and its pair similarities
 * 1 - hd(c_a, c_b) / dim. No score depends on the metric: it is checked as every call checks it, and the three metrics give the same
 * bytes. An add into a one-node graph gives the bytes of jv_graph_build_bq.
 * Rows [0, n0) of `bq` must be the graph's own nodes (the calls cannot check it). A BQ data set does not grow in place: encode the
 * new rows with jv_bq_encode_batch and register the longer word array with jv_dataset_register_bq.
 * No row may set a bit past dim in its last word (BinaryQuantization.encode and jv_bq_encode_* never do): the walk's query, re-encoded
 * from c_v, has those bits clear while the pair scores read the raw words. The calls check every row, with one small reduction before
 * any other device work.
 * The removal's prune runs at the smallest of 64 / 128 / 256 / 1024 / 2048 / 8192 candidate slots that holds a row's distinct
 * candidates; every degree up to 64 fits, so no candidate set is ever clipped and no call is refused for shared memory.
 * Errors: JV_ERR_INVALID for a null argument, a data set that is not BQ, a row with bits set past dim, n < n0 (add) or n != g's size
 * (remove), a device mismatch, a degree mismatch, a bad metric or alpha < 1; JV_ERR_UNSUPPORTED for a degree above 64. Every check
 * precedes the device work: a refused call has done none of it and leaves *out untouched. The fp32 and PQ calls keep refusing a BQ
 * data set with the codes they return for it. */
JV_API int jv_graph_build_bq(jv_dataset bq, int metric, const jv_build_params *params, jv_graph *out, double *device_ms);
/* the step-wise form of jv_graph_build_bq (same checks and errors); every other jv_builder_* call works on it unchanged */
JV_API int jv_builder_create_bq(jv_dataset bq, int metric, const jv_build_params *params, void *cuda_stream, jv_builder *out);
JV_API int jv_graph_add_nodes_bq(jv_graph g, jv_dataset bq, int metric, const jv_build_params *params, const uint32_t *deleted_bits,
                                 jv_graph *out, double *device_ms);
/* the step-wise form of jv_graph_add_nodes_bq, driven by the jv_builder_* calls like jv_builder_create_from_graph's builder */
JV_API int jv_builder_create_from_graph_bq(jv_graph g, jv_dataset bq, int metric, const jv_build_params *params, const uint32_t *deleted_bits,
                                           void *cuda_stream, jv_builder *out);
JV_API int jv_graph_remove_deleted_bq(jv_graph g, jv_dataset bq, int metric, float alpha, uint64_t seed,
                                      const uint32_t *deleted_bits /* host, bit (node & 31) of word (node >> 5) */,
                                      jv_graph *out, jv_remove_stats *stats);

/* ---- merging graphs: OnDiskGraphIndexCompactor's per-node work (graph/disk/OnDiskGraphIndexCompactor.java) on the device ----
 * S source graphs over fp32 rows become one graph over their live nodes, renumbered by each source's old_to_new. With
 * searchTopK = max(2, ceil(degree / S) * 4), every live node v of source s at level L gets as candidates its live neighbours at L
 * in s and, from every other source t that has a level L, the searchTopK best live members of t's level L: a search of t's graph
 * with v's row as the query (level 0), or a greedy descent from t's entry to level L + 1 and a beam of searchTopK on level L (upper
 * levels). When t has at most searchTopK live members at L, they are all candidates and no search runs (the set an exhaustive search
 * returns). Exact fp32 scores under `metric` order the candidates (equal scores: the lower new id first) and retainDiverse at
 * `alpha` picks the row, as the builder's prune does.
 * The new graph has a level L for every level some source has that keeps a live member; v sits at L iff it does in its source. Its
 * entry is the entry of the first source, in source order, whose top level is the merged top level and whose entry is live,
 * otherwise the lowest new id of the top level. It has no holes and no FusedPQ records. rows_out is a new fp32 data set of the live
 * rows in new-id order, the rows a search of the new graph needs. The sources are not modified.
 * Errors, all before any device work (a refused call leaves *graph_out and *rows_out as they were): JV_ERR_INVALID for a null
 * argument, nsources < 1, rows that are not fp32 or do not match their graph's size, unequal dims, degrees or devices, a bad
 * metric, alpha < 1, no live node, or new ids of the live nodes that are not exactly [0, live nodes); JV_ERR_UNSUPPORTED for a
 * degree above 64, or degree + (S - 1) * searchTopK above 8192 (more than 2033 sources at degree 64). JV_ERR_OVERFLOW when a search overflows its candidate list even after retries; what the call allocated is freed. */
typedef struct {
    jv_graph graph;            /* source graph; its holes (jv_graph_remove_deleted) count as dead */
    jv_dataset rows;           /* its fp32 rows (row i = node i); all sources on one device, with one dim */
    const uint32_t *live_bits; /* host, bit (node & 31) of word (node >> 5) over the graph's n; NULL = every node but holes live */
    const int32_t *old_to_new; /* host [n]; read for live nodes only */
} jv_compact_source;
typedef struct {
    int32_t nodes;          /* live nodes merged = the new graph's size */
    int levels;             /* levels of the new graph */
    int search_top_k;       /* the searchTopK used */
    int64_t searches;       /* (query, other source, level) searches run */
    int64_t exhaustive;     /* (query, other source, level) pairs answered by the whole live membership instead */
    int64_t candidates;     /* summed over all rows of all levels */
    int32_t max_candidates; /* largest candidate set of one row */
    int64_t visited;        /* summed visited counts of the searches */
    double device_ms;
} jv_compact_stats;
JV_API int jv_graph_compact(const jv_compact_source *sources, int nsources, int metric, float alpha, jv_graph *graph_out, jv_dataset *rows_out,
                            jv_compact_stats *stats);

/* Merging graphs whose nodes carry PQ codes (OnDiskGraphIndexCompactor's FusedPQ and sidecar compaction, DESIGN §4.3h). source_pq[i]
 * holds the codes of source i's n nodes, each source with codebooks of its own. Two forms:
 *   fused   every source graph carries FusedPQ records packed from its own source_pq[i] (jv_graph_fuse_pq): the search of another
 *           source t walks t's records (t's plain code rows above level 0) and reranks its searchTopK survivors exactly over t's rows;
 *           the merged graph is fused with the new codes;
 *   sidecar no source carries records: the merge is jv_graph_compact's, graph and rows byte for byte; the merged graph has no records.
 * Anything else (a mix, records packed from other codes) is refused. Either form then retrains PQ as PQRetrainer.retrain does: a
 * balanced sample of at most 128 000 live rows across the sources (PQRetrainer.sampleBalanced, chunks of 32 nodes in a Fisher-Yates
 * order drawn from `seed`), on which source 0's codebooks (and centroid) are refined by 6 unweighted Lloyd rounds (jv_pq_refine with
 * that seed). The merged rows, encoded with the new codebooks, become a new resident PQ data set in *pq_out (M, k and centroid are
 * source 0's). codebooks_out [k * dim] receives the new codebooks, centroid_out [dim] source 0's centroid (NULL allowed when source
 * 0 has none), samples_per_source_out [nsources] (or NULL) the rows sampled from each source.
 * Errors, all before any device work and leaving every output untouched: whatever jv_graph_compact refuses, with its codes, and
 * JV_ERR_INVALID for a null argument, a source_pq that is not PQ or differs from its graph in size, dim or device, sources of both
 * forms, a NULL centroid_out when source 0's PQ has a centroid, or fewer sampled rows than k. */
typedef struct {
    jv_compact_stats graph;    /* the merge's counters, as jv_graph_compact fills them (device_ms: the merge only) */
    int fused;                 /* 1: the sources' FusedPQ records were walked and the output is fused; 0: sidecar form */
    int64_t train_rows;        /* rows the codebooks were refined on */
    jv_pq_train_stats train;   /* the refine's counters */
    double retrain_ms, encode_ms, fuse_ms; /* stream time of the sample's gather and the refine, of the encoding, of the fuse */
} jv_compact_pq_stats;
JV_API int jv_graph_compact_pq(const jv_compact_source *sources, const jv_dataset *source_pq, int nsources, int metric, float alpha,
                               uint64_t seed, jv_graph *graph_out, jv_dataset *rows_out, jv_dataset *pq_out,
                               float *codebooks_out /* [k * dim] */, float *centroid_out /* [dim] or NULL when source 0 has none */,
                               int64_t *samples_per_source_out /* [nsources] or NULL */, jv_compact_pq_stats *stats);

/* The refinement pass on the device (DESIGN §4.3i). Returns a NEW graph in *out; g is untouched, its holes stay holes, and the entry
 * and the level membership are unchanged. The result has no FusedPQ records. ds holds g's rows (ds's n = g's n, same device).
 * JV_REFINE_BUILDER: GraphIndexBuilder.cleanup's improveConnections, over fp32, PQ or BQ data sets with the scores their builds use.
 *   Only a graph with upper levels is refined (a flat graph comes back as a copy): at level 0 every member of level 1, at each level
 *   L >= 1 every member of L, each with a non-empty row there. Per level the nodes go in ascending batches of params->max_batch (0:
 *   16384); each batch searches the level as the previous batches left it (level 0 from the entry, without descending; an upper level
 *   as a graph of its own), beam params->beam_width, excluding the node itself; its candidates are its current row plus the results
 *   not in it; the robust prune at params->alpha picks M; back-links follow (a row that already names the node is left as it is), rows
 *   past params->overflow * M are re-pruned, and after the last batch every row longer than M is.
 * JV_REFINE_COMPACTOR: OnDiskGraphIndexCompactor's refine pass, fp32 only. Level 0 only: the members of level 1, or every live node
 *   when g is flat; beam 8 M; every search reads g as it is and the rows replace the old ones at the end, with no back-links;
 *   params->alpha is the compactor's alpha. params->beam_width, overflow and max_batch still have to be valid.
 * params->degree must equal g's degree; params->add_hierarchy, seed and concurrent_window are not read.
 * Errors, all before any device work (a refused call leaves *out untouched): JV_ERR_INVALID for a null argument, a data set whose kind
 * the mode does not take, a size or device mismatch, a degree that differs from g's, bad build parameters, a bad metric or mode;
 * JV_ERR_UNSUPPORTED for a degree above 64, or a PQ LUT the prune cannot hold next to the candidates. */
#define JV_REFINE_BUILDER 0
#define JV_REFINE_COMPACTOR 1
#define JV_REFINE_MAX_LEVELS 64
typedef struct {
    int levels;                                   /* levels refined: g's levels (builder form), 1 (compactor form), 0 for a copy */
    int64_t nodes_refined[JV_REFINE_MAX_LEVELS];  /* per level; levels past the last entry are counted in it */
    int64_t candidates;                           /* candidates scored, summed over all refined nodes */
    int32_t max_candidates;                       /* the largest candidate set of one node */
    int64_t rows_changed;                         /* rows, over all levels, whose contents differ from g's */
    int64_t backlinks_added, backlinks_dropped;   /* builder form: back-links written, and dropped at a full row */
    int64_t rows_repruned;                        /* builder form: rows re-pruned past overflow * M and by the final cleanup */
    double device_ms;                             /* stream time of the refine's device work (searches, candidates, prunes, back-links,
                                                     re-prunes), summed between the host's waits for each batch's counts; the
                                                     host's work (node lists, the upper levels' rows and id mapping) is not in it */
} jv_refine_stats;
JV_API int jv_graph_refine(jv_graph g, jv_dataset ds, int metric, const jv_build_params *params, int mode, jv_graph *out, jv_refine_stats *stats);

/* device-memory helpers for callers that keep queries/results in HBM (bench `value` leg) */
JV_API int jv_device_malloc(void **out, size_t bytes);
JV_API int jv_device_free(void *p);
JV_API int jv_memcpy_h2d(void *dst_device, const void *src_host, size_t bytes);
JV_API int jv_memcpy_d2h(void *dst_host, const void *src_device, size_t bytes);
JV_API int jv_host_register(void *p, size_t bytes); /* pin a host buffer for faster copies */
JV_API int jv_host_unregister(void *p);
JV_API int jv_device_synchronize(void);
JV_API int64_t jv_kernel_launch_count(void); /* kernels this library has launched since load */

#ifdef __cplusplus
}
#endif
#endif /* JVECTOR_B200_H */
