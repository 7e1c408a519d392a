// kernels.h — host-callable launchers of the sm_90a kernels (internal; the public surface is include/jvector_b200.h)
#pragma once
#include <algorithm>
#include <atomic>
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>

#include "scorers.cuh"

namespace jv {

extern std::atomic<long long> g_launches;  // kernels launched by this library (jv_kernel_launch_count)
constexpr int MAX_DEGREE = 128;            // widest adjacency row the search kernel accepts

// Carves a device scratch block into pieces, each starting 256-byte aligned. Over base == nullptr the same sequence of take()
// calls only measures the block, so one layout gives both the block's size and its pointers.
struct Carver {
    uintptr_t base;
    size_t bytes = 0;
    explicit Carver(void *p) : base(reinterpret_cast<uintptr_t>(p)) {}
    template <typename T>
    T *take(size_t count)
    {
        T *r = reinterpret_cast<T *>(base + bytes);
        bytes += (count * sizeof(T) + 255) & ~(size_t)255;
        return r;
    }
};

struct GraphDesc {
    int32_t n;
    int degree;
    int levels;  // >= 1
    int32_t entry_node;
    int entry_level;
    const int32_t *adj0;       // [n][degree]
    const int32_t *upper_row;  // [(levels-1)][n] row index or -1 (nullptr when levels == 1)
    const int32_t *upper_adj;  // rows of all upper levels, concatenated
    const long long *upper_off;  // [(levels-1)] first row of each level in upper_adj (device)
    // FusedPQ feature (base:graph/disk/feature/FusedPQ.java): per node ONE record = [degree int32 neighbour ids][degree code rows
    // of fused_code_stride bytes, zero padded], so a level-0 hop of a PQ walk is one contiguous read. nullptr = not fused.
    const uint8_t *fused;
    const uint8_t *fused_codes_of;  // the PQ code array the records were packed from (identity of the data set they belong to)
    int fused_rec;                  // bytes per record (multiple of 16)
    int fused_code_stride;
    // low-rank edge bound (scorers.cuh lowrank_bound): [n][degree][LR_SLOT], slot t = the low-rank row of adj0[v][t]. Set per search
    // (api.cu search_device) for a sketched walk over the data set the records were built from; nullptr otherwise
    const uint8_t *edge_rec;
};

struct SearchCounters {  // device-side totals
    unsigned long long visited, expanded, expanded_base, reranked, overflowed;
    unsigned long long settled;  // new neighbours settled on their edge record (part of `visited`)
    unsigned long long direct, direct_dropped;  // new neighbours routed direct to their full row, and of them those the list refused
};

// ---- kernels_batch.cu ----
cudaError_t launch_prepare(const DataDesc &d, int metric, const float *queries_dev, int nq, float *blobs_dev, cudaStream_t s);
// ragged: query qi scores ids[offsets[qi]..offsets[qi+1]); offsets == nullptr: every query scores ids[0..n) -> scores[qi*n + i]
constexpr int HOP_MAX_IDS = 64;
struct HopIds { int32_t ids[HOP_MAX_IDS]; };
// one hop of one search with the ids in the kernel parameters and the scores stored to mapped host memory (latency path)
cudaError_t launch_score_hop(const DataDesc &d, int metric, const float *blob_dev, const int32_t *ids_host, int n, float *scores_mapped, cudaStream_t s);
cudaError_t launch_score_ragged(const DataDesc &d, int metric, const float *blobs_dev, int nq, const int32_t *ids_dev,
                                const int32_t *offsets_dev, int n_shared, int max_per_query, float *scores_dev, cudaStream_t s, int chunk = 0,
                                int *done_counter = nullptr, int *host_flag = nullptr, int seq = 0);
cudaError_t launch_score_pairs(const DataDesc &d, int metric, const int32_t *a_dev, const int32_t *b_dev, int n, float *out_dev, cudaStream_t s);

// sampled top-k: the rank j of the aggressive threshold among S sampled rows of n (k when the sample is the whole set)
int topk_aggressive_rank(int k, int S, long long n);
// device scratch of launch_topk_bruteforce for nq queries
size_t topk_scratch_bytes(const DataDesc &d, int nq, int k);
cudaError_t launch_topk_bruteforce(const DataDesc &d, int metric, const float *blobs_dev, int nq, int k, void *scratch_dev,
                                   long long *keys_out_dev, int *overflow_flag_dev, cudaStream_t s);

// acceptOrds-filtered top-k (jv_topk_bruteforce_ex). S = accept_sample_size(n) = launch_topk_bruteforce's sample size.
// launch_accept_compact: per bitset (bits + b * stride_words), cnt[b] = its rows < n whose bit is set, and ids[b * S + i],
// i < min(cnt, S): the accepted row of rank floor(i cnt / min(cnt, S)) (every accepted row in ascending order when cnt <= S).
int accept_sample_size(long long n);
cudaError_t launch_accept_compact(const uint32_t *bits_dev, long long stride_words, int nsets, long long n, int *cnt_dev, int32_t *ids_dev, cudaStream_t s);
struct AcceptLists {
    const uint32_t *bits;      // device: the bitsets
    long long stride_words;    // between two queries' bitsets; 0 = one bitset shared by the batch
    bool per_query;            // cnt / ids hold one entry per query (else one shared)
    const int *cnt;            // launch_accept_compact's counts
    const int32_t *ids;        // and lists
    int max_listed;            // max over the batch of min(cnt, S)
    const int *sampled;        // device: the queries with cnt > S (the sampled tier), n_sampled of them
    int n_sampled;
};
// keys of the k best accepted rows scoring >= the threshold (floor_key: its lowest key; KEY_MIN = none) per query, padded with KEY_MIN.
// scratch: topk_scratch_bytes(d, nq, k); *overflow_flag_dev as launch_topk_bruteforce's
cudaError_t launch_topk_accepted(const DataDesc &d, int metric, const float *blobs_dev, int nq, int k, const AcceptLists &acc, long long floor_key,
                                 void *scratch_dev, long long *keys_out_dev, int *overflow_flag_dev, cudaStream_t s);
// exhaustive search's last step over R sorted candidate keys per query: rr == nullptr: the first topK; else NodeQueue.rerank's take
// rule at `floor` (ids_dev [nq][R]: taken nodes, -1 elsewhere, offsets_dev [nq + 1]; *taken_dev += their count), their exact scores
// under the reranker (rblobs_dev: its prepared queries; exact_dev [nq][R]), the topK best exact keys. Out: nodes / scores [nq][topK],
// -1 / 0 padded
cudaError_t launch_rerank_accepted(const DataDesc *rr, int metric, const float *rblobs_dev, int nq, int R, int topK, float floor, const long long *cand_dev,
                                   int32_t *ids_dev, int32_t *offsets_dev, float *exact_dev, unsigned long long *taken_dev, int32_t *nodes_dev, float *scores_dev,
                                   cudaStream_t s);

cudaError_t launch_add_int(int *dst_dev, const int *src_dev, cudaStream_t s);
// keys[i] -> same score, node id + id_base (KEY_MIN pads untouched)
cudaError_t launch_key_rebase(long long *keys_dev, long long count, long long id_base, cudaStream_t s);
// per query: the k best of parts*k keys (the NCCL-gathered per-shard top-k), descending
cudaError_t launch_topk_merge(const long long *keys_in_dev, int nq, int parts, int k, long long *keys_out_dev, cudaStream_t s);
// the same for keys laid out [parts][nq][k] (shard-major, what peer copies / all_gather produce)
cudaError_t launch_topk_merge_strided(const long long *keys_in_dev, int nq, int parts, int k, long long *keys_out_dev, cudaStream_t s);
// the stable merge of per-segment answers nodes / scores [parts][nq][k] (node -1 = padding) into the k best per query: score
// descending, equal scores in segment order, then in list order; out: segment, node, score [nq][k], padded with -1, -1, 0.
// k <= SEGMENT_MERGE_MAX_K, parts * k <= SEGMENT_MERGE_MAX_KEYS (the keys are sorted in shared memory)
constexpr int SEGMENT_MERGE_MAX_K = 4096, SEGMENT_MERGE_MAX_KEYS = 16384;
cudaError_t launch_segment_merge(const int32_t *nodes_in_dev, const float *scores_in_dev, int nq, int parts, int k, int32_t *seg_out_dev, int32_t *nodes_out_dev,
                                 float *scores_out_dev, cudaStream_t s);

// int8 row sketch + {scale, radius} per row of an fp32 data set (the search kernel's sketch bound, see sketch_bound_pair)
cudaError_t launch_row_sketch(const float *rows_dev, long long n, int stride, int sketch_stride, int8_t *sketch_dev, float2 *meta_dev, cudaStream_t s);
// the low-rank edge bound (scorers.cuh lowrank_bound): one subspace-iteration step Y = X^T (X V) over the rows s * step, s < S
// (V, Y: [LR_K][stride] float64, Z: [S][LR_K] scratch); every row's codes and {t, rho, beta, xn} ([n][LR_SLOT]; nothing is launched for
// rows too wide to stage, lowrank_warps(stride) == 0); a graph's edge records ([n][degree][LR_SLOT], the rows of adj0's ids)
cudaError_t launch_lowrank_iteration(const float *rows_dev, int stride, long long step, int S, const double *V_dev, double *Z_dev, double *Y_dev, cudaStream_t s);
int lowrank_warps(int stride);
cudaError_t launch_lowrank_rows(const float *rows_dev, long long n, int stride, const float *B_dev, uint8_t *out_dev, cudaStream_t s);
// the low-rank bound as a DOT_PRODUCT score of row i against query i (rows_dev, queries_dev: [n][stride] zero padded), with the
// records of those rows in records_dev ([n][LR_SLOT], launch_lowrank_rows): one CTA per pair, the search kernel's device functions
cudaError_t launch_lowrank_bound_pairs(const float *B_dev, int dim, int stride, const float *queries_dev, const uint8_t *records_dev, long long n, float *out_dev, cudaStream_t s);
cudaError_t launch_edge_records(const int32_t *adj0_dev, long long n, int degree, const uint8_t *lr_rows_dev, uint8_t *rec_dev, cudaStream_t s);
cudaError_t launch_bq_encode(const float *rows_dev, long long n, int dim, int row_stride, unsigned long long *words_dev, cudaStream_t s);
cudaError_t launch_pq_encode(const DataDesc &pq, const float *rows_dev, long long n, int row_stride, uint8_t *codes_dev, cudaStream_t s);
cudaError_t launch_pq_self_magnitudes(const DataDesc &pq, float *mag_dev, cudaStream_t s);
cudaError_t launch_pq_pair_table(const DataDesc &pq, int euclidean, float *table_dev, cudaStream_t s);
cudaError_t launch_kmeans_assign(const float *points_dev, long long n, int dim, int point_stride, const float *centroids_dev, int k, int32_t *assign_dev, cudaStream_t s);
cudaError_t launch_nvq_encode(const float *rows_dev, long long n, int row_stride, int nsub, const int *sizes_dev, const int *offsets_dev,
                              const float *mean_dev, int learn, float *params_dev, uint8_t *bytes_dev, int byte_stride, cudaStream_t s);

// ---- bq_imma.cu: BQ Hamming top-k as an exact u8 contraction on the tensor cores (IMMA.16832) ----
constexpr int BQ_IMMA_CAP = 8192;  // captured keys per query in the filter pass
bool bq_imma_supported(const DataDesc &d, int k);
size_t bq_imma_scratch_bytes(long long n, int nq, int W);
// fully asynchronous on `s`: keys_out_dev [nq][k] best first with GLOBAL ids (row + id_base); *unresolved_dev = number of queries
// the integer-threshold path could not resolve (a Hamming bin wider than the buffer) — the caller falls back for those batches
cudaError_t launch_bq_topk_imma(const DataDesc &d, const float *queries_dev, int nq, int k, long long id_base, void *scratch_dev,
                                long long *keys_out_dev, int *unresolved_dev, int sm_count, cudaStream_t s);
// ---- bq_umma.cu: the filter pass of the same pipeline on the warpgroup MMA (wgmma u8, register accumulators) ----
bool bq_umma_supported(const DataDesc &d);
size_t bq_umma_image_bytes(int nq, int W);
cudaError_t launch_bq_umma_filter(const DataDesc &d, const uint32_t *qbits_dev, int nq, int nq_pad, const int *t2_dev, const int *pb_dev, long long *buf_dev,
                                  int *cnt_dev, int cap, long long id_base, uint8_t *images_dev, int sm_count, cudaStream_t s);

// FusedPQ.writeInline (FusedPQ.java:122-141) for every node: records[node] = ids + the neighbours' code rows in neighbour order
cudaError_t launch_fuse_pq(const GraphDesc &g, const DataDesc &pq, uint8_t *records_dev, int rec_bytes, cudaStream_t s);

// ---- search.cu ----
constexpr int MAX_LIST_CAP = 8192;  // longest candidate list (entries) the search kernel keeps in shared memory
struct SearchPlan {
    int threads;
    size_t smem_bytes;
    int ctas;
    int list_cap;     // entries the candidate list retains: rerankK + room for a tie tail
    int list_alloc;   // entries per list buffer (>= list_cap, >= sort_pow2)
    int sort_pow2;    // next power of two >= rerankK
    int visited_cap;  // power of two
    int blob_in_global;  // PQ: (part of) the LUT lives in an L2-resident global slice per CTA
    int pq_smem_m;       // PQ: LUT rows of sub-spaces [0, pq_smem_m) stay in shared memory
    int pq_wide;         // PQ: the 64-register build of the kernel (residency is limited by shared memory anyway)
    int blob_floats;
    int vis_slots_log, vis_rlog;  // visited set in shared memory: log2(slots), log2(slots per region); 0 = per-CTA global table
    unsigned vis_idmask;
    int row_prefetch;             // fp32 / NVQ walks: bulk L2 prefetch of newly visited rows
    int pq_rows;                  // PQ walk: lane = candidate, warp = partial sum
};
// acceptOrds / threshold / rerankFloor of GraphSearcher.search (base:graph/GraphSearcher.java:166-181,427-431, NodeQueue.java:168-230)
struct SearchFilter {
    const uint32_t *accept_bits;    // device; bit (node & 31) of word (node >> 5) set = acceptable; nullptr = Bits.ALL
    long long accept_stride_words;  // words between the bitsets of two queries; 0 = one bitset shared by the whole batch
    float threshold;                // minimum approximate score of a result; 0 = none
    float rerank_floor;             // NodeQueue.rerank's rerankFloor; 0 = none
    int lenient;                    // builder only: overflowing walks are cut short and counted instead of failing
    const int *arrived;             // device int or nullptr: queries [0, *arrived) are in place (host-pointer searches overlap the H2D copy)
    // device [nq] or nullptr: query q walks through node exclude_ids[q] but never accepts it (a refine search of a node's own row,
    // ExcludingBits); -1 excludes nothing
    const int32_t *exclude_ids;
};
// One walked segment of a multi-segment search (api.cu jv_segments_search_batch, the walk's SEG instantiations): its graph and data
// sets as search_walk_descs leaves them, its acceptOrds bitset (device, shared by the batch; nullptr = every node) and its slot: it
// adds to counters[slot] and writes output rows [slot * nq, (slot + 1) * nq)
struct SegmentDesc {
    GraphDesc g;
    DataDesc approx, rerank;
    const uint32_t *accept_bits;
    int slot;
};
// segments walked in one launch: descs_dev [nseg], all with edge records or all without; nq queries each
struct SegmentGroup {
    const SegmentDesc *descs_dev;
    int nseg, nq;
};
// the graph and data set a walk reads: FusedPQ records only over the codes they were packed from, the row sketch only when `sketch`,
// the edge records only next to the sketch and the low-rank basis of an fp32 DOT walk
void search_walk_descs(GraphDesc &g, DataDesc &approx, int metric, bool sketch);
cudaError_t plan_search(const DataDesc &approx, const DataDesc *rerank, const GraphDesc &g, int topK, int rerankK, int nq,
                        int visited_cap_hint, int list_cap_hint, int sm_count, SearchPlan *plan);
size_t search_scratch_bytes(const SearchPlan &p);
// whether a walk of nq queries under `plan` drops neighbours on the fp32 row sketch (launch_row_sketch) when DataDesc has one
bool search_uses_sketch(const DataDesc &approx, int metric, const SearchPlan &plan, int nq);
int sketch_stride(int stride);  // int8 sketch bytes per row of an fp32 data set of `stride` floats
cudaError_t launch_search(const GraphDesc &g, const DataDesc &approx, const DataDesc *rerank, int metric, const float *queries_dev,
                          int nq, int topK, int rerankK, const SearchPlan &plan, void *scratch_dev, int *work_counter_dev,
                          int32_t *nodes_out_dev, float *scores_out_dev, SearchCounters *counters_dev, uint8_t *overflow_flags_dev,
                          const int32_t *query_index_dev, int query_stride, const SearchFilter *filter, cudaStream_t s,
                          const SegmentGroup *segments = nullptr);

// ---- build.cu ----
struct BuildParams {
    int degree, beam;
    float overflow, alpha;
    int max_batch;
    int window;  // in-progress peers every insert sees besides its beam (-1 = default: what fits the 128-candidate tile, at most 32)
};
struct BuildStats {
    long long searched, pruned, dropped_backlinks, batches;
    long long truncated_searches;  // insert searches cut short by a full visited table / an oversized tie tail (pathological inputs)
};
// The state a builder starts from (addGraphNode into an existing graph). Rows [0, count) are seeded from rows_dev [count][width]
// (-1 = empty slot), their ids mapped through row_map_dev when given (an upper level's id -> row map); the valid entries move to
// the front of each row, in their order. Rows [count, n) start empty and are inserted in order. The insert searches start at
// `entry`; entry < 0 makes row `count` the entry with an empty row, as node 0 is for a build. accept (host, ceil(n / 32) words,
// nullptr = every row): the rows an insert may pick as neighbours; the others are still walked through.
// No seed = {nullptr, 0, 0, nullptr, -1, nullptr}: the build from nothing.
struct BuilderSeed {
    const int32_t *rows_dev;
    int count, width;
    const int32_t *row_map_dev;
    int32_t entry;
    const uint32_t *accept;
};
// flat Vamana graph over rows [0, n) of an f32 data set, of a PQ data set that carries the metric's pair table
// (pqBuildScoreProvider), or of a BQ data set (bqBuildScoreProvider); adj_out_dev [n][degree] (-1 padded); entry node is 0 (or the seed's)
cudaError_t build_graph_flat(const DataDesc &f32, int metric, const BuildParams &bp, int32_t *adj_out_dev, int sm_count,
                             BuildStats *stats, cudaStream_t s, const BuilderSeed *seed = nullptr);
// the same build advanced batch by batch; a sharded build calls the *_slice functions for its part of each batch and moves the
// rows between the replicas itself (see build.cu)
struct GraphBuilder;
cudaError_t builder_create(const DataDesc &d, int metric, const BuildParams &bp, int sm_count, GraphBuilder **out, cudaStream_t s,
                           const BuilderSeed *seed = nullptr);
void builder_destroy(GraphBuilder *B);
bool builder_next_batch(GraphBuilder *B, int *first, int *count);
cudaError_t builder_insert_slice(GraphBuilder *B, int first, int count, int lo, int hi, int32_t *rows_out, int *deg_out, cudaStream_t s);
cudaError_t builder_apply_new(GraphBuilder *B, int first, int count, const int32_t *rows, const int *rdeg, cudaStream_t s, const int32_t *ids = nullptr);
cudaError_t builder_reprune_slice(GraphBuilder *B, int lo, int hi, int32_t *rows_out, int *deg_out, cudaStream_t s);
cudaError_t builder_apply_repruned(GraphBuilder *B, int count, const int32_t *rows, const int *rdeg, cudaStream_t s);
cudaError_t builder_collect_over_degree(GraphBuilder *B, cudaStream_t s);
cudaError_t builder_list_count(GraphBuilder *B, int *count_host, cudaStream_t s);
cudaError_t builder_stats(GraphBuilder *B, BuildStats *stats, cudaStream_t s);
cudaError_t builder_finish(GraphBuilder *B, int32_t *adj_out_dev, BuildStats *stats, cudaStream_t s);
int builder_row_cap(const GraphBuilder *B);
int builder_degree(const GraphBuilder *B);
int builder_max_batch(const GraphBuilder *B);
// rows [ids[i]] of an fp32 data set into out_dev [count][stride], or into rows out_ids_dev[i] of out_dev when that is given
cudaError_t launch_gather_rows(const DataDesc &f32, const int32_t *ids_dev, int count, float *out_dev, cudaStream_t s, const int32_t *out_ids_dev = nullptr);
// PQ / BQ build (pqBuildScoreProvider, bqBuildScoreProvider): the fixed-size rows [ids[i]] of the code array (PQ code rows, BQ word rows,
// code_row_bytes each) into out_dev [count][code_row_bytes]; whether the PQ prune holds the data set's LUT
int code_row_bytes(const DataDesc &d);
cudaError_t launch_gather_codes(const DataDesc &d, const int32_t *ids_dev, int count, void *out_dev, cudaStream_t s);
bool pq_prune_fits(const DataDesc &pq);
// whether some row of a BQ data set has a bit set past dim (one reduction over the last word of every row; synchronises `s`)
cudaError_t bq_padding_set(const DataDesc &bq, bool *set, cudaStream_t s);
// whether the repair's PQ prune holds the LUT next to the largest candidate set a degree-`degree` row can gather
bool pq_repair_fits(const DataDesc &pq, int degree);
// whether the ragged prune's PQ tier for up to max_cands candidates per row holds the LUT
bool pq_ragged_fits(const DataDesc &pq, int max_cands);

// removeDeletedNodes on one level (see build.cu), over an fp32 data set, a PQ data set that carries the metric's pair table and
// passes pq_repair_fits, or a BQ data set. rows: members of the level; row r is node ids_dev[r] (nullptr: node r, level 0);
// rowmap_dev[node] = the node's row on this level (nullptr: identity). dead_dev: bitset of deleted nodes (bit node & 31 of word
// node >> 5). members_dev: the level's live members, ascending (random fallback). adj_new must hold a copy of adj_old: the repaired
// rows are written into it, every other row is left as it is. Synchronises `s`.
struct RepairStats {
    long long repaired_rows, candidates, random_fallbacks;
    int max_candidates;
    // fp32: rows pruned with <= 64, <= 128, <= 256, <= 1024, more candidates; PQ, BQ: <= 64, <= 128, <= 256, <= 1024, <= 2048, more
    long long tier_rows[6];
};
cudaError_t repair_level(const DataDesc &d, int metric, float alpha, int degree, int rows, const int32_t *adj_old, int32_t *adj_new, const int32_t *ids_dev,
                         const int32_t *rowmap_dev, const uint32_t *dead_dev, const int32_t *members_dev, int nmembers, uint64_t seed, int level,
                         int sm_count, RepairStats *st, cudaStream_t s);
cudaError_t launch_clear_dead_rows(int32_t *adj_dev, int n, int degree, const uint32_t *dead_dev, cudaStream_t s);

// OnDiskGraphIndexCompactor's per-node work on one level (DESIGN §4.3h, build.cu "Compaction"). The level's rows are handed over one
// source at a time: row i of a source block is the source's live member own_row[i] of its level adjacency own_adj; its candidates
// are its live neighbours mapped through old_to_new (-1 = dead), then, per other source t, targets[t]'s candidates: the search
// results res[i * K ..] mapped through map (-1 = dead or padding), or, when res is null, the `count` new ids of list for every row.
// The candidate segment of block row i goes to cand[(row0 + i) * cand_stride ..], its count to cand_cnt[i], its offset to cand_off[i].
struct CompactTarget {
    const int32_t *res, *map, *list;
    int count;
};
cudaError_t launch_compact_assemble(int rows, int degree, int K, const int32_t *own_adj, const int32_t *own_row, const int32_t *old_to_new,
                                    const CompactTarget *targets_dev, int ntargets, long long row0, int cand_stride, int32_t *cand, long long *cand_off,
                                    int *cand_cnt, cudaStream_t s);
// the builder's prune over `rows` ragged candidate rows (the repair's tiers, mode 2, out of place): row a is node row_node[a] of d,
// its candidates cand[cand_off[a] .. + cand_cnt[a]) (hcnt: the same counts on the host); the selected rows go to out_rows
// [rows][degree], -1 padded. Synchronises `s`.
cudaError_t prune_ragged_rows(const DataDesc &d, int metric, float alpha, int degree, int rows, const int32_t *cand, const int32_t *row_node,
                              const long long *cand_off, const int *cand_cnt, const std::vector<int> &hcnt, int32_t *out_rows, int sm_count, cudaStream_t s);
// The refine pass on one level (DESIGN §4.3i, build.cu "Refinement"): rows [0, d.n) of d with adjacency adj_in_dev [d.n][degree] (-1
// padded) and entry row `entry`; nodes (host, ascending rows) are refined in batches of bp.max_batch (0: 16384) with a search of
// beam `beam` and the ragged prune to degree at bp.alpha. Builder form (compactor false): back-links through the builder's sorted step,
// re-prunes past bp.overflow * degree and the final over-degree cleanup. Compactor form: every search reads adj_in, no back-links.
// The refined adjacency goes to adj_out_dev [d.n][degree]; the counters are added to *st. Synchronises `s`.
struct RefineStats {
    long long nodes, candidates, rows_changed, backlinks_added, backlinks_dropped, rows_repruned;
    int max_candidates;
    double device_ms;  // stream time of the refine's device work (see refine_level_enqueue)
};
cudaError_t refine_level(const DataDesc &d, int metric, const BuildParams &bp, int beam, bool compactor, const int32_t *adj_in_dev, int degree, int32_t entry,
                         const std::vector<int32_t> &nodes, int32_t *adj_out_dev, int sm_count, RefineStats *st, cudaStream_t s);
// adj_dev[rows_of[a] * degree ..] = rows_dev[a * degree ..] for a < count
cudaError_t launch_scatter_rows(int32_t *adj_dev, int degree, const int32_t *rows_of_dev, int count, const int32_t *rows_dev, cudaStream_t s);

// ---- pq_train.cu: ProductQuantization.compute / refine (UNWEIGHTED) ----
struct PqTrainArgs {
    int M, k;
    int globally_center;  // compute only
    int iters;            // Lloyd iterations (>= 0)
    long long cap;        // training rows at most (> 0)
    uint64_t seed;
    int aniso_iters;      // anisotropic rounds after Lloyd (0: none, UNWEIGHTED)
    float threshold;      // the anisotropic threshold T, -1 < T < 1 (aniso_iters > 0 only); sub-spaces of at most 64 floats
};
struct PqTrainStats {
    long long train_rows;
    int max_lloyd_updates;  // centroid updates of the sub-space that ran longest
    long long changed_last;  // summed over sub-spaces: rows that moved in the sub-space's last reassignment
    long long empty_reseeds, seeding_fallbacks;
    int aniso_updates;  // the same three for the anisotropic rounds
    long long aniso_changed_last, aniso_reseeds;
    double device_ms;
};
// KMeansPlusPlusClusterer.computeParallelCostMultiplier (base:quantization/KMeansPlusPlusClusterer.java:116-124), in double
inline float pq_parallel_cost_multiplier(double threshold, int dimensions)
{
    const double par = threshold * threshold, perp = (1 - par) / (dimensions - 1);
    return (float)std::max(1.0, par / perp);
}
// init_codebooks == nullptr: compute (sample, optional centring, k-means++ seeding, Lloyd); otherwise refine from those host
// codebooks, the training rows minus `centroid` (host, optional). Host outputs: codebooks_out [k * dim] (jv_dataset_register_pq
// layout), centroid_out [dim] (compute with centring). Synchronises `s`.
cudaError_t pq_train(const DataDesc &f32, const PqTrainArgs &p, const float *init_codebooks, const float *centroid, float *codebooks_out,
                     float *centroid_out, PqTrainStats *st, cudaStream_t s);

// ---- pq_encode_aniso.cu: ProductQuantization.encodeAnisotropic ----
struct PqEncodeStats {
    long long rows_moved, moves;  // rows whose code left its minimum-residual start; coordinate-descent moves in all
    int max_sweeps;               // sweeps of the row that ran longest (the last one changes nothing, or it is the 10th)
};
// pq: KIND_PQ descriptor with device codebooks, layout and optional centroid (its n is unused); rows_dev [n] rows of row_stride
// floats; pcm = pq_parallel_cost_multiplier(T, dim). scratch: pq_encode_aniso_scratch(dim, M, k) bytes. codes_dev [n][M].
// Does not synchronise; stats_dev: 3 uint64 counters, zeroed by the call.
size_t pq_encode_aniso_scratch(int dim, int M, int k);
cudaError_t launch_pq_encode_aniso(const DataDesc &pq, const float *rows_dev, long long n, int row_stride, float pcm, void *scratch,
                                   unsigned long long *stats_dev, uint8_t *codes_dev, cudaStream_t s);
}  // namespace jv
