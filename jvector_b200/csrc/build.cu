// build.cu — GraphIndexBuilder.build on the device, exact fp32 scoring
// (base:graph/GraphIndexBuilder.java:436-448 build, :605-671 addGraphNode / updateNeighborsOneLayer;
//  base:graph/OnHeapGraphIndex.java:279-282 addEdges; base:graph/ConcurrentNeighborMap.java:104-110 insertDiverse,
//  :158-165 backlink, :286-321 insert with overflow, :214-222 enforceDegree;
//  base:graph/diversity/VamanaDiversityProvider.java:45-95 retainDiverse / isDiverse).
//
// The reference inserts nodes concurrently from a ForkJoinPool; every insert is (1) a beam search of the graph as it
// stands, (2) a Vamana robust prune of the beam, (3) back-links into the chosen neighbours, re-pruning a neighbour
// whose list exceeds overflow * M. Here a BATCH of nodes plays the role of the concurrently inserting threads:
//   search  : graph_search_kernel (search.cu) over the batch, one CTA per inserted node, beam = efConstruction
//   prune   : prune_kernel, one CTA per node: scores -> sort by the reference key -> retainDiverse restated over a running
//             max-similarity per candidate, updated in bulk whenever a neighbour is selected (SURVEY §3.2 seam v)
//   backlink: append u to adj[v] for every chosen v (sorted (v, u) pairs, slot deg_before[v] + rank; a pair past the row's
//             capacity is dropped and counted), then prune_kernel again over every v whose list passed overflow * M
// Batches grow geometrically (x 33/32, JV_BUILD_BATCH_DIV) up to max_batch so early nodes see a connected graph. Neighbour lists in the
// reference are concurrency-order dependent, so parity is on scores and on the recall of the resulting graph
// (SURVEY §8d C5), not on identical adjacency.
// Over a PQ data set (BuildScoreProvider.pqBuildScoreProvider, DESIGN §4.3c) the same loop runs on the codes: the insert queries
// are decode(c_u) (pq_decode_kernel), the walk is the PQ walk, and the prune is prune_kernel<.., KIND_PQ> (ADC keys, pair table).
// Over a BQ data set (BuildScoreProvider.bqBuildScoreProvider, DESIGN §4.3g) the insert queries are c_u as +-1 (bq_decode_kernel), the
// walk is the BQ walk, and the prune is prune_kernel<.., KIND_BQ> (Hamming keys and pair scores).
#include <limits.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <vector>

#include <cub/cub.cuh>

#include "host_mem.h"
#include "kernels.h"

namespace jv {

constexpr int PRUNE_THREADS = 256;
constexpr int PRUNE_MAXC = 256;  // candidates per prune (beam or list capacity), power of two
// the PQ prune keeps v's whole LUT in shared memory next to its candidate state (the opt-in limit less the kernel's static shared
// memory): M * k up to ~56 K entries, M = 216 at k = 256
constexpr int PRUNE_PQ_SMEM_MAX = 226 * 1024;

struct PruneParams {
    DataDesc d;
    int metric;
    int degree;     // M: max selected
    int row_cap;    // slots per adjacency row
    float alpha;
    int32_t *adj;   // [n][row_cap]
    int *deg;       // [n]
    // mode 0: nodes = node_base + i, candidates = cand[i][0..cand_cnt) (search results, -1 padded)
    // mode 1: nodes = list[i], candidates = adj[v][0..min(deg, row_cap))
    int mode;
    int node_base;
    const int32_t *list;
    const int *count_ptr;  // number of nodes (device) or nullptr -> count
    int count;
    const int32_t *cand;
    int cand_stride;
    int *mark;  // cleared for pruned nodes in mode 1
    // mode 0: the W nodes around a batch node in insertion order are candidates too — the batch plays the reference's set of
    // concurrently inserting threads, whose in-progress nodes every insert scores and merges into its candidates
    // (GraphIndexBuilder.java:611-612,669,823-837 getConcurrentCandidates). Batch = nodes [batch_first, batch_first + batch_count).
    int window, batch_first, batch_count;
    // out-of-place results (sharded build: the slice's rows travel before they are applied): row i of this launch goes to
    // out_rows[(out_base + i) * out_stride ..] and out_deg[out_base + i]; nullptr = write adj / deg in place
    int32_t *out_rows;
    int *out_deg;
    int out_stride, out_base;
    int list_base;  // mode 1: nodes = list[list_base + i]
    // mode 2 (repair of deleted neighbours): row i of this launch is a = list[i] of the repaired rows, node = row_node[a], candidates =
    // cand[cand_off[a] .. + cand_cnt[a]) (ragged), result to out_rows[a * out_stride ..] and out_deg[a]
    const int32_t *row_node;
    const long long *cand_off;
    const int *cand_cnt;
};

// candidate i of node v: the search result while i < cand_stride, then the in-progress window (skipping v itself)
__device__ __forceinline__ int32_t prune_candidate(const PruneParams &P, const int32_t *cand, int nc_search, int v, int i)
{
    if (i < nc_search) return cand[i];
    if (P.mode != 0 || P.window <= 0) return -1;
    const int j = i - nc_search;  // 0 .. window-1
    const int half = P.window >> 1;
    int w = v - half + j;
    if (w >= v) w += 1;  // skip v: the window holds `window` OTHER nodes
    if (w < P.batch_first || w >= P.batch_first + P.batch_count) return -1;
    return w;
}

// decode(c_v) (ProductQuantization.decode, :454-471): per sub-space the codebook row, plus the global centroid when there is one —
// one fp32 add per element. The walk and prepare_blob then subtract the centroid again, as PQDecoder.CachingDecoder does, so both
// roundings are kept. Threads nt-strided over the sub-spaces; out[0, dim).
__device__ __forceinline__ void pq_decode_row(const DataDesc &d, int v, float *out, int tid, int nt)
{
    const uint8_t *c = d.codes + (size_t)v * d.code_stride;
    for (int m = tid; m < d.M; m += nt) {
        const int sz = d.sub_sizes[m], off = d.sub_offsets[m];
        const float *src = d.codebooks + (size_t)d.k * off + (size_t)c[m] * sz;
        for (int j = 0; j < sz; j++) out[off + j] = d.centroid ? __fadd_rn(src[j], d.centroid[off + j]) : src[j];
    }
}

// similarity score of candidate row `c` (global) against a cached row `srow` (shared or global), one warp
template <int METRIC>
__device__ __forceinline__ float pair_rows(const float4 *__restrict__ c, const float4 *srow, int n4, int lane)
{
    float s0 = 0.f, s1 = 0.f, aa = 0.f, bb = 0.f;
#pragma unroll 2
    for (int i = lane; i < n4; i += 32) {
        const float4 x = __ldg(c + i);
        const float4 y = srow[i];
        if (METRIC == JV_METRIC_EUCLIDEAN) {
            float d0 = x.x - y.x, d1 = x.y - y.y, d2 = x.z - y.z, d3 = x.w - y.w;
            s0 = fmaf(d0, d0, s0); s1 = fmaf(d1, d1, s1); s0 = fmaf(d2, d2, s0); s1 = fmaf(d3, d3, s1);
        } else {
            s0 = fmaf(x.x, y.x, s0); s1 = fmaf(x.y, y.y, s1); s0 = fmaf(x.z, y.z, s0); s1 = fmaf(x.w, y.w, s1);
            if (METRIC == JV_METRIC_COSINE) {
                aa = fmaf(x.x, x.x, aa); aa = fmaf(x.y, x.y, aa); aa = fmaf(x.z, x.z, aa); aa = fmaf(x.w, x.w, aa);
                bb = fmaf(y.x, y.x, bb); bb = fmaf(y.y, y.y, bb); bb = fmaf(y.z, y.z, bb); bb = fmaf(y.w, y.w, bb);
            }
        }
    }
    float s = group_sum<32>(s0 + s1);
    if (METRIC == JV_METRIC_COSINE) {
        aa = group_sum<32>(aa);
        bb = group_sum<32>(bb);
        s = __fdiv_rn(s, __fsqrt_rn(__fmul_rn(aa, bb)));
    }
    return score_map(METRIC, s);
}

// one BQ word row as floats in shared memory (2 W, rounded to 4 so that what follows stays 16-byte aligned)
__host__ __device__ inline int bq_row_floats(const DataDesc &d) { return (2 * d.W + 3) & ~3; }

// BQVectors.similarityBetween (BQVectors.java:116-118) of candidate row `a` (global) against a cached word row `srow` (shared), one warp
__device__ __forceinline__ float pair_bq_row(const DataDesc &d, int a, const unsigned long long *srow, int lane)
{
    const unsigned long long *x = d.words + (size_t)a * d.W;
    int hd = 0;
    for (int i = lane; i < d.W; i += 32) hd += __popcll(__ldg(x + i) ^ srow[i]);
    return bq_score_from_hd(group_sum_int<32>(hd), d.dim);
}

// ------------------------------------------------------------------------------------------------
// The steps the prune kernels share. Per row: the row's candidates (PruneRow), their keys against v (prune_keys_f32; prune_kernel
// has its own passes over codes), the sort and state reset, the selection (prune_select_gram over a Gram matrix; prune_kernel folds
// one selected row at a time) and the write-out (prune_write_row; prune_kernel's bounded tiers write with one thread per neighbour).
// The sort and prune_kernel's next-pick scan stay written out in each kernel: as shared functions they change the register
// allocation of the BQ and Gram instantiations, and the BQ ones already spill.
// ------------------------------------------------------------------------------------------------

// row `it` of a launch: node v, its candidates cand[0, ncs) followed (mode 0) by the in-progress window, nc of them in all up to
// the kernel's capacity; a is the repaired row's slot (mode 2)
struct PruneRow {
    int a, v, nc, ncs;
    const int32_t *cand;
    __device__ __forceinline__ PruneRow(const PruneParams &P, int it, int cap)
    {
        a = P.mode == 2 ? P.list[it] : 0;
        v = P.mode == 0 ? P.node_base + it : P.mode == 2 ? P.row_node[a] : P.list[P.list_base + it];
        if (P.mode == 0) {
            cand = P.cand + (size_t)it * P.cand_stride;
            ncs = P.cand_stride;
            nc = ncs + P.window;
        } else if (P.mode == 2) {
            cand = P.cand + P.cand_off[a];
            ncs = nc = P.cand_cnt[a];
        } else {
            cand = P.adj + (size_t)v * P.row_cap;
            ncs = nc = min(P.deg[v], P.row_cap);
        }
        nc = min(nc, cap);
    }
};

// the last alpha the reference loop reaches: 1.0, 1.2, ... while <= alpha + 1e-6
__device__ __forceinline__ float prune_alpha_max(float alpha)
{
    float alpha_max = 1.0f;
    for (float a = 1.0f; a <= alpha + 1e-6f; a += 0.2f) alpha_max = a;
    return alpha_max;
}

// exact fp32 scores of the row's candidates against v (blob: prepare_blob of v's row) as sortable keys in keys[0, CAP), two rows
// per warp at a time; KEY_MIN for an empty slot and for v itself
template <int METRIC, int CAP>
__device__ __forceinline__ void prune_keys_f32(const PruneParams &P, const PruneRow &r, const float *blob, long long *keys, int warp, int lane)
{
    constexpr int NW = PRUNE_THREADS / 32;
    for (int i = warp; i < CAP; i += 2 * NW) {
        const int i2 = i + NW;
        const int32_t ca = i < r.nc ? prune_candidate(P, r.cand, r.ncs, r.v, i) : -1, cb = (i2 < CAP && i2 < r.nc) ? prune_candidate(P, r.cand, r.ncs, r.v, i2) : -1;
        const bool va = ca >= 0 && ca != r.v, vb = cb >= 0 && cb != r.v;
        long long ka = KEY_MIN, kb = KEY_MIN;
        if (va || vb) {
            float sa, sb;
            score_f32_pair<METRIC>(P.d, blob, va ? ca : cb, vb ? cb : ca, lane, sa, sb);
            if (va) ka = topk_key(sa, ca);
            if (vb) kb = topk_key(sb, cb);
        }
        if (lane == 0) {
            keys[i] = ka;
            if (i2 < CAP) keys[i2] = kb;
        }
    }
}

// retainDiverse (VamanaDiversityProvider.java:45-95), restated so that the pair scores can be produced in bulk:
//   isDiverse(c) at alpha  <=>  max over the selected s of sim(c, s)  <=  score(c) * alpha.
// Keep M[c] = that running maximum (maxsim). Selecting a candidate s updates M[c] for every still-eligible c in parallel (the
// kernel's fold); the sequential part of the reference loop shrinks to "find the next c at or after the cursor with
// M[c] <= score(c) * alpha", a flag scan (prune_next). A candidate whose M[c] already exceeds score(c) * alpha_max can never be
// selected in any pass (M only grows) and is dropped from further updates. The selection sequence — and therefore the neighbour
// list — is exactly the reference loop's, including the alpha = 1.0, 1.2 passes.

// the next eligible candidate at or after the cursor that is diverse at alpha, INT_MAX if there is none; ends on a barrier
__device__ __forceinline__ int prune_next(const long long *keys, const float *maxsim, const uint8_t *state, int cursor, int nvalid, float alpha,
                                          int *s_next)
{
    if (threadIdx.x == 0) *s_next = INT_MAX;
    __syncthreads();
    for (int i = cursor + threadIdx.x; i < nvalid; i += PRUNE_THREADS)
        if (state[i] == 0 && !(maxsim[i] > __fmul_rn(key_score(keys[i]), alpha))) { atomicMin(s_next, i); break; }
    __syncthreads();
    return *s_next;
}

// the selection over a precomputed similarity matrix C (pitch CP, row i = sorted candidate i): the fold reads column `pick`
template <int CP>
__device__ __forceinline__ void prune_select_gram(const PruneParams &P, const float *C, const long long *keys, float *maxsim, uint8_t *state,
                                                  int nvalid, float alpha_max, int *s_next)
{
    int nsel = 0;
    float currentAlpha = 1.0f;
    while (currentAlpha <= P.alpha + 1e-6f && nsel < P.degree) {
        int cursor = 0;
        while (nsel < P.degree) {
            const int pick = prune_next(keys, maxsim, state, cursor, nvalid, currentAlpha, s_next);
            if (pick == INT_MAX) break;
            nsel++;
            cursor = pick + 1;
            for (int i = threadIdx.x; i < nvalid; i += PRUNE_THREADS) {
                if (i == pick) state[i] = 1;
                else if (state[i] == 0) {
                    const float m = fmaxf(maxsim[i], C[i * CP + pick]);
                    maxsim[i] = m;
                    if (m > __fmul_rn(key_score(keys[i]), alpha_max)) state[i] = 2;
                }
            }
            __syncthreads();
        }
        currentAlpha += 0.2f;
    }
}

// the selected neighbours (state 1) in score order (NodeArray.retain keeps the sorted order), -1 padded, to out_rows[oi] (a sharded
// build's slice, or the repair's row a) or in place to v's adjacency row; node_of(i) is the node of sorted candidate i. One thread.
template <typename NodeOf>
__device__ __forceinline__ void prune_write_row(const PruneParams &P, const PruneRow &r, int it, const uint8_t *state, int nvalid, NodeOf node_of)
{
    int w = 0;
    const int oi = P.mode == 2 ? r.a : P.out_base + it;
    int32_t *row = P.out_rows ? P.out_rows + (size_t)oi * P.out_stride : P.adj + (size_t)r.v * P.row_cap;
    const int width = P.out_rows ? P.out_stride : P.row_cap;
    for (int i = 0; i < nvalid; i++)
        if (state[i] == 1) row[w++] = node_of(i);
    for (int i = w; i < width; i++) row[i] = -1;
    if (P.out_rows) P.out_deg[oi] = w;
    else P.deg[r.v] = w;
    if (P.mode == 1 && P.mark) P.mark[r.v] = 0;
}

// MAXC: candidate capacity (power of two). The builder uses PRUNE_MAXC; the repair of deleted neighbours also instantiates
// larger capacities so that no candidate set is ever clipped.
// KIND_PQ (pqBuildScoreProvider, §4.3c): v's query is decode(c_v) (pq_decode_row, into the row slot), its LUT is prepare_blob's, the
// keys are score_pq's bits — the walk's — and the fold sums the centroid-pair table (pair_pq_table, ImmutablePQVectors' diversity).
// The PQ capacities above PRUNE_MAXC (the repair's upper tiers, §4.3e) work on the power of two that holds the row's own candidates
// instead of on MAXC — the key pass, the sort and the state reset shrink with it; a sort of KEY_MIN pads changes no result — and
// write the selected row with one thread per neighbour.
// KIND_BQ (bqBuildScoreProvider, §4.3g): the blob is v's own words c_v, the keys are score_bq's bits under it — the walk's, whose query
// decodes to c_v — and the fold is the Hamming score of two word rows (pair_bq_row). No score depends on the metric, so one METRIC
// instantiation serves all three. Its capacities above PRUNE_MAXC are bounded like PQ's.
template <int METRIC, int MAXC = PRUNE_MAXC, int KIND = KIND_F32>
__global__ void __launch_bounds__(PRUNE_THREADS) prune_kernel(PruneParams P)
{
    constexpr bool BOUNDED = (KIND == KIND_PQ || KIND == KIND_BQ) && MAXC > PRUNE_MAXC;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // f32: blob stride + 4, newrow stride (the most recently selected row). PQ: blob = the LUT, newrow = decode(c_v) (dim rounded to 4).
    // BQ: blob = c_v, newrow = the selected row's words (2 W floats each, rounded to 4)
    const int blob_fl = KIND == KIND_PQ ? blob_floats(P.d) : KIND == KIND_BQ ? bq_row_floats(P.d) : P.d.stride + 4;
    const int row_fl = KIND == KIND_PQ ? (P.d.dim + 3) & ~3 : KIND == KIND_BQ ? bq_row_floats(P.d) : P.d.stride;
    float *blob = reinterpret_cast<float *>(smem_raw);
    float *newrow = blob + blob_fl;
    long long *keys = reinterpret_cast<long long *>(newrow + row_fl);        // MAXC
    float *maxsim = reinterpret_cast<float *>(keys + MAXC);                  // MAXC
    int32_t *sel_ids = reinterpret_cast<int32_t *>(maxsim + MAXC);           // 128
    uint8_t *state = reinterpret_cast<uint8_t *>(sel_ids + 128);             // MAXC: 0 eligible, 1 selected, 2 dropped
    __shared__ float red[36];
    __shared__ int s_next;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NW = PRUNE_THREADS / 32;
    const int total = P.count_ptr ? *P.count_ptr : P.count;
    const int n4 = P.d.stride >> 2;
    const float alpha_max = prune_alpha_max(P.alpha);

    for (int it = blockIdx.x; it < total; it += gridDim.x) {
        const PruneRow r(P, it, MAXC);
        const int v = r.v;
        int cap = MAXC;
        if (BOUNDED)
            for (cap = PRUNE_MAXC; cap < r.nc;) cap <<= 1;
        // (if constexpr: the fp32 and PQ instantiations compile exactly as they did before the BQ branches existed)
        if constexpr (KIND == KIND_BQ) {
            const uint32_t *cv = reinterpret_cast<const uint32_t *>(P.d.words + (size_t)v * P.d.W);
            for (int t = tid; t < 2 * P.d.W; t += PRUNE_THREADS) reinterpret_cast<uint32_t *>(blob)[t] = __ldg(cv + t);
            __syncthreads();
            // the candidates' Hamming scores under c_v as sortable keys: 8 lanes per candidate, the walk's scorer and bits
            for (int i = tid >> 3; i < cap; i += PRUNE_THREADS / 8) {
                const int32_t c = i < r.nc ? prune_candidate(P, r.cand, r.ncs, v, i) : -1;
                long long kc = KEY_MIN;
                if (c >= 0 && c != v) kc = topk_key(score_bq(P.d, blob, c, lane & 7), c);
                if ((lane & 7) == 0) keys[i] = kc;
            }
        } else if (KIND == KIND_PQ) {
            pq_decode_row(P.d, v, newrow, tid, PRUNE_THREADS);
            __syncthreads();
            prepare_blob(P.d, P.metric, newrow, blob, red);
            // the candidates' ADC scores under v's LUT as sortable keys: 8 lanes per candidate, the walk's scorer and bits
            for (int i = tid >> 3; i < cap; i += PRUNE_THREADS / 8) {
                const int32_t c = i < r.nc ? prune_candidate(P, r.cand, r.ncs, v, i) : -1;
                long long kc = KEY_MIN;
                if (c >= 0 && c != v) kc = topk_key(score_pq<METRIC>(P.d, blob, c, lane & 7), c);
                if ((lane & 7) == 0) keys[i] = kc;
            }
        } else {
            prepare_blob(P.d, P.metric, P.d.rows + (size_t)v * P.d.stride, blob, red);
            prune_keys_f32<METRIC, MAXC>(P, r, blob, keys, warp, lane);
        }
        __syncthreads();
        bitonic_sort_desc(keys, cap);
        // valid keys form a prefix (KEY_MIN sorts last); duplicates are adjacent after the sort and are dropped
        int nvalid;
        {
            int lo = 0, hi = cap;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (keys[mid] != KEY_MIN) lo = mid + 1;
                else hi = mid;
            }
            nvalid = lo;
        }
        for (int i = tid; i < cap; i += PRUNE_THREADS) {
            maxsim[i] = -3.0e38f;
            state[i] = (i < nvalid && !(i > 0 && keys[i - 1] == keys[i])) ? 0 : 2;
        }
        __syncthreads();

        // the selection; the fold scores each still-eligible candidate against the new neighbour, one warp per candidate
        int nsel = 0;
        float currentAlpha = 1.0f;
        while (currentAlpha <= P.alpha + 1e-6f && nsel < P.degree) {
            int cursor = 0;
            while (nsel < P.degree) {
                // next eligible candidate at or after the cursor that is diverse at this alpha
                if (tid == 0) s_next = INT_MAX;
                __syncthreads();
                for (int i = cursor + tid; i < nvalid; i += PRUNE_THREADS)
                    if (state[i] == 0 && !(maxsim[i] > __fmul_rn(key_score(keys[i]), currentAlpha))) { atomicMin(&s_next, i); break; }
                __syncthreads();
                const int pick = s_next;
                if (pick == INT_MAX) break;
                const int32_t c = key_node(keys[pick]);
                const float4 *crow = reinterpret_cast<const float4 *>(P.d.rows + (size_t)c * P.d.stride);
                if (tid == 0) {
                    state[pick] = 1;
                    sel_ids[nsel] = c;
                    if (BOUNDED) sel_ids[64 + nsel] = pick;  // degree <= 64: the second half holds the picks' sorted positions
                }
                if constexpr (KIND == KIND_BQ) {
                    const uint32_t *cw = reinterpret_cast<const uint32_t *>(P.d.words + (size_t)c * P.d.W);
                    for (int t = tid; t < 2 * P.d.W; t += PRUNE_THREADS) reinterpret_cast<uint32_t *>(newrow)[t] = __ldg(cw + t);
                } else if (KIND != KIND_PQ)
                    for (int t = tid; t < n4; t += PRUNE_THREADS) reinterpret_cast<float4 *>(newrow)[t] = __ldg(crow + t);
                nsel++;
                cursor = pick + 1;
                __syncthreads();
                if (nsel >= P.degree) break;
                // fold the new neighbour into every still-eligible candidate's running maximum
                for (int i = warp; i < nvalid; i += NW) {
                    if (state[i] != 0) continue;
                    float ps;
                    if constexpr (KIND == KIND_BQ) {
                        ps = pair_bq_row(P.d, key_node(keys[i]), reinterpret_cast<const unsigned long long *>(newrow), lane);
                    } else if (KIND == KIND_PQ) {
                        ps = pair_pq_table<METRIC>(P.d, key_node(keys[i]), c, lane);
                    } else {
                        const float4 *row = reinterpret_cast<const float4 *>(P.d.rows + (size_t)key_node(keys[i]) * P.d.stride);
                        ps = pair_rows<METRIC>(row, reinterpret_cast<const float4 *>(newrow), n4, lane);
                    }
                    if (lane == 0) {
                        const float m = fmaxf(maxsim[i], ps);
                        maxsim[i] = m;
                        if (m > __fmul_rn(key_score(keys[i]), alpha_max)) state[i] = 2;  // can never become diverse
                    }
                }
                __syncthreads();
            }
            currentAlpha += 0.2f;
        }
        __syncthreads();
        if (BOUNDED) {
            // thread t places pick t at its rank among the picks' sorted positions instead of one thread scanning nvalid states
            const int oi = P.mode == 2 ? r.a : P.out_base + it;
            int32_t *row = P.out_rows ? P.out_rows + (size_t)oi * P.out_stride : P.adj + (size_t)v * P.row_cap;
            const int width = P.out_rows ? P.out_stride : P.row_cap;
            for (int t = tid; t < width; t += PRUNE_THREADS) {
                if (t < nsel) {
                    int rank = 0;
                    for (int j = 0; j < nsel; j++) rank += sel_ids[64 + j] < sel_ids[64 + t];
                    row[rank] = sel_ids[t];
                } else {
                    row[t] = -1;
                }
            }
            if (tid == 0) {
                if (P.out_rows) P.out_deg[oi] = nsel;
                else P.deg[v] = nsel;
                if (P.mode == 1 && P.mark) P.mark[v] = 0;
            }
        }
        if (!BOUNDED && tid == 0) prune_write_row(P, r, it, state, nvalid, [&](int i) { return key_node(keys[i]); });
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// prune_gram_kernel: the same retainDiverse, with the candidate x candidate similarity matrix produced up front by a
// shared-memory tiled Gram product on the CUDA cores (SURVEY §3.2 seam v: "compute the full candidate x candidate matrix
// and replay the sequential selection"). Rows are read ONCE (nc x 3 KB from L2) instead of once per selected neighbour;
// the selection loop then only touches shared memory. TILE = 128 candidates (beam) or 64 (re-prune of an adjacency row).
// Thread (ty, tx) of the 16 x 16 grid owns C[ty + 16 a][tx + 16 b]; K is walked in 32-float chunks staged in shared memory
// (row pitch 36 floats: 128-bit loads of a quarter-warp hit distinct banks).
// ------------------------------------------------------------------------------------------------
constexpr int GRAM_KC = 32;
constexpr int GRAM_PITCH = 36;

// floats [k, k + 4) of candidate `node` as the Gram product stages them. L2 takes x_node - x_v, the row translated by the pruned
// node's own: distances do not change, and G_ii + G_jj - 2 G_ij then carries an error relative to the neighbourhood's size
// (|x_i - x_v| + |x_j - x_v|)^2 instead of to |x|^2, which on rows sharing a large offset swamps the distances themselves.
template <int METRIC>
__device__ __forceinline__ float4 gram_row(const DataDesc &d, int32_t node, int v, int k)
{
    const float4 x = __ldg(reinterpret_cast<const float4 *>(d.rows + (size_t)node * d.stride + k));
    if (METRIC != JV_METRIC_EUCLIDEAN) return x;
    const float4 y = __ldg(reinterpret_cast<const float4 *>(d.rows + (size_t)v * d.stride + k));
    return make_float4(__fsub_rn(x.x, y.x), __fsub_rn(x.y, y.y), __fsub_rn(x.z, y.z), __fsub_rn(x.w, y.w));
}

// a Gram entry (the dot product of candidates i and j, diagonal entries di, dj) as the reference's similarity score; L2 and cosine
// need the diagonal, DOT ignores it
template <int METRIC>
__device__ __forceinline__ float gram_score(float dotv, float di, float dj)
{
    float raw;
    if (METRIC == JV_METRIC_EUCLIDEAN) raw = fmaxf(0.f, __fadd_rn(__fadd_rn(di, dj), -2.0f * dotv));
    else if (METRIC == JV_METRIC_COSINE) raw = __fdiv_rn(dotv, __fsqrt_rn(__fmul_rn(di, dj)));
    else raw = dotv;
    return score_map(METRIC, raw);
}

template <int METRIC, int TILE>
__global__ void __launch_bounds__(PRUNE_THREADS) prune_gram_kernel(PruneParams P)
{
    constexpr int NB = TILE / 16;       // rows / cols per thread
    constexpr int CP = TILE + 1;        // pitch of the similarity matrix
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *blob = reinterpret_cast<float *>(smem_raw);                         // stride + 4
    float *tileA = blob + P.d.stride + 4;                                      // TILE * GRAM_PITCH
    float *C = tileA + TILE * GRAM_PITCH;                                      // TILE * CP
    long long *keys = reinterpret_cast<long long *>(C + TILE * CP + ((TILE * CP) & 1));  // TILE (8-byte aligned)
    float *maxsim = reinterpret_cast<float *>(keys + TILE);                    // TILE
    int32_t *ids = reinterpret_cast<int32_t *>(maxsim + TILE);                 // TILE
    uint8_t *state = reinterpret_cast<uint8_t *>(ids + TILE);                  // TILE
    __shared__ float red[36];
    __shared__ int s_next;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ty = tid >> 4, tx = tid & 15;
    const int total = P.count_ptr ? *P.count_ptr : P.count;
    const float alpha_max = prune_alpha_max(P.alpha);

    for (int it = blockIdx.x; it < total; it += gridDim.x) {
        const PruneRow r(P, it, TILE);
        const int v = r.v;
        prepare_blob(P.d, P.metric, P.d.rows + (size_t)v * P.d.stride, blob, red);
        prune_keys_f32<METRIC, TILE>(P, r, blob, keys, warp, lane);
        __syncthreads();
        bitonic_sort_desc(keys, TILE);
        // valid keys form a prefix (KEY_MIN sorts last); duplicates are adjacent after the sort and are dropped
        int nvalid;
        {
            int lo = 0, hi = TILE;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (keys[mid] != KEY_MIN) lo = mid + 1;
                else hi = mid;
            }
            nvalid = lo;
        }
        for (int i = tid; i < TILE; i += PRUNE_THREADS) {
            maxsim[i] = -3.0e38f;
            state[i] = (i < nvalid && !(i > 0 && keys[i - 1] == keys[i])) ? 0 : 2;
            ids[i] = i < nvalid ? key_node(keys[i]) : -1;
        }
        __syncthreads();

        // ---- Gram matrix of the candidate rows (L2: translated by v's row, see gram_row) ----
        float acc[NB][NB];
#pragma unroll
        for (int a = 0; a < NB; a++)
#pragma unroll
            for (int b = 0; b < NB; b++) acc[a][b] = 0.f;
        for (int k0 = 0; k0 < P.d.stride; k0 += GRAM_KC) {
            // stage rows [0, TILE) x [k0, k0 + KC): TILE * 8 float4, zero beyond nvalid / beyond the row
            for (int t = tid; t < TILE * (GRAM_KC / 4); t += PRUNE_THREADS) {
                const int r = t / (GRAM_KC / 4), c4 = t - r * (GRAM_KC / 4);
                float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
                const int32_t node = ids[r];
                if (node >= 0 && k0 + 4 * c4 < P.d.stride) val = gram_row<METRIC>(P.d, node, v, k0 + 4 * c4);
                *reinterpret_cast<float4 *>(tileA + r * GRAM_PITCH + 4 * c4) = val;
            }
            __syncthreads();
#pragma unroll
            for (int k4 = 0; k4 < GRAM_KC / 4; k4++) {
                float4 av[NB], bv[NB];
#pragma unroll
                for (int a = 0; a < NB; a++) av[a] = *reinterpret_cast<const float4 *>(tileA + (ty + 16 * a) * GRAM_PITCH + 4 * k4);
#pragma unroll
                for (int b = 0; b < NB; b++) bv[b] = *reinterpret_cast<const float4 *>(tileA + (tx + 16 * b) * GRAM_PITCH + 4 * k4);
#pragma unroll
                for (int a = 0; a < NB; a++)
#pragma unroll
                    for (int b = 0; b < NB; b++) {
                        acc[a][b] = fmaf(av[a].x, bv[b].x, acc[a][b]);
                        acc[a][b] = fmaf(av[a].y, bv[b].y, acc[a][b]);
                        acc[a][b] = fmaf(av[a].z, bv[b].z, acc[a][b]);
                        acc[a][b] = fmaf(av[a].w, bv[b].w, acc[a][b]);
                    }
            }
            __syncthreads();
        }
#pragma unroll
        for (int a = 0; a < NB; a++)
#pragma unroll
            for (int b = 0; b < NB; b++) C[(ty + 16 * a) * CP + tx + 16 * b] = acc[a][b];
        __syncthreads();
        // raw dot products -> the reference's similarity scores (needs the diagonal for L2 / cosine)
        float diag_r[NB] = {}, diag_c[NB] = {};  // DOT reads no diagonal
        if (METRIC != JV_METRIC_DOT) {
#pragma unroll
            for (int a = 0; a < NB; a++) diag_r[a] = C[(ty + 16 * a) * CP + ty + 16 * a];
#pragma unroll
            for (int b = 0; b < NB; b++) diag_c[b] = C[(tx + 16 * b) * CP + tx + 16 * b];
            __syncthreads();
        }
#pragma unroll
        for (int a = 0; a < NB; a++)
#pragma unroll
            for (int b = 0; b < NB; b++) C[(ty + 16 * a) * CP + tx + 16 * b] = gram_score<METRIC>(acc[a][b], diag_r[a], diag_c[b]);
        __syncthreads();

        prune_select_gram<CP>(P, C, keys, maxsim, state, nvalid, alpha_max, &s_next);
        __syncthreads();
        if (tid == 0) prune_write_row(P, r, it, state, nvalid, [&](int i) { return ids[i]; });
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// prune_gram_tc_kernel: the same kernel with the Gram product on the tensor cores (Hopper wgmma). The candidate x candidate
// matrix is GEMM-shaped work (X X^T, X = the candidate rows). fp32 products are kept by the 3xTF32 split: x = hi + lo with
// hi = x truncated to tf32's 10 mantissa bits and lo = x - hi (exact), D += hi hi^T + hi lo^T + lo hi^T (the dropped lo lo^T term
// is 2^-22 relative), fp32 accumulation in registers. Per 32-float K chunk all 256 threads stage the rows into two K-major
// SWIZZLE_128B tiles (hi | lo, TILE rows x 128 B each; the same tile is the A and the B operand), double buffered, and each of
// the two warpgroups issues wgmma.m64nNk8.tf32 for its half of the columns (N = TILE / 2) over the TILE / 64 row blocks; the
// next chunk's global loads are in flight while they run. The similarity matrix C overlays the staging area once the last
// group has completed. The scores against v (the sort keys) stay exact fp32.
// ------------------------------------------------------------------------------------------------
namespace tc {
// D[64][N] (+)= A[64][8] * B[N][8]^T in tf32 with fp32 accumulation. Fragment: register 4 j + 2 h + e holds row
// 16 (warp % 4) + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e.
template <int N>
__device__ __forceinline__ void mma_tf32(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void mma_tf32<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void mma_tf32<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <int TILE>
struct Layout {
    static constexpr int TILE_BYTES = TILE * 128;                  // one operand tile: TILE rows x 32 floats
    static constexpr int STAGE_BYTES = 2 * TILE_BYTES;             // hi | lo
    static constexpr int STAGES_END = 2 * STAGE_BYTES;
    static constexpr int C_BYTES = (TILE * (TILE + 1) * 4 + 15) & ~15;
    static constexpr int AREA = ((STAGES_END > C_BYTES ? STAGES_END : C_BYTES) + 1023) & ~1023;
};
}  // namespace tc

template <int TILE>
static size_t gram_tc_smem_bytes(const DataDesc &d)
{
    size_t b = 1024 /* alignment slack */ + tc::Layout<TILE>::AREA + (size_t)(d.stride + 4) * 4 + (size_t)TILE * 8 + (size_t)TILE * 4 * 3 + TILE + 64;
    return (b + 15) & ~(size_t)15;
}

template <int METRIC, int TILE>
__global__ void __launch_bounds__(PRUNE_THREADS, TILE == 128 ? 2 : 3) prune_gram_tc_kernel(PruneParams P)
{
    using L = tc::Layout<TILE>;
    constexpr int CP = TILE + 1;
    constexpr int PASSES = TILE / 32;   // 256 threads stage 32 rows x 8 float4 per pass
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *area = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    float *C = reinterpret_cast<float *>(area);
    float *blob = reinterpret_cast<float *>(area + L::AREA);                   // stride + 4
    long long *keys = reinterpret_cast<long long *>(blob + ((P.d.stride + 4 + 1) & ~1));
    float *maxsim = reinterpret_cast<float *>(keys + TILE);
    float *diag = maxsim + TILE;
    int32_t *ids = reinterpret_cast<int32_t *>(diag + TILE);
    uint8_t *state = reinterpret_cast<uint8_t *>(ids + TILE);
    __shared__ float red[36];
    __shared__ int s_next;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int total = P.count_ptr ? *P.count_ptr : P.count;
    const float alpha_max = prune_alpha_max(P.alpha);

    // warpgroup wg computes columns [wg N, wg N + N) of every 64-row block of the Gram matrix
    constexpr int N = TILE / 2, MB = TILE / 64, R = N / 2;
    const int wg = warp >> 2;
    float acc[MB][R];
    const int nchunks = (P.d.stride + 31) / 32;
    const int c4 = tid & 7, r0 = tid >> 3;

    for (int it = blockIdx.x; it < total; it += gridDim.x) {
        const PruneRow r(P, it, TILE);
        const int v = r.v;
        prepare_blob(P.d, P.metric, P.d.rows + (size_t)v * P.d.stride, blob, red);
        prune_keys_f32<METRIC, TILE>(P, r, blob, keys, warp, lane);
        __syncthreads();
        bitonic_sort_desc(keys, TILE);
        // valid keys form a prefix (KEY_MIN sorts last); duplicates are adjacent after the sort and are dropped
        int nvalid;
        {
            int lo = 0, hi = TILE;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (keys[mid] != KEY_MIN) lo = mid + 1;
                else hi = mid;
            }
            nvalid = lo;
        }
        for (int i = tid; i < TILE; i += PRUNE_THREADS) {
            maxsim[i] = -3.0e38f;
            state[i] = (i < nvalid && !(i > 0 && keys[i - 1] == keys[i])) ? 0 : 2;
            ids[i] = i < nvalid ? key_node(keys[i]) : -1;
        }
        __syncthreads();

        // ---- Gram matrix of the candidate rows on the tensor cores (3xTF32; L2: translated by v's row, see gram_row) ----
        int32_t rnode[PASSES];
#pragma unroll
        for (int j = 0; j < PASSES; j++) rnode[j] = ids[r0 + 32 * j];
        float4 pre[PASSES];
#pragma unroll
        for (int j = 0; j < PASSES; j++) pre[j] = (rnode[j] >= 0 && 4 * c4 < P.d.stride) ? gram_row<METRIC>(P.d, rnode[j], v, 4 * c4) : make_float4(0.f, 0.f, 0.f, 0.f);
        for (int c = 0; c < nchunks; c++) {
            const int b = c & 1;
            if (c >= 2) {  // the MMAs of chunk c - 2 (both warpgroups) have read this buffer
                wgmma_wait<1>();
                __syncthreads();
            }
            unsigned char *hi_t = area + b * L::STAGE_BYTES, *lo_t = hi_t + L::TILE_BYTES;
#pragma unroll
            for (int j = 0; j < PASSES; j++) {
                const int r = r0 + 32 * j;
                const float4 x = pre[j];
                float4 h, l;
                h.x = __uint_as_float(__float_as_uint(x.x) & 0xffffe000u); l.x = __fsub_rn(x.x, h.x);
                h.y = __uint_as_float(__float_as_uint(x.y) & 0xffffe000u); l.y = __fsub_rn(x.y, h.y);
                h.z = __uint_as_float(__float_as_uint(x.z) & 0xffffe000u); l.z = __fsub_rn(x.z, h.z);
                h.w = __uint_as_float(__float_as_uint(x.w) & 0xffffe000u); l.w = __fsub_rn(x.w, h.w);
                const int off = (r >> 3) * 1024 + (r & 7) * 128 + ((c4 ^ (r & 7)) << 4);
                *reinterpret_cast<float4 *>(hi_t + off) = h;
                *reinterpret_cast<float4 *>(lo_t + off) = l;
            }
            if (c + 1 < nchunks) {
                const int k1 = (c + 1) * 32 + 4 * c4;
#pragma unroll
                for (int j = 0; j < PASSES; j++)
                    pre[j] = (rnode[j] >= 0 && k1 < P.d.stride) ? gram_row<METRIC>(P.d, rnode[j], v, k1) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            fence_proxy_async();
            __syncthreads();
            {
                const uint32_t ah = smem_u32(hi_t), al = smem_u32(lo_t);
#pragma unroll
                for (int mb = 0; mb < MB; mb++) acc_fence(acc[mb]);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 4; ks++) {
                    const uint64_t bh = wgmma_desc(ah + wg * (N / 8) * 1024 + 32 * ks), bl = wgmma_desc(al + wg * (N / 8) * 1024 + 32 * ks);
#pragma unroll
                    for (int mb = 0; mb < MB; mb++) {
                        const uint64_t dh = wgmma_desc(ah + mb * 8 * 1024 + 32 * ks), dl = wgmma_desc(al + mb * 8 * 1024 + 32 * ks);
                        tc::mma_tf32<N>(acc[mb], dh, bh, (c | ks) != 0 ? 1u : 0u);
                        tc::mma_tf32<N>(acc[mb], dh, bl, 1u);
                        tc::mma_tf32<N>(acc[mb], dl, bh, 1u);
                    }
                }
                wgmma_commit();
            }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int mb = 0; mb < MB; mb++) acc_fence(acc[mb]);
        __syncthreads();  // both warpgroups are past their waits: the staging area may now be overwritten by C
#pragma unroll
        for (int mb = 0; mb < MB; mb++) {
            const int i = 64 * mb + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
            for (int j = 0; j < N / 8; j++) {
                const int col = wg * N + 8 * j + 2 * (lane & 3);
                C[i * CP + col] = acc[mb][4 * j];
                C[i * CP + col + 1] = acc[mb][4 * j + 1];
                C[(i + 8) * CP + col] = acc[mb][4 * j + 2];
                C[(i + 8) * CP + col + 1] = acc[mb][4 * j + 3];
            }
        }
        __syncthreads();
        // raw dot products -> the reference's similarity scores (needs the diagonal for L2 / cosine)
        if (METRIC != JV_METRIC_DOT) {
            for (int i = tid; i < TILE; i += PRUNE_THREADS) diag[i] = C[i * CP + i];
            __syncthreads();
        }
        for (int idx = tid; idx < TILE * TILE; idx += PRUNE_THREADS) {
            const int i = idx / TILE, j = idx - i * TILE;
            C[i * CP + j] = gram_score<METRIC>(C[i * CP + j], diag[i], diag[j]);
        }
        __syncthreads();

        prune_select_gram<CP>(P, C, keys, maxsim, state, nvalid, alpha_max, &s_next);
        __syncthreads();
        if (tid == 0) prune_write_row(P, r, it, state, nvalid, [&](int i) { return ids[i]; });
        __syncthreads();
    }
}

template <int TILE>
static size_t gram_smem_bytes(const DataDesc &d)
{
    size_t b = (size_t)(d.stride + 4) * 4 + (size_t)TILE * GRAM_PITCH * 4 + ((size_t)TILE * (TILE + 1) + 1) * 4 + (size_t)TILE * 8 + (size_t)TILE * 4 + (size_t)TILE * 4 + TILE;
    return (b + 15) & ~(size_t)15;
}

// ------------------------------------------------------------------------------------------------
// back-links (ConcurrentNeighborMap.backlink, ConcurrentNeighborMap.java:158-165): for every selected neighbour t of a new
// node u, append u to t's row. Deterministic: the (t, u) pairs of a batch are SORTED, pair i lands at deg_before[t] + (rank of i
// inside t's segment), so every replica of a sharded build applies a batch to bit-identical adjacency (atomics would order the
// appends by timing, and which back-link a full row drops would differ between replicas).
// ------------------------------------------------------------------------------------------------
// position of node t in the ascending list ids[0, count), -1 if absent
__device__ __forceinline__ int batch_pos(const int32_t *ids, int count, int32_t t)
{
    int lo = 0, hi = count;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ids[mid] < t) lo = mid + 1;
        else hi = mid;
    }
    return lo < count && ids[lo] == t ? lo : -1;
}

// row i of a batch replaces node u's row: u = first + i (an insert), or with IDS u = ids[i] (a refine, ids ascending). (IDS is a
// template parameter so that the inserts' form compiles as it did without the id list.)
template <bool IDS>
__global__ void __launch_bounds__(256) apply_rows_kernel(int32_t *adj, int *deg, int row_cap, int degree, int first, int count, const int32_t *ids,
                                                         const int32_t *rows, const int *rdeg, unsigned long long *pairs)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count * row_cap) return;
    const int i = idx / row_cap, j = idx - i * row_cap;
    const int u = IDS ? ids[i] : first + i;
    const int32_t t = j < degree ? rows[(size_t)i * degree + j] : -1;
    adj[(size_t)u * row_cap + j] = t;
    if (j == 0) deg[u] = rdeg[i];
    if (j < degree) {
        bool link = t >= 0;
        if constexpr (!IDS) {
            if (link && t >= first && t < first + count) {
                // t was inserted in this very batch and may have chosen u itself (both sit in each other's in-progress window): then u is
                // already in t's row and the back-link would duplicate it (NodeArray.insertSorted refuses duplicates)
                const int32_t *trow = rows + (size_t)(t - first) * degree;
                for (int x = 0; x < degree; x++)
                    if (trow[x] == u) { link = false; break; }
            }
        } else if (link) {
            // a refine: a row that already names u takes no back-link (ConcurrentNeighborMap.java:305-309, a no-op) — t's new row when t
            // is in the batch, else its current one, which this launch does not write
            const int tp = batch_pos(ids, count, t);
            const int32_t *trow = tp >= 0 ? rows + (size_t)tp * degree : adj + (size_t)t * row_cap;
            const int w = tp >= 0 ? degree : row_cap;
            for (int x = 0; x < w; x++)
                if (trow[x] == u) { link = false; break; }
        }
        pairs[(size_t)i * degree + j] = link ? (((unsigned long long)(unsigned)t << 32) | (unsigned)u) : ~0ull;  // ~0 sorts last
    }
}

__device__ __forceinline__ int lower_bound_u64(const unsigned long long *a, int n, unsigned long long key)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// pairs sorted ascending. Thread i appends its u; the head of each segment publishes the new degree and flags the row when it
// passed overflow * M (ConcurrentNeighborMap.java:300: the row is then re-pruned).
__global__ void __launch_bounds__(256) backlink_sorted_kernel(int32_t *adj, int *deg, int row_cap, int hard_max, const unsigned long long *pairs, int npairs,
                                                              unsigned char *head_flag, int32_t *head_target, unsigned long long *dropped)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npairs) return;
    const unsigned long long p = pairs[i];
    head_flag[i] = 0;
    head_target[i] = -1;
    if (p == ~0ull) return;
    const int t = (int)(p >> 32), u = (int)(unsigned)p;
    const int seg0 = lower_bound_u64(pairs, npairs, (unsigned long long)(unsigned)t << 32);
    const int d0 = deg[t];  // no thread writes deg[t] before every pair of the segment has read it: see below
    const int pos = d0 + (i - seg0);
    if (pos < row_cap) adj[(size_t)t * row_cap + pos] = u;
    else atomicAdd(dropped, 1ull);
    if (i == seg0) {
        // segment head: remember the target and whether the row now passes overflow * M. The new degree itself is published by
        // publish_deg_kernel, a second launch, because the other pairs of the segment still read deg[t] in this one.
        const int seg1 = lower_bound_u64(pairs, npairs, (unsigned long long)((unsigned)t + 1u) << 32);
        const int nd = min(row_cap, d0 + (seg1 - seg0));
        head_target[i] = t;
        head_flag[i] = nd > hard_max ? 1 : 0;
    }
}

__global__ void __launch_bounds__(256) publish_deg_kernel(int *deg, int row_cap, const unsigned long long *pairs, int npairs)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npairs) return;
    const unsigned long long p = pairs[i];
    if (p == ~0ull) return;
    const int t = (int)(p >> 32);
    if (i > 0 && (int)(pairs[i - 1] >> 32) == t) return;  // not a segment head
    const int seg1 = lower_bound_u64(pairs, npairs, (unsigned long long)((unsigned)t + 1u) << 32);
    deg[t] = min(row_cap, deg[t] + (seg1 - i));
}

__global__ void __launch_bounds__(256) flag_over_degree_kernel(const int *deg, int n, int degree, unsigned char *flag)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flag[i] = deg[i] > degree ? 1 : 0;
}

__global__ void __launch_bounds__(256) iota_kernel(int32_t *a, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = i;
}

// re-pruned rows coming back from the exchange: row i replaces adj[list[i]]
__global__ void __launch_bounds__(256) scatter_rows_kernel(int32_t *adj, int *deg, int row_cap, const int32_t *list, int count, const int32_t *rows, const int *rdeg)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count * row_cap) return;
    const int i = idx / row_cap, j = idx - i * row_cap;
    const int v = list[i];
    adj[(size_t)v * row_cap + j] = rows[(size_t)i * row_cap + j];
    if (j == 0) deg[v] = rdeg[i];
}

// an existing graph's rows as the builder's first rows (BuilderSeed), one warp per row: the valid ids, mapped through row_map when
// given, are compacted by ballot to the front of the row_cap-wide row in their order; the rest of the row stays -1
__global__ void __launch_bounds__(256) seed_rows_kernel(const int32_t *__restrict__ rows, int count, int width, const int32_t *__restrict__ row_map,
                                                        int32_t *adj, int *deg, int row_cap)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= count) return;
    const int32_t *src = rows + (size_t)warp * width;
    int32_t *dst = adj + (size_t)warp * row_cap;
    int w = 0;
    for (int j0 = 0; j0 < width; j0 += 32) {
        int32_t id = j0 + lane < width ? src[j0 + lane] : -1;
        if (id >= 0 && row_map) id = row_map[id];
        const unsigned valid = __ballot_sync(FULL, id >= 0);
        if (id >= 0) dst[w + __popc(valid & ((1u << lane) - 1u))] = id;
        w += __popc(valid);
    }
    if (lane == 0) deg[warp] = w;
}

__global__ void __launch_bounds__(256) compact_adj_kernel(const int32_t *adj, const int *deg, int n, int row_cap, int degree, int32_t *out)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n * degree) return;
    const int v = (int)(idx / degree), j = (int)(idx % degree);
    out[idx] = j < min(deg[v], degree) ? adj[(size_t)v * row_cap + j] : -1;
}

// rows [ids[i]] of a data set gathered into a dense one (upper levels of the hierarchy, repair pass), or scattered to rows
// [out_ids[i]] of another (the merged rows of a compaction): one warp per row
__global__ void __launch_bounds__(256) gather_rows_kernel(const float *__restrict__ rows, int stride, const int32_t *__restrict__ ids, int count,
                                                          const int32_t *__restrict__ out_ids, float *__restrict__ out)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= count) return;
    const float4 *src = reinterpret_cast<const float4 *>(rows + (size_t)ids[warp] * stride);
    float4 *dst = reinterpret_cast<float4 *>(out + (size_t)(out_ids ? out_ids[warp] : warp) * stride);
    for (int i = lane; i < (stride >> 2); i += 32) dst[i] = ldg_stream(src + i);
}

cudaError_t launch_gather_rows(const DataDesc &f32, const int32_t *ids_dev, int count, float *out_dev, cudaStream_t s, const int32_t *out_ids_dev)
{
    if (count <= 0) return cudaSuccess;
    const long long blocks = ((long long)count * 32 + 255) / 256;
    gather_rows_kernel<<<(unsigned)blocks, 256, 0, s>>>(f32.rows, f32.stride, ids_dev, count, out_ids_dev, out_dev);
    g_launches++;
    return cudaGetLastError();
}

// fixed-size rows [ids[i]] of a code array (PQ code rows, BQ word rows) gathered into a dense one (upper levels of a PQ or BQ build):
// one thread per 32-bit word
__global__ void __launch_bounds__(256) gather_codes_kernel(const uint32_t *__restrict__ codes, int words, const int32_t *__restrict__ ids, int count,
                                                           uint32_t *__restrict__ out)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)count * words) return;
    const int i = (int)(idx / words), w = (int)(idx - (long long)i * words);
    out[idx] = __ldg(codes + (size_t)ids[i] * words + w);
}

int code_row_bytes(const DataDesc &d) { return d.kind == KIND_BQ ? 8 * d.W : d.code_stride; }

cudaError_t launch_gather_codes(const DataDesc &d, const int32_t *ids_dev, int count, void *out_dev, cudaStream_t s)
{
    if (count <= 0) return cudaSuccess;
    const int words = code_row_bytes(d) >> 2;
    const void *src = d.kind == KIND_BQ ? static_cast<const void *>(d.words) : static_cast<const void *>(d.codes);
    const long long total = (long long)count * words;
    gather_codes_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(reinterpret_cast<const uint32_t *>(src), words, ids_dev, count,
                                                                        reinterpret_cast<uint32_t *>(out_dev));
    g_launches++;
    return cudaGetLastError();
}

// the insert searches' queries of a PQ build: decode(c_u) for nodes first .. first + count - 1 (IDS, a refine's: nodes ids[i]) -> out
// [count][dim], one CTA per node. (IDS is a template parameter so that the build's form compiles as it did without the id list.)
template <bool IDS>
__global__ void __launch_bounds__(128) pq_decode_kernel(DataDesc d, int first, int count, const int32_t *ids, float *out)
{
    for (int i = blockIdx.x; i < count; i += gridDim.x) pq_decode_row(d, IDS ? ids[i] : first + i, out + (size_t)i * d.dim, threadIdx.x, blockDim.x);
}

// the insert searches' queries of a BQ build: c_u as fp32, +1 where bit j is set and -1 where it is clear, j < dim. The BQ walk
// re-encodes them (prepare_blob: v > 0) to exactly c_u when c_u has no bit set past dim (bq_padding_set).
// (IDS, a refine's: nodes ids[i], as pq_decode_kernel)
template <bool IDS>
__global__ void __launch_bounds__(128) bq_decode_kernel(DataDesc d, int first, int count, const int32_t *ids, float *out)
{
    for (int i = blockIdx.x; i < count; i += gridDim.x) {
        const unsigned long long *w = d.words + (size_t)(IDS ? ids[i] : first + i) * d.W;
        for (int j = threadIdx.x; j < d.dim; j += blockDim.x) out[(size_t)i * d.dim + j] = (__ldg(w + (j >> 6)) >> (j & 63)) & 1ull ? 1.0f : -1.0f;
    }
}

// whether some row of a BQ data set has a bit set past dim in its last word: one thread per row, the flags OR-ed into *any
__global__ void __launch_bounds__(256) bq_padding_kernel(const unsigned long long *__restrict__ words, long long n, int W, unsigned long long pad_mask, int *any)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool set = r < n && (__ldg(words + (size_t)r * W + W - 1) & pad_mask) != 0;
    if (__syncthreads_or(set) && threadIdx.x == 0) atomicOr(any, 1);
}

cudaError_t bq_padding_set(const DataDesc &bq, bool *set, cudaStream_t s)
{
    *set = false;
    if ((bq.dim & 63) == 0) return cudaSuccess;
    const unsigned long long pad_mask = ~0ull << (bq.dim & 63);
    DeviceBuffer flag;
    int h = 0;
    cudaError_t e = flag.alloc(sizeof(int));
    if (e == cudaSuccess) e = cudaMemsetAsync(flag.get(), 0, sizeof(int), s);
    if (e == cudaSuccess) {
        bq_padding_kernel<<<(unsigned)((bq.n + 255) / 256), 256, 0, s>>>(bq.words, bq.n, bq.W, pad_mask, flag.get<int>());
        g_launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h, flag.get(), sizeof(int), cudaMemcpyDeviceToHost, s);
    const cudaError_t drained = cudaStreamSynchronize(s);  // the flag goes when this returns
    if (e != cudaSuccess) return e;
    *set = h != 0;
    return drained;
}

// the prune's shared memory at capacity maxc: the query block of d's kind, then the candidate state of prune_kernel (13 B per slot).
// fp32: the staged row and v's row. PQ: v's LUT and decode(c_v). BQ: c_v and the selected row's words; at most 2 * 128 words
// (dim 8192) and 8192 slots make 111 KB, so every BQ call fits
static size_t prune_smem_bytes(const DataDesc &d, int maxc)
{
    size_t b;
    switch (d.kind) {
    case KIND_PQ: b = (size_t)blob_floats(d) * 4 + (size_t)((d.dim + 3) & ~3) * 4; break;
    case KIND_BQ: b = (size_t)bq_row_floats(d) * 4 * 2; break;
    default: b = (size_t)(d.stride + 4) * 4 + (size_t)d.stride * 4; break;
    }
    b += (size_t)maxc * 8 + (size_t)maxc * 4 + 128 * 4 + maxc;
    return (b + 15) & ~(size_t)15;
}

bool pq_prune_fits(const DataDesc &pq) { return prune_smem_bytes(pq, PRUNE_MAXC) <= (size_t)PRUNE_PQ_SMEM_MAX; }

template <typename Kernel>
static cudaError_t launch_prune_kernel(Kernel kernel, size_t smem, const PruneParams &P, int grid, cudaStream_t s)
{
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kernel<<<grid, PRUNE_THREADS, smem, s>>>(P);
    g_launches++;
    return cudaGetLastError();
}

// PQ and BQ: prune_kernel at the capacity, with no Gram tier (it would change the pair bits)
template <int METRIC, int KIND>
static cudaError_t launch_code_prune(const PruneParams &P, int maxc, int grid, cudaStream_t s)
{
#define JV_CODE_PRUNE(MAXC) launch_prune_kernel(prune_kernel<METRIC, MAXC, KIND>, prune_smem_bytes(P.d, MAXC), P, grid, s)
    switch (maxc) {
    case 64: return JV_CODE_PRUNE(64);
    case 128: return JV_CODE_PRUNE(128);
    case 256: return JV_CODE_PRUNE(256);
    case 1024: return JV_CODE_PRUNE(1024);
    case 2048: return JV_CODE_PRUNE(2048);
    default: return JV_CODE_PRUNE(8192);
    }
#undef JV_CODE_PRUNE
}

// fp32: candidate sets that fit a tile go through a Gram-matrix kernel, on the tensor cores (wgmma, 3xTF32) or the CUDA cores;
// anything larger keeps the incremental kernel
template <int METRIC>
static cudaError_t launch_prune_t(const PruneParams &P, int maxc, bool tc, int grid, cudaStream_t s)
{
    if (P.d.kind == KIND_PQ) return launch_code_prune<METRIC, KIND_PQ>(P, maxc, grid, s);
    if (maxc <= 64)
        return tc ? launch_prune_kernel(prune_gram_tc_kernel<METRIC, 64>, gram_tc_smem_bytes<64>(P.d), P, grid, s)
                  : launch_prune_kernel(prune_gram_kernel<METRIC, 64>, gram_smem_bytes<64>(P.d), P, grid, s);
    if (maxc <= 128)
        return tc ? launch_prune_kernel(prune_gram_tc_kernel<METRIC, 128>, gram_tc_smem_bytes<128>(P.d), P, grid, s)
                  : launch_prune_kernel(prune_gram_kernel<METRIC, 128>, gram_smem_bytes<128>(P.d), P, grid, s);
    switch (maxc) {
    case 256: return launch_prune_kernel(prune_kernel<METRIC, 256>, prune_smem_bytes(P.d, 256), P, grid, s);
    case 1024: return launch_prune_kernel(prune_kernel<METRIC, 1024>, prune_smem_bytes(P.d, 1024), P, grid, s);
    default: return launch_prune_kernel(prune_kernel<METRIC, 8192>, prune_smem_bytes(P.d, 8192), P, grid, s);
    }
}

// the prune of P.d's kind under P.metric at capacity maxc, the smallest of the caller's tiers that holds its candidates (the
// builder: 64, 128 or 256; the repair: its tier table). tc picks the tensor-core Gram kernels for fp32 up to 128 candidates. BQ
// scores do not depend on the metric: one instantiation serves all three
static cudaError_t launch_prune(const PruneParams &P, int maxc, bool tc, int grid, cudaStream_t s)
{
    if (P.d.kind == KIND_BQ) return launch_code_prune<JV_METRIC_DOT, KIND_BQ>(P, maxc, grid, s);
    if (P.metric == JV_METRIC_EUCLIDEAN) return launch_prune_t<JV_METRIC_EUCLIDEAN>(P, maxc, tc, grid, s);
    if (P.metric == JV_METRIC_DOT) return launch_prune_t<JV_METRIC_DOT>(P, maxc, tc, grid, s);
    return launch_prune_t<JV_METRIC_COSINE>(P, maxc, tc, grid, s);
}

// the builder's prune: the Gram kernels on the tensor cores unless JV_PRUNE_GRAM=ffma asks for the CUDA-core ones
static cudaError_t launch_build_prune(const PruneParams &P, int grid, cudaStream_t s)
{
    static const bool use_tc = !(getenv("JV_PRUNE_GRAM") && getenv("JV_PRUNE_GRAM")[0] == 'f');
    const int ncmax = P.mode == 0 ? P.cand_stride + P.window : P.row_cap;
    return launch_prune(P, ncmax <= 64 ? 64 : ncmax <= 128 ? 128 : 256, use_tc, grid, s);
}

#define JV_TRY(x)                      \
    do {                               \
        err = (x);                     \
        if (err != cudaSuccess) return err; \
    } while (0)

// ------------------------------------------------------------------------------------------------
// GraphBuilder: the device-resident state of one flat (single level) build, advanced batch by batch. One rank of a sharded
// build calls insert_slice / reprune_slice for ITS part of a batch; the rows travel (NCCL all-gather in jvector_b200/parallel.py,
// nothing at all on one GPU) and every replica applies the whole batch with apply_new / apply_repruned, deterministically.
// ------------------------------------------------------------------------------------------------
struct GraphBuilder {
    DataDesc d;
    int metric = 0, sm_count = 0;
    BuildParams bp;
    int n = 0, degree = 0, beam = 0, hard_max = 0, row_cap = 0, max_batch = 0, window = 0, batch_div = 32;
    int inserted = 1;  // rows [0, inserted) are in the graph: a build starts with node 0, the entry point, and an empty list
    int32_t entry = 0;  // where the insert searches start
    uint32_t *accept = nullptr;  // rows an insert may pick (nullptr = all): bit (row & 31) of word (row >> 5)
    int32_t *adj = nullptr, *res_nodes = nullptr, *list = nullptr, *head_target = nullptr, *iota = nullptr;
    int *deg = nullptr, *mark = nullptr, *list_count = nullptr, *work_counter = nullptr;
    float *res_scores = nullptr;
    unsigned long long *dropped = nullptr, *pairs = nullptr, *pairs_sorted = nullptr;
    unsigned char *head_flag = nullptr, *node_flag = nullptr;
    SearchCounters *counters = nullptr;
    uint8_t *overflow = nullptr;
    void *cub_tmp = nullptr;
    size_t cub_bytes = 0;
    int32_t *own_rows = nullptr;  // single-GPU path: the slice buffers are the builder's own
    int *own_deg = nullptr;
    float *qdec = nullptr;        // PQ / BQ: the insert searches' queries decode(c_u) / c_u as +-1, [max_batch][dim]
    std::vector<DeviceBuffer> mem;  // owns every block above
    DeviceBuffer scratch;           // the insert searches' scratch, grown with the slice
    BuildStats st = {0, 0, 0, 0, 0};
    int prune_grid = 0;
};

void builder_destroy(GraphBuilder *B) { delete B; }

cudaError_t builder_create(const DataDesc &d, int metric, const BuildParams &bp, int sm_count, GraphBuilder **out, cudaStream_t s,
                           const BuilderSeed *seed)
{
    const int n = (int)d.n;
    if ((d.kind != KIND_F32 && d.kind != KIND_PQ && d.kind != KIND_BQ) || bp.degree < 1 || bp.degree > 64 || bp.beam < 1 || bp.beam > PRUNE_MAXC) return cudaErrorInvalidValue;
    // PQ: with the centroid-pair table of this metric (jv_dataset_pq_pair_table) and a LUT the prune can hold
    if (d.kind == KIND_PQ && (!d.pair_table[metric == JV_METRIC_EUCLIDEAN ? 0 : 1] || !pq_prune_fits(d))) return cudaErrorInvalidValue;
    if (seed && (seed->count < 0 || seed->count > n || (seed->count > 0 && (!seed->rows_dev || seed->width < 1)) || seed->entry >= seed->count))
        return cudaErrorInvalidValue;
    std::unique_ptr<GraphBuilder> B(new GraphBuilder());
    B->d = d; B->metric = metric; B->bp = bp; B->sm_count = sm_count; B->n = n; B->degree = bp.degree; B->beam = bp.beam;
    B->hard_max = (int)(bp.overflow * bp.degree);  // ConcurrentNeighborMap.java:300
    B->row_cap = std::max(2 * bp.degree, B->hard_max + 1);
    if (B->row_cap > MAX_DEGREE || (seed && seed->width > B->row_cap)) return cudaErrorInvalidValue;
    B->max_batch = bp.max_batch > 0 ? bp.max_batch : 16384;
    if (const char *e = getenv("JV_BUILD_BATCH_DIV")) B->batch_div = atoi(e) > 0 ? atoi(e) : 32;  // tuning knob (tools/build_quality.py)
    // in-progress window: as many concurrently inserting peers as still fit the 128-candidate Gram tile next to the beam
    B->window = bp.window >= 0 ? bp.window : std::max(0, std::min(32, 128 - bp.beam));
    B->prune_grid = sm_count * 5;  // ~10 KB of shared memory per CTA: register-limited residency
    cudaError_t err = cudaSuccess;
    const size_t mb = (size_t)B->max_batch;
    auto &owned = B->mem;
    JV_TRY(alloc_owned(owned, B->adj, (size_t)n * B->row_cap * 4));
    JV_TRY(alloc_owned(owned, B->deg, (size_t)n * 4));
    JV_TRY(alloc_owned(owned, B->mark, (size_t)n * 4));
    JV_TRY(alloc_owned(owned, B->res_nodes, mb * B->beam * 4));
    JV_TRY(alloc_owned(owned, B->res_scores, mb * B->beam * 4));
    JV_TRY(alloc_owned(owned, B->list, (size_t)n * 4));
    JV_TRY(alloc_owned(owned, B->iota, (size_t)n * 4));
    JV_TRY(alloc_owned(owned, B->node_flag, (size_t)n));
    JV_TRY(alloc_owned(owned, B->list_count, 16));
    JV_TRY(alloc_owned(owned, B->work_counter, 16));
    JV_TRY(alloc_owned(owned, B->dropped, 16));
    JV_TRY(alloc_owned(owned, B->counters, sizeof(SearchCounters)));
    JV_TRY(alloc_owned(owned, B->overflow, mb));
    JV_TRY(alloc_owned(owned, B->pairs, mb * B->degree * 8));
    JV_TRY(alloc_owned(owned, B->pairs_sorted, mb * B->degree * 8));
    JV_TRY(alloc_owned(owned, B->head_flag, mb * B->degree));
    JV_TRY(alloc_owned(owned, B->head_target, mb * B->degree * 4));
    JV_TRY(alloc_owned(owned, B->own_rows, mb * B->degree * 4));
    JV_TRY(alloc_owned(owned, B->own_deg, mb * 4));
    if (d.kind == KIND_PQ || d.kind == KIND_BQ) JV_TRY(alloc_owned(owned, B->qdec, mb * d.dim * 4));
    {
        size_t b1 = 0, b2 = 0;
        cub::DeviceRadixSort::SortKeys(nullptr, b1, B->pairs, B->pairs_sorted, (int)(mb * B->degree), 0, 64, s);
        cub::DeviceSelect::Flagged(nullptr, b2, B->iota, B->node_flag, B->list, B->list_count, n, s);
        B->cub_bytes = std::max(b1, b2) + 256;
        JV_TRY(alloc_owned(owned, B->cub_tmp, B->cub_bytes));
    }
    JV_TRY(cudaMemsetAsync(B->adj, 0xff, (size_t)n * B->row_cap * 4, s));
    JV_TRY(cudaMemsetAsync(B->deg, 0, (size_t)n * 4, s));
    JV_TRY(cudaMemsetAsync(B->mark, 0, (size_t)n * 4, s));
    JV_TRY(cudaMemsetAsync(B->dropped, 0, 16, s));
    JV_TRY(cudaMemsetAsync(B->list_count, 0, 16, s));
    JV_TRY(cudaMemsetAsync(B->counters, 0, sizeof(SearchCounters), s));
    iota_kernel<<<(n + 255) / 256, 256, 0, s>>>(B->iota, n);
    g_launches++;
    JV_TRY(cudaGetLastError());
    if (seed) {
        if (seed->count > 0) {
            seed_rows_kernel<<<(unsigned)(((long long)seed->count * 32 + 255) / 256), 256, 0, s>>>(seed->rows_dev, seed->count, seed->width, seed->row_map_dev,
                                                                                                  B->adj, B->deg, B->row_cap);
            g_launches++;
            JV_TRY(cudaGetLastError());
        }
        if (seed->accept) {
            const size_t words = ((size_t)n + 31) / 32;
            JV_TRY(alloc_owned(owned, B->accept, words * 4));
            JV_TRY(cudaMemcpyAsync(B->accept, seed->accept, words * 4, cudaMemcpyHostToDevice, s));
        }
        // a graph without an entry (every node removed) takes its first new row as the entry, with an empty list
        B->entry = seed->entry >= 0 ? seed->entry : seed->count;
        B->inserted = std::min(n, seed->entry >= 0 ? seed->count : seed->count + 1);
    }
    *out = B.release();
    return cudaSuccess;
}

// the next batch: 1/32 of what is already inserted, at most max_batch — every batch searches a graph that already holds 97 % of the
// nodes a sequential build would show it. Measured on 100k rows: recall@10 at rerankK 100 is 0.950
// with inserted / 2, 0.9585 with / 8, 0.9624 with / 32, against 0.9631 for the reference-order (sequential) builder.
bool builder_next_batch(GraphBuilder *B, int *first, int *count)
{
    if (B->inserted >= B->n) return false;
    int batch = B->inserted / B->batch_div;
    if (batch < 1) batch = 1;
    if (batch > B->max_batch) batch = B->max_batch;
    if (batch > B->n - B->inserted) batch = B->n - B->inserted;
    *first = B->inserted;
    *count = batch;
    return true;
}

static PruneParams prune_params(const GraphBuilder *B)
{
    PruneParams P;
    memset(&P, 0, sizeof(P));
    P.d = B->d; P.metric = B->metric; P.degree = B->degree; P.row_cap = B->row_cap; P.alpha = B->bp.alpha; P.adj = B->adj; P.deg = B->deg; P.mark = B->mark;
    return P;
}

// batch positions [lo, hi): beam search of the graph as it stands + robust prune of (beam U in-progress window) -> rows_out
// [batch][degree] at positions lo..hi-1, deg_out likewise. Reads adjacency, writes none of it.
cudaError_t builder_insert_slice(GraphBuilder *B, int first, int count, int lo, int hi, int32_t *rows_out, int *deg_out, cudaStream_t s)
{
    cudaError_t err = cudaSuccess;
    if (!rows_out) { rows_out = B->own_rows; deg_out = B->own_deg; }
    const int m = hi - lo;
    if (m <= 0) return cudaSuccess;
    GraphDesc g = {};
    g.n = B->n; g.degree = B->row_cap; g.levels = 1; g.entry_node = B->entry; g.entry_level = 0; g.adj0 = B->adj;
    SearchPlan plan;
    JV_TRY(plan_search(B->d, nullptr, g, B->beam, B->beam, m, 0, 0, B->sm_count, &plan));
    JV_TRY(B->scratch.grow(search_scratch_bytes(plan)));
    SearchFilter lenient;
    memset(&lenient, 0, sizeof(lenient));
    lenient.lenient = 1;  // an insert search never fails the build: see SearchParams::lenient
    lenient.accept_bits = B->accept;  // an add into a graph with marked nodes walks through them but never links to them
    const float *queries = B->d.rows + (size_t)(first + lo) * B->d.stride;
    int query_stride = B->d.stride;
    if (B->d.kind == KIND_PQ) {
        // searchProviderFor over PQ: the walk scores with the codes only (no rerank), its query is decode(c_u)
        pq_decode_kernel<false><<<std::min(m, B->sm_count * 16), 128, 0, s>>>(B->d, first + lo, m, nullptr, B->qdec);
        g_launches++;
        JV_TRY(cudaGetLastError());
        queries = B->qdec;
        query_stride = B->d.dim;
    } else if (B->d.kind == KIND_BQ) {
        // searchProviderFor over BQ: the walk scores with the words only (no rerank), its query encodes to c_u
        bq_decode_kernel<false><<<std::min(m, B->sm_count * 16), 128, 0, s>>>(B->d, first + lo, m, nullptr, B->qdec);
        g_launches++;
        JV_TRY(cudaGetLastError());
        queries = B->qdec;
        query_stride = B->d.dim;
    }
    JV_TRY(launch_search(g, B->d, nullptr, B->metric, queries, m, B->beam, B->beam, plan, B->scratch.get(), B->work_counter,
                         B->res_nodes, B->res_scores, B->counters, B->overflow, nullptr, query_stride, &lenient, s));
    PruneParams P = prune_params(B);
    P.mode = 0; P.node_base = first + lo; P.count = m; P.cand = B->res_nodes; P.cand_stride = B->beam;
    P.window = B->window; P.batch_first = first; P.batch_count = count;
    P.out_rows = rows_out; P.out_deg = deg_out; P.out_stride = B->degree; P.out_base = lo;
    JV_TRY(launch_build_prune(P, m < B->prune_grid ? m : B->prune_grid, s));
    return cudaSuccess;
}

// the whole batch's rows (this rank's own slice + the gathered ones): write them, back-link them deterministically, and leave
// the SORTED list of rows that passed overflow * M in B->list (count in B->list_count[0])
// ids (device, ascending): the batch is those nodes' rows replaced (a refine) rather than nodes [first, first + count) inserted
cudaError_t builder_apply_new(GraphBuilder *B, int first, int count, const int32_t *rows, const int *rdeg, cudaStream_t s, const int32_t *ids)
{
    cudaError_t err = cudaSuccess;
    if (!rows) { rows = B->own_rows; rdeg = B->own_deg; }
    const int npairs = count * B->degree;
    const unsigned blocks = (count * B->row_cap + 255) / 256;
    if (ids) apply_rows_kernel<true><<<blocks, 256, 0, s>>>(B->adj, B->deg, B->row_cap, B->degree, first, count, ids, rows, rdeg, B->pairs);
    else apply_rows_kernel<false><<<blocks, 256, 0, s>>>(B->adj, B->deg, B->row_cap, B->degree, first, count, nullptr, rows, rdeg, B->pairs);
    g_launches++;
    size_t tb = B->cub_bytes;
    JV_TRY(cub::DeviceRadixSort::SortKeys(B->cub_tmp, tb, B->pairs, B->pairs_sorted, npairs, 0, 64, s));
    g_launches++;
    backlink_sorted_kernel<<<(npairs + 255) / 256, 256, 0, s>>>(B->adj, B->deg, B->row_cap, B->hard_max, B->pairs_sorted, npairs, B->head_flag, B->head_target, B->dropped);
    g_launches++;
    publish_deg_kernel<<<(npairs + 255) / 256, 256, 0, s>>>(B->deg, B->row_cap, B->pairs_sorted, npairs);
    g_launches++;
    tb = B->cub_bytes;
    JV_TRY(cub::DeviceSelect::Flagged(B->cub_tmp, tb, B->head_target, B->head_flag, B->list, B->list_count, npairs, s));  // sorted by target: heads are
    g_launches++;
    if (!ids) B->inserted = first + count;
    B->st.batches++;
    return cudaGetLastError();
}

// rows list[lo .. hi) re-pruned (VamanaDiversityProvider.retainDiverse over the row itself). rows_out == nullptr: in place, with
// the count read on the device (one-GPU path, no host round trip); otherwise out-of-place into rows_out [.][row_cap] at lo..hi-1.
cudaError_t builder_reprune_slice(GraphBuilder *B, int lo, int hi, int32_t *rows_out, int *deg_out, cudaStream_t s)
{
    PruneParams P = prune_params(B);
    P.mode = 1; P.list = B->list;
    if (!rows_out) {
        P.count_ptr = B->list_count;
        return launch_build_prune(P, B->prune_grid, s);
    }
    if (hi <= lo) return cudaSuccess;
    P.count = hi - lo; P.list_base = lo; P.out_rows = rows_out; P.out_deg = deg_out; P.out_stride = B->row_cap; P.out_base = lo;
    return launch_build_prune(P, std::min(hi - lo, B->prune_grid), s);
}

cudaError_t builder_apply_repruned(GraphBuilder *B, int count, const int32_t *rows, const int *rdeg, cudaStream_t s)
{
    if (count <= 0) return cudaSuccess;
    scatter_rows_kernel<<<(count * B->row_cap + 255) / 256, 256, 0, s>>>(B->adj, B->deg, B->row_cap, B->list, count, rows, rdeg);
    g_launches++;
    return cudaGetLastError();
}

// cleanup() of the reference: enforceDegree on every row longer than M. Leaves the sorted list of those rows in B->list.
cudaError_t builder_collect_over_degree(GraphBuilder *B, cudaStream_t s)
{
    cudaError_t err = cudaSuccess;
    flag_over_degree_kernel<<<(B->n + 255) / 256, 256, 0, s>>>(B->deg, B->n, B->degree, B->node_flag);
    g_launches++;
    size_t tb = B->cub_bytes;
    JV_TRY(cub::DeviceSelect::Flagged(B->cub_tmp, tb, B->iota, B->node_flag, B->list, B->list_count, B->n, s));
    g_launches++;
    return cudaGetLastError();
}

cudaError_t builder_list_count(GraphBuilder *B, int *count_host, cudaStream_t s)
{
    cudaError_t err = cudaSuccess;
    JV_TRY(cudaMemcpyAsync(count_host, B->list_count, sizeof(int), cudaMemcpyDeviceToHost, s));
    return cudaStreamSynchronize(s);
}

// the counters so far: batches applied, insert searches cut short, back-links dropped at a full row (synchronises `s`)
cudaError_t builder_stats(GraphBuilder *B, BuildStats *stats, cudaStream_t s)
{
    cudaError_t err = cudaSuccess;
    SearchCounters hc;
    unsigned long long hd = 0;
    JV_TRY(cudaMemcpyAsync(&hc, B->counters, sizeof(hc), cudaMemcpyDeviceToHost, s));
    JV_TRY(cudaMemcpyAsync(&hd, B->dropped, sizeof(hd), cudaMemcpyDeviceToHost, s));
    JV_TRY(cudaStreamSynchronize(s));
    B->st.searched = (long long)hc.visited;
    B->st.dropped_backlinks = (long long)hd;
    B->st.truncated_searches = (long long)hc.overflowed;
    if (stats) *stats = B->st;
    return cudaSuccess;
}

cudaError_t builder_finish(GraphBuilder *B, int32_t *adj_out_dev, BuildStats *stats, cudaStream_t s)
{
    const long long total = (long long)B->n * B->degree;
    compact_adj_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(B->adj, B->deg, B->n, B->row_cap, B->degree, adj_out_dev);
    g_launches++;
    const cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return err;
    return builder_stats(B, stats, s);
}

int builder_row_cap(const GraphBuilder *B) { return B->row_cap; }
int builder_degree(const GraphBuilder *B) { return B->degree; }
int builder_max_batch(const GraphBuilder *B) { return B->max_batch; }

// the whole build on one GPU: no exchange, no host synchronisation between batches. The same loop extends a seeded builder (an
// add into an existing graph): only the starting state differs.
cudaError_t build_graph_flat(const DataDesc &d, int metric, const BuildParams &bp, int32_t *adj_out_dev, int sm_count,
                             BuildStats *stats, cudaStream_t s, const BuilderSeed *seed)
{
    GraphBuilder *B = nullptr;
    cudaError_t err = builder_create(d, metric, bp, sm_count, &B, s, seed);
    if (err != cudaSuccess) return err;
    int first, count;
    while (err == cudaSuccess && builder_next_batch(B, &first, &count)) {
        err = builder_insert_slice(B, first, count, 0, count, nullptr, nullptr, s);
        if (err == cudaSuccess) err = builder_apply_new(B, first, count, nullptr, nullptr, s);
        if (err == cudaSuccess) err = builder_reprune_slice(B, 0, 0, nullptr, nullptr, s);
    }
    if (err == cudaSuccess) err = builder_collect_over_degree(B, s);
    if (err == cudaSuccess) err = builder_reprune_slice(B, 0, 0, nullptr, nullptr, s);
    if (err == cudaSuccess) err = builder_finish(B, adj_out_dev, stats, s);
    else if (stats) *stats = B->st;
    delete B;
    return err;
}

// ------------------------------------------------------------------------------------------------
// Repair of deleted neighbours (GraphIndexBuilder.removeDeletedNodes, base:graph/GraphIndexBuilder.java:689-799), one level at a time:
//   count  : one warp per row flags the live rows that name a deleted node and sizes their candidate segment
//   gather : one CTA per flagged row writes its live neighbours, the live 2-hop ids through its deleted neighbours (the FreshDiskANN
//            rule, :705-721) — or, when there are no such ids, random live members of the level (:743-759) — sorted and deduplicated
//   prune  : the builder's prune kernels (mode 2, ragged candidates, out of place), dispatched by candidate count so no set is clipped;
//            over a PQ data set the PQ prune at every tier, with the scores of the PQ build (query decode(c_v), ADC keys, pair table);
//            over a BQ data set the BQ prune at every tier, with Hamming scores
//   scatter: the pruned rows replace the old ones in the output adjacency
// Nothing depends on timing: compaction and offsets come from cub scans, the dedup from a sort, and the prune is deterministic.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool dead_bit(const uint32_t *bits, int v) { return (bits[v >> 5] >> (v & 31)) & 1u; }

__global__ void __launch_bounds__(256) repair_count_kernel(const int32_t *__restrict__ adj, int rows, int degree, const int32_t *__restrict__ ids,
                                                           const int32_t *__restrict__ rowmap, const uint32_t *__restrict__ dead, unsigned char *flag,
                                                           long long *cnt)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const int r = (int)warp;
    const int v = ids ? ids[r] : r;
    int live = 0, two = 0, hit = 0;
    if (!dead_bit(dead, v)) {
        for (int s = lane; s < degree; s += 32) {
            const int32_t j = adj[(size_t)r * degree + s];
            if (j < 0) continue;
            if (!dead_bit(dead, j)) { live++; continue; }
            hit = 1;
            const int rj = rowmap ? rowmap[j] : j;
            if (rj < 0) continue;
            for (int t = 0; t < degree; t++) {
                const int32_t k = adj[(size_t)rj * degree + t];
                if (k >= 0 && k != v && !dead_bit(dead, k)) two++;
            }
        }
    }
    live = group_sum<32>(live);
    two = group_sum<32>(two);
    hit = __any_sync(FULL, hit);
    if (lane == 0) {
        flag[r] = hit ? 1 : 0;
        // the random fallback adds at most `degree` picks; 2 * degree keeps the segment a multiple of the row width
        cnt[r] = hit ? (long long)live + two + (two == 0 ? 2 * degree : 0) : 0;
    }
}

__device__ __forceinline__ void bitonic_sort_asc_int(int32_t *keys, int n_pow2)
{
    for (int k = 2; k <= n_pow2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n_pow2; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const int32_t a = keys[i], b = keys[ixj];
                    const bool asc = (i & k) == 0;
                    if (asc ? (a > b) : (a < b)) { keys[i] = b; keys[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
}

// slot layout of a row's shared buffer (cap >= degree * (degree + 2), a power of two >= 256):
//   [0, degree)                           the live neighbours
//   degree + s * degree + t               entry t of the row of deleted neighbour s (live, != v)
//   degree * (degree + 1) + p             random pick p of the fallback
__global__ void __launch_bounds__(256) repair_gather_kernel(const int32_t *__restrict__ adj, int degree, const int32_t *__restrict__ ids,
                                                            const int32_t *__restrict__ rowmap, const uint32_t *__restrict__ dead,
                                                            const int32_t *__restrict__ aff, int naff, const long long *__restrict__ off_all, int cap,
                                                            const int32_t *__restrict__ members, int nmembers, unsigned long long seed, int level,
                                                            int32_t *cand, int32_t *row_node, long long *cand_off, int *cand_cnt, unsigned char *fallback)
{
    extern __shared__ int32_t buf[];
    __shared__ int32_t s_row[64];
    __shared__ int s_any;
    using BlockScan = cub::BlockScan<int, 256>;
    __shared__ typename BlockScan::TempStorage scan_tmp;
    const int tid = threadIdx.x;
    const int per = cap / 256;
    for (int a = blockIdx.x; a < naff; a += gridDim.x) {
        const int r = aff[a];
        const int v = ids ? ids[r] : r;
        for (int i = tid; i < cap; i += 256) buf[i] = INT_MAX;
        if (tid < degree) s_row[tid] = adj[(size_t)r * degree + tid];
        if (tid == 0) s_any = 0;
        __syncthreads();
        for (int x = tid; x < degree * (degree + 1); x += 256) {
            if (x < degree) {
                const int32_t j = s_row[x];
                if (j >= 0 && !dead_bit(dead, j)) buf[x] = j;
            } else {
                const int s = (x - degree) / degree, t = (x - degree) - s * degree;
                const int32_t j = s_row[s];
                if (j < 0 || !dead_bit(dead, j)) continue;
                const int rj = rowmap ? rowmap[j] : j;
                if (rj < 0) continue;
                const int32_t k = adj[(size_t)rj * degree + t];
                if (k >= 0 && k != v && !dead_bit(dead, k)) {
                    buf[x] = k;
                    s_any = 1;  // every writer stores the same value
                }
            }
        }
        __syncthreads();
        const bool fb = s_any == 0;
        if (fb && tid == 0 && nmembers > 0) {
            // no 2-hop candidate: up to 2 * degree random live members of the level, skipping v and repeats, until degree are found
            int32_t *pick = buf + degree * (degree + 1);
            int np = 0;
            for (int at = 0; at < 2 * degree && np < degree; at++) {
                const int32_t k = members[counter_random(seed, level, v, at) % (uint64_t)nmembers];
                bool dup = k == v;
                for (int p = 0; p < np && !dup; p++) dup = pick[p] == k;
                if (!dup) pick[np++] = k;
            }
        }
        __syncthreads();
        bitonic_sort_asc_int(buf, cap);
        // distinct ids, compacted in ascending order into the row's segment
        int c = 0;
        for (int i = tid * per; i < (tid + 1) * per; i++)
            c += buf[i] != INT_MAX && (i == 0 || buf[i - 1] != buf[i]);
        int pre, total;
        BlockScan(scan_tmp).ExclusiveSum(c, pre, total);
        const long long off = off_all[r];
        for (int i = tid * per; i < (tid + 1) * per; i++)
            if (buf[i] != INT_MAX && (i == 0 || buf[i - 1] != buf[i])) cand[off + pre++] = buf[i];
        if (tid == 0) {
            row_node[a] = v;
            cand_off[a] = off;
            cand_cnt[a] = total;
            fallback[a] = fb ? 1 : 0;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) repair_scatter_kernel(int32_t *adj, int degree, const int32_t *aff, int naff, const int32_t *rows)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)naff * degree) return;
    const int a = (int)(idx / degree), t = (int)(idx - (long long)a * degree);
    adj[(size_t)aff[a] * degree + t] = rows[idx];
}

__global__ void __launch_bounds__(256) clear_dead_rows_kernel(int32_t *adj, int n, int degree, const uint32_t *dead)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n * degree) return;
    if (dead_bit(dead, (int)(idx / degree))) adj[idx] = -1;
}

cudaError_t launch_clear_dead_rows(int32_t *adj_dev, int n, int degree, const uint32_t *dead_dev, cudaStream_t s)
{
    const long long total = (long long)n * degree;
    clear_dead_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(adj_dev, n, degree, dead_dev);
    g_launches++;
    return cudaGetLastError();
}

// the prune tiers of the repair: TILE-candidate Gram kernels on the tensor cores, then the incremental kernel at growing capacity
constexpr int REPAIR_TIERS = 5;
constexpr int REPAIR_TIER_MAX[REPAIR_TIERS] = {64, 128, 256, 1024, 8192};
// over a PQ data set (§4.3e) or a BQ data set (§4.3g) there is no Gram tier — it would change the pair bits — and every tier is
// prune_kernel<.., KIND_PQ> or <.., KIND_BQ>. The candidate state (13 B per slot) shares the CTA's shared memory with the whole LUT
// (PQ), so 2048 sits between 1024 and 8192: a degree-32 row has at most 32 * 34 = 1088 candidates and never pays for 8192 slots (106 KB)
constexpr int CODE_REPAIR_TIERS = 6;
constexpr int CODE_REPAIR_TIER_MAX[CODE_REPAIR_TIERS] = {64, 128, 256, 1024, 2048, 8192};
static_assert(CODE_REPAIR_TIERS <= (int)(sizeof(RepairStats::tier_rows) / sizeof(long long)), "RepairStats::tier_rows holds every tier");

// whether the repair of a degree-`degree` graph over `pq` can run: a row gathers up to degree * (degree + 2) candidates, and the tier
// that holds them must fit next to the LUT
bool pq_repair_fits(const DataDesc &pq, int degree) { return pq_ragged_fits(pq, degree * (degree + 2)); }

// whether the ragged prune's PQ tier that holds max_cands candidates fits next to the LUT
bool pq_ragged_fits(const DataDesc &pq, int max_cands)
{
    int t = 0;
    while (t < CODE_REPAIR_TIERS - 1 && max_cands > CODE_REPAIR_TIER_MAX[t]) t++;
    return prune_smem_bytes(pq, CODE_REPAIR_TIER_MAX[t]) <= (size_t)PRUNE_PQ_SMEM_MAX;
}

// the prune of ragged candidate rows (mode 2, out of place), each row at the smallest tier that holds its candidates: the repair's
// and the compaction's. tier_list: device scratch [rows]; tier_rows (optional) counts the rows of every tier
static cudaError_t prune_ragged_enqueue(const DataDesc &d, int metric, float alpha, int degree, int rows, const int32_t *cand, const int32_t *row_node,
                                        const long long *cand_off, const int *cand_cnt, const std::vector<int> &hcnt, int32_t *out_rows, int *out_deg,
                                        int32_t *tier_list, int sm_count, long long *tier_rows, cudaStream_t s)
{
    cudaError_t err = cudaSuccess;
    const bool codes = d.kind == KIND_PQ || d.kind == KIND_BQ;
    const int ntiers = codes ? CODE_REPAIR_TIERS : REPAIR_TIERS;
    const int *tier_max = codes ? CODE_REPAIR_TIER_MAX : REPAIR_TIER_MAX;
    std::vector<int32_t> tiers[CODE_REPAIR_TIERS];
    for (int a = 0; a < rows; a++) {
        int t = 0;
        while (t < ntiers - 1 && hcnt[a] > tier_max[t]) t++;
        tiers[t].push_back(a);
        if (tier_rows) tier_rows[t]++;
    }
    std::vector<int32_t> hlist;
    for (int t = 0; t < ntiers; t++) hlist.insert(hlist.end(), tiers[t].begin(), tiers[t].end());
    JV_TRY(cudaMemcpyAsync(tier_list, hlist.data(), (size_t)rows * 4, cudaMemcpyHostToDevice, s));
    PruneParams P;
    memset(&P, 0, sizeof(P));
    P.d = d; P.metric = metric; P.degree = degree; P.row_cap = degree; P.alpha = alpha; P.mode = 2;
    P.cand = cand; P.row_node = row_node; P.cand_off = cand_off; P.cand_cnt = cand_cnt;
    P.out_rows = out_rows; P.out_deg = out_deg; P.out_stride = degree;
    int first = 0;
    for (int t = 0; t < ntiers; t++) {
        const int c = (int)tiers[t].size();
        if (c == 0) continue;
        P.list = tier_list + first;
        P.count = c;
        JV_TRY(launch_prune(P, tier_max[t], true, std::min(c, sm_count * 5), s));
        first += c;
    }
    return cudaSuccess;
}

cudaError_t launch_scatter_rows(int32_t *adj_dev, int degree, const int32_t *rows_of_dev, int count, const int32_t *rows_dev, cudaStream_t s)
{
    if (count <= 0) return cudaSuccess;
    repair_scatter_kernel<<<(unsigned)(((long long)count * degree + 255) / 256), 256, 0, s>>>(adj_dev, degree, rows_of_dev, count, rows_dev);
    g_launches++;
    return cudaGetLastError();
}

// repair_level's work, enqueued on `s`; every block it allocates goes to `mem`
static cudaError_t repair_level_enqueue(const DataDesc &d, int metric, float alpha, int degree, int rows, const int32_t *adj_old, int32_t *adj_new,
                                        const int32_t *ids_dev, const int32_t *rowmap_dev, const uint32_t *dead_dev, const int32_t *members_dev,
                                        int nmembers, uint64_t seed, int level, int sm_count, RepairStats *st, std::vector<DeviceBuffer> &mem,
                                        cudaStream_t s)
{
    cudaError_t err = cudaSuccess;
    unsigned char *flag, *fallback;
    long long *cnt, *off_all, *cand_off;
    int32_t *iota, *aff, *cand, *row_node, *out_rows, *tier_list;
    int *naff_dev, *cand_cnt, *out_deg;
    void *tmp;
    JV_TRY(alloc_owned(mem, flag, (size_t)rows));
    JV_TRY(alloc_owned(mem, cnt, (size_t)rows * 8));
    JV_TRY(alloc_owned(mem, off_all, (size_t)rows * 8));
    JV_TRY(alloc_owned(mem, iota, (size_t)rows * 4));
    JV_TRY(alloc_owned(mem, aff, (size_t)rows * 4));
    JV_TRY(alloc_owned(mem, naff_dev, 16));
    repair_count_kernel<<<(unsigned)(((long long)rows * 32 + 255) / 256), 256, 0, s>>>(adj_old, rows, degree, ids_dev, rowmap_dev, dead_dev, flag, cnt);
    g_launches++;
    iota_kernel<<<(rows + 255) / 256, 256, 0, s>>>(iota, rows);
    g_launches++;
    JV_TRY(cudaGetLastError());
    size_t t1 = 0, t2 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, t1, cnt, off_all, rows, s);
    cub::DeviceSelect::Flagged(nullptr, t2, iota, flag, aff, naff_dev, rows, s);
    const size_t tb = std::max(t1, t2) + 256;
    JV_TRY(alloc_owned(mem, tmp, tb));
    t1 = tb;
    JV_TRY(cub::DeviceScan::ExclusiveSum(tmp, t1, cnt, off_all, rows, s));
    g_launches++;
    t2 = tb;
    JV_TRY(cub::DeviceSelect::Flagged(tmp, t2, iota, flag, aff, naff_dev, rows, s));
    g_launches++;
    int naff = 0;
    long long last[2] = {0, 0};
    JV_TRY(cudaMemcpyAsync(&naff, naff_dev, sizeof(int), cudaMemcpyDeviceToHost, s));
    JV_TRY(cudaMemcpyAsync(&last[0], off_all + rows - 1, 8, cudaMemcpyDeviceToHost, s));
    JV_TRY(cudaMemcpyAsync(&last[1], cnt + rows - 1, 8, cudaMemcpyDeviceToHost, s));
    JV_TRY(cudaStreamSynchronize(s));
    const long long total = last[0] + last[1];
    if (naff == 0) return cudaSuccess;
    JV_TRY(alloc_owned(mem, cand, (size_t)std::max(total, 1ll) * 4));
    JV_TRY(alloc_owned(mem, row_node, (size_t)naff * 4));
    JV_TRY(alloc_owned(mem, cand_off, (size_t)naff * 8));
    JV_TRY(alloc_owned(mem, cand_cnt, (size_t)naff * 4));
    JV_TRY(alloc_owned(mem, fallback, (size_t)naff));
    JV_TRY(alloc_owned(mem, out_rows, (size_t)naff * degree * 4));
    JV_TRY(alloc_owned(mem, out_deg, (size_t)naff * 4));
    JV_TRY(alloc_owned(mem, tier_list, (size_t)naff * 4));
    {
        int cap = 256;
        while (cap < degree * (degree + 2)) cap <<= 1;
        const size_t gsm = (size_t)cap * 4;
        JV_TRY(cudaFuncSetAttribute(repair_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gsm));
        repair_gather_kernel<<<std::min(naff, sm_count * 8), 256, gsm, s>>>(adj_old, degree, ids_dev, rowmap_dev, dead_dev, aff, naff, off_all, cap, members_dev,
                                                                           nmembers, (unsigned long long)seed, level, cand, row_node, cand_off, cand_cnt, fallback);
        g_launches++;
        JV_TRY(cudaGetLastError());
    }
    std::vector<int> hcnt(naff);
    std::vector<unsigned char> hfb(naff);
    JV_TRY(cudaMemcpyAsync(hcnt.data(), cand_cnt, (size_t)naff * 4, cudaMemcpyDeviceToHost, s));
    JV_TRY(cudaMemcpyAsync(hfb.data(), fallback, (size_t)naff, cudaMemcpyDeviceToHost, s));
    JV_TRY(cudaStreamSynchronize(s));
    for (int a = 0; a < naff; a++) {
        st->candidates += hcnt[a];
        st->max_candidates = std::max(st->max_candidates, hcnt[a]);
        st->random_fallbacks += hfb[a];
    }
    st->repaired_rows += naff;
    JV_TRY(prune_ragged_enqueue(d, metric, alpha, degree, naff, cand, row_node, cand_off, cand_cnt, hcnt, out_rows, out_deg, tier_list, sm_count,
                                st->tier_rows, s));
    return launch_scatter_rows(adj_new, degree, aff, naff, out_rows, s);
}

cudaError_t repair_level(const DataDesc &d, int metric, float alpha, int degree, int rows, const int32_t *adj_old, int32_t *adj_new, const int32_t *ids_dev,
                         const int32_t *rowmap_dev, const uint32_t *dead_dev, const int32_t *members_dev, int nmembers, uint64_t seed, int level,
                         int sm_count, RepairStats *st, cudaStream_t s)
{
    if (rows <= 0) return cudaSuccess;
    if (degree < 1 || degree > 64 || (d.kind != KIND_F32 && d.kind != KIND_PQ && d.kind != KIND_BQ)) return cudaErrorInvalidValue;
    if (d.kind == KIND_PQ && (!d.pair_table[metric == JV_METRIC_EUCLIDEAN ? 0 : 1] || !pq_repair_fits(d, degree))) return cudaErrorInvalidValue;
    std::vector<DeviceBuffer> mem;  // the scratch goes when this returns: the stream drains first, on success and on error
    const cudaError_t err = repair_level_enqueue(d, metric, alpha, degree, rows, adj_old, adj_new, ids_dev, rowmap_dev, dead_dev, members_dev, nmembers,
                                                 seed, level, sm_count, st, mem, s);
    const cudaError_t drained = cudaStreamSynchronize(s);
    return err != cudaSuccess ? err : drained;
}

// ------------------------------------------------------------------------------------------------
// Compaction (OnDiskGraphIndexCompactor's per-node work, DESIGN §4.3h). The searches into the other sources run in api.cu (the search
// kernel over each source, or over a source's sub-hierarchy for an upper level); here every merged row of a level gets its candidate
// segment and the repair's ragged prune picks its neighbours. The candidates are the node's live neighbours in its own source and,
// per other source, the search results or that source's whole live membership of the level, each under its new id. Distinct
// sources map to distinct new ids, so no segment holds an id twice and none needs a dedup. One warp per row; the ballot compaction
// keeps the order of its inputs, so the segment is a pure function of them.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) compact_assemble_kernel(int rows, int degree, int K, const int32_t *__restrict__ own_adj,
                                                               const int32_t *__restrict__ own_row, const int32_t *__restrict__ old_to_new,
                                                               const CompactTarget *__restrict__ targets, int ntargets, long long row0, int cand_stride,
                                                               int32_t *__restrict__ cand, long long *__restrict__ cand_off, int *__restrict__ cand_cnt)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const int i = (int)warp;
    const long long off = (row0 + i) * cand_stride;
    int32_t *seg = cand + off;
    int w = 0;
    // every lane offers one id (-1: none); the kept ones are appended in lane order
    auto put = [&](int32_t id) {
        const unsigned b = __ballot_sync(FULL, id >= 0);
        if (id >= 0) seg[w + __popc(b & ((1u << lane) - 1u))] = id;
        w += __popc(b);
    };
    const int32_t *row = own_adj + (size_t)own_row[i] * degree;
    for (int j0 = 0; j0 < degree; j0 += 32) {
        const int32_t nb = j0 + lane < degree ? row[j0 + lane] : -1;
        put(nb >= 0 ? old_to_new[nb] : -1);
    }
    for (int t = 0; t < ntargets; t++) {
        const CompactTarget T = targets[t];
        if (T.res) {
            const int32_t *r = T.res + (size_t)i * K;
            for (int j0 = 0; j0 < K; j0 += 32) {
                const int32_t p = j0 + lane < K ? r[j0 + lane] : -1;
                put(p >= 0 ? T.map[p] : -1);
            }
        } else {
            for (int j0 = 0; j0 < T.count; j0 += 32) put(j0 + lane < T.count ? T.list[j0 + lane] : -1);
        }
    }
    if (lane == 0) {
        cand_off[i] = off;
        cand_cnt[i] = w;
    }
}

cudaError_t launch_compact_assemble(int rows, int degree, int K, const int32_t *own_adj, const int32_t *own_row, const int32_t *old_to_new,
                                    const CompactTarget *targets_dev, int ntargets, long long row0, int cand_stride, int32_t *cand, long long *cand_off,
                                    int *cand_cnt, cudaStream_t s)
{
    if (rows <= 0) return cudaSuccess;
    compact_assemble_kernel<<<(unsigned)(((long long)rows * 32 + 255) / 256), 256, 0, s>>>(rows, degree, K, own_adj, own_row, old_to_new, targets_dev,
                                                                                          ntargets, row0, cand_stride, cand, cand_off, cand_cnt);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t prune_ragged_rows(const DataDesc &d, int metric, float alpha, int degree, int rows, const int32_t *cand, const int32_t *row_node,
                              const long long *cand_off, const int *cand_cnt, const std::vector<int> &hcnt, int32_t *out_rows, int sm_count, cudaStream_t s)
{
    if (rows <= 0) return cudaSuccess;
    if (degree < 1 || degree > 64 || d.kind != KIND_F32) return cudaErrorInvalidValue;
    std::vector<DeviceBuffer> mem;  // the scratch goes when this returns: the stream drains first, on success and on error
    cudaError_t err = cudaSuccess;
    int *out_deg = nullptr;
    int32_t *tier_list = nullptr;
    if ((err = alloc_owned(mem, out_deg, (size_t)rows * 4)) == cudaSuccess && (err = alloc_owned(mem, tier_list, (size_t)rows * 4)) == cudaSuccess)
        err = prune_ragged_enqueue(d, metric, alpha, degree, rows, cand, row_node, cand_off, cand_cnt, hcnt, out_rows, out_deg, tier_list, sm_count, nullptr, s);
    const cudaError_t drained = cudaStreamSynchronize(s);
    return err != cudaSuccess ? err : drained;
}

// ------------------------------------------------------------------------------------------------
// Refinement (GraphIndexBuilder.cleanup's improveConnections, OnDiskGraphIndexCompactor's refine pass; DESIGN §4.3i), one level at a
// time. The level's rows seed a GraphBuilder; the nodes to refine go through it in ascending batches of at most max_batch:
//   search  : graph_search_kernel over the level from its entry, the node's own row (decode(c_v), c_v as +-1) as the query and the
//             node itself walked through but never accepted (SearchFilter::exclude_ids), topK = rerankK = beam
//   assemble: refine_assemble_kernel, one warp per node: its current row, then the results that are not in it
//   prune   : the ragged prune (prune_ragged_enqueue) to M, which sorts the candidates by the top-k key
//   builder form  : the batch's rows are applied with their back-links (builder_apply_new over the id list, a link into a row that
//                   already names the node skipped), the rows that passed overflow * M are re-pruned, so the next batch searches the
//                   level as this one left it; after the last batch every row longer than M is re-pruned
//   compactor form: every search reads the level as it was given; the rows replace the old ones at the end, with no back-links
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) refine_assemble_kernel(int rows, const int32_t *__restrict__ ids, const int32_t *__restrict__ adj,
                                                              const int *__restrict__ deg, int row_cap, const int32_t *__restrict__ res, int K,
                                                              int cand_stride, int32_t *__restrict__ cand, long long *__restrict__ cand_off,
                                                              int *__restrict__ cand_cnt)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const int i = (int)warp;
    const int32_t *row = adj + (size_t)ids[i] * row_cap;
    const int d = min(deg[ids[i]], row_cap);
    int32_t *seg = cand + (size_t)i * cand_stride;
    int w = 0;
    // every lane offers one id (-1: none); the kept ones are appended in lane order
    auto put = [&](int32_t id) {
        const unsigned b = __ballot_sync(FULL, id >= 0);
        if (id >= 0) seg[w + __popc(b & ((1u << lane) - 1u))] = id;
        w += __popc(b);
    };
    for (int j0 = 0; j0 < d; j0 += 32) put(j0 + lane < d ? row[j0 + lane] : -1);
    for (int j0 = 0; j0 < K; j0 += 32) {
        int32_t id = j0 + lane < K ? res[(size_t)i * K + j0 + lane] : -1;
        for (int x = 0; x < d && id >= 0; x++)
            if (row[x] == id) id = -1;
        put(id);
    }
    if (lane == 0) {
        cand_off[i] = (long long)i * cand_stride;
        cand_cnt[i] = w;
    }
}

// the back-link pairs of a batch that were not skipped: the sorted pairs end in ~0 entries
__global__ void count_links_kernel(const unsigned long long *pairs_sorted, int npairs, unsigned long long *count)
{
    atomicAdd(count, (unsigned long long)lower_bound_u64(pairs_sorted, npairs, ~0ull));
}

// rows of a [n][degree] adjacency that differ from those of b, one thread per row
__global__ void __launch_bounds__(256) count_changed_rows_kernel(const int32_t *a, const int32_t *b, int n, int degree, unsigned long long *count)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    bool changed = false;
    if (v < n)
        for (int j = 0; j < degree && !changed; j++) changed = a[(size_t)v * degree + j] != b[(size_t)v * degree + j];
    const unsigned m = __ballot_sync(FULL, changed);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(count, (unsigned long long)__popc(m));
}

static cudaError_t refine_level_enqueue(const DataDesc &d, int metric, const BuildParams &bp, int beam, bool compactor, const int32_t *adj_in,
                                        int degree, int32_t entry, const std::vector<int32_t> &nodes, int32_t *adj_out, int sm_count, RefineStats *st,
                                        GraphBuilder **Bp, std::vector<DeviceBuffer> &mem, cudaStream_t s)
{
    cudaError_t err = cudaSuccess;
    const int n = (int)d.n, nn = (int)nodes.size();
    // the builder holds the level's rows, degrees, back-link and re-prune state; its own insert buffers go unused
    BuildParams cp = bp;
    cp.beam = std::min(beam, PRUNE_MAXC);
    cp.window = 0;
    const BuilderSeed seed = {adj_in, n, degree, nullptr, entry, nullptr};
    JV_TRY(builder_create(d, metric, cp, sm_count, Bp, s, &seed));
    GraphBuilder *B = *Bp;
    const int mb = std::min(B->max_batch, std::max(nn, 1)), row_cap = B->row_cap, cand_stride = row_cap + beam;
    const bool codes = d.kind == KIND_PQ || d.kind == KIND_BQ;
    int32_t *list, *res, *cand, *out_rows, *tier_list;
    float *qrows = B->qdec, *scores;
    long long *cand_off;
    int *cand_cnt, *out_deg;
    unsigned long long *counts;  // back-links kept, rows changed
    JV_TRY(alloc_owned(mem, list, (size_t)std::max(nn, 1) * 4));
    if (!codes) JV_TRY(alloc_owned(mem, qrows, (size_t)mb * d.stride * 4));
    JV_TRY(alloc_owned(mem, res, (size_t)mb * beam * 4));
    JV_TRY(alloc_owned(mem, scores, (size_t)mb * beam * 4));
    JV_TRY(alloc_owned(mem, cand, (size_t)mb * cand_stride * 4));
    JV_TRY(alloc_owned(mem, cand_off, (size_t)mb * 8));
    JV_TRY(alloc_owned(mem, cand_cnt, (size_t)mb * 4));
    JV_TRY(alloc_owned(mem, tier_list, (size_t)mb * 4));
    // compactor form: every refined row is kept until the end
    JV_TRY(alloc_owned(mem, out_rows, (size_t)(compactor ? std::max(nn, 1) : mb) * degree * 4));
    JV_TRY(alloc_owned(mem, out_deg, (size_t)(compactor ? std::max(nn, 1) : mb) * 4));
    JV_TRY(alloc_owned(mem, counts, 16));
    // st->device_ms: the stream time of the device work, lap by lap between the host's waits (the batch's candidate counts, the
    // re-prune list's length); the allocations above and the host's work while the stream is idle are outside it
    StreamTimer timer;
    auto lap_end = [&]() -> cudaError_t {
        cudaError_t e = timer.stop(s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e == cudaSuccess) st->device_ms += timer.ms();
        return e;
    };
    JV_TRY(timer.start(s));
    JV_TRY(cudaMemsetAsync(counts, 0, 16, s));
    if (nn > 0) JV_TRY(cudaMemcpyAsync(list, nodes.data(), (size_t)nn * 4, cudaMemcpyHostToDevice, s));
    GraphDesc g = {};
    g.n = n; g.degree = row_cap; g.levels = 1; g.entry_node = B->entry; g.entry_level = 0; g.adj0 = B->adj;
    SearchFilter f;
    memset(&f, 0, sizeof(f));
    f.lenient = 1;  // as an insert search: a full visited table ends the walk with what it has
    std::vector<int> hcnt;
    for (int b0 = 0; b0 < nn; b0 += mb) {
        const int m = std::min(mb, nn - b0);
        const int32_t *ids = list + b0;
        int query_stride = d.stride;
        if (d.kind == KIND_PQ) pq_decode_kernel<true><<<std::min(m, sm_count * 16), 128, 0, s>>>(d, 0, m, ids, qrows);
        else if (d.kind == KIND_BQ) bq_decode_kernel<true><<<std::min(m, sm_count * 16), 128, 0, s>>>(d, 0, m, ids, qrows);
        if (codes) {
            g_launches++;
            JV_TRY(cudaGetLastError());
            query_stride = d.dim;
        } else {
            JV_TRY(launch_gather_rows(d, ids, m, qrows, s));
        }
        SearchPlan plan;
        JV_TRY(plan_search(d, nullptr, g, beam, beam, m, 0, 0, sm_count, &plan));
        JV_TRY(B->scratch.grow(search_scratch_bytes(plan)));
        f.exclude_ids = ids;
        JV_TRY(launch_search(g, d, nullptr, metric, qrows, m, beam, beam, plan, B->scratch.get(), B->work_counter, res, scores, B->counters, B->overflow,
                             nullptr, query_stride, &f, s));
        refine_assemble_kernel<<<(unsigned)(((long long)m * 32 + 255) / 256), 256, 0, s>>>(m, ids, B->adj, B->deg, row_cap, res, beam, cand_stride, cand,
                                                                                         cand_off, cand_cnt);
        g_launches++;
        JV_TRY(cudaGetLastError());
        hcnt.resize(m);
        JV_TRY(cudaMemcpyAsync(hcnt.data(), cand_cnt, (size_t)m * 4, cudaMemcpyDeviceToHost, s));
        JV_TRY(lap_end());
        JV_TRY(timer.start(s));
        for (int a = 0; a < m; a++) {
            st->candidates += hcnt[a];
            st->max_candidates = std::max(st->max_candidates, hcnt[a]);
        }
        int32_t *rows = compactor ? out_rows + (size_t)b0 * degree : out_rows;
        int *rdeg = compactor ? out_deg + b0 : out_deg;
        JV_TRY(prune_ragged_enqueue(d, metric, bp.alpha, degree, m, cand, ids, cand_off, cand_cnt, hcnt, rows, rdeg, tier_list, sm_count, nullptr, s));
        if (compactor) continue;
        JV_TRY(builder_apply_new(B, 0, m, rows, rdeg, s, ids));
        count_links_kernel<<<1, 1, 0, s>>>(B->pairs_sorted, m * degree, counts);
        g_launches++;
        int over = 0;
        JV_TRY(lap_end());
        JV_TRY(builder_list_count(B, &over, s));
        JV_TRY(timer.start(s));
        st->rows_repruned += over;
        JV_TRY(builder_reprune_slice(B, 0, 0, nullptr, nullptr, s));
    }
    st->nodes += nn;
    if (!compactor) {
        int over = 0;
        JV_TRY(builder_collect_over_degree(B, s));
        JV_TRY(lap_end());
        JV_TRY(builder_list_count(B, &over, s));
        JV_TRY(timer.start(s));
        st->rows_repruned += over;
        JV_TRY(builder_reprune_slice(B, 0, 0, nullptr, nullptr, s));
    }
    const long long total = (long long)n * degree;
    compact_adj_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(B->adj, B->deg, n, row_cap, degree, adj_out);
    g_launches++;
    JV_TRY(cudaGetLastError());
    if (compactor) JV_TRY(launch_scatter_rows(adj_out, degree, list, nn, out_rows, s));
    count_changed_rows_kernel<<<(n + 255) / 256, 256, 0, s>>>(adj_in, adj_out, n, degree, counts + 1);
    g_launches++;
    JV_TRY(cudaGetLastError());
    unsigned long long h[2];
    JV_TRY(cudaMemcpyAsync(h, counts, 16, cudaMemcpyDeviceToHost, s));
    JV_TRY(lap_end());
    BuildStats bs;
    JV_TRY(builder_stats(B, &bs, s));
    st->backlinks_added += (long long)h[0] - bs.dropped_backlinks;
    st->backlinks_dropped += bs.dropped_backlinks;
    st->rows_changed += (long long)h[1];
    return cudaSuccess;
}

cudaError_t refine_level(const DataDesc &d, int metric, const BuildParams &bp, int beam, bool compactor, const int32_t *adj_in_dev, int degree, int32_t entry,
                         const std::vector<int32_t> &nodes, int32_t *adj_out_dev, int sm_count, RefineStats *st, cudaStream_t s)
{
    if (degree < 1 || degree > 64 || beam < 1 || entry < 0 || entry >= d.n) return cudaErrorInvalidValue;
    GraphBuilder *B = nullptr;
    std::vector<DeviceBuffer> mem;  // the scratch goes when this returns: the stream drains first, on success and on error
    const cudaError_t err = refine_level_enqueue(d, metric, bp, beam, compactor, adj_in_dev, degree, entry, nodes, adj_out_dev, sm_count, st, &B, mem, s);
    const cudaError_t drained = cudaStreamSynchronize(s);
    delete B;
    return err != cudaSuccess ? err : drained;
}

}  // namespace jv
