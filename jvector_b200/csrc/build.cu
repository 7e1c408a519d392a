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
//   backlink: append u to adj[v] for every chosen v (atomic slot), then prune_kernel again over every v whose list
//             passed overflow * M
// Batches grow geometrically (x 33/32, JV_BUILD_BATCH_DIV) up to max_batch so early nodes see a connected graph. Neighbour lists in the
// reference are concurrency-order dependent, so parity is on scores and on the recall of the resulting graph
// (SURVEY §8d C5), not on identical adjacency.
#include <limits.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include <cub/cub.cuh>

#include "kernels.h"

namespace jv {

constexpr int PRUNE_THREADS = 256;
constexpr int PRUNE_MAXC = 256;  // candidates per prune (beam or list capacity), power of two

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

__device__ __forceinline__ void bitonic_sort_desc_prune(long long *keys, int n_pow2)
{
    for (int k = 2; k <= n_pow2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n_pow2; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const long long a = keys[i], b = keys[ixj];
                    const bool desc = (i & k) == 0;
                    if (desc ? (a < b) : (a > b)) { keys[i] = b; keys[ixj] = a; }
                }
            }
            __syncthreads();
        }
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

// retainDiverse (VamanaDiversityProvider.java:45-95), restated so that the pair scores can be produced in bulk:
//   isDiverse(c) at alpha  <=>  max over the selected s of sim(c, s)  <=  score(c) * alpha.
// Keep M[c] = that running maximum. Selecting a candidate s updates M[c] for every still-eligible c in parallel (one warp
// per candidate, the new row cached in shared memory); the sequential part of the reference loop shrinks to "find the next
// c at or after the cursor with M[c] <= score(c) * alpha", a flag scan. A candidate whose M[c] already exceeds
// score(c) * alpha_max can never be selected in any pass (M only grows) and is dropped from further updates. The selection
// sequence — and therefore the neighbour list — is exactly the reference loop's, including the alpha = 1.0, 1.2 passes.
// MAXC: candidate capacity (power of two). The builder uses PRUNE_MAXC; the repair of deleted neighbours also instantiates
// larger capacities so that no candidate set is ever clipped.
template <int METRIC, int MAXC = PRUNE_MAXC>
__global__ void __launch_bounds__(PRUNE_THREADS) prune_kernel(PruneParams P)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *blob = reinterpret_cast<float *>(smem_raw);                       // stride + 4
    float *newrow = blob + P.d.stride + 4;                                   // stride: the most recently selected row
    long long *keys = reinterpret_cast<long long *>(newrow + P.d.stride);    // MAXC
    float *maxsim = reinterpret_cast<float *>(keys + MAXC);                  // MAXC
    int32_t *sel_ids = reinterpret_cast<int32_t *>(maxsim + MAXC);           // 128
    uint8_t *state = reinterpret_cast<uint8_t *>(sel_ids + 128);             // MAXC: 0 eligible, 1 selected, 2 dropped
    __shared__ float red[36];
    __shared__ int s_next;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NW = PRUNE_THREADS / 32;
    const int total = P.count_ptr ? *P.count_ptr : P.count;
    const int n4 = P.d.stride >> 2;
    // the last alpha the reference loop reaches: 1.0, 1.2, ... while <= alpha + 1e-6
    float alpha_max = 1.0f;
    for (float a = 1.0f; a <= P.alpha + 1e-6f; a += 0.2f) alpha_max = a;

    for (int it = blockIdx.x; it < total; it += gridDim.x) {
        const int a = P.mode == 2 ? P.list[it] : 0;
        const int v = P.mode == 0 ? P.node_base + it : P.mode == 2 ? P.row_node[a] : P.list[P.list_base + it];
        const int32_t *cand;
        int nc, ncs;
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
        nc = min(nc, MAXC);
        prepare_blob(P.d, P.metric, P.d.rows + (size_t)v * P.d.stride, blob, red);
        // exact scores of the candidates against v, as sortable keys (two rows per warp at a time)
        for (int i = warp; i < MAXC; i += 2 * NW) {
            const int i2 = i + NW;
            const int32_t ca = i < nc ? prune_candidate(P, cand, ncs, v, i) : -1, cb = i2 < nc ? prune_candidate(P, cand, ncs, v, i2) : -1;
            const bool va = ca >= 0 && ca != v, vb = cb >= 0 && cb != v;
            long long ka = KEY_MIN, kb = KEY_MIN;
            if (va || vb) {
                float sa, sb;
                score_f32_pair<METRIC>(P.d, blob, va ? ca : cb, vb ? cb : ca, lane, sa, sb);
                if (va) ka = topk_key(sa, ca);
                if (vb) kb = topk_key(sb, cb);
            }
            if (lane == 0) {
                keys[i] = ka;
                if (i2 < MAXC) keys[i2] = kb;
            }
        }
        __syncthreads();
        bitonic_sort_desc_prune(keys, MAXC);
        // valid keys form a prefix (KEY_MIN sorts last); duplicates are adjacent after the sort and are dropped
        int nvalid;
        {
            int lo = 0, hi = MAXC;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (keys[mid] != KEY_MIN) lo = mid + 1;
                else hi = mid;
            }
            nvalid = lo;
        }
        for (int i = tid; i < MAXC; i += PRUNE_THREADS) {
            maxsim[i] = -3.0e38f;
            state[i] = (i < nvalid && !(i > 0 && keys[i - 1] == keys[i])) ? 0 : 2;
        }
        __syncthreads();

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
                if (tid == 0) { state[pick] = 1; sel_ids[nsel] = c; }
                for (int t = tid; t < n4; t += PRUNE_THREADS) reinterpret_cast<float4 *>(newrow)[t] = __ldg(crow + t);
                nsel++;
                cursor = pick + 1;
                __syncthreads();
                if (nsel >= P.degree) break;
                // fold the new neighbour into every still-eligible candidate's running maximum
                for (int i = warp; i < nvalid; i += NW) {
                    if (state[i] != 0) continue;
                    const float4 *row = reinterpret_cast<const float4 *>(P.d.rows + (size_t)key_node(keys[i]) * P.d.stride);
                    const float ps = pair_rows<METRIC>(row, reinterpret_cast<const float4 *>(newrow), n4, lane);
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
        // the selected neighbours, in score order (NodeArray.retain keeps the sorted order)
        __syncthreads();
        if (tid == 0) {
            int w = 0;
            const int oi = P.mode == 2 ? a : P.out_base + it;
            int32_t *row = P.out_rows ? P.out_rows + (size_t)oi * P.out_stride : P.adj + (size_t)v * P.row_cap;
            const int width = P.out_rows ? P.out_stride : P.row_cap;
            for (int i = 0; i < nvalid; i++)
                if (state[i] == 1) row[w++] = key_node(keys[i]);
            for (int i = w; i < width; i++) row[i] = -1;
            if (P.out_rows) P.out_deg[oi] = w;
            else P.deg[v] = w;
            if (P.mode == 1 && P.mark) P.mark[v] = 0;
        }
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
    constexpr int NW = PRUNE_THREADS / 32;
    const int total = P.count_ptr ? *P.count_ptr : P.count;
    float alpha_max = 1.0f;
    for (float a = 1.0f; a <= P.alpha + 1e-6f; a += 0.2f) alpha_max = a;

    for (int it = blockIdx.x; it < total; it += gridDim.x) {
        const int a = P.mode == 2 ? P.list[it] : 0;
        const int v = P.mode == 0 ? P.node_base + it : P.mode == 2 ? P.row_node[a] : P.list[P.list_base + it];
        const int32_t *cand;
        int nc, ncs;
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
        nc = min(nc, TILE);
        prepare_blob(P.d, P.metric, P.d.rows + (size_t)v * P.d.stride, blob, red);
        for (int i = warp; i < TILE; i += 2 * NW) {
            const int i2 = i + NW;
            const int32_t ca = i < nc ? prune_candidate(P, cand, ncs, v, i) : -1, cb = (i2 < TILE && i2 < nc) ? prune_candidate(P, cand, ncs, v, i2) : -1;
            const bool va = ca >= 0 && ca != v, vb = cb >= 0 && cb != v;
            long long ka = KEY_MIN, kb = KEY_MIN;
            if (va || vb) {
                float sa, sb;
                score_f32_pair<METRIC>(P.d, blob, va ? ca : cb, vb ? cb : ca, lane, sa, sb);
                if (va) ka = topk_key(sa, ca);
                if (vb) kb = topk_key(sb, cb);
            }
            if (lane == 0) {
                keys[i] = ka;
                if (i2 < TILE) keys[i2] = kb;
            }
        }
        __syncthreads();
        bitonic_sort_desc_prune(keys, TILE);
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

        // ---- Gram matrix of the candidate rows ----
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
                if (node >= 0 && k0 + 4 * c4 < P.d.stride) val = __ldg(reinterpret_cast<const float4 *>(P.d.rows + (size_t)node * P.d.stride + k0) + c4);
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
        if (METRIC != JV_METRIC_DOT) {
            float diag_r[NB], diag_c[NB];
#pragma unroll
            for (int a = 0; a < NB; a++) diag_r[a] = C[(ty + 16 * a) * CP + ty + 16 * a];
#pragma unroll
            for (int b = 0; b < NB; b++) diag_c[b] = C[(tx + 16 * b) * CP + tx + 16 * b];
            __syncthreads();
#pragma unroll
            for (int a = 0; a < NB; a++)
#pragma unroll
                for (int b = 0; b < NB; b++) {
                    float raw;
                    if (METRIC == JV_METRIC_EUCLIDEAN) raw = fmaxf(0.f, __fadd_rn(__fadd_rn(diag_r[a], diag_c[b]), -2.0f * acc[a][b]));
                    else raw = __fdiv_rn(acc[a][b], __fsqrt_rn(__fmul_rn(diag_r[a], diag_c[b])));
                    C[(ty + 16 * a) * CP + tx + 16 * b] = score_map(METRIC, raw);
                }
        } else {
#pragma unroll
            for (int a = 0; a < NB; a++)
#pragma unroll
                for (int b = 0; b < NB; b++) C[(ty + 16 * a) * CP + tx + 16 * b] = score_map(METRIC, acc[a][b]);
        }
        __syncthreads();

        // ---- the sequential selection, now over shared memory only ----
        int nsel = 0;
        float currentAlpha = 1.0f;
        while (currentAlpha <= P.alpha + 1e-6f && nsel < P.degree) {
            int cursor = 0;
            while (nsel < P.degree) {
                if (tid == 0) s_next = INT_MAX;
                __syncthreads();
                for (int i = cursor + tid; i < nvalid; i += PRUNE_THREADS)
                    if (state[i] == 0 && !(maxsim[i] > __fmul_rn(key_score(keys[i]), currentAlpha))) { atomicMin(&s_next, i); break; }
                __syncthreads();
                const int pick = s_next;
                if (pick == INT_MAX) break;
                nsel++;
                cursor = pick + 1;
                for (int i = tid; i < nvalid; i += PRUNE_THREADS) {
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
        __syncthreads();
        if (tid == 0) {
            int w = 0;
            const int oi = P.mode == 2 ? a : P.out_base + it;
            int32_t *row = P.out_rows ? P.out_rows + (size_t)oi * P.out_stride : P.adj + (size_t)v * P.row_cap;
            const int width = P.out_rows ? P.out_stride : P.row_cap;
            for (int i = 0; i < nvalid; i++)
                if (state[i] == 1) row[w++] = ids[i];
            for (int i = w; i < width; i++) row[i] = -1;
            if (P.out_rows) P.out_deg[oi] = w;
            else P.deg[v] = w;
            if (P.mode == 1 && P.mark) P.mark[v] = 0;
        }
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
__device__ __forceinline__ uint64_t desc_sw128(uint32_t smem_addr)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3ffff) >> 4);  // start address
    d |= (uint64_t)1 << 16;                       // leading byte offset (unused by swizzled K-major layouts)
    d |= (uint64_t)(1024 >> 4) << 32;             // stride byte offset: 8-row atoms 1024 B apart
    d |= (uint64_t)1 << 62;                       // SWIZZLE_128B
    return d;
}
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
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
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
    constexpr int NW = PRUNE_THREADS / 32;
    const int total = P.count_ptr ? *P.count_ptr : P.count;
    float alpha_max = 1.0f;
    for (float a = 1.0f; a <= P.alpha + 1e-6f; a += 0.2f) alpha_max = a;

    // warpgroup wg computes columns [wg N, wg N + N) of every 64-row block of the Gram matrix
    constexpr int N = TILE / 2, MB = TILE / 64, R = N / 2;
    const int wg = warp >> 2;
    float acc[MB][R];
    const int nchunks = (P.d.stride + 31) / 32;
    const int c4 = tid & 7, r0 = tid >> 3;

    for (int it = blockIdx.x; it < total; it += gridDim.x) {
        const int a = P.mode == 2 ? P.list[it] : 0;
        const int v = P.mode == 0 ? P.node_base + it : P.mode == 2 ? P.row_node[a] : P.list[P.list_base + it];
        const int32_t *cand;
        int nc, ncs;
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
        nc = min(nc, TILE);
        prepare_blob(P.d, P.metric, P.d.rows + (size_t)v * P.d.stride, blob, red);
        for (int i = warp; i < TILE; i += 2 * NW) {
            const int i2 = i + NW;
            const int32_t ca = i < nc ? prune_candidate(P, cand, ncs, v, i) : -1, cb = (i2 < TILE && i2 < nc) ? prune_candidate(P, cand, ncs, v, i2) : -1;
            const bool va = ca >= 0 && ca != v, vb = cb >= 0 && cb != v;
            long long ka = KEY_MIN, kb = KEY_MIN;
            if (va || vb) {
                float sa, sb;
                score_f32_pair<METRIC>(P.d, blob, va ? ca : cb, vb ? cb : ca, lane, sa, sb);
                if (va) ka = topk_key(sa, ca);
                if (vb) kb = topk_key(sb, cb);
            }
            if (lane == 0) {
                keys[i] = ka;
                if (i2 < TILE) keys[i2] = kb;
            }
        }
        __syncthreads();
        bitonic_sort_desc_prune(keys, TILE);
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

        // ---- Gram matrix of the candidate rows on the tensor cores (3xTF32) ----
        const float *rowp[PASSES];
#pragma unroll
        for (int j = 0; j < PASSES; j++) {
            const int32_t node = ids[r0 + 32 * j];
            rowp[j] = node >= 0 ? P.d.rows + (size_t)node * P.d.stride + 4 * c4 : nullptr;
        }
        float4 pre[PASSES];
#pragma unroll
        for (int j = 0; j < PASSES; j++) pre[j] = (rowp[j] && 4 * c4 < P.d.stride) ? __ldg(reinterpret_cast<const float4 *>(rowp[j])) : make_float4(0.f, 0.f, 0.f, 0.f);
        for (int c = 0; c < nchunks; c++) {
            const int b = c & 1;
            if (c >= 2) {  // the MMAs of chunk c - 2 (both warpgroups) have read this buffer
                asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
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
                    pre[j] = (rowp[j] && k1 < P.d.stride) ? __ldg(reinterpret_cast<const float4 *>(rowp[j] + (c + 1) * 32)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            {
                const uint32_t ah = smem_u32(hi_t), al = smem_u32(lo_t);
#pragma unroll
                for (int mb = 0; mb < MB; mb++) tc::acc_fence(acc[mb]);
                asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
                for (int ks = 0; ks < 4; ks++) {
                    const uint64_t bh = tc::desc_sw128(ah + wg * (N / 8) * 1024 + 32 * ks), bl = tc::desc_sw128(al + wg * (N / 8) * 1024 + 32 * ks);
#pragma unroll
                    for (int mb = 0; mb < MB; mb++) {
                        const uint64_t dh = tc::desc_sw128(ah + mb * 8 * 1024 + 32 * ks), dl = tc::desc_sw128(al + mb * 8 * 1024 + 32 * ks);
                        tc::mma_tf32<N>(acc[mb], dh, bh, (c | ks) != 0 ? 1u : 0u);
                        tc::mma_tf32<N>(acc[mb], dh, bl, 1u);
                        tc::mma_tf32<N>(acc[mb], dl, bh, 1u);
                    }
                }
                asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            }
        }
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
        for (int mb = 0; mb < MB; mb++) tc::acc_fence(acc[mb]);
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
            const float dotv = C[i * CP + j];
            float raw;
            if (METRIC == JV_METRIC_EUCLIDEAN) raw = fmaxf(0.f, __fadd_rn(__fadd_rn(diag[i], diag[j]), -2.0f * dotv));
            else if (METRIC == JV_METRIC_COSINE) raw = __fdiv_rn(dotv, __fsqrt_rn(__fmul_rn(diag[i], diag[j])));
            else raw = dotv;
            C[i * CP + j] = score_map(METRIC, raw);
        }
        __syncthreads();

        // ---- the sequential selection, over shared memory only ----
        int nsel = 0;
        float currentAlpha = 1.0f;
        while (currentAlpha <= P.alpha + 1e-6f && nsel < P.degree) {
            int cursor = 0;
            while (nsel < P.degree) {
                if (tid == 0) s_next = INT_MAX;
                __syncthreads();
                for (int i = cursor + tid; i < nvalid; i += PRUNE_THREADS)
                    if (state[i] == 0 && !(maxsim[i] > __fmul_rn(key_score(keys[i]), currentAlpha))) { atomicMin(&s_next, i); break; }
                __syncthreads();
                const int pick = s_next;
                if (pick == INT_MAX) break;
                nsel++;
                cursor = pick + 1;
                for (int i = tid; i < nvalid; i += PRUNE_THREADS) {
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
        __syncthreads();
        if (tid == 0) {
            int w = 0;
            const int oi = P.mode == 2 ? a : P.out_base + it;
            int32_t *row = P.out_rows ? P.out_rows + (size_t)oi * P.out_stride : P.adj + (size_t)v * P.row_cap;
            const int width = P.out_rows ? P.out_stride : P.row_cap;
            for (int i = 0; i < nvalid; i++)
                if (state[i] == 1) row[w++] = ids[i];
            for (int i = w; i < width; i++) row[i] = -1;
            if (P.out_rows) P.out_deg[oi] = w;
            else P.deg[v] = w;
            if (P.mode == 1 && P.mark) P.mark[v] = 0;
        }
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
__global__ void __launch_bounds__(256) apply_rows_kernel(int32_t *adj, int *deg, int row_cap, int degree, int first, int count, const int32_t *rows,
                                                         const int *rdeg, unsigned long long *pairs)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= count * row_cap) return;
    const int i = idx / row_cap, j = idx - i * row_cap;
    const int u = first + i;
    const int32_t t = j < degree ? rows[(size_t)i * degree + j] : -1;
    adj[(size_t)u * row_cap + j] = t;
    if (j == 0) deg[u] = rdeg[i];
    if (j < degree) {
        bool link = t >= 0;
        if (link && t >= first && t < first + count) {
            // t was inserted in this very batch and may have chosen u itself (both sit in each other's in-progress window): then u is
            // already in t's row and the back-link would duplicate it (NodeArray.insertSorted refuses duplicates)
            const int32_t *trow = rows + (size_t)(t - first) * degree;
            for (int x = 0; x < degree; x++)
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

__global__ void __launch_bounds__(256) compact_adj_kernel(const int32_t *adj, const int *deg, int n, int row_cap, int degree, int32_t *out)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n * degree) return;
    const int v = (int)(idx / degree), j = (int)(idx % degree);
    out[idx] = j < min(deg[v], degree) ? adj[(size_t)v * row_cap + j] : -1;
}

// rows [ids[i]] of a data set gathered into a dense one (upper levels of the hierarchy, repair pass): one warp per row
__global__ void __launch_bounds__(256) gather_rows_kernel(const float *__restrict__ rows, int stride, const int32_t *__restrict__ ids, int count, float *__restrict__ out)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= count) return;
    const float4 *src = reinterpret_cast<const float4 *>(rows + (size_t)ids[warp] * stride);
    float4 *dst = reinterpret_cast<float4 *>(out + (size_t)warp * stride);
    for (int i = lane; i < (stride >> 2); i += 32) dst[i] = ldg_stream(src + i);
}

cudaError_t launch_gather_rows(const DataDesc &f32, const int32_t *ids_dev, int count, float *out_dev, cudaStream_t s)
{
    if (count <= 0) return cudaSuccess;
    const long long blocks = ((long long)count * 32 + 255) / 256;
    gather_rows_kernel<<<(unsigned)blocks, 256, 0, s>>>(f32.rows, f32.stride, ids_dev, count, out_dev);
    g_launches++;
    return cudaGetLastError();
}

static size_t prune_smem_bytes(const DataDesc &d, int maxc = PRUNE_MAXC)
{
    size_t b = (size_t)(d.stride + 4) * 4 + (size_t)d.stride * 4 + (size_t)maxc * 8 + (size_t)maxc * 4 + 128 * 4 + maxc;
    return (b + 15) & ~(size_t)15;
}

template <int METRIC>
static cudaError_t launch_prune_t(const PruneParams &P, int grid, size_t smem, cudaStream_t s)
{
    // candidate sets that fit a tile go through the Gram-matrix kernel; anything larger keeps the incremental kernel
    const int ncmax = P.mode == 0 ? P.cand_stride + P.window : P.row_cap;
    cudaError_t e;
    // Gram products on the tensor cores (wgmma, 3xTF32) unless JV_PRUNE_GRAM=ffma asks for the CUDA-core kernel
    static const bool use_tc = !(getenv("JV_PRUNE_GRAM") && getenv("JV_PRUNE_GRAM")[0] == 'f');
    if (ncmax <= 64 && use_tc) {
        const size_t gs = gram_tc_smem_bytes<64>(P.d);
        if ((e = cudaFuncSetAttribute(prune_gram_tc_kernel<METRIC, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gs)) != cudaSuccess) return e;
        prune_gram_tc_kernel<METRIC, 64><<<grid, PRUNE_THREADS, gs, s>>>(P);
    } else if (ncmax <= 128 && use_tc) {
        const size_t gs = gram_tc_smem_bytes<128>(P.d);
        if ((e = cudaFuncSetAttribute(prune_gram_tc_kernel<METRIC, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gs)) != cudaSuccess) return e;
        prune_gram_tc_kernel<METRIC, 128><<<grid, PRUNE_THREADS, gs, s>>>(P);
    } else if (ncmax <= 64) {
        const size_t gs = gram_smem_bytes<64>(P.d);
        if ((e = cudaFuncSetAttribute(prune_gram_kernel<METRIC, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gs)) != cudaSuccess) return e;
        prune_gram_kernel<METRIC, 64><<<grid, PRUNE_THREADS, gs, s>>>(P);
    } else if (ncmax <= 128) {
        const size_t gs = gram_smem_bytes<128>(P.d);
        if ((e = cudaFuncSetAttribute(prune_gram_kernel<METRIC, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gs)) != cudaSuccess) return e;
        prune_gram_kernel<METRIC, 128><<<grid, PRUNE_THREADS, gs, s>>>(P);
    } else {
        if ((e = cudaFuncSetAttribute(prune_kernel<METRIC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
        prune_kernel<METRIC><<<grid, PRUNE_THREADS, smem, s>>>(P);
    }
    g_launches++;
    return cudaGetLastError();
}

static cudaError_t launch_prune(const PruneParams &P, int grid, size_t smem, cudaStream_t s)
{
    if (P.metric == JV_METRIC_EUCLIDEAN) return launch_prune_t<JV_METRIC_EUCLIDEAN>(P, grid, smem, s);
    if (P.metric == JV_METRIC_DOT) return launch_prune_t<JV_METRIC_DOT>(P, grid, smem, s);
    return launch_prune_t<JV_METRIC_COSINE>(P, grid, smem, s);
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
    int inserted = 1;  // node 0 is the entry point with an empty list
    int32_t *adj = nullptr, *res_nodes = nullptr, *list = nullptr, *head_target = nullptr, *iota = nullptr;
    int *deg = nullptr, *mark = nullptr, *list_count = nullptr, *work_counter = nullptr;
    float *res_scores = nullptr;
    unsigned long long *dropped = nullptr, *pairs = nullptr, *pairs_sorted = nullptr;
    unsigned char *head_flag = nullptr, *node_flag = nullptr;
    SearchCounters *counters = nullptr;
    uint8_t *overflow = nullptr;
    void *scratch = nullptr, *cub_tmp = nullptr;
    size_t scratch_bytes = 0, cub_bytes = 0;
    int32_t *own_rows = nullptr;  // single-GPU path: the slice buffers are the builder's own
    int *own_deg = nullptr;
    int32_t *own_rp_rows = nullptr;
    int *own_rp_deg = nullptr;
    size_t own_rp_cap = 0;
    BuildStats st = {0, 0, 0, 0, 0};
    size_t psmem = 0;
    int prune_grid = 0;
};

static void builder_free(GraphBuilder *B)
{
    if (!B) return;
    cudaFree(B->adj); cudaFree(B->res_nodes); cudaFree(B->list); cudaFree(B->head_target); cudaFree(B->iota); cudaFree(B->deg); cudaFree(B->mark);
    cudaFree(B->list_count); cudaFree(B->work_counter); cudaFree(B->res_scores); cudaFree(B->dropped); cudaFree(B->pairs); cudaFree(B->pairs_sorted);
    cudaFree(B->head_flag); cudaFree(B->node_flag); cudaFree(B->counters); cudaFree(B->overflow); cudaFree(B->scratch); cudaFree(B->cub_tmp);
    cudaFree(B->own_rows); cudaFree(B->own_deg); cudaFree(B->own_rp_rows); cudaFree(B->own_rp_deg);
    delete B;
}

void builder_destroy(GraphBuilder *B) { builder_free(B); }

cudaError_t builder_create(const DataDesc &d, int metric, const BuildParams &bp, int sm_count, GraphBuilder **out, cudaStream_t s)
{
    const int n = (int)d.n;
    if (d.kind != KIND_F32 || bp.degree < 1 || bp.degree > 64 || bp.beam < 1 || bp.beam > PRUNE_MAXC) return cudaErrorInvalidValue;
    GraphBuilder *B = new GraphBuilder();
    B->d = d; B->metric = metric; B->bp = bp; B->sm_count = sm_count; B->n = n; B->degree = bp.degree; B->beam = bp.beam;
    B->hard_max = (int)(bp.overflow * bp.degree);  // ConcurrentNeighborMap.java:300
    B->row_cap = std::max(2 * bp.degree, B->hard_max + 1);
    if (B->row_cap > MAX_DEGREE) { delete B; return cudaErrorInvalidValue; }
    B->max_batch = bp.max_batch > 0 ? bp.max_batch : 16384;
    if (const char *e = getenv("JV_BUILD_BATCH_DIV")) B->batch_div = atoi(e) > 0 ? atoi(e) : 32;  // tuning knob (tools/build_quality.py)
    // in-progress window: as many concurrently inserting peers as still fit the 128-candidate Gram tile next to the beam
    B->window = bp.window >= 0 ? bp.window : std::max(0, std::min(32, 128 - bp.beam));
    B->psmem = prune_smem_bytes(d);
    B->prune_grid = sm_count * 5;  // ~10 KB of shared memory per CTA: register-limited residency
    cudaError_t err = cudaSuccess;
    const size_t mb = (size_t)B->max_batch;
#define ALLOC(ptr, bytes)                                                  \
    do {                                                                   \
        err = cudaMalloc((void **)&(ptr), (bytes));                        \
        if (err != cudaSuccess) { builder_free(B); return err; }           \
    } while (0)
    ALLOC(B->adj, (size_t)n * B->row_cap * 4);
    ALLOC(B->deg, (size_t)n * 4);
    ALLOC(B->mark, (size_t)n * 4);
    ALLOC(B->res_nodes, mb * B->beam * 4);
    ALLOC(B->res_scores, mb * B->beam * 4);
    ALLOC(B->list, (size_t)n * 4);
    ALLOC(B->iota, (size_t)n * 4);
    ALLOC(B->node_flag, (size_t)n);
    ALLOC(B->list_count, 16);
    ALLOC(B->work_counter, 16);
    ALLOC(B->dropped, 16);
    ALLOC(B->counters, sizeof(SearchCounters));
    ALLOC(B->overflow, mb);
    ALLOC(B->pairs, mb * B->degree * 8);
    ALLOC(B->pairs_sorted, mb * B->degree * 8);
    ALLOC(B->head_flag, mb * B->degree);
    ALLOC(B->head_target, mb * B->degree * 4);
    ALLOC(B->own_rows, mb * B->degree * 4);
    ALLOC(B->own_deg, mb * 4);
#undef ALLOC
    {
        size_t b1 = 0, b2 = 0;
        cub::DeviceRadixSort::SortKeys(nullptr, b1, B->pairs, B->pairs_sorted, (int)(mb * B->degree), 0, 64, s);
        cub::DeviceSelect::Flagged(nullptr, b2, B->iota, B->node_flag, B->list, B->list_count, n, s);
        B->cub_bytes = std::max(b1, b2) + 256;
        err = cudaMalloc(&B->cub_tmp, B->cub_bytes);
        if (err != cudaSuccess) { builder_free(B); return err; }
    }
    JV_TRY(cudaMemsetAsync(B->adj, 0xff, (size_t)n * B->row_cap * 4, s));
    JV_TRY(cudaMemsetAsync(B->deg, 0, (size_t)n * 4, s));
    JV_TRY(cudaMemsetAsync(B->mark, 0, (size_t)n * 4, s));
    JV_TRY(cudaMemsetAsync(B->dropped, 0, 16, s));
    JV_TRY(cudaMemsetAsync(B->list_count, 0, 16, s));
    JV_TRY(cudaMemsetAsync(B->counters, 0, sizeof(SearchCounters), s));
    iota_kernel<<<(n + 255) / 256, 256, 0, s>>>(B->iota, n);
    g_launches++;
    *out = B;
    return cudaGetLastError();
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
    g.n = B->n; g.degree = B->row_cap; g.levels = 1; g.entry_node = 0; g.entry_level = 0; g.adj0 = B->adj;
    SearchPlan plan;
    JV_TRY(plan_search(B->d, nullptr, g, B->beam, B->beam, m, 0, 0, B->sm_count, &plan));
    const size_t need = search_scratch_bytes(plan);
    if (need > B->scratch_bytes) {
        if (B->scratch) cudaFree(B->scratch);
        B->scratch = nullptr;
        B->scratch_bytes = 0;
        JV_TRY(cudaMalloc(&B->scratch, need));
        B->scratch_bytes = need;
    }
    SearchFilter lenient;
    memset(&lenient, 0, sizeof(lenient));
    lenient.lenient = 1;  // an insert search never fails the build: see SearchParams::lenient
    JV_TRY(launch_search(g, B->d, nullptr, B->metric, B->d.rows + (size_t)(first + lo) * B->d.stride, m, B->beam, B->beam, plan, B->scratch, B->work_counter,
                         B->res_nodes, B->res_scores, B->counters, B->overflow, nullptr, B->d.stride, &lenient, s));
    PruneParams P = prune_params(B);
    P.mode = 0; P.node_base = first + lo; P.count = m; P.cand = B->res_nodes; P.cand_stride = B->beam;
    P.window = B->window; P.batch_first = first; P.batch_count = count;
    P.out_rows = rows_out; P.out_deg = deg_out; P.out_stride = B->degree; P.out_base = lo;
    JV_TRY(launch_prune(P, m < B->prune_grid ? m : B->prune_grid, B->psmem, s));
    return cudaSuccess;
}

// the whole batch's rows (this rank's own slice + the gathered ones): write them, back-link them deterministically, and leave
// the SORTED list of rows that passed overflow * M in B->list (count in B->list_count[0])
cudaError_t builder_apply_new(GraphBuilder *B, int first, int count, const int32_t *rows, const int *rdeg, cudaStream_t s)
{
    cudaError_t err = cudaSuccess;
    if (!rows) { rows = B->own_rows; rdeg = B->own_deg; }
    const int npairs = count * B->degree;
    apply_rows_kernel<<<(count * B->row_cap + 255) / 256, 256, 0, s>>>(B->adj, B->deg, B->row_cap, B->degree, first, count, rows, rdeg, B->pairs);
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
    B->inserted = first + count;
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
        return launch_prune(P, B->prune_grid, B->psmem, s);
    }
    if (hi <= lo) return cudaSuccess;
    P.count = hi - lo; P.list_base = lo; P.out_rows = rows_out; P.out_deg = deg_out; P.out_stride = B->row_cap; P.out_base = lo;
    return launch_prune(P, std::min(hi - lo, B->prune_grid), B->psmem, s);
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

cudaError_t builder_finish(GraphBuilder *B, int32_t *adj_out_dev, BuildStats *stats, cudaStream_t s)
{
    cudaError_t err = cudaSuccess;
    const long long total = (long long)B->n * B->degree;
    compact_adj_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(B->adj, B->deg, B->n, B->row_cap, B->degree, adj_out_dev);
    g_launches++;
    JV_TRY(cudaGetLastError());
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

int builder_row_cap(const GraphBuilder *B) { return B->row_cap; }
int builder_degree(const GraphBuilder *B) { return B->degree; }
int builder_max_batch(const GraphBuilder *B) { return B->max_batch; }

// the whole build on one GPU: no exchange, no host synchronisation between batches
cudaError_t build_graph_flat(const DataDesc &d, int metric, const BuildParams &bp, int32_t *adj_out_dev, int sm_count,
                             BuildStats *stats, cudaStream_t s)
{
    GraphBuilder *B = nullptr;
    cudaError_t err = builder_create(d, metric, bp, sm_count, &B, s);
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
    builder_free(B);
    return err;
}

// ------------------------------------------------------------------------------------------------
// Repair of deleted neighbours (GraphIndexBuilder.removeDeletedNodes, base:graph/GraphIndexBuilder.java:689-799), one level at a time:
//   count  : one warp per row flags the live rows that name a deleted node and sizes their candidate segment
//   gather : one CTA per flagged row writes its live neighbours, the live 2-hop ids through its deleted neighbours (the FreshDiskANN
//            rule, :705-721) — or, when there are no such ids, random live members of the level (:743-759) — sorted and deduplicated
//   prune  : the builder's prune kernels (mode 2, ragged candidates, out of place), dispatched by candidate count so no set is clipped
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

// the counter-based generator of the random fallback: a pure function of (seed, level, node, attempt)
__host__ __device__ __forceinline__ uint64_t repair_mix(uint64_t x)
{
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
__host__ __device__ __forceinline__ uint64_t repair_random(uint64_t seed, int level, int node, int attempt)
{
    return repair_mix(repair_mix(repair_mix(seed ^ (uint64_t)(uint32_t)level) ^ (uint64_t)(uint32_t)node) ^ (uint64_t)(uint32_t)attempt);
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
                const int32_t k = members[repair_random(seed, level, v, at) % (uint64_t)nmembers];
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

template <int METRIC>
static cudaError_t launch_repair_prune_t(const PruneParams &P, int tier, int grid, cudaStream_t s)
{
    cudaError_t e;
#define JV_PRUNE_LAUNCH(KERNEL, SMEM)                                                                                   \
    do {                                                                                                                \
        const size_t sm_ = (SMEM);                                                                                      \
        if ((e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_)) != cudaSuccess) return e; \
        KERNEL<<<grid, PRUNE_THREADS, sm_, s>>>(P);                                                                     \
    } while (0)
    switch (tier) {
    case 0: JV_PRUNE_LAUNCH((prune_gram_tc_kernel<METRIC, 64>), gram_tc_smem_bytes<64>(P.d)); break;
    case 1: JV_PRUNE_LAUNCH((prune_gram_tc_kernel<METRIC, 128>), gram_tc_smem_bytes<128>(P.d)); break;
    case 2: JV_PRUNE_LAUNCH((prune_kernel<METRIC, 256>), prune_smem_bytes(P.d, 256)); break;
    case 3: JV_PRUNE_LAUNCH((prune_kernel<METRIC, 1024>), prune_smem_bytes(P.d, 1024)); break;
    default: JV_PRUNE_LAUNCH((prune_kernel<METRIC, 8192>), prune_smem_bytes(P.d, 8192)); break;
    }
#undef JV_PRUNE_LAUNCH
    g_launches++;
    return cudaGetLastError();
}

static cudaError_t launch_repair_prune(const PruneParams &P, int tier, int grid, cudaStream_t s)
{
    if (P.metric == JV_METRIC_EUCLIDEAN) return launch_repair_prune_t<JV_METRIC_EUCLIDEAN>(P, tier, grid, s);
    if (P.metric == JV_METRIC_DOT) return launch_repair_prune_t<JV_METRIC_DOT>(P, tier, grid, s);
    return launch_repair_prune_t<JV_METRIC_COSINE>(P, tier, grid, s);
}

cudaError_t repair_level(const DataDesc &d, int metric, float alpha, int degree, int rows, const int32_t *adj_old, int32_t *adj_new, const int32_t *ids_dev,
                         const int32_t *rowmap_dev, const uint32_t *dead_dev, const int32_t *members_dev, int nmembers, uint64_t seed, int level,
                         int sm_count, RepairStats *st, cudaStream_t s)
{
    cudaError_t err = cudaSuccess;
    if (rows <= 0) return cudaSuccess;
    if (degree < 1 || degree > 64) return cudaErrorInvalidValue;
    unsigned char *flag = nullptr, *fallback = nullptr;
    long long *cnt = nullptr, *off_all = nullptr, *cand_off = nullptr;
    int32_t *iota = nullptr, *aff = nullptr, *cand = nullptr, *row_node = nullptr, *out_rows = nullptr, *tier_list = nullptr;
    int *naff_dev = nullptr, *cand_cnt = nullptr, *out_deg = nullptr;
    void *tmp = nullptr;
    int naff = 0;
    long long total = 0;
    std::vector<int> hcnt;
    std::vector<unsigned char> hfb;
    std::vector<int32_t> tiers[REPAIR_TIERS];
    std::vector<int32_t> hlist;
    size_t tb = 0, t1 = 0, t2 = 0;
#define R_TRY(x)                                 \
    do {                                         \
        err = (x);                               \
        if (err != cudaSuccess) goto done;       \
    } while (0)
    R_TRY(cudaMalloc(&flag, (size_t)rows));
    R_TRY(cudaMalloc(&cnt, (size_t)rows * 8));
    R_TRY(cudaMalloc(&off_all, (size_t)rows * 8));
    R_TRY(cudaMalloc(&iota, (size_t)rows * 4));
    R_TRY(cudaMalloc(&aff, (size_t)rows * 4));
    R_TRY(cudaMalloc(&naff_dev, 16));
    repair_count_kernel<<<(unsigned)(((long long)rows * 32 + 255) / 256), 256, 0, s>>>(adj_old, rows, degree, ids_dev, rowmap_dev, dead_dev, flag, cnt);
    g_launches++;
    iota_kernel<<<(rows + 255) / 256, 256, 0, s>>>(iota, rows);
    g_launches++;
    R_TRY(cudaGetLastError());
    cub::DeviceScan::ExclusiveSum(nullptr, t1, cnt, off_all, rows, s);
    cub::DeviceSelect::Flagged(nullptr, t2, iota, flag, aff, naff_dev, rows, s);
    tb = std::max(t1, t2) + 256;
    R_TRY(cudaMalloc(&tmp, tb));
    t1 = tb;
    R_TRY(cub::DeviceScan::ExclusiveSum(tmp, t1, cnt, off_all, rows, s));
    g_launches++;
    t2 = tb;
    R_TRY(cub::DeviceSelect::Flagged(tmp, t2, iota, flag, aff, naff_dev, rows, s));
    g_launches++;
    {
        long long last[2] = {0, 0};
        R_TRY(cudaMemcpyAsync(&naff, naff_dev, sizeof(int), cudaMemcpyDeviceToHost, s));
        R_TRY(cudaMemcpyAsync(&last[0], off_all + rows - 1, 8, cudaMemcpyDeviceToHost, s));
        R_TRY(cudaMemcpyAsync(&last[1], cnt + rows - 1, 8, cudaMemcpyDeviceToHost, s));
        R_TRY(cudaStreamSynchronize(s));
        total = last[0] + last[1];
    }
    if (naff == 0) goto done;
    R_TRY(cudaMalloc(&cand, (size_t)std::max(total, 1ll) * 4));
    R_TRY(cudaMalloc(&row_node, (size_t)naff * 4));
    R_TRY(cudaMalloc(&cand_off, (size_t)naff * 8));
    R_TRY(cudaMalloc(&cand_cnt, (size_t)naff * 4));
    R_TRY(cudaMalloc(&fallback, (size_t)naff));
    R_TRY(cudaMalloc(&out_rows, (size_t)naff * degree * 4));
    R_TRY(cudaMalloc(&out_deg, (size_t)naff * 4));
    R_TRY(cudaMalloc(&tier_list, (size_t)naff * 4));
    {
        int cap = 256;
        while (cap < degree * (degree + 2)) cap <<= 1;
        const size_t gsm = (size_t)cap * 4;
        R_TRY(cudaFuncSetAttribute(repair_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gsm));
        repair_gather_kernel<<<std::min(naff, sm_count * 8), 256, gsm, s>>>(adj_old, degree, ids_dev, rowmap_dev, dead_dev, aff, naff, off_all, cap, members_dev,
                                                                           nmembers, (unsigned long long)seed, level, cand, row_node, cand_off, cand_cnt, fallback);
        g_launches++;
        R_TRY(cudaGetLastError());
    }
    hcnt.resize(naff);
    hfb.resize(naff);
    R_TRY(cudaMemcpyAsync(hcnt.data(), cand_cnt, (size_t)naff * 4, cudaMemcpyDeviceToHost, s));
    R_TRY(cudaMemcpyAsync(hfb.data(), fallback, (size_t)naff, cudaMemcpyDeviceToHost, s));
    R_TRY(cudaStreamSynchronize(s));
    for (int a = 0; a < naff; a++) {
        int t = 0;
        while (t < REPAIR_TIERS - 1 && hcnt[a] > REPAIR_TIER_MAX[t]) t++;
        tiers[t].push_back(a);
        st->candidates += hcnt[a];
        st->max_candidates = std::max(st->max_candidates, hcnt[a]);
        st->random_fallbacks += hfb[a];
        st->tier_rows[t]++;
    }
    st->repaired_rows += naff;
    for (int t = 0; t < REPAIR_TIERS; t++) hlist.insert(hlist.end(), tiers[t].begin(), tiers[t].end());
    R_TRY(cudaMemcpyAsync(tier_list, hlist.data(), (size_t)naff * 4, cudaMemcpyHostToDevice, s));
    {
        PruneParams P;
        memset(&P, 0, sizeof(P));
        P.d = d; P.metric = metric; P.degree = degree; P.row_cap = degree; P.alpha = alpha; P.mode = 2;
        P.cand = cand; P.row_node = row_node; P.cand_off = cand_off; P.cand_cnt = cand_cnt;
        P.out_rows = out_rows; P.out_deg = out_deg; P.out_stride = degree;
        int first = 0;
        for (int t = 0; t < REPAIR_TIERS; t++) {
            const int c = (int)tiers[t].size();
            if (c == 0) continue;
            P.list = tier_list + first;
            P.count = c;
            R_TRY(launch_repair_prune(P, t, std::min(c, sm_count * 5), s));
            first += c;
        }
    }
    repair_scatter_kernel<<<(unsigned)(((long long)naff * degree + 255) / 256), 256, 0, s>>>(adj_new, degree, aff, naff, out_rows);
    g_launches++;
    R_TRY(cudaGetLastError());
    R_TRY(cudaStreamSynchronize(s));  // the scratch below is freed on return
done:
#undef R_TRY
    if (err != cudaSuccess) cudaStreamSynchronize(s);
    cudaFree(flag); cudaFree(cnt); cudaFree(off_all); cudaFree(iota); cudaFree(aff); cudaFree(naff_dev); cudaFree(tmp);
    cudaFree(cand); cudaFree(row_node); cudaFree(cand_off); cudaFree(cand_cnt); cudaFree(fallback); cudaFree(out_rows); cudaFree(out_deg); cudaFree(tier_list);
    return err;
}

}  // namespace jv
