// kernels_batch.cu — batched scoring kernels: one launch per hop / rerank list / multi-query step / brute-force pass.
// HBM-bound reductions and gathers: CUDA cores, 128-bit loads, shuffle reductions; no tensor cores (SURVEY §8d).
#include "kernels.h"

namespace jv {

std::atomic<long long> g_launches{0};

#define JV_DISPATCH_KIND_METRIC(kind, metric, CALL)                                            \
    do {                                                                                        \
        if ((kind) == KIND_F32) {                                                               \
            if ((metric) == JV_METRIC_EUCLIDEAN) { CALL(KIND_F32, JV_METRIC_EUCLIDEAN); }       \
            else if ((metric) == JV_METRIC_DOT) { CALL(KIND_F32, JV_METRIC_DOT); }              \
            else { CALL(KIND_F32, JV_METRIC_COSINE); }                                          \
        } else if ((kind) == KIND_PQ) {                                                         \
            if ((metric) == JV_METRIC_EUCLIDEAN) { CALL(KIND_PQ, JV_METRIC_EUCLIDEAN); }        \
            else if ((metric) == JV_METRIC_DOT) { CALL(KIND_PQ, JV_METRIC_DOT); }               \
            else { CALL(KIND_PQ, JV_METRIC_COSINE); }                                           \
        } else if ((kind) == KIND_BQ) {                                                         \
            CALL(KIND_BQ, JV_METRIC_COSINE);                                                    \
        } else {                                                                                \
            if ((metric) == JV_METRIC_EUCLIDEAN) { CALL(KIND_NVQ, JV_METRIC_EUCLIDEAN); }       \
            else if ((metric) == JV_METRIC_DOT) { CALL(KIND_NVQ, JV_METRIC_DOT); }              \
            else { CALL(KIND_NVQ, JV_METRIC_COSINE); }                                          \
        }                                                                                       \
    } while (0)

// ------------------------------------------------------------------------------------------------
// query preparation: one CTA per query (LUT build = the M calculatePartialSums calls of PQDecoder.java:48-53)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) prepare_kernel(DataDesc d, int metric, const float *__restrict__ queries, float *__restrict__ blobs, int blob_stride)
{
    __shared__ float red[36];
    prepare_blob(d, metric, queries + (size_t)blockIdx.x * d.dim, blobs + (size_t)blockIdx.x * blob_stride, red);
}

cudaError_t launch_prepare(const DataDesc &d, int metric, const float *queries_dev, int nq, float *blobs_dev, cudaStream_t s)
{
    if (nq <= 0) return cudaSuccess;
    prepare_kernel<<<nq, 256, 0, s>>>(d, metric, queries_dev, blobs_dev, blob_floats(d));
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// ragged scoring: grid = (chunks, nq); each CTA scores up to CHUNK ids of one query, one lane-group per id
// ------------------------------------------------------------------------------------------------
constexpr int RAGGED_THREADS = 128;
constexpr int RAGGED_CHUNK = 128;

template <int KIND, int METRIC>
__global__ void __launch_bounds__(RAGGED_THREADS) score_ragged_kernel(DataDesc d, const float *__restrict__ blobs, int blob_stride,
                                                                      const int32_t *__restrict__ ids, const int32_t *__restrict__ offsets,
                                                                      int n_shared, float *__restrict__ scores, int chunk, int *done_counter,
                                                                      int *host_flag, int seq)
{
    constexpr int G = GroupOf<KIND>::value;
    const int q = blockIdx.y;
    int begin, count;
    size_t out_base;
    if (offsets) {
        begin = offsets[q];
        count = offsets[q + 1] - begin;
        out_base = (size_t)begin;
    } else {
        begin = 0;
        count = n_shared;
        out_base = (size_t)q * n_shared;
    }
    const int c0 = blockIdx.x * chunk;
    if (c0 < count) {
        const int c1 = min(count, c0 + chunk);
        const float *blob = blobs + (size_t)q * blob_stride;
        const int group = threadIdx.x / G, lane = threadIdx.x % G;
        constexpr int NG = RAGGED_THREADS / G;
        for (int i = c0 + group; i < c1; i += NG) {
            const int node = ids[begin + i];
            float sc = 0.f;
            if (node >= 0 && node < d.n) sc = score_row<KIND, METRIC>(d, blob, node, lane);
            if (lane == 0) {
                scores[out_base + i] = sc;
                if (host_flag) __threadfence_system();
            }
        }
    }
    if (host_flag) {
        // completion signal for a host that spins on mapped memory instead of synchronising the stream: the last CTA to finish
        // publishes `seq` after every score (written to mapped host memory too) has been fenced to the system scope
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence_system();
            if (atomicAdd(done_counter, 1) == (int)(gridDim.x * gridDim.y) - 1) {
                *done_counter = 0;
                __threadfence_system();
                *(volatile int *)host_flag = seq;
            }
        }
    }
}

cudaError_t launch_score_ragged(const DataDesc &d, int metric, const float *blobs_dev, int nq, const int32_t *ids_dev,
                                const int32_t *offsets_dev, int n_shared, int max_per_query, float *scores_dev, cudaStream_t s, int chunk,
                                int *done_counter, int *host_flag, int seq)
{
    if (nq <= 0 || max_per_query <= 0) return cudaSuccess;
    if (chunk <= 0) chunk = RAGGED_CHUNK;
    dim3 grid((max_per_query + chunk - 1) / chunk, nq);
    if (grid.y > 65535u) return cudaErrorInvalidValue;
#define CALL(K, M) \
    score_ragged_kernel<K, M><<<grid, RAGGED_THREADS, 0, s>>>(d, blobs_dev, blob_floats(d), ids_dev, offsets_dev, n_shared, scores_dev, chunk, done_counter, host_flag, seq)
    JV_DISPATCH_KIND_METRIC(d.kind, metric, CALL);
#undef CALL
    g_launches++;
    return cudaGetLastError();
}

// one hop of one search, latency path: the candidate ids travel in the kernel parameters (no PCIe read before the rows can be
// fetched), one lane group per id, and every score is stored straight into mapped host memory, where the host polls for the
// sentinel it left there to disappear (no fence / counter / flag chain at the end of the kernel).
template <int KIND, int METRIC>
__global__ void __launch_bounds__(RAGGED_THREADS) score_hop_kernel(DataDesc d, const float *__restrict__ blob, HopIds h, int n, float *__restrict__ scores)
{
    constexpr int G = GroupOf<KIND>::value;
    constexpr int NG = RAGGED_THREADS / G;
    const int i = blockIdx.x * NG + threadIdx.x / G, lane = threadIdx.x % G;
    if (i >= n) return;
    const int node = h.ids[i];
    float sc = 0.f;
    if (node >= 0 && node < d.n) sc = score_row<KIND, METRIC>(d, blob, node, lane);
    if (lane == 0) scores[i] = sc;
}

cudaError_t launch_score_hop(const DataDesc &d, int metric, const float *blob_dev, const int32_t *ids_host, int n, float *scores_mapped, cudaStream_t s)
{
    if (n <= 0) return cudaSuccess;
    if (n > HOP_MAX_IDS) return cudaErrorInvalidValue;
    HopIds h;
    memcpy(h.ids, ids_host, (size_t)n * 4);
    const int G = d.kind == KIND_F32 ? GroupOf<KIND_F32>::value : d.kind == KIND_PQ ? GroupOf<KIND_PQ>::value : d.kind == KIND_BQ ? GroupOf<KIND_BQ>::value : GroupOf<KIND_NVQ>::value;
    const int per_cta = RAGGED_THREADS / G;
    const int grid = (n + per_cta - 1) / per_cta;
#define CALL(K, M) score_hop_kernel<K, M><<<grid, RAGGED_THREADS, 0, s>>>(d, blob_dev, h, n, scores_mapped)
    JV_DISPATCH_KIND_METRIC(d.kind, metric, CALL);
#undef CALL
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// pairs: one warp per (a, b) pair — the candidate x selected scores of VamanaDiversityProvider.retainDiverse
// ------------------------------------------------------------------------------------------------
template <int KIND, int METRIC>
__global__ void __launch_bounds__(128) score_pairs_kernel(DataDesc d, const int32_t *__restrict__ a, const int32_t *__restrict__ b, int n, float *__restrict__ out)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= n) return;
    const int x = a[warp], y = b[warp];
    float sc;
    if (KIND == KIND_F32) sc = pair_f32<METRIC>(d, x, y, lane);
    else if (KIND == KIND_PQ) sc = d.pair_table[METRIC == JV_METRIC_EUCLIDEAN ? 0 : 1] ? pair_pq_table<METRIC>(d, x, y, lane) : pair_pq<METRIC>(d, x, y, lane);
    else sc = pair_bq(d, x, y, lane);
    if (lane == 0) out[warp] = sc;
}

cudaError_t launch_score_pairs(const DataDesc &d, int metric, const int32_t *a_dev, const int32_t *b_dev, int n, float *out_dev, cudaStream_t s)
{
    if (n <= 0) return cudaSuccess;
    if (d.kind == KIND_NVQ) return cudaErrorNotSupported;
    const int blocks = (n * 32 + 127) / 128;
#define CALL(K, M) score_pairs_kernel<K, M><<<blocks, 128, 0, s>>>(d, a_dev, b_dev, n, out_dev)
    if (d.kind == KIND_F32) {
        if (metric == JV_METRIC_EUCLIDEAN) CALL(KIND_F32, JV_METRIC_EUCLIDEAN);
        else if (metric == JV_METRIC_DOT) CALL(KIND_F32, JV_METRIC_DOT);
        else CALL(KIND_F32, JV_METRIC_COSINE);
    } else if (d.kind == KIND_PQ) {
        if (metric == JV_METRIC_EUCLIDEAN) CALL(KIND_PQ, JV_METRIC_EUCLIDEAN);
        else if (metric == JV_METRIC_DOT) CALL(KIND_PQ, JV_METRIC_DOT);
        else CALL(KIND_PQ, JV_METRIC_COSINE);
    } else CALL(KIND_BQ, JV_METRIC_COSINE);
#undef CALL
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// brute-force top-k: sample -> per-query threshold -> filtered full pass -> per-query sort.
// Keys are the reference's 64-bit ordering key (NodeQueue.java:125-137), so ties go to the smaller node id.
// ------------------------------------------------------------------------------------------------
// Leaves the P largest of keys[0..n_pow2) sorted descending in keys[0..P) (P, n_pow2 powers of two, P <= n_pow2):
// sort every P-chunk (alternating directions), then halve: element-wise max of neighbouring chunks is a bitonic sequence
// holding the best P of the pair; re-sort it with one bitonic merge. ~ (log^2 P + 2 log P) / 2 full-width stages instead of
// log^2 n / 2 — the thresholds only need the top max(j, k) of the sample / candidate buffer, not a full sort.
__device__ __forceinline__ void bitonic_top_desc(long long *keys, int n_pow2, int P)
{
    if (P >= n_pow2) { bitonic_sort_desc(keys, n_pow2); return; }
    // phase 1: bitonic sort of each P-chunk; chunk c descending when c is even, ascending when odd
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n_pow2; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const long long a = keys[i], b = keys[ixj];
                    const bool desc = (i & k) == 0;  // at k == P this alternates per chunk: even chunks descending, odd ascending
                    if (desc ? (a < b) : (a > b)) { keys[i] = b; keys[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
    // phase 2: repeatedly merge chunk pairs (desc, asc) -> best P of the pair, compacted to the front
    for (int len = n_pow2; len > P; len >>= 1) {
        const int chunks = len / P;  // even
        // max(desc chunk 2c, asc chunk 2c+1) element-wise is bitonic and holds the best P of the 2P
        for (int i = threadIdx.x; i < (chunks >> 1) * P; i += blockDim.x) {
            const int c = i / P, o = i - c * P;
            const long long a = keys[(2 * c) * P + o], b = keys[(2 * c + 1) * P + o];
            keys[(2 * c) * P + o] = a > b ? a : b;
        }
        __syncthreads();
        // compact surviving chunks to the front: chunk 2c -> chunk c (c > 0 only; in-place copy is ordered by a barrier)
        for (int c = 1; c < (chunks >> 1); c++) {
            for (int o = threadIdx.x; o < P; o += blockDim.x) keys[c * P + o] = keys[(2 * c) * P + o];
            __syncthreads();
        }
        // bitonic merge of every surviving chunk; alternate directions again unless it is the last one
        const int surv = chunks >> 1;
        for (int j = P >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < surv * P; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const long long a = keys[i], b = keys[ixj];
                    const bool desc = surv == 1 || (((i / P) & 1) == 0);
                    if (desc ? (a < b) : (a > b)) { keys[i] = b; keys[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(256) topk_sample_ids_kernel(int32_t *ids, int S, long long n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < S) ids[i] = (int32_t)(((long long)i * n) / S);
}

constexpr long long KEY_DONE = 0x7fffffffffffffffLL;  // thr value of a finished query: nothing passes the filter

// Per query: sort the sample; thr = an AGGRESSIVE threshold (the j-th best of the sample, j ~ 3 k S / n + 2 < k), thr_safe = the
// k-th best of the sample (a guaranteed lower bound of the final k-th best). The filtered pass is exact whenever it finds at
// least k keys >= thr; otherwise the query is redone with thr_safe (topk_select_kernel decides).
__global__ void __launch_bounds__(256) topk_threshold_kernel(const float *__restrict__ sample_scores, const int32_t *__restrict__ sample_ids, int S, int S_pow2,
                                                             int k, int j_aggr, int whole, long long *__restrict__ thr, long long *__restrict__ thr_safe,
                                                             int *__restrict__ cnt)
{
    extern __shared__ long long skeys[];
    const int q = blockIdx.x;
    for (int i = threadIdx.x; i < S_pow2; i += blockDim.x)
        skeys[i] = i < S ? topk_key(sample_scores[(size_t)q * S + i], sample_ids[i]) : KEY_MIN;
    __syncthreads();
    bitonic_top_desc(skeys, S_pow2, next_pow2(k));  // j_aggr <= k: both thresholds live in the top k of the sample
    if (threadIdx.x == 0) {
        const long long safe = (!whole && k <= S) ? skeys[k - 1] : KEY_MIN;
        thr_safe[q] = safe;
        thr[q] = (!whole && j_aggr < k && j_aggr <= S) ? skeys[j_aggr - 1] : safe;
        cnt[q] = 0;
    }
}

constexpr int BF_THREADS = 256;
constexpr int BF_TILE = 2048;  // rows per CTA

// word w of an accept bitset over n rows, the bits at positions >= n cleared
__device__ __forceinline__ uint32_t accept_word(const uint32_t *__restrict__ bits, long long w, long long n)
{
    uint32_t x = __ldg(bits + w);
    const long long left = n - w * 32;
    if (left < 32) x &= (1u << (int)left) - 1u;
    return x;
}

// ACC (jv_topk_bruteforce_ex): only the rows whose bit is set in the query's accept bitset (acc + q * acc_stride words) are scored;
// each warp takes one 32-row word of the tile at a time, so an all-zero word costs the warp one load
template <int KIND, int METRIC, bool ACC = false>
__global__ void __launch_bounds__(BF_THREADS) topk_filter_kernel(DataDesc d, const float *__restrict__ blobs, int blob_stride, const long long *__restrict__ thr,
                                                                 long long *__restrict__ buf, int *__restrict__ cnt, int cap, const int *__restrict__ qlist,
                                                                 const uint32_t *__restrict__ acc = nullptr, long long acc_stride = 0)
{
    constexpr int G = GroupOf<KIND>::value;
    constexpr int NG = BF_THREADS / G;
    const int q = qlist ? qlist[blockIdx.x] : blockIdx.x;
    const long long r0 = (long long)blockIdx.y * BF_TILE;
    const long long r1 = min(d.n, r0 + BF_TILE);
    const float *blob = blobs + (size_t)q * blob_stride;
    const long long t = thr[q];
    if (t == KEY_DONE) return;
    const int group = threadIdx.x / G, lane = threadIdx.x % G;
    if constexpr (!ACC) {
        for (long long r = r0 + group; r < r1; r += NG) {
            const float sc = score_row<KIND, METRIC>(d, blob, (int)r, lane);
            if (lane == 0) {
                const long long key = topk_key(sc, (int32_t)r);
                if (key >= t) {
                    const int pos = atomicAdd(&cnt[q], 1);
                    if (pos < cap) buf[(size_t)q * cap + pos] = key;
                }
            }
        }
    } else {
        const uint32_t *bits = acc + (size_t)q * acc_stride;
        constexpr int GPW = 32 / G;  // lane groups per warp
        const int gw = (threadIdx.x & 31) / G;
        for (long long w = r0 / 32 + (threadIdx.x >> 5); w * 32 < r1; w += BF_THREADS / 32) {
            const uint32_t x = accept_word(bits, w, d.n);
            const int p = __popc(x);
            for (int i = gw; i < p; i += GPW) {
                const int r = (int)(w * 32) + (int)__fns(x, 0, i + 1);
                const float sc = score_row<KIND, METRIC>(d, blob, r, lane);
                if (lane == 0) {
                    const long long key = topk_key(sc, r);
                    if (key >= t) {
                        const int pos = atomicAdd(&cnt[q], 1);
                        if (pos < cap) buf[(size_t)q * cap + pos] = key;
                    }
                }
            }
        }
    }
}

// Hamming distance of MAXW 64-bit words by a Harley-Seal carry-save adder tree over the 32-bit halves: 16 XORed words are
// compressed into ones/twos/fours/eights/sixteens bit-planes with 15 CSAs (2 LOP3 each) and ONE popcount, instead of 16
// popcounts. POPC issues at a quarter of the LOP3 rate on this part, so the pair loop moves from the popcount pipe to the
// ALU pipe. Exact integer arithmetic: the result equals sum(popcll(r[w] ^ q[w])).
__device__ __forceinline__ void csa32(unsigned &h, unsigned &l, unsigned a, unsigned b, unsigned c)
{
    const unsigned u = a ^ b;
    h = (a & b) | (u & c);
    l = u ^ c;
}

template <int MAXW>
__device__ __forceinline__ int hamming_csa(const unsigned long long (&r)[MAXW], const unsigned long long *q)
{
    static_assert(MAXW % 8 == 0, "16 32-bit halves per block");
    unsigned ones = 0, twos = 0, fours = 0, eights = 0;
    int total16 = 0;
#pragma unroll
    for (int b = 0; b < MAXW / 8; b++) {
        unsigned d[16];
        const ulonglong2 *q2 = reinterpret_cast<const ulonglong2 *>(q) + b * 4;  // 128-bit shared loads: half the LDS issue slots
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const ulonglong2 qq = q2[i];
            const unsigned long long x = r[b * 8 + 2 * i] ^ qq.x, y = r[b * 8 + 2 * i + 1] ^ qq.y;
            d[4 * i] = (unsigned)x;
            d[4 * i + 1] = (unsigned)(x >> 32);
            d[4 * i + 2] = (unsigned)y;
            d[4 * i + 3] = (unsigned)(y >> 32);
        }
        unsigned twosA, twosB, foursA, foursB, eightsA, eightsB, sixteens;
        csa32(twosA, ones, ones, d[0], d[1]);
        csa32(twosB, ones, ones, d[2], d[3]);
        csa32(foursA, twos, twos, twosA, twosB);
        csa32(twosA, ones, ones, d[4], d[5]);
        csa32(twosB, ones, ones, d[6], d[7]);
        csa32(foursB, twos, twos, twosA, twosB);
        csa32(eightsA, fours, fours, foursA, foursB);
        csa32(twosA, ones, ones, d[8], d[9]);
        csa32(twosB, ones, ones, d[10], d[11]);
        csa32(foursA, twos, twos, twosA, twosB);
        csa32(twosA, ones, ones, d[12], d[13]);
        csa32(twosB, ones, ones, d[14], d[15]);
        csa32(foursB, twos, twos, twosA, twosB);
        csa32(eightsB, fours, fours, foursA, foursB);
        csa32(sixteens, eights, eights, eightsA, eightsB);
        total16 += __popc(sixteens);
    }
    return 16 * total16 + 8 * __popc(eights) + 4 * __popc(fours) + 2 * __popc(twos) + __popc(ones);
}

// ---- BQ specialisation: Hamming brute force is popcount-bound, not HBM-bound (SURVEY §8d C4): one ROW per thread, its
// words held in registers, the query bit-packs staged in shared memory and read by broadcast; no shuffles. A pair costs
// W x (LDS.64 broadcast / 32 rows + XOR + POPC + ADD). The exact key is formed only for pairs under the per-query
// Hamming bound derived from the sample threshold.
constexpr int BQF_THREADS = 256;

// ACC: a row is scored against a query only when its bit is set in that query's accept bitset. A warp's 32 rows are one bitset word:
// a shared bitset's all-zero word skips the warp's row loads, a per-query bitset's all-zero word skips that query for the warp.
template <int MAXW, bool ACC = false>
__global__ void __launch_bounds__(BQF_THREADS) topk_filter_bq_kernel(DataDesc d, const float *__restrict__ blobs, int blob_stride, int nq,
                                                                     const long long *__restrict__ thr, long long *__restrict__ buf,
                                                                     int *__restrict__ cnt, int cap, const int *__restrict__ qlist,
                                                                     const uint32_t *__restrict__ acc = nullptr, long long acc_stride = 0)
{
    constexpr int BQF_QCHUNK = MAXW <= 16 ? 256 : 128;  // queries staged per pass (<= 32 KB of bit packs)
    __shared__ __align__(16) unsigned long long qs[BQF_QCHUNK * MAXW];
    __shared__ int hdmax[BQF_QCHUNK];
    __shared__ int sq[BQF_QCHUNK];
    __shared__ long long sthr[BQF_QCHUNK];
    const int W = d.W;
    const long long row_stride = (long long)gridDim.x * BQF_THREADS;
    for (long long r = (long long)blockIdx.x * BQF_THREADS + threadIdx.x; r - threadIdx.x < d.n; r += row_stride) {
        unsigned long long rw[MAXW];
        bool live = r < d.n;
        if (ACC && acc_stride == 0) live = live && ((accept_word(acc, r >> 5, d.n) >> (r & 31)) & 1u);
        const unsigned long long *row = d.words + (size_t)(live ? r : 0) * W;
#pragma unroll
        for (int w = 0; w < MAXW; w++) rw[w] = (live && w < W) ? __ldg(row + w) : 0ull;
        for (int q0 = 0; q0 < nq; q0 += BQF_QCHUNK) {
            const int qc = min(BQF_QCHUNK, nq - q0);
            __syncthreads();
            for (int i = threadIdx.x; i < qc * MAXW; i += BQF_THREADS) {
                const int q = i / MAXW, w = i - q * MAXW;
                const int qq = qlist ? qlist[q0 + q] : q0 + q;
                qs[i] = w < W ? reinterpret_cast<const unsigned long long *>(blobs + (size_t)qq * blob_stride)[w] : 0ull;
            }
            for (int q = threadIdx.x; q < qc; q += BQF_THREADS) {
                const int qq = qlist ? qlist[q0 + q] : q0 + q;
                sq[q] = qq;
                const long long t = thr[qq];
                sthr[q] = t;
                // largest Hamming distance whose score can still reach the threshold key
                int h = d.dim;
                if (t == KEY_DONE) h = -1;
                else if (t != KEY_MIN) {
                    const float ts = key_score(t);
                    h = (int)((1.0f - ts) * (float)d.dim) + 2;
                    if (h > d.dim) h = d.dim;
                    while (h >= 0 && bq_score_from_hd(h, d.dim) < ts) h--;
                }
                hdmax[q] = h;
            }
            __syncthreads();
            if (live) {
                for (int q = 0; q < qc; q++) {
                    if (ACC && acc_stride != 0) {
                        const uint32_t x = accept_word(acc + (size_t)sq[q] * acc_stride, r >> 5, d.n);
                        if (!((x >> (r & 31)) & 1u)) continue;
                    }
                    int hd;
                    if constexpr (MAXW >= 8) hd = hamming_csa<MAXW>(rw, qs + q * MAXW);
                    else {
                        hd = 0;
#pragma unroll
                        for (int w = 0; w < MAXW; w++) hd += __popcll(rw[w] ^ qs[q * MAXW + w]);
                    }
                    if (hd <= hdmax[q]) {
                        const long long key = topk_key(bq_score_from_hd(hd, d.dim), (int32_t)r);
                        if (key >= sthr[q]) {
                            const int qq = sq[q];
                            const int pos = atomicAdd(&cnt[qq], 1);
                            if (pos < cap) buf[(size_t)qq * cap + pos] = key;
                        }
                    }
                }
            }
        }
    }
}

// ---- PQ specialisation: the per-query partial-sums table (LUT, M*k fp32 = 96 KB at M=96) is staged into shared memory
// with TMA bulk copies (cp.async.bulk + mbarrier; SASS UBLKCP), then code rows stream through 8-lane groups.
constexpr int PQF_THREADS = 256;
constexpr int PQF_TILE = 16384;

// ACC: as topk_filter_kernel's, one warp per 32-row bitset word
template <int METRIC, bool ACC = false>
__global__ void __launch_bounds__(PQF_THREADS) topk_filter_pq_kernel(DataDesc d, const float *__restrict__ blobs, int blob_stride,
                                                                     const long long *__restrict__ thr, long long *__restrict__ buf,
                                                                     int *__restrict__ cnt, int cap, const int *__restrict__ qlist,
                                                                     const uint32_t *__restrict__ acc = nullptr, long long acc_stride = 0)
{
    extern __shared__ __align__(128) unsigned char pq_smem[];
    float *lut = reinterpret_cast<float *>(pq_smem);
    __shared__ __align__(8) uint64_t bar;
    const int q = qlist ? qlist[blockIdx.x] : blockIdx.x;
    if (thr[q] == KEY_DONE) return;
    const unsigned bytes = (unsigned)blob_stride * 4u;
    if (threadIdx.x == 0) {
        mbar_init(&bar, 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(&bar, bytes);
        const char *src = reinterpret_cast<const char *>(blobs + (size_t)q * blob_stride);
        for (unsigned off = 0; off < bytes; off += 32768u) bulk_g2s(pq_smem + off, src + off, min(32768u, bytes - off), &bar);
    }
    mbar_wait(&bar, 0);
    constexpr int G = 8, NG = PQF_THREADS / G;
    const long long r0 = (long long)blockIdx.y * PQF_TILE;
    const long long r1 = min(d.n, r0 + PQF_TILE);
    const long long t = thr[q];
    const int group = threadIdx.x / G, lane = threadIdx.x % G;
    if constexpr (!ACC) {
        for (long long r = r0 + group; r < r1; r += NG) {
            const float sc = score_pq<METRIC>(d, lut, (int)r, lane);
            if (lane == 0) {
                const long long key = topk_key(sc, (int32_t)r);
                if (key >= t) {
                    const int pos = atomicAdd(&cnt[q], 1);
                    if (pos < cap) buf[(size_t)q * cap + pos] = key;
                }
            }
        }
    } else {
        const uint32_t *bits = acc + (size_t)q * acc_stride;
        constexpr int GPW = 32 / G;
        const int gw = (threadIdx.x & 31) / G;
        for (long long w = r0 / 32 + (threadIdx.x >> 5); w * 32 < r1; w += PQF_THREADS / 32) {
            const uint32_t x = accept_word(bits, w, d.n);
            const int p = __popc(x);
            for (int i = gw; i < p; i += GPW) {
                const int r = (int)(w * 32) + (int)__fns(x, 0, i + 1);
                const float sc = score_pq<METRIC>(d, lut, r, lane);
                if (lane == 0) {
                    const long long key = topk_key(sc, r);
                    if (key >= t) {
                        const int pos = atomicAdd(&cnt[q], 1);
                        if (pos < cap) buf[(size_t)q * cap + pos] = key;
                    }
                }
            }
        }
    }
}

__global__ void __launch_bounds__(256) topk_select_kernel(const long long *__restrict__ buf, int *__restrict__ cnt, int cap, int cap_pow2, int k,
                                                          long long n_rows, long long *__restrict__ thr, const long long *__restrict__ thr_safe,
                                                          long long *__restrict__ keys_out, int *__restrict__ n_redo, const int *__restrict__ qlist,
                                                          int *__restrict__ qlist_next)
{
    extern __shared__ long long skeys[];
    const int q = qlist ? qlist[blockIdx.x] : blockIdx.x;
    const long long t = thr[q];
    if (t == KEY_DONE) return;
    const int c = cnt[q];
    const int m = min(c, cap);
    for (int i = threadIdx.x; i < cap_pow2; i += blockDim.x) skeys[i] = i < m ? buf[(size_t)q * cap + i] : KEY_MIN;
    __syncthreads();
    bitonic_top_desc(skeys, cap_pow2, next_pow2(k));  // only the best k are emitted (or used as the tightened threshold)
    const long long need = n_rows < (long long)k ? n_rows : (long long)k;
    if (c <= cap && (c >= need || t == thr_safe[q])) {
        // exact: every key >= thr was captured and there are at least k of them (or the threshold was the guaranteed one)
        for (int i = threadIdx.x; i < k; i += blockDim.x) keys_out[(size_t)q * k + i] = i < m ? skeys[i] : KEY_MIN;
        if (threadIdx.x == 0) thr[q] = KEY_DONE;
    } else if (threadIdx.x == 0) {
        // too many (buffer overflowed): the k-th best of what was captured is a tighter valid bound; too few: fall back
        thr[q] = c > cap ? skeys[k - 1] : thr_safe[q];
        cnt[q] = 0;
        qlist_next[atomicAdd(n_redo, 1)] = q;
    }
}

// aggressive threshold = j-th best of the sample with the smallest j such that j - 6 sqrt(j) >= k S / n: the j-th best of a
// random sample has rank ~ j n / S (std sqrt(j) n / S) in the full set, so fewer than k survivors is a > 6 sigma event
__host__ __device__ inline int aggressive_rank(int k, int S, long long n)
{
    if (n <= S) return k;
    const double kf = (double)k * S / (double)n;
    for (int j = 1; j < k; j++)
        if ((double)j - 6.0 * sqrt((double)j) >= kf) return j;
    return k;
}
int topk_aggressive_rank(int k, int S, long long n) { return aggressive_rank(k, S, n); }

// launch_topk_bruteforce's device scratch for nq queries, carved from `base` (nullptr: only measured)
struct TopkScratch {
    int S, cap;              // sampled rows, captured keys per query
    int32_t *sample_ids;     // [S]
    float *sample_scores;    // [nq][S]
    long long *thr;          // [nq]
    long long *thr_safe;     // [nq]
    long long *buf;          // [nq][cap]
    int *cnt;                // [nq]
    int *qlist_a, *qlist_b;  // [nq] each: queries still unresolved after a pass
    size_t bytes;
    TopkScratch(const DataDesc &d, int nq, int k, void *base)
    {
        S = d.n < 16384 ? (int)d.n : 16384;
        // room for twice the expected survivors of the aggressive threshold (j n / S); a whole-set sample captures every row
        const double f = (double)S / (double)d.n;
        const double expect = d.n <= S ? (double)d.n : topk_aggressive_rank(k, S, d.n) / f;
        cap = expect * 2 > 8192 ? 16384 : (expect * 2 > 4096 ? 8192 : 4096);
        if (cap < S && d.n <= S) cap = 16384;
        Carver c(base);
        sample_ids = c.take<int32_t>(S);
        sample_scores = c.take<float>((size_t)nq * S);
        thr = c.take<long long>(nq);
        thr_safe = c.take<long long>(nq);
        buf = c.take<long long>((size_t)nq * cap);
        cnt = c.take<int>(nq);
        qlist_a = c.take<int>(nq);
        qlist_b = c.take<int>(nq);
        bytes = c.bytes;
    }
};

size_t topk_scratch_bytes(const DataDesc &d, int nq, int k) { return TopkScratch(d, nq, k, nullptr).bytes; }

// The filtered passes of the sampled top-k: `active` queries (qlist, nullptr = 0 .. active) hold thresholds in ts.thr; each pass
// captures the keys >= thr, then topk_select_kernel finishes the exact queries and lists the rest for the next pass. acc != nullptr:
// only the rows accepted by each query's bitset (acc + q * acc_stride words) take part (the ACC kernel instantiations).
template <bool ACC>
static cudaError_t topk_filter_passes(const DataDesc &d, int metric, const float *blobs_dev, int active, const int *qlist, int k, const TopkScratch &ts,
                                      const uint32_t *acc, long long acc_stride, long long *keys_out_dev, int *overflow_flag_dev, cudaStream_t s)
{
    cudaError_t e;
    const int cap2 = next_pow2(ts.cap);
    if ((size_t)cap2 * sizeof(long long) > 48 * 1024)
        if ((e = cudaFuncSetAttribute(topk_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cap2 * (int)sizeof(long long))) != cudaSuccess) return e;
    for (int pass = 0; pass < 8; pass++) {
        int *qnext = (pass & 1) ? ts.qlist_a : ts.qlist_b;
        if ((e = cudaMemsetAsync(overflow_flag_dev, 0, sizeof(int), s)) != cudaSuccess) return e;
        if (d.kind == KIND_BQ && d.W <= 32) {
            // popcount-bound: every CTA walks a slice of the rows against ALL active queries (rows in registers, queries in smem)
            long long want = (d.n + BQF_THREADS - 1) / BQF_THREADS;
            int dev = 0, sms = 0;
            if ((e = cudaGetDevice(&dev)) != cudaSuccess || (e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return e;
            int gridx = (int)(want < sms * 8LL ? want : sms * 8LL);
#define CALLBQ(MW) topk_filter_bq_kernel<MW, ACC><<<gridx, BQF_THREADS, 0, s>>>(d, blobs_dev, blob_floats(d), active, ts.thr, ts.buf, ts.cnt, ts.cap, qlist, acc, acc_stride)
            if (d.W <= 4) CALLBQ(4);
            else if (d.W <= 8) CALLBQ(8);
            else if (d.W <= 16) CALLBQ(16);
            else if (d.W <= 24) CALLBQ(24);
            else CALLBQ(32);
#undef CALLBQ
        } else if (d.kind == KIND_PQ && (size_t)blob_floats(d) * 4 <= 200 * 1024) {
            dim3 grid(active, (unsigned)((d.n + PQF_TILE - 1) / PQF_TILE));
            const int smem = blob_floats(d) * 4;
#define CALLPQ(M)                                                                                                             \
    do {                                                                                                                      \
        if ((e = cudaFuncSetAttribute(topk_filter_pq_kernel<M, ACC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)) != cudaSuccess) return e; \
        topk_filter_pq_kernel<M, ACC><<<grid, PQF_THREADS, smem, s>>>(d, blobs_dev, blob_floats(d), ts.thr, ts.buf, ts.cnt, ts.cap, qlist, acc, acc_stride); \
    } while (0)
            if (metric == JV_METRIC_EUCLIDEAN) CALLPQ(JV_METRIC_EUCLIDEAN);
            else if (metric == JV_METRIC_DOT) CALLPQ(JV_METRIC_DOT);
            else CALLPQ(JV_METRIC_COSINE);
#undef CALLPQ
        } else {
            dim3 grid(active, (unsigned)((d.n + BF_TILE - 1) / BF_TILE));
            if (grid.y > 65535u) return cudaErrorInvalidValue;
#define CALL(K, M) topk_filter_kernel<K, M, ACC><<<grid, BF_THREADS, 0, s>>>(d, blobs_dev, blob_floats(d), ts.thr, ts.buf, ts.cnt, ts.cap, qlist, acc, acc_stride)
            JV_DISPATCH_KIND_METRIC(d.kind, metric, CALL);
#undef CALL
        }
        g_launches++;
        topk_select_kernel<<<active, 256, (size_t)cap2 * sizeof(long long), s>>>(ts.buf, ts.cnt, ts.cap, cap2, k, d.n, ts.thr, ts.thr_safe, keys_out_dev, overflow_flag_dev,
                                                                                qlist, qnext);
        g_launches++;
        int redo = 0;
        if ((e = cudaMemcpyAsync(&redo, overflow_flag_dev, sizeof(int), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
        if (redo == 0) return cudaGetLastError();  // overflow_flag_dev is left at 0
        active = redo;
        qlist = qnext;
    }
    return cudaGetLastError();  // overflow_flag_dev still holds the number of unresolved queries
}

cudaError_t launch_topk_bruteforce(const DataDesc &d, int metric, const float *blobs_dev, int nq, int k, void *scratch_dev,
                                   long long *keys_out_dev, int *overflow_flag_dev, cudaStream_t s)
{
    if (nq <= 0) return cudaSuccess;
    cudaError_t e;
    const TopkScratch ts(d, nq, k, scratch_dev);
    const int S = ts.S;
    topk_sample_ids_kernel<<<(S + 255) / 256, 256, 0, s>>>(ts.sample_ids, S, d.n);
    g_launches++;
    if ((e = launch_score_ragged(d, metric, blobs_dev, nq, ts.sample_ids, nullptr, S, S, ts.sample_scores, s)) != cudaSuccess) return e;
    const int S2 = next_pow2(S);
    if ((size_t)S2 * sizeof(long long) > 48 * 1024)
        if ((e = cudaFuncSetAttribute(topk_threshold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, S2 * (int)sizeof(long long))) != cudaSuccess) return e;
    const int whole = d.n <= S ? 1 : 0;
    const int ja = topk_aggressive_rank(k, S, d.n);
    topk_threshold_kernel<<<nq, 256, (size_t)S2 * sizeof(long long), s>>>(ts.sample_scores, ts.sample_ids, S, S2, k, ja, whole, ts.thr, ts.thr_safe, ts.cnt);
    g_launches++;
    return topk_filter_passes<false>(d, metric, blobs_dev, nq, nullptr, k, ts, nullptr, 0, keys_out_dev, overflow_flag_dev, s);
}

// ---- acceptOrds-filtered top-k (jv_topk_bruteforce_ex, DESIGN §4.2a)
constexpr int ACC_THREADS = 1024;  // 32 warps: the block scan's second level is one warp

int accept_sample_size(long long n) { return n < 16384 ? (int)n : 16384; }  // = TopkScratch::S

// One CTA per bitset: the popcounts of its words (bits at positions >= n cleared), an exclusive scan over the CTA, then the
// accepted rows in ascending order. cnt[b] = accepted rows; ids[b * S + i], i < m = min(cnt, S) = the row of accepted rank
// floor(i cnt / m): every accepted row when cnt <= S, else S evenly spaced ranks (the sampled tier's sample).
__global__ void __launch_bounds__(ACC_THREADS) accept_compact_kernel(const uint32_t *__restrict__ bits, long long stride, long long n, int S,
                                                                     int *__restrict__ cnt, int32_t *__restrict__ ids)
{
    __shared__ int warp_base[32];
    __shared__ int s_total;
    const uint32_t *b = bits + (size_t)blockIdx.x * stride;
    const long long words = (n + 31) / 32;
    const long long per = (words + ACC_THREADS - 1) / ACC_THREADS;
    const long long w0 = min(words, (long long)threadIdx.x * per), w1 = min(words, w0 + per);
    int c = 0;
    for (long long w = w0; w < w1; w++) c += __popc(accept_word(b, w, n));
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int inc = c;
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(FULL, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) warp_base[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        const int t = warp_base[lane];
        int ti = t;
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(FULL, ti, o);
            if (lane >= o) ti += v;
        }
        warp_base[lane] = ti - t;
        if (lane == 31) s_total = ti;
    }
    __syncthreads();
    const long long total = s_total, base = warp_base[wid] + inc - c;
    if (threadIdx.x == 0) cnt[blockIdx.x] = (int)total;
    const long long m = total < S ? total : S;
    if (c == 0) return;
    int32_t *out = ids + (size_t)blockIdx.x * S;
    // the samples whose rank falls in this thread's [base, base + c): the first is i = ceil(base m / total)
    long long i = (base * m + total - 1) / total, r = i * total / m, rank = base;
    for (long long w = w0; w < w1 && i < m; w++) {
        const uint32_t x = accept_word(b, w, n);
        const int p = __popc(x);
        while (i < m && r < rank + p) {
            out[i] = (int32_t)(w * 32 + __fns(x, 0, (int)(r - rank) + 1));
            i++;
            r = i * total / m;
        }
        rank += p;
    }
}

cudaError_t launch_accept_compact(const uint32_t *bits_dev, long long stride_words, int nsets, long long n, int *cnt_dev, int32_t *ids_dev, cudaStream_t s)
{
    if (nsets <= 0) return cudaSuccess;
    accept_compact_kernel<<<nsets, ACC_THREADS, 0, s>>>(bits_dev, stride_words, n, accept_sample_size(n), cnt_dev, ids_dev);
    g_launches++;
    return cudaGetLastError();
}

// the rows of accept_compact_kernel's lists, scored by gather: grid = (chunks, nq); query q scores ids[q * ids_stride + i],
// i < min(cnt[q * cnt_stride], S), into scores[q * S + i]
template <int KIND, int METRIC>
__global__ void __launch_bounds__(RAGGED_THREADS) score_accepted_kernel(DataDesc d, const float *__restrict__ blobs, int blob_stride, const int32_t *__restrict__ ids,
                                                                        long long ids_stride, const int *__restrict__ cnt, int cnt_stride, int S,
                                                                        float *__restrict__ scores)
{
    constexpr int G = GroupOf<KIND>::value;
    constexpr int NG = RAGGED_THREADS / G;
    const int q = blockIdx.y;
    const int m = min(cnt[q * cnt_stride], S);
    const int c0 = blockIdx.x * RAGGED_CHUNK, c1 = min(m, c0 + RAGGED_CHUNK);
    const float *blob = blobs + (size_t)q * blob_stride;
    const int32_t *qi = ids + (size_t)q * ids_stride;
    const int group = threadIdx.x / G, lane = threadIdx.x % G;
    for (int i = c0 + group; i < c1; i += NG) {
        const float sc = score_row<KIND, METRIC>(d, blob, qi[i], lane);
        if (lane == 0) scores[(size_t)q * S + i] = sc;
    }
}

// Per query: the keys of its accepted list (keys below floor_key, the score threshold, masked), their best next_pow2(k) sorted.
// cnt <= S (whole tier): the list held every accepted row, so the best k are the answer. Otherwise the sampled thresholds of
// topk_threshold_kernel with the 6-sigma rank taken over the accepted count, each raised to floor_key.
__global__ void __launch_bounds__(256) topk_threshold_acc_kernel(const float *__restrict__ sample_scores, const int32_t *__restrict__ ids, long long ids_stride,
                                                                 const int *__restrict__ acc_cnt, int cnt_stride, int S, int S_pow2, int k, long long floor_key,
                                                                 long long *__restrict__ thr, long long *__restrict__ thr_safe, int *__restrict__ cnt,
                                                                 long long *__restrict__ keys_out)
{
    extern __shared__ long long skeys[];
    const int q = blockIdx.x;
    const int total = acc_cnt[q * cnt_stride], m = min(total, S);
    const int32_t *qi = ids + (size_t)q * ids_stride;
    for (int i = threadIdx.x; i < S_pow2; i += blockDim.x) {
        long long key = KEY_MIN;
        if (i < m) {
            key = topk_key(sample_scores[(size_t)q * S + i], qi[i]);
            if (key < floor_key) key = KEY_MIN;
        }
        skeys[i] = key;
    }
    __syncthreads();
    bitonic_top_desc(skeys, S_pow2, next_pow2(k));
    if (total <= S) {
        for (int i = threadIdx.x; i < k; i += blockDim.x) keys_out[(size_t)q * k + i] = skeys[i];
        if (threadIdx.x == 0) thr[q] = KEY_DONE;
        return;
    }
    if (threadIdx.x == 0) {
        const int j = aggressive_rank(k, S, total);
        const long long safe = max(skeys[k - 1], floor_key);
        thr_safe[q] = safe;
        thr[q] = j < k ? max(skeys[j - 1], floor_key) : safe;
        cnt[q] = 0;
    }
}

cudaError_t launch_topk_accepted(const DataDesc &d, int metric, const float *blobs_dev, int nq, int k, const AcceptLists &acc, long long floor_key,
                                 void *scratch_dev, long long *keys_out_dev, int *overflow_flag_dev, cudaStream_t s)
{
    if (nq <= 0) return cudaSuccess;
    cudaError_t e;
    const TopkScratch ts(d, nq, k, scratch_dev);
    const int S = ts.S;
    const int cs = acc.per_query ? 1 : 0;
    const long long is = acc.per_query ? S : 0;
    if (acc.max_listed > 0) {
        dim3 grid((acc.max_listed + RAGGED_CHUNK - 1) / RAGGED_CHUNK, nq);
        if (grid.y > 65535u) return cudaErrorInvalidValue;
#define CALL(K, M) score_accepted_kernel<K, M><<<grid, RAGGED_THREADS, 0, s>>>(d, blobs_dev, blob_floats(d), acc.ids, is, acc.cnt, cs, S, ts.sample_scores)
        JV_DISPATCH_KIND_METRIC(d.kind, metric, CALL);
#undef CALL
        g_launches++;
    }
    const int S2 = next_pow2(std::max(std::max(acc.max_listed, k), 1));
    if ((size_t)S2 * sizeof(long long) > 48 * 1024)
        if ((e = cudaFuncSetAttribute(topk_threshold_acc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, S2 * (int)sizeof(long long))) != cudaSuccess) return e;
    topk_threshold_acc_kernel<<<nq, 256, (size_t)S2 * sizeof(long long), s>>>(ts.sample_scores, acc.ids, is, acc.cnt, cs, S, S2, k, floor_key, ts.thr, ts.thr_safe, ts.cnt,
                                                                              keys_out_dev);
    g_launches++;
    if (acc.n_sampled == 0) return cudaGetLastError();
    return topk_filter_passes<true>(d, metric, blobs_dev, acc.n_sampled, acc.sampled, k, ts, acc.bits, acc.stride_words, keys_out_dev, overflow_flag_dev, s);
}

// ---- exhaustive search: NodeQueue.rerank's take rule over the candidates, exact rescoring, key order
// ids[q][i] = the candidate's node when it is reranked, else -1: a candidate is taken when its approximate score is >= floor, and the
// best one (i = 0, the keys are sorted) when none is
__global__ void __launch_bounds__(256) rerank_take_kernel(const long long *__restrict__ cand, int nq, int R, float floor, int32_t *__restrict__ ids,
                                                          int32_t *__restrict__ offsets, unsigned long long *__restrict__ taken)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t <= nq) offsets[t] = (int32_t)(t * R);  // query q's candidates are ids[q R .. (q + 1) R)
    bool take = false;
    if (t < (long long)nq * R) {
        const long long key = cand[t];
        take = key != KEY_MIN && (t % R == 0 || key_score(key) >= floor);
        ids[t] = take ? key_node(key) : -1;
    }
    const unsigned b = __ballot_sync(FULL, take);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(taken, (unsigned long long)__popc(b));
}

// one CTA per query: the topK best of its taken candidates by exact key (exact == nullptr: the first topK candidates as they are),
// nodes -1 and scores 0 past the end
__global__ void __launch_bounds__(256) rerank_finish_kernel(const long long *__restrict__ cand, const int32_t *__restrict__ ids, const float *__restrict__ exact, int R,
                                                            int R_pow2, int topK, int32_t *__restrict__ nodes, float *__restrict__ scores)
{
    extern __shared__ long long skeys[];
    const int q = blockIdx.x;
    const long long *src = cand + (size_t)q * R;
    if (exact) {
        for (int i = threadIdx.x; i < R_pow2; i += blockDim.x) {
            const int32_t f = i < R ? ids[(size_t)q * R + i] : -1;
            skeys[i] = f >= 0 ? topk_key(exact[(size_t)q * R + i], f) : KEY_MIN;
        }
        __syncthreads();
        bitonic_top_desc(skeys, R_pow2, next_pow2(topK));
        src = skeys;
    }
    for (int i = threadIdx.x; i < topK; i += blockDim.x) {
        const long long key = src[i];
        nodes[(size_t)q * topK + i] = key == KEY_MIN ? -1 : key_node(key);
        scores[(size_t)q * topK + i] = key == KEY_MIN ? 0.f : key_score(key);
    }
}

cudaError_t launch_rerank_accepted(const DataDesc *rr, int metric, const float *rblobs_dev, int nq, int R, int topK, float floor, const long long *cand_dev,
                                   int32_t *ids_dev, int32_t *offsets_dev, float *exact_dev, unsigned long long *taken_dev, int32_t *nodes_dev, float *scores_dev,
                                   cudaStream_t s)
{
    if (nq <= 0) return cudaSuccess;
    cudaError_t e;
    int R2 = 0;
    if (rr) {
        const long long threads = std::max((long long)nq * R, (long long)nq + 1);
        rerank_take_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(cand_dev, nq, R, floor, ids_dev, offsets_dev, taken_dev);
        g_launches++;
        if ((e = launch_score_ragged(*rr, metric, rblobs_dev, nq, ids_dev, offsets_dev, 0, R, exact_dev, s)) != cudaSuccess) return e;
        R2 = next_pow2(std::max(R, topK));
        if ((size_t)R2 * sizeof(long long) > 48 * 1024)
            if ((e = cudaFuncSetAttribute(rerank_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, R2 * (int)sizeof(long long))) != cudaSuccess) return e;
    }
    rerank_finish_kernel<<<nq, 256, (size_t)R2 * sizeof(long long), s>>>(cand_dev, ids_dev, rr ? exact_dev : nullptr, R, R2, topK, nodes_dev, scores_dev);
    g_launches++;
    return cudaGetLastError();
}

__global__ void add_int_kernel(int *dst, const int *src) { *dst += *src; }
cudaError_t launch_add_int(int *dst_dev, const int *src_dev, cudaStream_t s)
{
    add_int_kernel<<<1, 1, 0, s>>>(dst_dev, src_dev);
    g_launches++;
    return cudaGetLastError();
}

// the low word of a key is ~node: adding id_base to the node subtracts it from the key (no borrow: node + base < 2^31)
__global__ void __launch_bounds__(256) key_rebase_kernel(long long *keys, long long count, long long id_base)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count && keys[i] != KEY_MIN) keys[i] -= id_base;
}

cudaError_t launch_key_rebase(long long *keys_dev, long long count, long long id_base, cudaStream_t s)
{
    if (count <= 0) return cudaSuccess;
    key_rebase_kernel<<<(unsigned)((count + 255) / 256), 256, 0, s>>>(keys_dev, count, id_base);
    g_launches++;
    return cudaGetLastError();
}

// the only exchange step of the path (SURVEY §8e): per-shard top-k key arrays are all-gathered over NCCL, then merged here
__global__ void __launch_bounds__(256) topk_merge_kernel(const long long *__restrict__ in, int total, int total_pow2, int k, long long *__restrict__ out)
{
    extern __shared__ long long skeys[];
    const int q = blockIdx.x;
    for (int i = threadIdx.x; i < total_pow2; i += blockDim.x) skeys[i] = i < total ? in[(size_t)q * total + i] : KEY_MIN;
    __syncthreads();
    bitonic_sort_desc(skeys, total_pow2);
    for (int i = threadIdx.x; i < k; i += blockDim.x) out[(size_t)q * k + i] = i < total ? skeys[i] : KEY_MIN;
}

// the sort step of the strided merges: skeys[i] = load(p, j) for entry j of part p (i = p * k + j < parts * k), KEY_MIN past
// them, sorted descending
template <typename Load>
__device__ __forceinline__ void strided_load_sort(long long *skeys, int parts, int k, int total_pow2, Load load)
{
    const int total = parts * k;
    for (int i = threadIdx.x; i < total_pow2; i += blockDim.x) {
        const int p = i / k, j = i - p * k;
        skeys[i] = i < total ? load(p, j) : KEY_MIN;
    }
    __syncthreads();
    bitonic_sort_desc(skeys, total_pow2);
}

// same merge over the layout the peer copies produce: in [parts][nq][k]
__global__ void __launch_bounds__(256) topk_merge_strided_kernel(const long long *__restrict__ in, int nq, int parts, int k, int total_pow2, long long *__restrict__ out)
{
    extern __shared__ long long skeys[];
    const int q = blockIdx.x, total = parts * k;
    strided_load_sort(skeys, parts, k, total_pow2, [&](int p, int j) { return in[((size_t)p * nq + q) * k + j]; });
    for (int i = threadIdx.x; i < k; i += blockDim.x) out[(size_t)q * k + i] = i < total ? skeys[i] : KEY_MIN;
}

// the stable merge of jv_segments_search_batch over the segments' answers nodes_in / scores_in [parts][nq][k] (node -1 = padding):
// entry j of segment p is keyed (float_to_sortable(score) << 32) | ~((p << 12) | j), so that the key order (the greater key first)
// is the score descending, then the lower segment, then the earlier entry of that segment's list; padding is KEY_MIN. The first k
// keys are unpacked into (segment, node, score) read back from the inputs, padded with -1, -1, 0.
__global__ void __launch_bounds__(256) segment_merge_kernel(const int32_t *__restrict__ nodes_in, const float *__restrict__ scores_in, int nq, int parts, int k,
                                                            int total_pow2, int32_t *__restrict__ seg_out, int32_t *__restrict__ nodes_out,
                                                            float *__restrict__ scores_out)
{
    extern __shared__ long long skeys[];
    const int q = blockIdx.x;
    strided_load_sort(skeys, parts, k, total_pow2, [&](int p, int j) {
        const size_t at = ((size_t)p * nq + q) * k + j;
        if (nodes_in[at] < 0) return KEY_MIN;
        return (long long)(((unsigned long long)(uint32_t)float_to_sortable(scores_in[at]) << 32) | (unsigned long long)(uint32_t)~(uint32_t)((p << 12) | j));
    });
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        const long long key = skeys[i];
        const size_t o = (size_t)q * k + i;
        if (key == KEY_MIN) {
            seg_out[o] = -1;
            nodes_out[o] = -1;
            scores_out[o] = 0.f;
        } else {
            const uint32_t tag = ~(uint32_t)((unsigned long long)key & 0xffffffffull);
            const int p = (int)(tag >> 12), j = (int)(tag & 4095u);
            const size_t at = ((size_t)p * nq + q) * k + j;
            seg_out[o] = p;
            nodes_out[o] = nodes_in[at];
            scores_out[o] = scores_in[at];
        }
    }
}

cudaError_t launch_segment_merge(const int32_t *nodes_in_dev, const float *scores_in_dev, int nq, int parts, int k, int32_t *seg_out_dev, int32_t *nodes_out_dev,
                                 float *scores_out_dev, cudaStream_t s)
{
    if (k > SEGMENT_MERGE_MAX_K || (long long)parts * k > SEGMENT_MERGE_MAX_KEYS) return cudaErrorInvalidValue;
    const int p2 = next_pow2(parts * k);
    cudaError_t e;
    if ((size_t)p2 * 8 > 48 * 1024)
        if ((e = cudaFuncSetAttribute(segment_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, p2 * 8)) != cudaSuccess) return e;
    segment_merge_kernel<<<nq, 256, (size_t)p2 * 8, s>>>(nodes_in_dev, scores_in_dev, nq, parts, k, p2, seg_out_dev, nodes_out_dev, scores_out_dev);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_topk_merge_strided(const long long *keys_in_dev, int nq, int parts, int k, long long *keys_out_dev, cudaStream_t s)
{
    const int total = parts * k, p2 = next_pow2(total);
    cudaError_t e;
    if ((size_t)p2 * 8 > 48 * 1024)
        if ((e = cudaFuncSetAttribute(topk_merge_strided_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, p2 * 8)) != cudaSuccess) return e;
    topk_merge_strided_kernel<<<nq, 256, (size_t)p2 * 8, s>>>(keys_in_dev, nq, parts, k, p2, keys_out_dev);
    g_launches++;
    return cudaGetLastError();
}

cudaError_t launch_topk_merge(const long long *keys_in_dev, int nq, int parts, int k, long long *keys_out_dev, cudaStream_t s)
{
    const int total = parts * k, p2 = next_pow2(total);
    cudaError_t e;
    if ((size_t)p2 * 8 > 48 * 1024)
        if ((e = cudaFuncSetAttribute(topk_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, p2 * 8)) != cudaSuccess) return e;
    topk_merge_kernel<<<nq, 256, (size_t)p2 * 8, s>>>(keys_in_dev, total, p2, k, keys_out_dev);
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// FusedPQ.writeInline (base:graph/disk/feature/FusedPQ.java:122-141): one record per node = its level-0 neighbour ids followed by
// the neighbours' PQ codes in neighbour order, zero padded to the full degree. One warp per (node, neighbour slot) code row.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) fuse_pq_kernel(const int32_t *__restrict__ adj0, int n, int degree, const uint8_t *__restrict__ codes, int code_stride,
                                                      uint8_t *__restrict__ records, int rec_bytes)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= (long long)n * degree) return;
    const int node = (int)(warp / degree), slot = (int)(warp - (long long)node * degree);
    uint8_t *rec = records + (size_t)node * rec_bytes;
    const int32_t f = adj0[(size_t)node * degree + slot];
    if (lane == 0) reinterpret_cast<int32_t *>(rec)[slot] = f;
    uint32_t *dst = reinterpret_cast<uint32_t *>(rec + 4 * degree + (size_t)slot * code_stride);
    const uint32_t *src = f >= 0 ? reinterpret_cast<const uint32_t *>(codes + (size_t)f * code_stride) : nullptr;
    for (int i = lane; i < (code_stride >> 2); i += 32) dst[i] = src ? src[i] : 0u;
    // bytes between the last code row and the 16-byte rounded record end
    if (slot == degree - 1)
        for (int o = 4 * degree + degree * code_stride + lane; o < rec_bytes; o += 32) rec[o] = 0;
}

cudaError_t launch_fuse_pq(const GraphDesc &g, const DataDesc &pq, uint8_t *records_dev, int rec_bytes, cudaStream_t s)
{
    const long long warps = (long long)g.n * g.degree;
    const long long blocks = (warps * 32 + 255) / 256;
    if (blocks > 0x7fffffffLL) return cudaErrorInvalidValue;
    fuse_pq_kernel<<<(unsigned)blocks, 256, 0, s>>>(g.adj0, g.n, g.degree, pq.codes, pq.code_stride, records_dev, rec_bytes);
    g_launches++;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// bulk encoders
// ------------------------------------------------------------------------------------------------
// BinaryQuantization.encodeTo (BinaryQuantization.java:96-109): one warp per 32 dimensions via ballot
__global__ void __launch_bounds__(256) bq_encode_kernel(const float *__restrict__ rows, long long n, int dim, int row_stride, unsigned *__restrict__ halves, int halves_per_row)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const long long total = n * halves_per_row;
    if (warp >= total) return;
    const long long r = warp / halves_per_row;
    const int h = (int)(warp - r * halves_per_row);
    const int idx = h * 32 + lane;
    const bool bit = idx < dim && rows[r * row_stride + idx] > 0.f;
    const unsigned b = __ballot_sync(FULL, bit);
    if (lane == 0) halves[warp] = b;
}

cudaError_t launch_bq_encode(const float *rows_dev, long long n, int dim, int row_stride, unsigned long long *words_dev, cudaStream_t s)
{
    if (n <= 0) return cudaSuccess;
    const int hp = 2 * ((dim + 63) / 64);
    const long long warps = n * hp;
    const long long blocks = (warps * 32 + 255) / 256;
    bq_encode_kernel<<<(unsigned)blocks, 256, 0, s>>>(rows_dev, n, dim, row_stride, reinterpret_cast<unsigned *>(words_dev), hp);
    g_launches++;
    return cudaGetLastError();
}

// Row sketch of an fp32 data set (the bound of sketch_bound_pair, scorers.cuh): one warp per row. s = max|x| / 127, codes
// round(x / s) in [-127, 127] (all 0 for a zero row), x_hat = s c. The radius r = ||x - x_hat|| + gamma (||x|| + ||x_hat||),
// gamma = (stride + 8) 2^-23, is summed in fp64 rounding every step upward (x - x_hat itself is exact in fp64) and rounded up to
// fp32. Padding codes up to sketch_stride are zero.
__global__ void __launch_bounds__(256) row_sketch_kernel(const float *__restrict__ rows, long long n, int stride, int sketch_stride, int8_t *__restrict__ sketch,
                                                         float2 *__restrict__ meta)
{
    const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n) return;
    const float *x = rows + r * stride;
    float m = 0.f;
    for (int i = lane; i < stride; i += 32) m = fmaxf(m, fabsf(x[i]));
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(FULL, m, o));
    const float s = __fdiv_rn(m, 127.0f);
    double dd = 0.0, xx = 0.0, hh = 0.0;
    for (int i = lane; i < sketch_stride; i += 32) {
        const float v = i < stride ? x[i] : 0.f;
        const int c = s > 0.f ? min(127, max(-127, __float2int_rn(__fdiv_rn(v, s)))) : 0;
        sketch[r * sketch_stride + i] = (int8_t)c;
        const double xh = (double)c * (double)s, df = (double)v - xh;
        dd = __dadd_ru(dd, __dmul_ru(df, df));
        xx = __dadd_ru(xx, __dmul_ru((double)v, (double)v));
        hh = __dadd_ru(hh, __dmul_ru(xh, xh));
    }
    for (int o = 16; o; o >>= 1) {
        dd = __dadd_ru(dd, __shfl_xor_sync(FULL, dd, o));
        xx = __dadd_ru(xx, __shfl_xor_sync(FULL, xx, o));
        hh = __dadd_ru(hh, __shfl_xor_sync(FULL, hh, o));
    }
    if (lane == 0) {
        const double gamma = (double)(stride + 8) * 0x1p-23;
        const double rad = __dadd_ru(__dsqrt_ru(dd), __dmul_ru(gamma, __dadd_ru(__dsqrt_ru(xx), __dsqrt_ru(hh))));
        meta[r] = make_float2(s, __double2float_ru(rad));
    }
}

cudaError_t launch_row_sketch(const float *rows_dev, long long n, int stride, int sketch_stride, int8_t *sketch_dev, float2 *meta_dev, cudaStream_t s)
{
    if (n <= 0) return cudaSuccess;
    const long long blocks = (n * 32 + 255) / 256;
    row_sketch_kernel<<<(unsigned)blocks, 256, 0, s>>>(rows_dev, n, stride, sketch_stride, sketch_dev, meta_dev);
    g_launches++;
    return cudaGetLastError();
}

// Basis of the low-rank edge bound (scorers.cuh lowrank_bound): subspace iteration V <- orth(X^T (X V)) over the rows s * step,
// s < S, in float64; the orthonormalisation of the LR_K columns runs on the host (api.cu ensure_lowrank). Z = X V: one warp per
// sampled row. Y = X^T Z: one thread per (column j, coordinate i).
__global__ void __launch_bounds__(256) lowrank_project_kernel(const float *__restrict__ rows, int stride, long long step, int S, const double *__restrict__ V,
                                                              double *__restrict__ Z)
{
    const int sr = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (sr >= S) return;
    const float *x = rows + (size_t)sr * step * stride;
    for (int j = 0; j < LR_K; j++) {
        double a = 0.0;
        for (int i = lane; i < stride; i += 32) a = fma((double)x[i], V[(size_t)j * stride + i], a);
        for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(FULL, a, o);
        if (lane == 0) Z[(size_t)sr * LR_K + j] = a;
    }
}

__global__ void __launch_bounds__(256) lowrank_gram_kernel(const float *__restrict__ rows, int stride, long long step, int S, const double *__restrict__ Z,
                                                           double *__restrict__ Y)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
    if (i >= stride) return;
    double a = 0.0;
    for (int sr = 0; sr < S; sr++) a = fma((double)rows[(size_t)sr * step * stride + i], Z[(size_t)sr * LR_K + j], a);
    Y[(size_t)j * stride + i] = a;
}

cudaError_t launch_lowrank_iteration(const float *rows_dev, int stride, long long step, int S, const double *V_dev, double *Z_dev, double *Y_dev, cudaStream_t s)
{
    lowrank_project_kernel<<<(unsigned)((S * 32 + 255) / 256), 256, 0, s>>>(rows_dev, stride, step, S, V_dev, Z_dev);
    lowrank_gram_kernel<<<dim3((unsigned)((stride + 127) / 128), LR_K), 128, 0, s>>>(rows_dev, stride, step, S, Z_dev, Y_dev);
    g_launches += 2;
    return cudaGetLastError();
}

// Low-rank rows (scorers.cuh lowrank_bound): one warp per row, float64 throughout. a = B^T x, t = max|a_j| / 127 rounded to fp32,
// c = round(a / t) in [-127, 127] (0 when t = 0), w = x - t B c with each w_i within lr_g64(LR_K + 2) A_i, A_i = |x_i| + t sum_j |B_ij c_j|,
// so rho = ||w~|| + g ||A|| >= ||w||; |(B^T w)_j| <= |(B^T w~)_j| + lr_g64(stride + LR_K + 2) sum_i |B_ij| (|w~_i| + A_i) gives beta.
// Out: [n][LR_SLOT] = LR_K int8 codes, then {t, rho, beta, xn} rounded up. w~ and A are staged in shared memory, 2 stride doubles
// per warp.
__global__ void lowrank_rows_kernel(const float *__restrict__ rows, long long n, int stride, const float *__restrict__ B, uint8_t *__restrict__ out)
{
    extern __shared__ double lr_stage[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + wib;
    if (r >= n) return;
    double *ws = lr_stage + (size_t)wib * 2 * stride, *as = ws + stride;
    const float *x = rows + r * stride;
    double aj = 0.0;  // lane j: a_j
    for (int j = 0; j < LR_K; j++) {
        double a = 0.0;
        for (int i = lane; i < stride; i += 32) a = fma((double)__ldg(B + (size_t)j * stride + i), (double)x[i], a);
        for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(FULL, a, o);
        if (lane == j) aj = a;
    }
    double amax = fabs(aj);
    for (int o = 16; o; o >>= 1) amax = fmax(amax, __shfl_xor_sync(FULL, amax, o));
    const float t = (float)(amax / 127.0);
    const int cj = t > 0.f ? (int)fmin(127.0, fmax(-127.0, rint(aj / (double)t))) : 0;
    out[r * LR_SLOT + lane] = (uint8_t)(int8_t)cj;
    double w2 = 0.0, a2 = 0.0, x2 = 0.0;
    for (int i0 = 0; i0 < stride; i0 += 32) {  // every lane runs every step: the code shuffles below name the whole warp
        const int i = i0 + lane;
        double v = 0.0, av = 0.0;
        for (int j = 0; j < LR_K; j++) {
            const double c = (double)__shfl_sync(FULL, cj, j);
            const double bc = i < stride ? (double)__ldg(B + (size_t)j * stride + i) * c : 0.0;
            v += bc;
            av += fabs(bc);
        }
        if (i >= stride) continue;
        const double xi = (double)x[i];
        const double w = xi - (double)t * v, A = fabs(xi) + (double)t * av;
        ws[i] = w;
        as[i] = A;
        w2 = fma(w, w, w2);
        a2 = fma(A, A, a2);
        x2 = fma(xi, xi, x2);
    }
    __syncwarp();
    double bj = 0.0;  // lane j: |(B^T w~)_j| + its error bound
    const double gb = lr_g64(stride + LR_K + 2);
    for (int j = 0; j < LR_K; j++) {
        double bw = 0.0, ab = 0.0;
        for (int i = lane; i < stride; i += 32) {
            const double b = (double)__ldg(B + (size_t)j * stride + i);
            bw = fma(b, ws[i], bw);
            ab = fma(fabs(b), fabs(ws[i]) + as[i], ab);
        }
        for (int o = 16; o; o >>= 1) {
            bw += __shfl_xor_sync(FULL, bw, o);
            ab += __shfl_xor_sync(FULL, ab, o);
        }
        if (lane == j) bj = fabs(bw) + gb * ab;
    }
    double b2 = bj * bj;
    for (int o = 16; o; o >>= 1) {
        b2 += __shfl_xor_sync(FULL, b2, o);
        w2 += __shfl_xor_sync(FULL, w2, o);
        a2 += __shfl_xor_sync(FULL, a2, o);
        x2 += __shfl_xor_sync(FULL, x2, o);
    }
    if (lane == 0) {
        const float rho = __double2float_ru((sqrt(w2 * LR_PAD) + lr_g64(LR_K + 2) * sqrt(a2 * LR_PAD)) * LR_PAD);
        const float beta = __double2float_ru(sqrt(b2 * LR_PAD) * LR_PAD), xn = __double2float_ru(sqrt(x2 * LR_PAD) * LR_PAD);
        *reinterpret_cast<float4 *>(out + r * LR_SLOT + LR_K) = make_float4(t, rho, beta, xn);
    }
}

// rows per block of lowrank_rows_kernel for rows of `stride` floats (0: the staging does not fit in shared memory)
int lowrank_warps(int stride)
{
    const long long per = 16ll * stride;
    return per > 200 * 1024 ? 0 : (int)std::min(4ll, (200 * 1024) / per);
}

cudaError_t launch_lowrank_rows(const float *rows_dev, long long n, int stride, const float *B_dev, uint8_t *out_dev, cudaStream_t s)
{
    const int w = lowrank_warps(stride);
    if (w == 0 || n <= 0) return cudaSuccess;
    const size_t smem = (size_t)w * 16 * stride;
    cudaError_t e = cudaFuncSetAttribute(lowrank_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    lowrank_rows_kernel<<<(unsigned)((n + w - 1) / w), 32 * w, smem, s>>>(rows_dev, n, stride, B_dev, out_dev);
    g_launches++;
    return cudaGetLastError();
}

__global__ void __launch_bounds__(128) lowrank_bound_pairs_kernel(DataDesc d, const float *__restrict__ queries, const uint8_t *__restrict__ records, float *__restrict__ out)
{
    extern __shared__ __align__(16) float pair_blob[];
    __shared__ float red[36], lr[LR_QUERY];
    const long long i = blockIdx.x;
    prepare_blob<128>(d, JV_METRIC_DOT, queries + i * d.stride, pair_blob, red);
    prepare_lowrank<128>(d.lr_basis, d.stride, pair_blob, lr);
    if (threadIdx.x == 0) {
        const uint4 *e = reinterpret_cast<const uint4 *>(records + i * LR_SLOT);
        float est;
        out[i] = lowrank_bound(d, pair_blob, lr, e[0], e[1], *reinterpret_cast<const float4 *>(e + 2), est);
    }
}

cudaError_t launch_lowrank_bound_pairs(const float *B_dev, int dim, int stride, const float *queries_dev, const uint8_t *records_dev, long long n, float *out_dev, cudaStream_t s)
{
    if (n <= 0) return cudaSuccess;
    DataDesc d;
    memset(&d, 0, sizeof(d));
    d.kind = KIND_F32;
    d.dim = dim;
    d.stride = stride;
    d.n = n;
    d.lr_basis = B_dev;
    lowrank_bound_pairs_kernel<<<(unsigned)n, 128, (size_t)(stride + 4) * 4, s>>>(d, queries_dev, records_dev, out_dev);
    g_launches++;
    return cudaGetLastError();
}

// a graph's edge records: slot t of node v = the low-rank row of adj0[v][t] (zeros for an empty slot), 16 bytes per thread
__global__ void __launch_bounds__(256) edge_records_kernel(const int32_t *__restrict__ adj0, long long slots, const uint4 *__restrict__ lr_rows, uint4 *__restrict__ rec)
{
    constexpr int P = LR_SLOT / 16;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= slots * P) return;
    const int32_t f = __ldg(adj0 + i / P);
    rec[i] = f >= 0 ? __ldg(lr_rows + (size_t)f * P + i % P) : make_uint4(0, 0, 0, 0);
}

cudaError_t launch_edge_records(const int32_t *adj0_dev, long long n, int degree, const uint8_t *lr_rows_dev, uint8_t *rec_dev, cudaStream_t s)
{
    const long long items = n * degree * (LR_SLOT / 16);
    if (items <= 0) return cudaSuccess;
    edge_records_kernel<<<(unsigned)((items + 255) / 256), 256, 0, s>>>(adj0_dev, n * degree, reinterpret_cast<const uint4 *>(lr_rows_dev), reinterpret_cast<uint4 *>(rec_dev));
    g_launches++;
    return cudaGetLastError();
}

// ProductQuantization.encode (ProductQuantization.java:507-520): code[m] = argmin_c ||v[off_m..] - centroid_{m,c}||^2, first
// minimum wins. One warp per (row, subspace); lanes stride over the k centroids, then an arg-min shuffle that prefers
// the smaller index on ties.
__global__ void __launch_bounds__(256) pq_encode_kernel(DataDesc pq, const float *__restrict__ rows, long long n, int row_stride, uint8_t *__restrict__ codes)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= n * pq.M) return;
    const long long r = warp / pq.M;
    const int m = (int)(warp - r * pq.M);
    const int sz = pq.sub_sizes[m], off = pq.sub_offsets[m];
    const float *v = rows + r * row_stride + off;
    const float *cb = pq.codebooks + (size_t)pq.k * off;
    float best = __int_as_float(0x7f800000);
    int bi = 0x7fffffff;
    for (int c = lane; c < pq.k; c += 32) {
        const float *cen = cb + (size_t)c * sz;
        float s = 0.f;
        for (int j = 0; j < sz; j++) {
            float x = v[j];
            if (pq.centroid) x = __fsub_rn(x, pq.centroid[off + j]);
            // squareDistance(codebook, c*size, vector, off, size): (a - b)^2 accumulated in order
            const float df = __fsub_rn(cen[j], x);
            s = __fadd_rn(s, __fmul_rn(df, df));
        }
        if (s < best) { best = s; bi = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(FULL, best, o);
        const int oi = __shfl_xor_sync(FULL, bi, o);
        if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) codes[r * pq.M + m] = (uint8_t)(bi == 0x7fffffff ? 0 : bi);
}

cudaError_t launch_pq_encode(const DataDesc &pq, const float *rows_dev, long long n, int row_stride, uint8_t *codes_dev, cudaStream_t s)
{
    if (n <= 0) return cudaSuccess;
    const long long warps = n * pq.M;
    const long long blocks = (warps * 32 + 255) / 256;
    if (blocks > 0x7fffffffLL) return cudaErrorInvalidValue;
    pq_encode_kernel<<<(unsigned)blocks, 256, 0, s>>>(pq, rows_dev, n, row_stride, codes_dev);
    g_launches++;
    return cudaGetLastError();
}

// ProductQuantization.createCodebookPartialSums (ProductQuantization.java:609-628): for every sub-space the upper triangle
// (i <= j) of centroid-vs-centroid dot products or squared L2 distances, rows in order. One thread per entry.
__global__ void __launch_bounds__(256) pq_pair_table_kernel(DataDesc pq, int euclidean, float *__restrict__ table)
{
    const int block = pq.k * (pq.k + 1) / 2;
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)pq.M * block) return;
    const int m = (int)(e / block), t = (int)(e - (long long)m * block);
    // invert t = i k - i (i - 1) / 2 + (j - i): i = the largest row whose first entry is <= t
    int i = (int)((2.0 * pq.k + 1.0 - sqrt((2.0 * pq.k + 1.0) * (2.0 * pq.k + 1.0) - 8.0 * t)) / 2.0);
    while (i > 0 && i * pq.k - i * (i - 1) / 2 > t) i--;
    while ((i + 1) * pq.k - (i + 1) * i / 2 <= t) i++;
    const int j = i + (t - (i * pq.k - i * (i - 1) / 2));
    const int sz = pq.sub_sizes[m];
    const float *cb = pq.codebooks + (size_t)pq.k * pq.sub_offsets[m];
    const float *x = cb + (size_t)i * sz, *y = cb + (size_t)j * sz;
    float s = 0.f;
    for (int c = 0; c < sz; c++) {
        if (euclidean) {
            const float df = __fsub_rn(x[c], y[c]);
            s = fmaf(df, df, s);
        } else s = fmaf(x[c], y[c], s);
    }
    table[e] = s;
}

cudaError_t launch_pq_pair_table(const DataDesc &pq, int euclidean, float *table_dev, cudaStream_t s)
{
    const long long total = (long long)pq.M * (pq.k * (pq.k + 1) / 2);
    pq_pair_table_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(pq, euclidean, table_dev);
    g_launches++;
    return cudaGetLastError();
}

// KMeansPlusPlusClusterer.getNearestCluster (base:quantization/KMeansPlusPlusClusterer.java:329-342) for a batch of points: the
// assignment step of Lloyd's iterations (and, per sub-space, what ProductQuantization.encode does). One warp per point, lanes
// stride over the centroids, first minimum wins.
__global__ void __launch_bounds__(256) kmeans_assign_kernel(const float *__restrict__ points, long long n, int dim, int point_stride,
                                                            const float *__restrict__ centroids, int k, int32_t *__restrict__ assign)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= n) return;
    const float *v = points + warp * point_stride;
    float best = 3.402823466e+38f;  // Float.MAX_VALUE
    int bi = 0x7fffffff;
    for (int c = lane; c < k; c += 32) {
        const float *cen = centroids + (size_t)c * dim;
        float s = 0.f;
        for (int j = 0; j < dim; j++) {
            const float df = __fsub_rn(v[j], cen[j]);
            s = __fadd_rn(s, __fmul_rn(df, df));
        }
        if (s < best) { best = s; bi = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(FULL, best, o);
        const int oi = __shfl_xor_sync(FULL, bi, o);
        if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) assign[warp] = bi == 0x7fffffff ? 0 : bi;
}

cudaError_t launch_kmeans_assign(const float *points_dev, long long n, int dim, int point_stride, const float *centroids_dev, int k, int32_t *assign_dev, cudaStream_t s)
{
    if (n <= 0) return cudaSuccess;
    const long long blocks = (n * 32 + 255) / 256;
    if (blocks > 0x7fffffffLL) return cudaErrorInvalidValue;
    kmeans_assign_kernel<<<(unsigned)blocks, 256, 0, s>>>(points_dev, n, dim, point_stride, centroids_dev, k, assign_dev);
    g_launches++;
    return cudaGetLastError();
}

// calculatePartialSelfMagnitudes (PQDecoder.java:93-105): mag[m*k + c] = ||centroid_{m,c}||^2, query independent
__global__ void __launch_bounds__(256) pq_self_mag_kernel(DataDesc pq, float *__restrict__ mag)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= pq.M * pq.k) return;
    const int m = e / pq.k, c = e - m * pq.k;
    const int sz = pq.sub_sizes[m];
    const float *cen = pq.codebooks + (size_t)pq.k * pq.sub_offsets[m] + (size_t)c * sz;
    float s = 0.f;
    for (int j = 0; j < sz; j++) s = fmaf(cen[j], cen[j], s);
    mag[e] = s;
}

cudaError_t launch_pq_self_magnitudes(const DataDesc &pq, float *mag_dev, cudaStream_t s)
{
    const int total = pq.M * pq.k;
    pq_self_mag_kernel<<<(total + 255) / 256, 256, 0, s>>>(pq, mag_dev);
    g_launches++;
    return cudaGetLastError();
}

// NVQuantization.encodeTo + QuantizedSubVector.quantizeTo (NVQuantization.java:211-214,524-578): one warp per
// (row, sub-vector): min/max, optional growth-rate grid search (20 coarse + 20 fine nvqLoss evaluations against the
// uniform-loss baseline), then nvqQuantize8bit. Follows the native kernels' arithmetic (native-c:...:1149-1303).
__device__ __forceinline__ float nvq_loss_warp(const float *v, const float *mean, int n, float alpha, float minv, float maxv, int lane)
{
    const NvqConsts c = nvq_setup(minv, maxv, alpha, 0.f, 255.0f);
    const float inv = __fdiv_rn(1.0f, c.scale);
    float s = 0.f;
    for (int i = lane; i < n; i += 32) {
        const float x = __fsub_rn(v[i], mean[i]);
        const float r = __fmul_rn(__fsub_rn(nvq_logistic(x, c.sa, c.sx0), c.bias), inv);
        const float rq = (float)__float2int_rz(__fadd_rn(r, 0.5f));
        const float df = __fsub_rn(x, nvq_dequant(c, rq));
        s = __fmaf_rn(df, df, s);
    }
    return group_sum<32>(s);
}

__global__ void __launch_bounds__(256) nvq_encode_kernel(const float *__restrict__ rows, long long n, int row_stride, int nsub, const int *__restrict__ sizes,
                                                         const int *__restrict__ offsets, const float *__restrict__ mean, int learn,
                                                         float *__restrict__ params, uint8_t *__restrict__ bytes, int byte_stride)
{
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= n * nsub) return;
    const long long r = warp / nsub;
    const int sv = (int)(warp - r * nsub);
    const int sz = sizes[sv], off = offsets[sv];
    const float *v = rows + r * row_stride + off;
    const float *mu = mean + off;
    float minv = 3.402823466e+38f, maxv = -3.402823466e+38f;
    for (int i = lane; i < sz; i += 32) {
        const float x = __fsub_rn(v[i], mu[i]);
        minv = fminf(minv, x);
        maxv = fmaxf(maxv, x);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        minv = fminf(minv, __shfl_xor_sync(FULL, minv, o));
        maxv = fmaxf(maxv, __shfl_xor_sync(FULL, maxv, o));
    }
    float growth = 1e-2f;
    if (learn) {
        // baseline = nvqUniformLoss (native-c:...:1258-1303)
        const float constant = 255.0f, delta = __fsub_rn(maxv, minv);
        float us = 0.f;
        for (int i = lane; i < sz; i += 32) {
            const float x = __fsub_rn(v[i], mu[i]);
            const float rr = __fmul_rn(__fsub_rn(x, minv), __fdiv_rn(constant, delta));
            const float rq = (float)__float2int_rz(__fadd_rn(rr, 0.5f));
            const float rec = __fmaf_rn(rq, __fdiv_rn(delta, constant), minv);
            const float df = __fsub_rn(x, rec);
            us = __fmaf_rn(df, df, us);
        }
        const float baseline = group_sum<32>(us);
        float coarse = 1e-2f, best = 1.40129846e-45f;
        for (float gr = 1e-6f; gr < 20.f; gr = __fadd_rn(gr, 1.f)) {
            const float lv = __fdiv_rn(baseline, nvq_loss_warp(v, mu, sz, gr, minv, maxv, lane));
            if (lv > best) { best = lv; coarse = gr; }
        }
        float fine = coarse;
        for (float gr = __fsub_rn(coarse, 1.f); gr < __fadd_rn(coarse, 1.f); gr = __fadd_rn(gr, 0.1f)) {
            const float lv = __fdiv_rn(baseline, nvq_loss_warp(v, mu, sz, gr, minv, maxv, lane));
            if (lv > best) { best = lv; fine = gr; }
        }
        growth = fine;
    }
    // nvq_quantize_8bit (native-c:...:1149-1197); the reference build fuses (L - bias) * inv + 0.5 into one fma
    {
        const float delta = __fsub_rn(maxv, minv), sa = __fdiv_rn(growth, delta), sx0 = __fmul_rn(0.f, delta);
        const float bias = nvq_logistic(minv, sa, sx0);
        const float inv = __fdiv_rn(255.0f, __fsub_rn(nvq_logistic(maxv, sa, sx0), bias));
        uint8_t *dst = bytes + r * byte_stride + off;
        for (int i = lane; i < sz; i += 32) {
            const float x = __fsub_rn(v[i], mu[i]);
            const float a = __fmaf_rn(__fsub_rn(nvq_logistic(x, sa, sx0), bias), inv, 0.5f);
            const int qv = __float2int_rz(a);
            dst[i] = (uint8_t)(qv < 0 ? 0 : qv > 255 ? 255 : qv);
        }
    }
    if (lane == 0) {
        float4 p = make_float4(minv, maxv, growth, 0.f);
        reinterpret_cast<float4 *>(params)[warp] = p;
    }
}

cudaError_t launch_nvq_encode(const float *rows_dev, long long n, int row_stride, int nsub, const int *sizes_dev, const int *offsets_dev,
                              const float *mean_dev, int learn, float *params_dev, uint8_t *bytes_dev, int byte_stride, cudaStream_t s)
{
    if (n <= 0) return cudaSuccess;
    const long long warps = n * nsub;
    const long long blocks = (warps * 32 + 255) / 256;
    if (blocks > 0x7fffffffLL) return cudaErrorInvalidValue;
    nvq_encode_kernel<<<(unsigned)blocks, 256, 0, s>>>(rows_dev, n, row_stride, nsub, sizes_dev, offsets_dev, mean_dev, learn, params_dev, bytes_dev, byte_stride);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace jv
