// bq_imma.cu — exhaustive BQ (Hamming) top-k as an exact integer contraction on the tensor cores.
//
// BQVectors.similarityBetween (base:quantization/BQVectors.java:116-118) scores a pair by 1 - hd / dim with
// hd = popcount(a ^ b) (base:vector/DefaultVectorUtilSupport.java:342-348). For a batch of queries against every row that is
// a dense binary contraction: hd = popc(a) + popc(b) - 2 * <a, b> over {0,1} operands, and <a, b> accumulates exactly in
// int32. The kernel expands bit words to {0,1} bytes in registers and feeds IMMA.16832 (mma.sync m16n8k32 u8 x u8 -> s32,
// native SASS on sm_90a), so a popcount loop (POPC / LOP3 bound) becomes tensor-pipe bound. Integer arithmetic: keys are bit-identical to the
// scalar restatement.
//
// Top-k without a sort of the scores: Hamming distances live in [0, dim], so thresholds are integers.
//   1. pack the queries to bit words, popcount them;
//   2. SAMPLE pass: the same contraction over S strided rows -> hd matrix [nq][S] (u16);
//   3. per query, a histogram of the sample over [0, dim] gives thr (aggressive: the j-th smallest sample distance with
//      j - 6 sqrt(j) >= k S / n, so fewer than k survivors is a > 6 sigma event) and safe (the k-th smallest: a guaranteed bound);
//   4. FILTER pass over all rows: (row, query) pairs with hd <= thr[q] append their 64-bit reference key to a per-query buffer;
//   5. per query: histogram of the captured keys over hd -> boundary bin -> the few keys at or under it are sorted (<= 2 k).
//      A query with fewer than k survivors (or an overflowed buffer) is redone with the safe (or a tightened) threshold by
//      the same kernels over a query list; the redo launches are unconditional and exit at once when the list is empty, so
//      the common path has no host synchronisation.
// Row ids inside the keys are global (local row + id_base), so the keys can be the NCCL send buffer of a range-sharded base.
#include <limits.h>
#include <stdlib.h>

#include "kernels.h"

namespace jv {

namespace {

constexpr int BM = 128;        // rows per CTA tile
constexpr int BN = 128;        // queries per CTA tile
constexpr int IMMA_THREADS = 256;
constexpr int WM = 32, WN = 64;  // warp tile: 2 m16 x 8 n8 IMMA tiles, 64 int32 accumulators per thread
constexpr long long KEY_DONE = 0x7fffffffffffffffLL;

__device__ __forceinline__ void imma_16832(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// BinaryQuantization.encodeTo for the queries (BQVectors.java:109 encodes the query like a row): one warp per 32 dimensions.
// qbits [nq_pad][W32] (rows >= nq are zero), pb[q] = popcount of the query's bits.
__global__ void __launch_bounds__(256) bq_pack_queries_kernel(const float *__restrict__ queries, int nq, int nq_pad, int dim, int W32,
                                                              uint32_t *__restrict__ qbits, int *__restrict__ pb)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= nq_pad) return;
    int pc = 0;
    for (int h = 0; h < W32; h++) {
        const int idx = h * 32 + lane;
        const bool bit = warp < nq && idx < dim && queries[(size_t)warp * dim + idx] > 0.f;
        const unsigned b = __ballot_sync(FULL, bit);
        if (lane == 0) qbits[(size_t)warp * W32 + h] = b;
        pc += __popc(b);
    }
    if (lane == 0) pb[warp] = pc;
}

struct ImmaParams {
    const uint32_t *rows;   // [n][W32] (the registered BQ words viewed as 32-bit halves)
    long long n;
    int W32, dim;
    const uint32_t *qbits;  // [nq_pad][W32]
    int nq_pad, nq;
    const int *qlist;       // redo passes: the query tile gathers qlist[0 .. *n_active); nullptr = identity over nq_pad
    const int *n_active;    // device count of active queries (nullptr: nq_pad)
    // MODE 0 (filter)
    const int *t2;          // [nq_pad] thr[q] - pb[q]; a pair passes iff pa[row] - 2 <a,b> <= t2[q]
    const int *pb;          // [nq_pad]
    long long *buf;         // [nq][cap]
    int *cnt;               // [nq]
    int cap;
    long long id_base;
    // MODE 1 (sample)
    int S;                  // sampled rows: row(s) = s * n / S
    unsigned short *hdm;    // [nq_pad][S]
};

// One CTA: BM rows x BN queries over the whole K = 32 * W32 bits. Bit words of both tiles sit in shared memory (row pitch W32 + 4
// words: 128-bit loads of 8 rows hit 32 distinct banks); every k-step expands 4 row words and 8 query words per lane into
// IMMA fragments: lane (g = lane / 4, t = lane % 4) takes bits {2t + 8m} and {2t + 1 + 8m} (m = 0..3) of the word of row g —
// the same positions on both operands, which is all an inner product needs.
template <int MODE>
__global__ void __launch_bounds__(IMMA_THREADS, 2) bq_imma_kernel(ImmaParams P)
{
    extern __shared__ __align__(16) uint32_t sm[];
    const int pitch = P.W32 + 4;
    uint32_t *As = sm;                          // [BM][pitch]
    uint32_t *Bs = As + BM * pitch;             // [BN][pitch]
    int *pa = reinterpret_cast<int *>(Bs + BN * pitch);  // [BM] popcount of each row
    int *t2s = pa + BM;                         // [BN]
    int *qid = t2s + BN;                        // [BN] query index of each tile column (-1 = padding)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = warp & 3, wn = warp >> 2;
    const int nact = P.n_active ? *P.n_active : P.nq;  // tile columns past the active queries are padding (qid = -1, never pass)
    const long long rows_total = MODE == 1 ? (long long)P.S : P.n;
    const long long r0 = ((long long)blockIdx.y + (long long)blockIdx.z * gridDim.y) * BM;  // row tiles fold over y and z (gridDim.y <= 65535)
    if (r0 >= rows_total) return;
    const int W4 = P.W32 >> 2;  // W32 = 2 W is a multiple of 4 (bq_imma_supported: W even), so every row is a whole number of uint4

    bool a_loaded = false;
    for (int qt = blockIdx.x; qt * BN < nact; qt += gridDim.x) {
        __syncthreads();
        if (!a_loaded) {
            // row tile: 128-bit copies + per-row popcount (4 lanes per row, each every fourth uint4)
            for (int i = tid; i < BM * W4; i += IMMA_THREADS) {
                const int r = i / W4, c = i - r * W4;
                const long long rr = r0 + r;
                uint4 v = make_uint4(0u, 0u, 0u, 0u);
                if (rr < rows_total) {
                    const long long src = MODE == 1 ? (rr * P.n) / P.S : rr;
                    v = __ldg(reinterpret_cast<const uint4 *>(P.rows + (size_t)src * P.W32) + c);
                }
                *reinterpret_cast<uint4 *>(As + r * pitch + 4 * c) = v;
            }
            a_loaded = true;
        }
        for (int i = tid; i < BN * W4; i += IMMA_THREADS) {
            const int r = i / W4, c = i - r * W4;
            const int slot = qt * BN + r;
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (slot < nact) {
                const int q = P.qlist ? P.qlist[slot] : slot;
                v = __ldg(reinterpret_cast<const uint4 *>(P.qbits + (size_t)q * P.W32) + c);
            }
            *reinterpret_cast<uint4 *>(Bs + r * pitch + 4 * c) = v;
        }
        for (int r = tid; r < BN; r += IMMA_THREADS) {
            const int slot = qt * BN + r;
            const int q = slot < nact ? (P.qlist ? P.qlist[slot] : slot) : -1;
            qid[r] = q;
            if (MODE == 0) t2s[r] = q >= 0 ? P.t2[q] : INT_MIN;
        }
        __syncthreads();
        if (MODE == 0 && qt == blockIdx.x) {
            for (int r = tid; r < BM; r += IMMA_THREADS) {
                int pc = 0;
                for (int c = 0; c < P.W32; c++) pc += __popc(As[r * pitch + c]);
                pa[r] = pc;
            }
        }

        int acc[2][8][4];
#pragma unroll
        for (int i = 0; i < 2; i++)
#pragma unroll
            for (int j = 0; j < 8; j++)
#pragma unroll
                for (int e = 0; e < 4; e++) acc[i][j][e] = 0;
        const uint32_t *arow = As + (wm * WM + g) * pitch;
        const uint32_t *brow = Bs + (wn * WN + g) * pitch;
        const int sh = 2 * t;
        const int W2 = P.W32 >> 1;
        for (int k2 = 0; k2 < W2; k2++) {
            uint2 aw[4], bw[8];  // two k-steps (64 bits) of rows g, g+8, g+16, g+24 and of queries g + 8 j: conflict-free 64-bit loads
#pragma unroll
            for (int i = 0; i < 4; i++) aw[i] = *reinterpret_cast<const uint2 *>(arow + (8 * i) * pitch + 2 * k2);
#pragma unroll
            for (int j = 0; j < 8; j++) bw[j] = *reinterpret_cast<const uint2 *>(brow + (8 * j) * pitch + 2 * k2);
#pragma unroll
            for (int kk = 0; kk < 2; kk++) {
                uint32_t a[2][4];
#pragma unroll
                for (int i = 0; i < 2; i++) {
                    const uint32_t lo = (kk == 0 ? aw[2 * i].x : aw[2 * i].y) >> sh;
                    const uint32_t hi = (kk == 0 ? aw[2 * i + 1].x : aw[2 * i + 1].y) >> sh;
                    a[i][0] = lo & 0x01010101u;         // row g,     bits 2t + 8m
                    a[i][1] = hi & 0x01010101u;         // row g + 8, bits 2t + 8m
                    a[i][2] = (lo >> 1) & 0x01010101u;  // row g,     bits 2t + 1 + 8m
                    a[i][3] = (hi >> 1) & 0x01010101u;  // row g + 8, bits 2t + 1 + 8m
                }
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const uint32_t w = (kk == 0 ? bw[j].x : bw[j].y) >> sh;
                    const uint32_t b0 = w & 0x01010101u, b1 = (w >> 1) & 0x01010101u;
                    imma_16832(acc[0][j], a[0], b0, b1);
                    imma_16832(acc[1][j], a[1], b0, b1);
                }
            }
        }
        // epilogue. Accumulator (i, j, e): row = wm*32 + 16 i + g + 8 (e >> 1), column = wn*64 + 8 j + 2 t + (e & 1)
        if (MODE == 0) {
            __syncthreads();  // pa
#pragma unroll
            for (int i = 0; i < 2; i++)
#pragma unroll
                for (int e2 = 0; e2 < 2; e2++) {
                    const int rl = wm * WM + 16 * i + g + 8 * e2;
                    const long long rr = r0 + rl;
                    if (rr >= rows_total) continue;
                    const int par = pa[rl];
#pragma unroll
                    for (int j = 0; j < 8; j++)
#pragma unroll
                        for (int e1 = 0; e1 < 2; e1++) {
                            const int cl = wn * WN + 8 * j + 2 * t + e1;
                            const int dot = acc[i][j][2 * e2 + e1];
                            if (par - 2 * dot <= t2s[cl]) {
                                const int q = qid[cl];
                                const int hd = par + P.pb[q] - 2 * dot;
                                const long long key = topk_key(bq_score_from_hd(hd, P.dim), (int32_t)(rr + P.id_base));
                                const int pos = atomicAdd(&P.cnt[q], 1);
                                if (pos < P.cap) P.buf[(size_t)q * P.cap + pos] = key;
                            }
                        }
                }
        } else {
            // sample: hd needs popc(row) too; cheaper here: hd = popc(a) + popc(b) - 2 dot with popc(a) recomputed per row by its 4 lanes
#pragma unroll
            for (int i = 0; i < 2; i++)
#pragma unroll
                for (int e2 = 0; e2 < 2; e2++) {
                    const int rl = wm * WM + 16 * i + g + 8 * e2;
                    const long long rr = r0 + rl;
                    int par = 0;
                    for (int c = t; c < P.W32; c += 4) par += __popc(As[rl * pitch + c]);
                    par += __shfl_xor_sync(FULL, par, 1);
                    par += __shfl_xor_sync(FULL, par, 2);
                    if (rr >= rows_total) continue;
#pragma unroll
                    for (int j = 0; j < 8; j++)
#pragma unroll
                        for (int e1 = 0; e1 < 2; e1++) {
                            const int cl = wn * WN + 8 * j + 2 * t + e1;
                            const int q = qid[cl];
                            if (q >= 0) P.hdm[(size_t)q * P.S + rr] = (unsigned short)(par + P.pb[q] - 2 * acc[i][j][2 * e2 + e1]);
                        }
                }
        }
    }
}

// block-wide exclusive scan helper over `bins` counters in shared memory (bins <= 256 * per): returns through `pre`
// (pre[i] = sum of hist[0 .. i)). 256 threads.
__device__ __forceinline__ void block_scan_exclusive(const int *hist, int *pre, int bins, int *wsum /* 9 ints */)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int per = (bins + 255) / 256;
    const int b0 = tid * per, b1 = min(bins, b0 + per);
    int s = 0;
    for (int i = b0; i < b1; i++) s += hist[i];
    int inc = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(FULL, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    if (tid == 0) {
        int run = 0;
        for (int w = 0; w < 8; w++) { const int v = wsum[w]; wsum[w] = run; run += v; }
        wsum[8] = run;
    }
    __syncthreads();
    int run = wsum[warp] + inc - s;
    for (int i = b0; i < b1; i++) { pre[i] = run; run += hist[i]; }
    __syncthreads();
}

// smallest h with (number of values <= h) >= want, given the exclusive prefix pre[] and hist[]; bins values 0 .. bins-1.
// Returns bins - 1 when the total is smaller than want.
__device__ __forceinline__ int first_bin_reaching(const int *hist, const int *pre, int bins, int want, int *s_res)
{
    if (threadIdx.x == 0) *s_res = bins - 1;
    __syncthreads();
    for (int i = threadIdx.x; i < bins; i += blockDim.x)
        if (pre[i] < want && pre[i] + hist[i] >= want) *s_res = i;  // exactly one bin crosses `want`
    __syncthreads();
    return *s_res;
}

// step 3: per query, thresholds from the sample's histogram. S sample distances in hdm[q][0..S).
__global__ void __launch_bounds__(256) bq_threshold_kernel(const unsigned short *__restrict__ hdm, int S, int dim, int k, int j_aggr, int whole,
                                                           const int *__restrict__ pb, int *__restrict__ thr, int *__restrict__ safe,
                                                           int *__restrict__ t2, int *__restrict__ cnt, int *__restrict__ counters)
{
    extern __shared__ int hsm[];
    const int bins = dim + 1;
    int *hist = hsm, *pre = hsm + bins;
    __shared__ int wsum[9];
    __shared__ int s_res;
    const int q = blockIdx.x;
    for (int i = threadIdx.x; i < bins; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < S; i += blockDim.x) atomicAdd(&hist[min((int)hdm[(size_t)q * S + i], dim)], 1);
    __syncthreads();
    block_scan_exclusive(hist, pre, bins, wsum);
    const int kk = min(k, S);
    const int hs = first_bin_reaching(hist, pre, bins, kk, &s_res);
    __syncthreads();
    int ha = hs;
    if (!whole && j_aggr < kk) ha = first_bin_reaching(hist, pre, bins, j_aggr, &s_res);
    if (threadIdx.x == 0) {
        if (S < k) { ha = dim; }  // fewer sampled rows than k: everything passes (n <= S here)
        const int hsafe = S < k ? dim : hs;
        thr[q] = ha;
        safe[q] = hsafe;
        t2[q] = ha - pb[q];
        cnt[q] = 0;
        if (q == 0) { counters[0] = 0; counters[1] = 0; counters[2] = 0; }
    }
}

// step 5: exact top-k of one query from its captured keys. hd of a key is recovered from the stored score bits by inverting
// the monotone map through a per-block table? No need: keys order by (score desc, node asc) and score is a decreasing function
// of hd, so the histogram runs over hd recomputed as round((1 - score) * dim) — exact for every representable hd / dim
// (checked against the forward map below).
__device__ __forceinline__ int hd_of_key(long long key, int dim)
{
    const float s = key_score(key);
    int h = __float2int_rn(__fmul_rn(__fsub_rn(1.0f, s), (float)dim));
    h = max(0, min(dim, h));
    // the forward map is what defines the key: correct a possible off-by-one of the inverse
    if (bq_score_from_hd(h, dim) != s) {
        if (h > 0 && bq_score_from_hd(h - 1, dim) == s) h -= 1;
        else if (h < dim && bq_score_from_hd(h + 1, dim) == s) h += 1;
    }
    return h;
}

// pass: 0 = after the aggressive filter, 1 = after the first redo. Writes keys_out[q][0..k) when the query is resolved;
// otherwise sets the next threshold and appends q to qlist_next (count in counters[pass + 1... see launcher]).
__global__ void __launch_bounds__(256) bq_select_kernel(const long long *__restrict__ buf, int *__restrict__ cnt, int cap, int k, long long n_rows, int dim,
                                                        const int *__restrict__ pb, int *__restrict__ thr, const int *__restrict__ safe,
                                                        int *__restrict__ t2, long long *__restrict__ keys_out, const int *__restrict__ qlist,
                                                        const int *__restrict__ n_active, int *__restrict__ qlist_next, int *__restrict__ n_next,
                                                        int sort_cap, int *__restrict__ unresolved)
{
    extern __shared__ __align__(16) unsigned char ssm[];
    const int bins = dim + 1;
    int *hist = reinterpret_cast<int *>(ssm);
    int *pre = hist + bins;
    long long *skeys = reinterpret_cast<long long *>(pre + bins + ((2 * bins) & 1));
    __shared__ int wsum[9];
    __shared__ int s_res, s_m;
    const int nact = n_active ? *n_active : (int)gridDim.x;
    if ((int)blockIdx.x >= nact) return;
    const int q = qlist ? qlist[blockIdx.x] : blockIdx.x;
    const int t = thr[q];
    if (t < 0) return;  // already resolved
    const int c = cnt[q];
    const int m = min(c, cap);
    const long long need = n_rows < (long long)k ? n_rows : (long long)k;
    const long long *kb = buf + (size_t)q * cap;
    for (int i = threadIdx.x; i < bins; i += blockDim.x) hist[i] = 0;
    if (threadIdx.x == 0) s_m = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += blockDim.x) atomicAdd(&hist[hd_of_key(kb[i], dim)], 1);
    __syncthreads();
    block_scan_exclusive(hist, pre, bins, wsum);
    const bool complete = c <= cap;  // every row with hd <= thr was captured
    if (complete && (long long)c >= need) {
        // boundary bin: the smallest h whose cumulative count reaches min(k, m); keys at or under it are the only contenders
        const int want = (int)min((long long)m, need);
        const int hb = want > 0 ? first_bin_reaching(hist, pre, bins, want, &s_res) : -1;
        __syncthreads();
        const int take = want > 0 ? pre[hb] + hist[hb] : 0;  // contenders
        if (take <= sort_cap) {
            for (int i = threadIdx.x; i < m; i += blockDim.x) {
                const long long key = kb[i];
                if (hd_of_key(key, dim) <= hb) skeys[atomicAdd(&s_m, 1)] = key;
            }
            __syncthreads();
            const int p2 = next_pow2(take);
            for (int i = take + threadIdx.x; i < p2; i += blockDim.x) skeys[i] = KEY_MIN;
            __syncthreads();
            bitonic_sort_desc(skeys, p2);
            for (int i = threadIdx.x; i < k; i += blockDim.x) keys_out[(size_t)q * k + i] = i < want ? skeys[i] : KEY_MIN;
            if (threadIdx.x == 0) thr[q] = -1;
            return;
        }
        // a boundary bin wider than the sort buffer: adversarial ties; fall through to "unresolved"
    }
    if (threadIdx.x == 0) {
        int next;
        if (!complete) {
            // too many survivors: the k-th smallest CAPTURED distance is a valid, tighter bound
            int hb = dim;
            for (int h = 0; h < bins; h++)
                if (pre[h] + hist[h] >= k) { hb = h; break; }
            next = hb < t ? hb : -2;  // no progress possible: give up on this query
        } else next = t < safe[q] ? safe[q] : -2;
        if (next == -2 || qlist_next == nullptr) {
            atomicAdd(unresolved, 1);
            thr[q] = -1;
            for (int i = 0; i < k; i++) keys_out[(size_t)q * k + i] = KEY_MIN;
        } else {
            thr[q] = next;
            t2[q] = next - pb[q];
            cnt[q] = 0;
            qlist_next[atomicAdd(n_next, 1)] = q;
        }
    }
}

}  // namespace

// sampled rows: enough that the aggressive threshold (>= 37 sample ranks at 6 sigma) leaves about cap / 3 survivors per query
static int bq_imma_sample_rows(long long n)
{
    long long s = (n / 64 + 127) & ~127LL;
    if (s < 16384) s = 16384;
    if (s > 262144) s = 262144;
    return (int)(n < s ? n : s);
}

constexpr int NQ_ALIGN = 256;  // query count padded to the wgmma tile (a multiple of the IMMA tile)

// launch_bq_topk_imma's device scratch for nq queries, carved from `base` (nullptr: only measured)
struct BqScratch {
    uint32_t *qbits;                                    // [nq_pad][W32]
    int *pb, *thr, *safe, *t2, *cnt, *qla, *qlb;        // [nq_pad] each
    int *counters;                                      // redo list lengths
    unsigned short *hdm;                                // [nq_pad][S]
    long long *buf;                                     // [nq][BQ_IMMA_CAP]
    uint8_t *images;                                    // pre-swizzled query images of the wgmma filter pass
    size_t bytes;
    BqScratch(long long n, int nq, int W, void *base)
    {
        const int nq_pad = (nq + NQ_ALIGN - 1) / NQ_ALIGN * NQ_ALIGN;
        Carver c(base);
        qbits = c.take<uint32_t>((size_t)nq_pad * 2 * W);
        pb = c.take<int>(nq_pad);
        thr = c.take<int>(nq_pad);
        safe = c.take<int>(nq_pad);
        t2 = c.take<int>(nq_pad);
        cnt = c.take<int>(nq_pad);
        qla = c.take<int>(nq_pad);
        qlb = c.take<int>(nq_pad);
        counters = c.take<int>(16);
        hdm = c.take<unsigned short>((size_t)nq_pad * bq_imma_sample_rows(n));
        buf = c.take<long long>((size_t)nq * BQ_IMMA_CAP);
        images = c.take<uint8_t>(bq_umma_image_bytes(nq, W));
        bytes = c.bytes;
    }
};

size_t bq_imma_scratch_bytes(long long n, int nq, int W) { return BqScratch(n, nq, W, nullptr).bytes; }

bool bq_imma_supported(const DataDesc &d, int k)
{
    // rows are read as 128-bit chunks of 32-bit halves: W even (W32 = 2 W multiple of 4) keeps every row 16-byte aligned
    return d.kind == KIND_BQ && (d.W % 2) == 0 && d.W <= 32 && d.n >= 4096 && k <= BQ_IMMA_CAP / 4 && d.n < 0x7fffffffLL;
}

cudaError_t launch_bq_topk_imma(const DataDesc &d, const float *queries_dev, int nq, int k, long long id_base, void *scratch_dev,
                                long long *keys_out_dev, int *unresolved_dev, int sm_count, cudaStream_t s)
{
    if (nq <= 0) return cudaSuccess;
    const int nq_pad = (nq + NQ_ALIGN - 1) / NQ_ALIGN * NQ_ALIGN, W32 = 2 * d.W;
    // the full filter pass runs on the warpgroup MMA (bq_umma.cu) whenever the shape allows;
    // JV_BQ_FILTER=imma forces the legacy-MMA kernel (the sample pass and the redo passes always use it)
    const char *fm = getenv("JV_BQ_FILTER");
    const bool use_umma = !(fm && fm[0] == 'i') && bq_umma_supported(d);
    const BqScratch b(d.n, nq, d.W, scratch_dev);
    const int S = bq_imma_sample_rows(d.n);
    cudaError_t e;

    bq_pack_queries_kernel<<<(nq_pad * 32 + 255) / 256, 256, 0, s>>>(queries_dev, nq, nq_pad, d.dim, W32, b.qbits, b.pb);
    g_launches++;
    ImmaParams P;
    P.rows = reinterpret_cast<const uint32_t *>(d.words);
    P.n = d.n; P.W32 = W32; P.dim = d.dim; P.qbits = b.qbits; P.nq_pad = nq_pad; P.nq = nq; P.qlist = nullptr; P.n_active = nullptr;
    P.t2 = b.t2; P.pb = b.pb; P.buf = b.buf; P.cnt = b.cnt; P.cap = BQ_IMMA_CAP; P.id_base = id_base; P.S = S; P.hdm = b.hdm;
    const size_t smem = (size_t)(BM + BN) * (W32 + 4) * 4 + (size_t)(BM + 2 * BN) * 4;
    if ((e = cudaFuncSetAttribute(bq_imma_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(bq_imma_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
    auto row_grid = [](unsigned qtiles, long long rows) {
        const long long tiles = (rows + BM - 1) / BM;
        const unsigned gy = (unsigned)(tiles < 32768 ? tiles : 32768);
        return dim3(qtiles, gy, (unsigned)((tiles + gy - 1) / gy));
    };
    // 2. sample pass
    {
        dim3 grid = row_grid(nq_pad / BN, S);
        bq_imma_kernel<1><<<grid, IMMA_THREADS, smem, s>>>(P);
        g_launches++;
    }
    // 3. thresholds
    const int whole = d.n <= S ? 1 : 0;
    const int ja = topk_aggressive_rank(k, S, d.n);
    const size_t hsm = (size_t)2 * (d.dim + 1) * 4;
    bq_threshold_kernel<<<nq, 256, hsm, s>>>(b.hdm, S, d.dim, k, ja, whole, b.pb, b.thr, b.safe, b.t2, b.cnt, b.counters);
    g_launches++;
    if ((e = cudaMemsetAsync(unresolved_dev, 0, sizeof(int), s)) != cudaSuccess) return e;
    // 4./5. filter + select, then two unconditional redo rounds over the (normally empty) lists
    const int sort_cap = 4096;
    const size_t ssm = hsm + 8 + (size_t)sort_cap * 8;
    if ((e = cudaFuncSetAttribute(bq_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssm)) != cudaSuccess) return e;
    for (int pass = 0; pass < 3; pass++) {
        const int *qlist = pass == 0 ? nullptr : (pass == 1 ? b.qla : b.qlb);
        const int *nact = pass == 0 ? nullptr : &b.counters[pass - 1];
        int *qnext = pass == 0 ? b.qla : (pass == 1 ? b.qlb : nullptr);
        int *nnext = pass == 2 ? nullptr : &b.counters[pass];
        P.qlist = qlist;
        P.n_active = nact;
        if (pass == 0 && use_umma) {
            if ((e = launch_bq_umma_filter(d, b.qbits, nq, nq_pad, b.t2, b.pb, b.buf, b.cnt, BQ_IMMA_CAP, id_base, b.images, sm_count, s)) != cudaSuccess) return e;
        } else {
            dim3 grid = row_grid(pass == 0 ? nq_pad / BN : 1, d.n);
            bq_imma_kernel<0><<<grid, IMMA_THREADS, smem, s>>>(P);
            g_launches++;
        }
        bq_select_kernel<<<pass == 0 ? nq : min(nq, 65535), 256, ssm, s>>>(b.buf, b.cnt, BQ_IMMA_CAP, k, d.n, d.dim, b.pb, b.thr, b.safe, b.t2, keys_out_dev, qlist, nact, qnext,
                                                                           nnext, sort_cap, unresolved_dev);
        g_launches++;
    }
    return cudaGetLastError();
}

}  // namespace jv
