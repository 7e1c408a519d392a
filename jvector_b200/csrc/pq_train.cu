// pq_train.cu — ProductQuantization.compute / refine with isotropic (UNWEIGHTED) loss on the device
// (base:quantization/ProductQuantization.java:109-221, KMeansPlusPlusClusterer.java:131-376).
//
// One definition, restated bit for bit by tests/pq_train_model.py:
//   1. sample   n > cap: Floyd's algorithm over counter_random(seed, TAG_SAMPLE, j, 0), ordinals sorted ascending; the rows are
//               gathered (centred) into a sub-space-major training buffer [M][n_train][size_m] by one kernel.
//   2. centre   per-dimension int64 fixed-point sums (fixed_exp / to_fixed / from_fixed): a pure function of the rows.
//   3. seeding  k-means++ as an exponential race: pick argmin E_j / D_j, E_j = -ln u_j, u_j a 24-bit uniform of (seed, m, round, j).
//               One streaming pass per round updates D with the previous pick and reduces packed (key bits, j) with atomicMin.
//   4. Lloyd    KMeansPlusPlusClusterer.cluster(iterations, 0): initial assignment; then per iteration centroid update (fixed-point
//               sums per (sub-space, cluster), empty clusters reseeded), reassignment, and a sub-space stops once
//               changed <= 0.01 n_train.
//   5. anisotropic (T > UNWEIGHTED only) KMeansPlusPlusClusterer.cluster(.., anisotropicIterations), from the assignment step 4
//               left: per round, for every active sub-space, the fixed-point means and counts of step 4, int64 fixed-point sums of
//               fl(fl(x_a x_b) * fl(1 / |x|^2)) per (cluster, a <= b), one Gauss-Jordan solve per (sub-space, cluster) in the
//               reference's order (Matrix.invert, then the row-wise product with the mean), then the weighted reassignment;
//               a sub-space stops once changed <= 0.01 n_train. pcm uses the sub-space's own size, as the reference does.
#include <algorithm>
#include <unordered_set>
#include <vector>

#include "host_mem.h"
#include "kernels.h"

namespace jv {
namespace {

constexpr int TAG_RESEED = 0x40000000;  // first counter of the empty-cluster reseed draws: sub-space | TAG_RESEED
constexpr int TAG_ARESEED = 0x20000000; // the same for the anisotropic rounds: sub-space | TAG_ARESEED never equals a Lloyd,
                                        // seeding (sub-space < 2^29) or sampling counter
constexpr int ANISO_MAX_SUB = 64;       // largest sub-space the anisotropic solve holds in shared memory (N x 2N floats)
constexpr int PAIR_TILE = 512;          // (a, b) pairs per outer-product block at most
constexpr int TAG_SAMPLE = 0x7fffffff;  // first counter of Floyd's draws
constexpr int SAMPLE_ROWS = 256;        // training rows per block of the gather / column passes
constexpr int TILE_FLOATS = 12288;      // centroid floats per shared-memory tile of the assignment (48 KB)
constexpr int SUM_TILE = 5632;          // int64 sums per centroid-update block (44 KB, + 1 KB of counts)
constexpr int UPDATE_ROWS = 4096;       // training rows per centroid-update block
constexpr int REG_X = 16;               // sub-vectors up to this size stay in registers during the assignment

// ProductQuantization.getSubvectorSizesAndOffsets (ProductQuantization.java:535-550)
__device__ __forceinline__ void sub_layout(int dim, int M, int m, int &size, int &off)
{
    const int base = dim / M, rem = dim % M;
    size = base + (m < rem ? 1 : 0);
    off = m * base + min(m, rem);
}
__device__ __forceinline__ int sub_of(int dim, int M, int d)
{
    const int base = dim / M, rem = dim % M, split = rem * (base + 1);
    return d < split ? d / (base + 1) : rem + (d - split) / base;
}

// int64 fixed point of one column: x -> rint(x 2^e). With |x| <= colmax < 2^ea and n < 2^L, e = 62 - ea - L keeps every term
// below 2^(62 - L), so n terms never overflow, in any order. colmax = 0 (an all-zero column) sums zeros.
__device__ __forceinline__ int fixed_exp(unsigned colmax_bits, long long n)
{
    if (colmax_bits == 0) return 0;
    const int E = (colmax_bits >> 23) & 0xff;
    return 62 - (E > 0 ? E - 126 : -126) - (64 - __clzll(n));
}
__device__ __forceinline__ double pow2(int e) { return __longlong_as_double((long long)(1023 + e) << 52); }
__device__ __forceinline__ long long to_fixed(float x, int e) { return __double2ll_rn(__dmul_rn((double)x, pow2(e))); }
__device__ __forceinline__ float from_fixed(long long sum, int e, long long count)
{
    return __double2float_rn(__ddiv_rn(__dmul_rn(__ll2double_rn(sum), pow2(-e)), __ll2double_rn(count)));
}

__device__ __forceinline__ unsigned long long race_key(float key, long long j)
{
    return ((unsigned long long)__float_as_uint(key) << 32) | (unsigned long long)(uint32_t)j;
}
// the pick of one round: the least finite key, else (every D_j = 0) the least E_j
__device__ __forceinline__ bool race_fallback(unsigned long long best) { return (uint32_t)(best >> 32) >= 0x7f800000u; }
__device__ __forceinline__ long long race_pick(unsigned long long best, unsigned long long ebest)
{
    return (long long)(uint32_t)(race_fallback(best) ? ebest : best);
}
__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(FULL, v, o);
        v = w < v ? w : v;
    }
    return v;
}

// KMeansPlusPlusClusterer's squareL2Distance as kmeans_assign_kernel computes it: (x - c)^2 accumulated in order
__device__ __forceinline__ float sq_dist(const float *x, const float *c, int sz)
{
    float s = 0.f;
    for (int t = 0; t < sz; t++) {
        const float df = __fsub_rn(x[t], c[t]);
        s = __fadd_rn(s, __fmul_rn(df, df));
    }
    return s;
}

// Step 1 (and the column pass of step 2): rows ord[i] (i when ord is null), minus `center` when given, into the training buffer
// when `train` is given; colmax[d] = max |value| of column d. Block: 128 columns x SAMPLE_ROWS rows.
__global__ void __launch_bounds__(128) pq_train_gather_kernel(const float *__restrict__ rows, int stride, const int32_t *__restrict__ ord, long long nt,
                                                              int dim, int M, const float *__restrict__ center, float *__restrict__ train,
                                                              unsigned *__restrict__ colmax)
{
    const int d = blockIdx.x * 128 + threadIdx.x;
    if (d >= dim) return;
    int sz, off;
    sub_layout(dim, M, sub_of(dim, M, d), sz, off);
    const int t = d - off;
    const long long i0 = (long long)blockIdx.y * SAMPLE_ROWS, i1 = min(nt, i0 + SAMPLE_ROWS);
    const float c = center ? center[d] : 0.f;
    float mx = 0.f;
    for (long long i = i0; i < i1; i++) {
        float x = rows[(size_t)(ord ? ord[i] : i) * stride + d];
        if (center) x = __fsub_rn(x, c);
        if (train) train[(size_t)nt * off + (size_t)i * sz + t] = x;
        mx = fmaxf(mx, fabsf(x));
    }
    atomicMax(colmax + d, __float_as_uint(mx));
}

// step 2: per-column fixed-point sums of the sampled rows
__global__ void __launch_bounds__(128) pq_train_colsum_kernel(const float *__restrict__ rows, int stride, const int32_t *__restrict__ ord, long long nt,
                                                              int dim, const unsigned *__restrict__ colmax, long long *__restrict__ sums)
{
    const int d = blockIdx.x * 128 + threadIdx.x;
    if (d >= dim) return;
    const int e = fixed_exp(colmax[d], nt);
    const long long i0 = (long long)blockIdx.y * SAMPLE_ROWS, i1 = min(nt, i0 + SAMPLE_ROWS);
    long long s = 0;
    for (long long i = i0; i < i1; i++) s += to_fixed(rows[(size_t)(ord ? ord[i] : i) * stride + d], e);
    atomicAdd((unsigned long long *)(sums + d), (unsigned long long)s);
}

__global__ void pq_train_mean_kernel(const long long *__restrict__ sums, const unsigned *__restrict__ colmax, long long nt, int dim, float *__restrict__ mean)
{
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d < dim) mean[d] = from_fixed(sums[d], fixed_exp(colmax[d], nt), nt);
}

// step 3, one round of the race for every sub-space (grid.y): D_j = min(D_j, |x_j - x_pick(round - 1)|^2), key = E_j / D_j
// (+inf where D_j = 0; round 0: key = E_j). best / ebest: this round's packed (key, j) and (E_j, j) minima.
__global__ void __launch_bounds__(256) pq_train_seed_kernel(const float *__restrict__ train, long long nt, int dim, int M, int round, uint64_t seed,
                                                            float *__restrict__ D, unsigned long long *__restrict__ best, unsigned long long *__restrict__ ebest)
{
    const int m = blockIdx.y;
    int sz, off;
    sub_layout(dim, M, m, sz, off);
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long kb = ~0ull, eb = ~0ull;
    if (j < nt) {
        const float *sub = train + (size_t)nt * off;
        const uint64_t r = counter_random(seed, m, round, (int)j);
        const float E = neg_ln_unit(__fmul_rn((float)((r >> 40) + 1), 0x1p-24f));  // u in (0, 1], exact
        float key = E;
        if (round > 0) {
            const size_t prev = (size_t)(round - 1) * M + m;
            const float *c = sub + (size_t)race_pick(best[prev], ebest[prev]) * sz;
            const float dj = sq_dist(sub + (size_t)j * sz, c, sz);
            float Dj = dj;
            if (round > 1) {
                const float old = D[(size_t)m * nt + j];
                if (!(dj < old)) Dj = old;
            }
            D[(size_t)m * nt + j] = Dj;
            key = Dj > 0.f ? __fdiv_rn(E, Dj) : __int_as_float(0x7f800000);
            eb = race_key(E, j);
        }
        kb = race_key(key, j);
    }
    kb = warp_min_u64(kb);
    eb = warp_min_u64(eb);
    if ((threadIdx.x & 31) == 0) {
        const size_t slot = (size_t)round * M + m;
        if (kb != ~0ull) atomicMin(best + slot, kb);
        if (eb != ~0ull) atomicMin(ebest + slot, eb);
    }
}

// the picks of all k rounds -> the initial centroids, in the codebook layout [k][size_m] at k * off_m
__global__ void pq_train_seed_finish_kernel(const float *__restrict__ train, long long nt, int dim, int M, int k, const unsigned long long *__restrict__ best,
                                            const unsigned long long *__restrict__ ebest, float *__restrict__ cent, unsigned long long *__restrict__ fallbacks)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= M * k) return;
    const int m = idx / k, c = idx - m * k;
    int sz, off;
    sub_layout(dim, M, m, sz, off);
    const size_t slot = (size_t)c * M + m;
    if (race_fallback(best[slot])) atomicAdd(fallbacks, 1ull);
    const float *x = train + (size_t)nt * off + (size_t)race_pick(best[slot], ebest[slot]) * sz;
    float *dst = cent + (size_t)k * off + (size_t)c * sz;
    for (int t = 0; t < sz; t++) dst[t] = x[t];
}

// step 4, assignment: one thread per (sub-space = grid.y, training row), the sub-space's centroids staged in shared memory tile by
// tile (read from global memory when one centroid exceeds a tile); first minimum wins. changed (optional): per sub-space count of
// rows whose assignment moved. Sub-spaces with active[m] == 0 are skipped.
template <bool REG>
__global__ void __launch_bounds__(256) pq_train_assign_kernel(const float *__restrict__ train, long long nt, int dim, int M, int k,
                                                              const float *__restrict__ cent, const int *__restrict__ active, int32_t *__restrict__ assign,
                                                              unsigned long long *__restrict__ changed)
{
    extern __shared__ float s_cent[];
    const int m = blockIdx.y;
    if (active && !active[m]) return;
    int sz, off;
    sub_layout(dim, M, m, sz, off);
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = j < nt;
    const float *x = train + (size_t)nt * off + (size_t)(valid ? j : 0) * sz;
    float xr[REG ? REG_X : 1];
    if (REG) {
#pragma unroll
        for (int t = 0; t < REG_X; t++) xr[t] = valid && t < sz ? x[t] : 0.f;
    }
    const float *cb = cent + (size_t)k * off;
    const bool staged = sz <= TILE_FLOATS;
    const int ct = staged ? TILE_FLOATS / sz : k;
    float best = 3.402823466e+38f;  // Float.MAX_VALUE
    int bi = 0;
    for (int c0 = 0; c0 < k; c0 += ct) {
        const int c1 = min(k, c0 + ct);
        const float *tile = cb + (size_t)c0 * sz;
        if (staged) {
            __syncthreads();
            for (int q = threadIdx.x; q < (c1 - c0) * sz; q += blockDim.x) s_cent[q] = tile[q];
            __syncthreads();
            tile = s_cent;
        }
        if (!valid) continue;
        for (int c = c0; c < c1; c++) {
            const float *cen = tile + (size_t)(c - c0) * sz;
            float s = 0.f;
            if (REG) {
#pragma unroll
                for (int t = 0; t < REG_X; t++)
                    if (t < sz) {
                        const float df = __fsub_rn(xr[t], cen[t]);
                        s = __fadd_rn(s, __fmul_rn(df, df));
                    }
            } else s = sq_dist(x, cen, sz);
            if (s < best) { best = s; bi = c; }
        }
    }
    bool moved = false;
    if (valid) {
        int32_t *a = assign + (size_t)m * nt + j;
        moved = *a != bi;
        *a = bi;
    }
    if (changed) {
        const unsigned b = __ballot_sync(FULL, moved);
        if ((threadIdx.x & 31) == 0 && b) atomicAdd(changed + m, (unsigned long long)__popc(b));
    }
}

// step 4, centroid update: fixed-point sums per (sub-space = grid.z, cluster, dimension tile = grid.y) over UPDATE_ROWS rows
// (grid.x), aggregated in shared memory, then added to sums (the codebook layout) and counts [M][k]
__global__ void __launch_bounds__(256) pq_train_update_kernel(const float *__restrict__ train, long long nt, int dim, int M, int k, int tlen,
                                                              const int32_t *__restrict__ assign, const int *__restrict__ active,
                                                              const unsigned *__restrict__ colmax, long long *__restrict__ sums, int *__restrict__ counts)
{
    __shared__ long long s_sum[SUM_TILE];
    __shared__ int s_cnt[256];
    const int m = blockIdx.z;
    if (active && !active[m]) return;
    int sz, off;
    sub_layout(dim, M, m, sz, off);
    const int t0 = blockIdx.y * tlen;
    if (t0 >= sz) return;
    const int tl = min(tlen, sz - t0);
    const bool count = blockIdx.y == 0;
    for (int q = threadIdx.x; q < k * tl; q += blockDim.x) s_sum[q] = 0;
    for (int q = threadIdx.x; q < k; q += blockDim.x) s_cnt[q] = 0;
    __syncthreads();
    const long long i0 = (long long)blockIdx.x * UPDATE_ROWS, i1 = min(nt, i0 + UPDATE_ROWS);
    const int32_t *a = assign + (size_t)m * nt;
    const float *x = train + (size_t)nt * off;
    for (long long q = threadIdx.x; q < (i1 - i0) * tl; q += blockDim.x) {
        const long long i = i0 + q / tl;
        const int t = (int)(q % tl);
        const int c = a[i];
        const float v = x[(size_t)i * sz + t0 + t];
        atomicAdd((unsigned long long *)&s_sum[c * tl + t], (unsigned long long)to_fixed(v, fixed_exp(colmax[off + t0 + t], nt)));
        if (count && t == 0) atomicAdd(&s_cnt[c], 1);
    }
    __syncthreads();
    for (int q = threadIdx.x; q < k * tl; q += blockDim.x) {
        const long long v = s_sum[q];
        if (v) atomicAdd((unsigned long long *)&sums[(size_t)k * off + (size_t)(q / tl) * sz + t0 + q % tl], (unsigned long long)v);
    }
    if (count)
        for (int c = threadIdx.x; c < k; c += blockDim.x)
            if (s_cnt[c]) atomicAdd(&counts[(size_t)m * k + c], s_cnt[c]);
}

// step 4, the new centroids (KMeansPlusPlusClusterer.updateCentroidsUnweighted): sum / count, or for an empty cluster training
// row counter_random(seed, m | TAG_RESEED, iteration, cluster) % n_train. One thread per codebook float.
__global__ void pq_train_finalize_kernel(const float *__restrict__ train, long long nt, int dim, int M, int k, const int *__restrict__ active,
                                         const long long *__restrict__ sums, const int *__restrict__ counts, const unsigned *__restrict__ colmax,
                                         uint64_t seed, int it, float *__restrict__ cent, unsigned long long *__restrict__ reseeds)
{
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= (long long)k * dim) return;
    const int m = sub_of(dim, M, (int)(q / k));
    if (!active[m]) return;
    int sz, off;
    sub_layout(dim, M, m, sz, off);
    const int local = (int)(q - (long long)k * off), c = local / sz, t = local - c * sz;
    const int cnt = counts[(size_t)m * k + c];
    if (cnt == 0) {
        const long long r = (long long)(counter_random(seed, m | TAG_RESEED, it, c) % (uint64_t)nt);
        cent[q] = train[(size_t)nt * off + (size_t)r * sz + t];
        if (t == 0) atomicAdd(reseeds, 1ull);
    } else cent[q] = from_fixed(sums[q], fixed_exp(colmax[off + t], nt), cnt);
}

// step 5: |x|^2 of every (sub-space = grid.y, training row), accumulated in order, and fl(1 / |x|^2) where |x|^2 > 0 (else 0)
__global__ void __launch_bounds__(256) pq_train_norm_kernel(const float *__restrict__ train, long long nt, int dim, int M, float *__restrict__ xn,
                                                            float *__restrict__ rinv)
{
    const int m = blockIdx.y;
    int sz, off;
    sub_layout(dim, M, m, sz, off);
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nt) return;
    const float *x = train + (size_t)nt * off + (size_t)j * sz;
    float s = 0.f;
    for (int t = 0; t < sz; t++) s = __fadd_rn(s, __fmul_rn(x[t], x[t]));
    xn[(size_t)m * nt + j] = s;
    rinv[(size_t)m * nt + j] = s > 0.f ? __fdiv_rn(1.f, s) : 0.f;
}

// the upper-triangle pair index of (a, b), a <= b < n, rows in order
__device__ __forceinline__ int pair_index(int a, int b, int n) { return a * n - a * (a - 1) / 2 + (b - a); }

// step 5, outer-product sums: int64 fixed point of fl(fl(x_a x_b) * rinv) for the pairs [p0, p0 + ptile) of sub-space grid.z, summed
// per cluster over UPDATE_ROWS rows (grid.x) in shared memory, then added to osum [M][k][npair_max]. |term| < 2, so one exponent
// (fixed_exp of 1.0f) serves every term; rows with |x|^2 = 0 add nothing (KMeansPlusPlusClusterer skips them).
__global__ void __launch_bounds__(256) pq_train_outer_kernel(const float *__restrict__ train, long long nt, int dim, int M, int k, int ptile, int npmax,
                                                             const int32_t *__restrict__ assign, const int *__restrict__ active,
                                                             const float *__restrict__ rinv, long long *__restrict__ osum)
{
    __shared__ long long s_sum[SUM_TILE];
    __shared__ unsigned char s_a[PAIR_TILE], s_b[PAIR_TILE];
    const int m = blockIdx.z;
    if (!active[m]) return;
    int sz, off;
    sub_layout(dim, M, m, sz, off);
    const int np = sz * (sz + 1) / 2, p0 = blockIdx.y * ptile;
    if (p0 >= np) return;
    const int pl = min(ptile, np - p0);
    for (int q = threadIdx.x; q < k * pl; q += blockDim.x) s_sum[q] = 0;
    for (int p = threadIdx.x; p < pl; p += blockDim.x) {
        int a = 0, r = p0 + p;
        while (r >= sz - a) { r -= sz - a; a++; }
        s_a[p] = (unsigned char)a;
        s_b[p] = (unsigned char)(a + r);
    }
    __syncthreads();
    const int e = fixed_exp(0x3f800000u, nt);
    const long long i0 = (long long)blockIdx.x * UPDATE_ROWS, i1 = min(nt, i0 + UPDATE_ROWS);
    const int32_t *as = assign + (size_t)m * nt;
    const float *ri = rinv + (size_t)m * nt;
    const float *x = train + (size_t)nt * off;
    for (long long q = threadIdx.x; q < (i1 - i0) * pl; q += blockDim.x) {
        const long long i = i0 + q / pl;
        const int p = (int)(q % pl);
        const float r = ri[i];
        if (r == 0.f) continue;
        const float *xi = x + (size_t)i * sz;
        const float term = __fmul_rn(__fmul_rn(xi[s_a[p]], xi[s_b[p]]), r);
        atomicAdd((unsigned long long *)&s_sum[as[i] * pl + p], (unsigned long long)to_fixed(term, e));
    }
    __syncthreads();
    for (int q = threadIdx.x; q < k * pl; q += blockDim.x) {
        const long long v = s_sum[q];
        if (v) atomicAdd((unsigned long long *)&osum[((size_t)m * k + q / pl) * npmax + p0 + q % pl], (unsigned long long)v);
    }
}

// step 5, the new centroid of (cluster = grid.x, sub-space = grid.y) (KMeansPlusPlusClusterer.updateCentroidsAnisotropic):
//   A = fl(S * fl(fl(1 - ocm) / |L|)) (+ ocm on the diagonal), S the outer-product sums, ocm = fl(1 / pcm);
//   c = invert(A) * mean, Matrix.invert's Gauss-Jordan (largest |pivot|, the first row on a tie; the pivot row times fl(1 / pivot);
//   every other row plus fl(-factor * pivot row)), then row-wise dot products accumulated in order. Every element sees the same
//   sequence of roundings whichever thread applies it. Columns left of the pivot are never read again and are not updated.
//   An empty cluster takes training row counter_random(seed, m | TAG_ARESEED, round, cluster) % n_train.
__global__ void __launch_bounds__(256) pq_train_solve_kernel(const float *__restrict__ train, long long nt, int dim, int M, int k, int npmax,
                                                             const int *__restrict__ active, const long long *__restrict__ sums,
                                                             const int *__restrict__ counts, const unsigned *__restrict__ colmax,
                                                             const long long *__restrict__ osum, float pcm_big, float pcm_small, uint64_t seed, int round,
                                                             float *__restrict__ cent, unsigned long long *__restrict__ reseeds)
{
    __shared__ float a[ANISO_MAX_SUB * 2 * ANISO_MAX_SUB];
    __shared__ float mean[ANISO_MAX_SUB], fac[ANISO_MAX_SUB];
    __shared__ int s_piv;
    const int c = blockIdx.x, m = blockIdx.y;
    if (!active[m]) return;
    int N, off;
    sub_layout(dim, M, m, N, off);
    const int W = 2 * N;
    float *dst = cent + (size_t)k * off + (size_t)c * N;
    const int cnt = counts[(size_t)m * k + c];
    if (cnt == 0) {
        const long long r = (long long)(counter_random(seed, m | TAG_ARESEED, round, c) % (uint64_t)nt);
        for (int t = threadIdx.x; t < N; t += blockDim.x) dst[t] = train[(size_t)nt * off + (size_t)r * N + t];
        if (threadIdx.x == 0) atomicAdd(reseeds, 1ull);
        return;
    }
    const float pcm = m < dim % M ? pcm_big : pcm_small;
    const float ocm = __fdiv_rn(1.f, pcm);
    const float scale = __fdiv_rn(__fsub_rn(1.f, ocm), (float)cnt);
    const int eo = fixed_exp(0x3f800000u, nt);
    const long long *os = osum + ((size_t)m * k + c) * npmax;
    for (int t = threadIdx.x; t < N; t += blockDim.x) mean[t] = from_fixed(sums[(size_t)k * off + (size_t)c * N + t], fixed_exp(colmax[off + t], nt), cnt);
    for (int q = threadIdx.x; q < N * N; q += blockDim.x) {
        const int i = q / N, j = q - i * N;
        const float S = __double2float_rn(__dmul_rn(__ll2double_rn(os[pair_index(min(i, j), max(i, j), N)]), pow2(-eo)));
        float v = __fmul_rn(S, scale);
        if (i == j) v = __fadd_rn(v, ocm);
        a[i * W + j] = v;
        a[i * W + N + j] = i == j ? 1.f : 0.f;
    }
    __syncthreads();
    for (int i = 0; i < N; i++) {
        if (threadIdx.x == 0) {
            int mr = i;
            for (int r = i + 1; r < N; r++)
                if (fabsf(a[r * W + i]) > fabsf(a[mr * W + i])) mr = r;
            s_piv = mr;
        }
        __syncthreads();
        const int mr = s_piv;
        if (mr != i)
            for (int j = i + threadIdx.x; j < W; j += blockDim.x) {
                const float t = a[i * W + j];
                a[i * W + j] = a[mr * W + j];
                a[mr * W + j] = t;
            }
        __syncthreads();
        const float rp = __fdiv_rn(1.f, a[i * W + i]);
        for (int r = threadIdx.x; r < N; r += blockDim.x) fac[r] = a[r * W + i];
        __syncthreads();
        for (int j = i + 1 + threadIdx.x; j < W; j += blockDim.x) a[i * W + j] = __fmul_rn(a[i * W + j], rp);
        __syncthreads();
        const int cols = W - i - 1;
        for (int q = threadIdx.x; q < (N - 1) * cols; q += blockDim.x) {
            int r = q / cols;
            const int j = i + 1 + (q - r * cols);
            r += r >= i;
            a[r * W + j] = __fadd_rn(a[r * W + j], __fmul_rn(-fac[r], a[i * W + j]));
        }
        __syncthreads();
    }
    for (int t = threadIdx.x; t < N; t += blockDim.x) {
        float s = 0.f;
        for (int u = 0; u < N; u++) s = __fadd_rn(s, __fmul_rn(a[t * W + N + u], mean[u]));
        dst[t] = s;
    }
}

// step 5, weighted reassignment (KMeansPlusPlusClusterer.updateAssignedPointsAnisotropic): argmin over c of
//   fl(fl(pcm * fl(e * e)) + fl(fl(fl(|c|^2 - fl(2 dot)) + |x|^2) - fl(e * e))),  dot = c.x in order, e = fl(dot - |x|^2),
// starting from the current cluster at Float.MAX_VALUE, first minimum wins. Centroid tiles and their |c|^2 in shared memory.
template <bool REG>
__global__ void __launch_bounds__(256) pq_train_assign_aniso_kernel(const float *__restrict__ train, long long nt, int dim, int M, int k,
                                                                    const float *__restrict__ cent, const int *__restrict__ active,
                                                                    const float *__restrict__ xn, float pcm_big, float pcm_small,
                                                                    int32_t *__restrict__ assign, unsigned long long *__restrict__ changed)
{
    extern __shared__ float s_cent[];
    const int m = blockIdx.y;
    if (!active[m]) return;
    int sz, off;
    sub_layout(dim, M, m, sz, off);
    const float pcm = m < dim % M ? pcm_big : pcm_small;
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = j < nt;
    const float *x = train + (size_t)nt * off + (size_t)(valid ? j : 0) * sz;
    float xr[REG ? REG_X : 1];
    if (REG) {
#pragma unroll
        for (int t = 0; t < REG_X; t++) xr[t] = valid && t < sz ? x[t] : 0.f;
    }
    const float xx = valid ? xn[(size_t)m * nt + j] : 0.f;
    const float *cb = cent + (size_t)k * off;
    const int ct = TILE_FLOATS / (sz + 1);
    float *s_norm = s_cent + (size_t)ct * sz;
    int32_t *a = assign + (size_t)m * nt + (valid ? j : 0);
    const int old = valid ? *a : 0;
    float best = 3.402823466e+38f;  // Float.MAX_VALUE
    int bi = old;
    for (int c0 = 0; c0 < k; c0 += ct) {
        const int c1 = min(k, c0 + ct);
        __syncthreads();
        for (int q = threadIdx.x; q < (c1 - c0) * sz; q += blockDim.x) s_cent[q] = cb[(size_t)c0 * sz + q];
        __syncthreads();
        for (int c = threadIdx.x; c < c1 - c0; c += blockDim.x) {
            float s = 0.f;
            for (int t = 0; t < sz; t++) s = __fadd_rn(s, __fmul_rn(s_cent[c * sz + t], s_cent[c * sz + t]));
            s_norm[c] = s;
        }
        __syncthreads();
        if (!valid) continue;
        for (int c = c0; c < c1; c++) {
            const float *cen = s_cent + (size_t)(c - c0) * sz;
            float dot = 0.f;
            if (REG) {
#pragma unroll
                for (int t = 0; t < REG_X; t++)
                    if (t < sz) dot = __fadd_rn(dot, __fmul_rn(cen[t], xr[t]));
            } else
                for (int t = 0; t < sz; t++) dot = __fadd_rn(dot, __fmul_rn(cen[t], x[t]));
            const float e = __fsub_rn(dot, xx);
            const float resid = __fadd_rn(__fsub_rn(s_norm[c - c0], __fmul_rn(2.f, dot)), xx);
            const float par = __fmul_rn(e, e);
            const float d = __fadd_rn(__fmul_rn(pcm, par), __fsub_rn(resid, par));
            if (d < best) { best = d; bi = c; }
        }
    }
    const bool moved = valid && bi != old;
    if (valid) *a = bi;
    const unsigned b = __ballot_sync(FULL, moved);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(changed + m, (unsigned long long)__popc(b));
}

#define LAUNCHED()                                  \
    do {                                            \
        g_launches++;                               \
        cudaError_t e_ = cudaGetLastError();        \
        if (e_ != cudaSuccess) return e_;           \
    } while (0)
#define TRY(x)                                      \
    do {                                            \
        cudaError_t e_ = (x);                       \
        if (e_ != cudaSuccess) return e_;           \
    } while (0)

}  // namespace

static std::vector<int32_t> pq_train_sample(long long n, long long cap, uint64_t seed)
{
    std::vector<int32_t> ord;
    if (n <= cap) return ord;
    // extractTrainingVectors (ProductQuantization.java:141-179): Floyd's algorithm, j from n - cap to n - 1
    std::unordered_set<int32_t> chosen;
    chosen.reserve((size_t)cap * 2);
    for (long long j = n - cap; j < n; j++) {
        const int32_t t = (int32_t)(counter_random(seed, TAG_SAMPLE, (int)j, 0) % (uint64_t)(j + 1));
        chosen.insert(chosen.count(t) ? (int32_t)j : t);
    }
    ord.assign(chosen.begin(), chosen.end());
    std::sort(ord.begin(), ord.end());
    return ord;
}

cudaError_t pq_train(const DataDesc &f32, const PqTrainArgs &p, const float *init_codebooks, const float *centroid, float *codebooks_out,
                     float *centroid_out, PqTrainStats *st, cudaStream_t s)
{
    const long long n = f32.n;
    const int dim = f32.dim, M = p.M, k = p.k;
    const std::vector<int32_t> ord = pq_train_sample(n, p.cap, p.seed);
    const long long nt = ord.empty() ? n : (long long)ord.size();
    const bool seeding = init_codebooks == nullptr;
    const bool center = seeding ? p.globally_center != 0 : centroid != nullptr;
    const bool aniso = p.aniso_iters > 0;
    const int szmax = (dim + M - 1) / M, npmax = aniso ? szmax * (szmax + 1) / 2 : 0;
    int32_t *d_ord, *d_assign, *d_counts, *d_active;
    float *d_train, *d_D, *d_cent, *d_mean, *d_xn, *d_rinv;
    long long *d_sums, *d_csum, *d_osum;
    unsigned long long *d_best, *d_ebest, *d_changed, *d_counters;
    unsigned *d_colmax;
    auto carve = [&](void *base) {
        Carver c(base);
        d_ord = c.take<int32_t>(ord.size());
        d_train = c.take<float>((size_t)nt * dim);
        d_D = c.take<float>(seeding ? (size_t)nt * M : 0);
        d_assign = c.take<int32_t>((size_t)nt * M);
        d_cent = c.take<float>((size_t)k * dim);
        d_sums = c.take<long long>((size_t)k * dim);
        d_counts = c.take<int32_t>((size_t)M * k);
        d_best = c.take<unsigned long long>(seeding ? 2 * (size_t)k * M : 0);
        d_ebest = d_best + (size_t)k * M;
        d_colmax = c.take<unsigned>(2 * (size_t)dim);  // raw rows (the centring pass), training rows
        d_csum = c.take<long long>(dim);
        d_mean = c.take<float>(dim);
        d_changed = c.take<unsigned long long>(M);
        d_active = c.take<int32_t>(M);
        d_counters = c.take<unsigned long long>(3);  // seeding fallbacks, empty reseeds, anisotropic reseeds
        d_xn = c.take<float>(aniso ? (size_t)nt * M : 0);
        d_rinv = c.take<float>(aniso ? (size_t)nt * M : 0);
        d_osum = c.take<long long>((size_t)M * k * npmax);
        return c.bytes;
    };
    DeviceBuffer mem;
    if (const cudaError_t e = mem.alloc(carve(nullptr)); e != cudaSuccess) {
        cudaGetLastError();  // a failed cudaMalloc is not sticky: clear it so the next launch check does not report it
        return e;
    }
    carve(mem.get());
    StreamTimer timer;
    TRY(timer.start(s));
    TRY(cudaMemsetAsync(d_colmax, 0, 2 * (size_t)dim * 4, s));
    TRY(cudaMemsetAsync(d_csum, 0, (size_t)dim * 8, s));
    TRY(cudaMemsetAsync(d_counters, 0, 24, s));
    if (!ord.empty()) TRY(cudaMemcpyAsync(d_ord, ord.data(), ord.size() * 4, cudaMemcpyHostToDevice, s));
    const int32_t *ordp = ord.empty() ? nullptr : d_ord;
    const dim3 col_grid((dim + 127) / 128, (unsigned)((nt + SAMPLE_ROWS - 1) / SAMPLE_ROWS));
    if (seeding && center) {
        pq_train_gather_kernel<<<col_grid, 128, 0, s>>>(f32.rows, f32.stride, ordp, nt, dim, M, nullptr, nullptr, d_colmax + dim);
        LAUNCHED();
        pq_train_colsum_kernel<<<col_grid, 128, 0, s>>>(f32.rows, f32.stride, ordp, nt, dim, d_colmax + dim, d_csum);
        LAUNCHED();
        pq_train_mean_kernel<<<(dim + 255) / 256, 256, 0, s>>>(d_csum, d_colmax + dim, nt, dim, d_mean);
        LAUNCHED();
    } else if (center) TRY(cudaMemcpyAsync(d_mean, centroid, (size_t)dim * 4, cudaMemcpyHostToDevice, s));
    pq_train_gather_kernel<<<col_grid, 128, 0, s>>>(f32.rows, f32.stride, ordp, nt, dim, M, center ? d_mean : nullptr, d_train, d_colmax);
    LAUNCHED();

    const dim3 row_grid((unsigned)((nt + 255) / 256), M);
    if (seeding) {
        TRY(cudaMemsetAsync(d_best, 0xff, 2 * (size_t)k * M * 8, s));
        for (int r = 0; r < k; r++) {
            pq_train_seed_kernel<<<row_grid, 256, 0, s>>>(d_train, nt, dim, M, r, p.seed, d_D, d_best, d_ebest);
            LAUNCHED();
        }
        pq_train_seed_finish_kernel<<<(M * k + 255) / 256, 256, 0, s>>>(d_train, nt, dim, M, k, d_best, d_ebest, d_cent, d_counters);
        LAUNCHED();
    } else TRY(cudaMemcpyAsync(d_cent, init_codebooks, (size_t)k * dim * 4, cudaMemcpyHostToDevice, s));

    const size_t assign_smem = (size_t)TILE_FLOATS * 4;
    auto assign = [&](const int *active, unsigned long long *changed) -> cudaError_t {
        if (szmax <= REG_X) pq_train_assign_kernel<true><<<row_grid, 256, assign_smem, s>>>(d_train, nt, dim, M, k, d_cent, active, d_assign, changed);
        else pq_train_assign_kernel<false><<<row_grid, 256, assign_smem, s>>>(d_train, nt, dim, M, k, d_cent, active, d_assign, changed);
        LAUNCHED();
        return cudaSuccess;
    };
    TRY(assign(nullptr, nullptr));

    // Lloyd (KMeansPlusPlusClusterer.cluster(iterations, 0)): one host sync per iteration reads the changed counts
    std::vector<int32_t> active(M, 1);
    std::vector<unsigned long long> changed(M);
    std::vector<int> updates(M, 0);
    std::vector<long long> last(M, 0);
    const int tlen = std::max(1, std::min(szmax, SUM_TILE / k));
    const dim3 upd_grid((unsigned)((nt + UPDATE_ROWS - 1) / UPDATE_ROWS), (unsigned)((szmax + tlen - 1) / tlen), M);
    for (int it = 0; it < p.iters; it++) {
        if (std::find(active.begin(), active.end(), 1) == active.end()) break;
        TRY(cudaMemcpyAsync(d_active, active.data(), (size_t)M * 4, cudaMemcpyHostToDevice, s));
        TRY(cudaMemsetAsync(d_sums, 0, (size_t)k * dim * 8, s));
        TRY(cudaMemsetAsync(d_counts, 0, (size_t)M * k * 4, s));
        TRY(cudaMemsetAsync(d_changed, 0, (size_t)M * 8, s));
        pq_train_update_kernel<<<upd_grid, 256, 0, s>>>(d_train, nt, dim, M, k, tlen, d_assign, d_active, d_colmax, d_sums, d_counts);
        LAUNCHED();
        const long long total = (long long)k * dim;
        pq_train_finalize_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(d_train, nt, dim, M, k, d_active, d_sums, d_counts, d_colmax, p.seed, it,
                                                                                 d_cent, d_counters + 1);
        LAUNCHED();
        TRY(assign(d_active, d_changed));
        TRY(cudaMemcpyAsync(changed.data(), d_changed, (size_t)M * 8, cudaMemcpyDeviceToHost, s));
        TRY(cudaStreamSynchronize(s));
        for (int m = 0; m < M; m++) {
            if (!active[m]) continue;
            updates[m]++;
            last[m] = (long long)changed[m];
            if ((double)changed[m] <= 0.01 * (double)nt) active[m] = 0;
        }
    }
    // anisotropic rounds (KMeansPlusPlusClusterer.cluster(.., aniso_iters)) for every sub-space, from the assignment above
    std::vector<int> aupdates(M, 0);
    std::vector<long long> alast(M, 0);
    if (aniso) {
        const float pcm_big = pq_parallel_cost_multiplier(p.threshold, szmax), pcm_small = pq_parallel_cost_multiplier(p.threshold, dim / M);
        pq_train_norm_kernel<<<row_grid, 256, 0, s>>>(d_train, nt, dim, M, d_xn, d_rinv);
        LAUNCHED();
        const int ptile = std::max(1, std::min({npmax, SUM_TILE / k, PAIR_TILE}));
        const dim3 outer_grid(upd_grid.x, (unsigned)((npmax + ptile - 1) / ptile), M);
        std::fill(active.begin(), active.end(), 1);
        for (int r = 0; r < p.aniso_iters; r++) {
            if (std::find(active.begin(), active.end(), 1) == active.end()) break;
            TRY(cudaMemcpyAsync(d_active, active.data(), (size_t)M * 4, cudaMemcpyHostToDevice, s));
            TRY(cudaMemsetAsync(d_sums, 0, (size_t)k * dim * 8, s));
            TRY(cudaMemsetAsync(d_counts, 0, (size_t)M * k * 4, s));
            TRY(cudaMemsetAsync(d_osum, 0, (size_t)M * k * npmax * 8, s));
            TRY(cudaMemsetAsync(d_changed, 0, (size_t)M * 8, s));
            pq_train_update_kernel<<<upd_grid, 256, 0, s>>>(d_train, nt, dim, M, k, tlen, d_assign, d_active, d_colmax, d_sums, d_counts);
            LAUNCHED();
            pq_train_outer_kernel<<<outer_grid, 256, 0, s>>>(d_train, nt, dim, M, k, ptile, npmax, d_assign, d_active, d_rinv, d_osum);
            LAUNCHED();
            pq_train_solve_kernel<<<dim3(k, M), 256, 0, s>>>(d_train, nt, dim, M, k, npmax, d_active, d_sums, d_counts, d_colmax, d_osum, pcm_big, pcm_small,
                                                             p.seed, r, d_cent, d_counters + 2);
            LAUNCHED();
            if (szmax <= REG_X)
                pq_train_assign_aniso_kernel<true><<<row_grid, 256, assign_smem, s>>>(d_train, nt, dim, M, k, d_cent, d_active, d_xn, pcm_big, pcm_small,
                                                                                      d_assign, d_changed);
            else
                pq_train_assign_aniso_kernel<false><<<row_grid, 256, assign_smem, s>>>(d_train, nt, dim, M, k, d_cent, d_active, d_xn, pcm_big, pcm_small,
                                                                                       d_assign, d_changed);
            LAUNCHED();
            TRY(cudaMemcpyAsync(changed.data(), d_changed, (size_t)M * 8, cudaMemcpyDeviceToHost, s));
            TRY(cudaStreamSynchronize(s));
            for (int m = 0; m < M; m++) {
                if (!active[m]) continue;
                aupdates[m]++;
                alast[m] = (long long)changed[m];
                if ((double)changed[m] <= 0.01 * (double)nt) active[m] = 0;
            }
        }
    }
    unsigned long long counters[3];
    TRY(cudaMemcpyAsync(codebooks_out, d_cent, (size_t)k * dim * 4, cudaMemcpyDeviceToHost, s));
    if (seeding && center && centroid_out) TRY(cudaMemcpyAsync(centroid_out, d_mean, (size_t)dim * 4, cudaMemcpyDeviceToHost, s));
    TRY(cudaMemcpyAsync(counters, d_counters, 24, cudaMemcpyDeviceToHost, s));
    TRY(timer.stop(s));
    TRY(cudaStreamSynchronize(s));
    st->train_rows = nt;
    st->max_lloyd_updates = *std::max_element(updates.begin(), updates.end());
    st->changed_last = 0;
    for (long long c : last) st->changed_last += c;
    st->seeding_fallbacks = (long long)counters[0];
    st->empty_reseeds = (long long)counters[1];
    st->aniso_updates = *std::max_element(aupdates.begin(), aupdates.end());
    st->aniso_changed_last = 0;
    for (long long c : alast) st->aniso_changed_last += c;
    st->aniso_reseeds = (long long)counters[2];
    st->device_ms = timer.ms();
    return cudaSuccess;
}

}  // namespace jv
