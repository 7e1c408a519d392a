// scorers.cuh — the per-candidate scoring functions of the hot path as device code.
//
// One "row scorer" per storage kind; each is executed by a GROUP of lanes (32 for fp32 rows and NVQ bytes, 8 for
// PQ code rows and BQ words) and returns, in every lane of the group, the reference's similarity SCORE
// (base:vector/VectorSimilarityFunction.java:37-69). The same scorers are used by the batch kernels
// (kernels_batch.cu), the device-resident GraphSearcher (search.cu) and the builder (build.cu).
//
// A query is first "prepared" into a blob (prepare_blob): the fp32 query itself (+ ||q||^2), the PQ partial-sums
// table (PQDecoder.java:41-54), the BQ bit pack (BQVectors.java:109), or the NVQ shifted query (+ <q,mean>, ||q||)
// (NVQScorer.java:46-137). The blob may live in global or shared memory.
#pragma once
#include "common.cuh"

namespace jv {

enum { KIND_F32 = 0, KIND_PQ = 1, KIND_BQ = 2, KIND_NVQ = 3 };

struct DataDesc {
    int kind;
    int dim;
    long long n;
    // f32: rows [n][stride] fp32, stride = dim rounded up to 4, zero padded
    const float *rows;
    int stride;
    // f32 row sketch (row_sketch_kernel): [n][sketch_stride] int8 codes round(x / s), s = max|x| / 127 (sketch_stride = stride
    // rounded up to 8, zero padded) and [n] {s, radius}. Set only for the search kernel's fp32 DOT walks that fill the GPU (api.cu,
    // search.cu); nullptr elsewhere
    const int8_t *sketch;
    const float2 *sketch_meta;
    int sketch_stride;
    // pq: codes [n][code_stride] u8 (code_stride = M rounded up to 4), codebooks concatenated, codebook m at k*sub_offsets[m]
    const uint8_t *codes;
    int M, k, code_stride;
    const float *codebooks;
    const int *sub_sizes;    // [M] (pq) or [nsub] (nvq)
    const int *sub_offsets;  // [M] (pq) or [nsub] (nvq)
    const float *centroid;   // pq global centroid or nullptr
    const float *mag;        // pq ||centroid||^2 table [M*k] (cosine)
    // pq centroid-vs-centroid tables of ProductQuantization.createCodebookPartialSums (ProductQuantization.java:609-628):
    // [M][k (k + 1) / 2] upper triangles, [0] squared L2, [1] dot product; nullptr until jv_dataset_pq_pair_table builds one
    const float *pair_table[2];
    // bq: words [n][W] u64
    const unsigned long long *words;
    int W;
    // nvq: bytes [n][byte_stride] u8 (byte_stride = dim rounded up to 4), params [n][nsub][4] {min,max,growth,midpoint}
    const uint8_t *bytes;
    int byte_stride;
    const float *params;
    int nsub;
    const float *mean;
};

template <int KIND>
struct GroupOf {
    static constexpr int value = (KIND == KIND_F32 || KIND == KIND_NVQ) ? 32 : 8;
};

__host__ __device__ inline int blob_floats(const DataDesc &d)
{
    switch (d.kind) {
    case KIND_F32: return d.stride + 4;
    case KIND_PQ: return (d.M * d.k + 1 + 3) & ~3;
    case KIND_BQ: return ((2 * d.W + 3) & ~3) + 4;
    default: return d.stride + 4;
    }
}

// ------------------------------------------------------------------------------------------------
// block-wide sum, result broadcast to all threads. red: >= 33 floats of shared memory.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_sum(float v, float *red)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = group_sum<32>(v);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        float t = lane < nw ? red[lane] : 0.f;
        t = group_sum<32>(t);
        if (lane == 0) red[32] = t;
    }
    __syncthreads();
    return red[32];
}

// ------------------------------------------------------------------------------------------------
// prepare_blob: whole CTA. q: raw query [dim] in global memory. blob: global or shared, blob_floats() long.
// ------------------------------------------------------------------------------------------------
// PQ only: sub-spaces m < split_m write their k entries through `blob` (shared memory in the search kernel), the others and the
// trailing <q', q'> through `blob_hi` (a per-CTA global slice that stays in L2); both are indexed m * k + c. Default: one array.
__device__ inline void prepare_blob(const DataDesc &d, int metric, const float *__restrict__ q, float *blob, float *red, float *blob_hi = nullptr, int split_m = 1 << 30)
{
    if (!blob_hi) blob_hi = blob;
    const int tid = threadIdx.x, nt = blockDim.x;
    if (d.kind == KIND_F32) {
        float acc = 0.f;
        for (int i = tid; i < d.stride; i += nt) {
            float v = i < d.dim ? q[i] : 0.f;
            blob[i] = v;
            acc = fmaf(v, v, acc);
        }
        float qn = block_sum(acc, red);
        // blob[stride + 1] = an upper bound of ||q|| for the row-sketch bound (sketch_bound_pair): qn is q . q summed in fp32, within
        // gamma = (stride + 8) 2^-23 relative (any order of depth < stride + 8) plus what underflow can drop, (stride + 512) 2^-149
        if (tid == 0) {
            const float kq = __fmul_rn((float)(d.stride + 512), 0x1p-149f);
            const float g2 = __fadd_rn(1.0f, __fmul_rn((float)(d.stride + 8), 0x1p-22f));  // 1 + 2 gamma, exact
            blob[d.stride] = qn; blob[d.stride + 1] = __fsqrt_ru(__fmul_ru(__fadd_ru(qn, kq), g2)); blob[d.stride + 2] = 0.f; blob[d.stride + 3] = 0.f;
        }
    } else if (d.kind == KIND_PQ) {
        // LUT[m*k + c] = metric(centroid_{m,c}, q'[off_m..]) — PQDecoder.java:48-53, DefaultVectorUtilSupport.java:351-365.
        // One warp per sub-space m (its sizes / offset / query fragment are warp-uniform), lanes stride over the k centroids:
        // every lane streams one contiguous centroid, 128-bit loads when the sub-vector allows it. Accumulation order over the
        // sub-vector is sequential (j = 0..sz-1) for every entry.
        const int total = d.M * d.k;
        const int lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
        for (int m = warp; m < d.M; m += nw) {
            const int sz = d.sub_sizes[m], off = d.sub_offsets[m];
            const float *cb = d.codebooks + (size_t)d.k * off;
            if (sz == 8 && ((off & 3) == 0)) {
                float qv[8];
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    float qq = q[off + j];
                    if (d.centroid) qq = __fsub_rn(qq, d.centroid[off + j]);
                    qv[j] = qq;
                }
#pragma unroll 4
                for (int c = lane; c < d.k; c += 32) {
                    const float4 a = __ldg(reinterpret_cast<const float4 *>(cb + (size_t)c * 8));
                    const float4 b = __ldg(reinterpret_cast<const float4 *>(cb + (size_t)c * 8) + 1);
                    const float cen[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
                    float s = 0.f;
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        if (metric == JV_METRIC_EUCLIDEAN) {
                            const float df = __fsub_rn(cen[j], qv[j]);
                            s = fmaf(df, df, s);
                        } else s = fmaf(cen[j], qv[j], s);
                    }
                    (m < split_m ? blob : blob_hi)[m * d.k + c] = s;
                }
            } else {
                for (int c = lane; c < d.k; c += 32) {
                    const float *cen = cb + (size_t)c * sz;
                    float s = 0.f;
                    for (int j = 0; j < sz; j++) {
                        float qq = q[off + j];
                        if (d.centroid) qq = __fsub_rn(qq, d.centroid[off + j]);
                        if (metric == JV_METRIC_EUCLIDEAN) {
                            const float df = __fsub_rn(cen[j], qq);
                            s = fmaf(df, df, s);
                        } else s = fmaf(cen[j], qq, s);
                    }
                    (m < split_m ? blob : blob_hi)[m * d.k + c] = s;
                }
            }
        }
        float acc = 0.f;  // bMagnitude = <q', q'> (PQDecoder.java:119)
        for (int i = tid; i < d.dim; i += nt) {
            float qq = q[i];
            if (d.centroid) qq = __fsub_rn(qq, d.centroid[i]);
            acc = fmaf(qq, qq, acc);
        }
        float bm = block_sum(acc, red);
        if (tid == 0) blob_hi[total] = bm;
    } else if (d.kind == KIND_BQ) {
        // BinaryQuantization.java:96-109: bit j of word i = (v[64 i + j] > 0)
        unsigned long long *w = reinterpret_cast<unsigned long long *>(blob);
        const int lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
        for (int i = warp; i < 2 * d.W; i += nw) {  // 32-bit halves
            int idx = i * 32 + lane;
            bool bit = idx < d.dim && q[idx] > 0.f;
            unsigned b = __ballot_sync(FULL, bit);
            if (lane == 0) reinterpret_cast<unsigned *>(w)[i] = b;
        }
    } else {
        // NVQScorer.java: DOT keeps q and adds <q,mean>; L2 shifts q by mean; COSINE keeps q, needs ||q||
        float a0 = 0.f, a1 = 0.f;
        for (int i = tid; i < d.stride; i += nt) {
            float v = i < d.dim ? q[i] : 0.f;
            float mu = i < d.dim ? d.mean[i] : 0.f;
            a0 = fmaf(v, mu, a0);
            a1 = fmaf(v, v, a1);
            blob[i] = metric == JV_METRIC_EUCLIDEAN ? __fsub_rn(v, mu) : v;
        }
        float qb = block_sum(a0, red);
        float qq = block_sum(a1, red);
        if (tid == 0) { blob[d.stride] = qb; blob[d.stride + 1] = __fsqrt_rn(qq); blob[d.stride + 2] = 0.f; blob[d.stride + 3] = 0.f; }
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// fp32 rows — VectorUtilSupport.dotProduct / squareDistance / cosine (native-c:src/jvector_simd_kernels.cpp:208-287)
// one warp per row, 128-bit streaming loads, 4 independent accumulators, xor-shuffle reduction
// ------------------------------------------------------------------------------------------------
template <int METRIC>
__device__ __forceinline__ float score_f32_vec(const float4 *__restrict__ row, const float4 *__restrict__ q4, int n4, float qnorm2, int lane)
{
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f, b0 = 0.f, b1 = 0.f;
#pragma unroll 4
    for (int i = lane; i < n4; i += 32) {
        const float4 b = ldg_stream(row + i);
        const float4 a = q4[i];
        if (METRIC == JV_METRIC_EUCLIDEAN) {
            float d0 = a.x - b.x, d1 = a.y - b.y, d2 = a.z - b.z, d3 = a.w - b.w;
            s0 = fmaf(d0, d0, s0); s1 = fmaf(d1, d1, s1); s2 = fmaf(d2, d2, s2); s3 = fmaf(d3, d3, s3);
        } else {
            s0 = fmaf(a.x, b.x, s0); s1 = fmaf(a.y, b.y, s1); s2 = fmaf(a.z, b.z, s2); s3 = fmaf(a.w, b.w, s3);
            if (METRIC == JV_METRIC_COSINE) {
                b0 = fmaf(b.x, b.x, b0); b1 = fmaf(b.y, b.y, b1); b0 = fmaf(b.z, b.z, b0); b1 = fmaf(b.w, b.w, b1);
            }
        }
    }
    float s = group_sum<32>((s0 + s1) + (s2 + s3));
    if (METRIC == JV_METRIC_COSINE) {
        float bb = group_sum<32>(b0 + b1);
        s = __fdiv_rn(s, __fsqrt_rn(__fmul_rn(qnorm2, bb)));  // native: sum / sqrtf(aMag * bMag)
    }
    return s;
}

template <int METRIC>
__device__ __forceinline__ float score_f32(const DataDesc &d, const float *blob, int node, int lane)
{
    const float4 *row = reinterpret_cast<const float4 *>(d.rows + (size_t)node * d.stride);
    float raw = score_f32_vec<METRIC>(row, reinterpret_cast<const float4 *>(blob), d.stride >> 2, blob[d.stride], lane);
    return score_map(METRIC, raw);
}

// two rows against one query: both rows' loads are issued before either reduction, the query fragment is read once.
// Accumulation order per row is exactly score_f32_vec's, so a row scores identically in every kernel.
template <int METRIC>
__device__ __forceinline__ void score_f32_pair(const DataDesc &d, const float *blob, int nodeA, int nodeB, int lane, float &outA, float &outB)
{
    const float4 *ra = reinterpret_cast<const float4 *>(d.rows + (size_t)nodeA * d.stride);
    const float4 *rb = reinterpret_cast<const float4 *>(d.rows + (size_t)nodeB * d.stride);
    const float4 *q4 = reinterpret_cast<const float4 *>(blob);
    const int n4 = d.stride >> 2;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f, na0 = 0.f, na1 = 0.f, nb0 = 0.f, nb1 = 0.f;
#pragma unroll 3
    for (int i = lane; i < n4; i += 32) {
        const float4 x = ldg_stream(ra + i);
        const float4 y = ldg_stream(rb + i);
        const float4 q = q4[i];
        if (METRIC == JV_METRIC_EUCLIDEAN) {
            float d0 = q.x - x.x, d1 = q.y - x.y, d2 = q.z - x.z, d3 = q.w - x.w;
            a0 = fmaf(d0, d0, a0); a1 = fmaf(d1, d1, a1); a2 = fmaf(d2, d2, a2); a3 = fmaf(d3, d3, a3);
            d0 = q.x - y.x; d1 = q.y - y.y; d2 = q.z - y.z; d3 = q.w - y.w;
            b0 = fmaf(d0, d0, b0); b1 = fmaf(d1, d1, b1); b2 = fmaf(d2, d2, b2); b3 = fmaf(d3, d3, b3);
        } else {
            a0 = fmaf(q.x, x.x, a0); a1 = fmaf(q.y, x.y, a1); a2 = fmaf(q.z, x.z, a2); a3 = fmaf(q.w, x.w, a3);
            b0 = fmaf(q.x, y.x, b0); b1 = fmaf(q.y, y.y, b1); b2 = fmaf(q.z, y.z, b2); b3 = fmaf(q.w, y.w, b3);
            if (METRIC == JV_METRIC_COSINE) {
                na0 = fmaf(x.x, x.x, na0); na1 = fmaf(x.y, x.y, na1); na0 = fmaf(x.z, x.z, na0); na1 = fmaf(x.w, x.w, na1);
                nb0 = fmaf(y.x, y.x, nb0); nb1 = fmaf(y.y, y.y, nb1); nb0 = fmaf(y.z, y.z, nb0); nb1 = fmaf(y.w, y.w, nb1);
            }
        }
    }
    float sa = group_sum<32>((a0 + a1) + (a2 + a3)), sb = group_sum<32>((b0 + b1) + (b2 + b3));
    if (METRIC == JV_METRIC_COSINE) {
        const float qn = blob[d.stride];
        sa = __fdiv_rn(sa, __fsqrt_rn(__fmul_rn(qn, group_sum<32>(na0 + na1))));
        sb = __fdiv_rn(sb, __fsqrt_rn(__fmul_rn(qn, group_sum<32>(nb0 + nb1))));
    }
    outA = score_map(METRIC, sa);
    outB = score_map(METRIC, sb);
}

// Upper bounds of the DOT_PRODUCT scores score_f32 would give two rows, from their int8 sketches (row_sketch_kernel) at a quarter
// of the bytes. With c the codes as fp32, s_c = fl(q . c) in any order, x_hat = s c, gamma = (stride + 8) 2^-23 (the relative error
// bound of an fp32 sum of depth < stride + 8, met by this sum and by score_f32's) and kd = (stride + 512) 2^-149 (what underflow can
// add to one such sum):
//   fl(q . x) <= q . x + gamma ||q|| ||x|| + kd = q . x_hat + q . (x - x_hat) + gamma ||q|| ||x|| + kd
//             <= s s_c + ||q|| (||x - x_hat|| + gamma (||x|| + ||x_hat||)) + kd (1 + s) = s s_c + ||q|| r + kd (1 + s),
// evaluated rounding upward; score_map is monotone, so the bound survives it. blob[stride + 1] is ||q|| rounded up (prepare_blob).
// Both rows' loads are in flight before either reduction, as in score_f32_pair.
__device__ __forceinline__ void sketch_bound_pair(const DataDesc &d, const float *blob, int nodeA, int nodeB, int lane, float &outA, float &outB)
{
    const uint2 *ra = reinterpret_cast<const uint2 *>(d.sketch + (size_t)nodeA * d.sketch_stride);
    const uint2 *rb = reinterpret_cast<const uint2 *>(d.sketch + (size_t)nodeB * d.sketch_stride);
    const float2 ma = __ldg(d.sketch_meta + nodeA), mb = __ldg(d.sketch_meta + nodeB);  // {s, r}
    const float4 *q4 = reinterpret_cast<const float4 *>(blob);
    const int n8 = d.sketch_stride >> 3;  // 8 codes per load; a stride of 8 m + 4 ends in 4 padding codes, read against q = 0
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
#pragma unroll 3
    for (int i = lane; i < n8; i += 32) {
        const uint2 x = ldg_stream_u2(ra + i);
        const uint2 y = ldg_stream_u2(rb + i);
        const float4 qa = q4[2 * i], qb = 8 * i + 4 < d.stride ? q4[2 * i + 1] : z4;
        const float q[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            const unsigned wx = j < 4 ? x.x : x.y, wy = j < 4 ? y.x : y.y;
            const int sh = 8 * (j & 3);
            a0 = fmaf(q[j], (float)(int8_t)(wx >> sh), a0); a1 = fmaf(q[j + 1], (float)(int8_t)(wx >> (sh + 8)), a1);
            b0 = fmaf(q[j], (float)(int8_t)(wy >> sh), b0); b1 = fmaf(q[j + 1], (float)(int8_t)(wy >> (sh + 8)), b1);
        }
    }
    const float sa = group_sum<32>(a0 + a1), sb = group_sum<32>(b0 + b1);
    const float qn = blob[d.stride + 1];
    const float kd = __fmul_rn((float)(d.stride + 512), 0x1p-149f);
    const float ua = __fadd_ru(__fmaf_ru(qn, ma.y, __fmul_ru(sa, ma.x)), __fmaf_ru(kd, ma.x, kd));
    const float ub = __fadd_ru(__fmaf_ru(qn, mb.y, __fmul_ru(sb, mb.x)), __fmaf_ru(kd, mb.x, kd));
    outA = score_map(JV_METRIC_DOT, ua);
    outB = score_map(JV_METRIC_DOT, ub);
}

// ------------------------------------------------------------------------------------------------
// PQ ADC — VectorUtilSupport.assembleAndSum / pqDecodedCosineSimilarity
// (DefaultVectorUtilSupport.java:303-309; native-c:...:662-724,821-879). 8 lanes per code row, 4 codes per 32-bit load.
// ------------------------------------------------------------------------------------------------
template <int METRIC>
__device__ __forceinline__ float score_pq_codes(const DataDesc &d, const float *lut_lo, const uint8_t *__restrict__ c, int g, const float *lut_hi = nullptr,
                                                int split_m = 1 << 30)
{
    // sub-spaces m < split_m (a multiple of 4) are looked up in lut_lo, the rest (and the cosine query norm) in lut_hi
    if (!lut_hi) lut_hi = lut_lo;
    const int k = d.k, M = d.M;
    float s = 0.f, a = 0.f;
    const int M4 = M >> 2;
    const uint32_t *c4 = reinterpret_cast<const uint32_t *>(c);
    for (int j = g; j < M4; j += 8) {
        const uint32_t w = __ldg(c4 + j);
        const int base = (4 * j) * k;
        const float *lut = 4 * j < split_m ? lut_lo : lut_hi;
        const int i0 = base + (int)(w & 255u), i1 = base + k + (int)((w >> 8) & 255u), i2 = base + 2 * k + (int)((w >> 16) & 255u),
                  i3 = base + 3 * k + (int)(w >> 24);
        s = __fadd_rn(s, lut[i0]); s = __fadd_rn(s, lut[i1]); s = __fadd_rn(s, lut[i2]); s = __fadd_rn(s, lut[i3]);
        if (METRIC == JV_METRIC_COSINE) {
            a = __fadd_rn(a, __ldg(d.mag + i0)); a = __fadd_rn(a, __ldg(d.mag + i1));
            a = __fadd_rn(a, __ldg(d.mag + i2)); a = __fadd_rn(a, __ldg(d.mag + i3));
        }
    }
    for (int m = 4 * M4 + g; m < M; m += 8) {
        const int idx = m * k + (int)c[m];
        s = __fadd_rn(s, (m < split_m ? lut_lo : lut_hi)[idx]);
        if (METRIC == JV_METRIC_COSINE) a = __fadd_rn(a, __ldg(d.mag + idx));
    }
    s = group_sum<8>(s);
    if (METRIC == JV_METRIC_COSINE) {
        a = group_sum<8>(a);
        s = __fdiv_rn(s, __fsqrt_rn(__fmul_rn(a, lut_hi[M * k])));  // native-c:...:879
    }
    return score_map(METRIC, s);
}

// The same score split the way the butterfly of score_pq_codes splits it: lane g of the 8 keeps the running sum of words g, g + 8, ...
// (then tail element g), and the 8 sums are folded by xor 4, 2, 1. score_pq_partial computes sum g alone (codes already in
// shared memory), pq_fold8 folds eight of them in the same tree, so partial sums computed by eight different WARPS give the same
// bits. The search kernel uses this to make every gather instruction of a warp stay inside one 1 KB LUT row (lane = candidate,
// warp = partial sum): at most 8 lines per instruction instead of 32.
template <int METRIC>
__device__ __forceinline__ void score_pq_partial(const DataDesc &d, const float *lut_lo, const float *lut_hi, int split_m, const uint8_t *c, int g, float &s_out,
                                                 float &a_out)
{
    const int k = d.k, M = d.M, M4 = M >> 2;
    float s = 0.f, a = 0.f;
    const uint32_t *c4 = reinterpret_cast<const uint32_t *>(c);
    for (int j = g; j < M4; j += 8) {
        const uint32_t w = c4[j];
        const int base = (4 * j) * k;
        const float *lut = 4 * j < split_m ? lut_lo : lut_hi;
        const int i0 = base + (int)(w & 255u), i1 = base + k + (int)((w >> 8) & 255u), i2 = base + 2 * k + (int)((w >> 16) & 255u),
                  i3 = base + 3 * k + (int)(w >> 24);
        s = __fadd_rn(s, lut[i0]); s = __fadd_rn(s, lut[i1]); s = __fadd_rn(s, lut[i2]); s = __fadd_rn(s, lut[i3]);
        if (METRIC == JV_METRIC_COSINE) {
            a = __fadd_rn(a, __ldg(d.mag + i0)); a = __fadd_rn(a, __ldg(d.mag + i1));
            a = __fadd_rn(a, __ldg(d.mag + i2)); a = __fadd_rn(a, __ldg(d.mag + i3));
        }
    }
    const int m = 4 * M4 + g;
    if (m < M) {
        const int idx = m * k + (int)c[m];
        s = __fadd_rn(s, (m < split_m ? lut_lo : lut_hi)[idx]);
        if (METRIC == JV_METRIC_COSINE) a = __fadd_rn(a, __ldg(d.mag + idx));
    }
    s_out = s;
    a_out = a;
}
// p[g * stride], g = 0..7 -> group_sum<8>'s tree (xor 4, xor 2, xor 1)
__device__ __forceinline__ float pq_fold8(const float *p, int stride)
{
    return __fadd_rn(__fadd_rn(__fadd_rn(p[0], p[4 * stride]), __fadd_rn(p[2 * stride], p[6 * stride])),
                     __fadd_rn(__fadd_rn(p[stride], p[5 * stride]), __fadd_rn(p[3 * stride], p[7 * stride])));
}

template <int METRIC>
__device__ __forceinline__ float score_pq(const DataDesc &d, const float *lut, int node, int g, const float *lut_hi = nullptr, int split_m = 1 << 30)
{
    return score_pq_codes<METRIC>(d, lut, d.codes + (size_t)node * d.code_stride, g, lut_hi, split_m);
}

// ------------------------------------------------------------------------------------------------
// BQ Hamming — VectorUtilSupport.hammingDistance + BQVectors.similarityBetween
// (DefaultVectorUtilSupport.java:342-348, BQVectors.java:116-118): integer exact
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float bq_score_from_hd(int hd, int dim) { return __fsub_rn(1.0f, __fdiv_rn((float)hd, (float)dim)); }

__device__ __forceinline__ float score_bq(const DataDesc &d, const float *blob, int node, int g)
{
    const unsigned long long *q = reinterpret_cast<const unsigned long long *>(blob);
    const unsigned long long *w = d.words + (size_t)node * d.W;
    int hd = 0;
    for (int i = g; i < d.W; i += 8) hd += __popcll(__ldg(w + i) ^ q[i]);
    hd = group_sum_int<8>(hd);
    return bq_score_from_hd(hd, d.dim);
}

// ------------------------------------------------------------------------------------------------
// NVQ 8-bit — VectorUtilSupport.nvqDotProduct8bit / nvqSquareL2Distance8bit / nvqCosine8bit, SIMD/native form
// (PanamaVectorUtilSupport.java:1164-1237, native-c:...:1047-1111,1359-1641); dequantisation fused into the sum.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float nvq_logistic(float v, float alpha, float x0)
{
    const float t = __fmaf_rn(v, alpha, __fmul_rn(-alpha, x0));
    const int p = (__float_as_int(t) < 0) ? __float2int_rz(t) : __float2int_rz(__fadd_rn(t, 1.0f));
    const float e = (float)p;
    const int m = __float_as_int(__fmaf_rn(__fsub_rn(t, e), 0.5f, 1.0f));
    const float r = __int_as_float((int)((unsigned)m + ((unsigned)p << 23)));
    return __fdiv_rn(r, __fadd_rn(r, 1.0f));
}

__device__ __forceinline__ float nvq_logit(float v, float inv_alpha, float x0)
{
    const float z = __fdiv_rn(v, __fsub_rn(1.0f, v));
    const int t = __float_as_int(z);
    const int p = ((t & 0x7f800000) >> 23) - 128;
    const float m = __int_as_float((t & 0x007fffff) + 0x3f800000);
    return __fmaf_rn(__fadd_rn(m, (float)p), inv_alpha, x0);
}

struct NvqConsts {
    float sa, isa, sx0, bias, scale;
};

__device__ __forceinline__ NvqConsts nvq_setup(float minv, float maxv, float alpha, float x0, float levels)
{
    NvqConsts c;
    const float delta = __fsub_rn(maxv, minv);
    c.sa = __fdiv_rn(alpha, delta);
    c.isa = __fdiv_rn(delta, alpha);  // native-c:...:1380
    c.sx0 = __fmul_rn(x0, delta);
    c.bias = nvq_logistic(minv, c.sa, c.sx0);
    c.scale = __fdiv_rn(__fsub_rn(nvq_logistic(maxv, c.sa, c.sx0), c.bias), levels);
    return c;
}

__device__ __forceinline__ float nvq_dequant(const NvqConsts &c, float byteval)
{
    return nvq_logit(__fmaf_rn(byteval, c.scale, c.bias), c.isa, c.sx0);
}

template <int METRIC>
__device__ __forceinline__ void nvq_accum(float q, float dq, float mu, float &s, float &nm)
{
    if (METRIC == JV_METRIC_DOT) s = __fmaf_rn(q, dq, s);
    else if (METRIC == JV_METRIC_EUCLIDEAN) {
        const float df = __fsub_rn(q, dq);
        s = __fmaf_rn(df, df, s);
    } else {
        const float e = __fadd_rn(dq, mu);
        s = __fmaf_rn(q, e, s);
        nm = __fmaf_rn(e, e, nm);
    }
}

template <int METRIC>
__device__ __forceinline__ float score_nvq(const DataDesc &d, const float *blob, int node, int lane)
{
    const uint8_t *row = d.bytes + (size_t)node * d.byte_stride;
    const float *prm = d.params + (size_t)node * 4 * d.nsub;
    float s = 0.f, nm = 0.f;
    for (int sv = 0; sv < d.nsub; sv++) {
        const float4 p4 = __ldg(reinterpret_cast<const float4 *>(prm) + sv);  // {min, max, growthRate, midpoint}
        const NvqConsts c = nvq_setup(p4.x, p4.y, p4.z, p4.w, 255.0f);
        const int off = d.sub_offsets[sv], sz = d.sub_sizes[sv];
        if (((off | sz) & 3) == 0) {
            const uint32_t *b4 = reinterpret_cast<const uint32_t *>(row + off);
            const float4 *q4 = reinterpret_cast<const float4 *>(blob + off);
            const float4 *m4 = reinterpret_cast<const float4 *>(d.mean + off);
#pragma unroll 2
            for (int i = lane; i < (sz >> 2); i += 32) {
                const uint32_t w = __ldg(b4 + i);
                const float4 q = q4[i];
                float4 mu = make_float4(0.f, 0.f, 0.f, 0.f);
                if (METRIC == JV_METRIC_COSINE) mu = __ldg(m4 + i);
                nvq_accum<METRIC>(q.x, nvq_dequant(c, (float)(w & 255u)), mu.x, s, nm);
                nvq_accum<METRIC>(q.y, nvq_dequant(c, (float)((w >> 8) & 255u)), mu.y, s, nm);
                nvq_accum<METRIC>(q.z, nvq_dequant(c, (float)((w >> 16) & 255u)), mu.z, s, nm);
                nvq_accum<METRIC>(q.w, nvq_dequant(c, (float)(w >> 24)), mu.w, s, nm);
            }
        } else {
            for (int i = lane; i < sz; i += 32) {
                const float mu = METRIC == JV_METRIC_COSINE ? __ldg(d.mean + off + i) : 0.f;
                nvq_accum<METRIC>(blob[off + i], nvq_dequant(c, (float)row[off + i]), mu, s, nm);
            }
        }
    }
    s = group_sum<32>(s);
    if (METRIC == JV_METRIC_DOT) return __fdiv_rn(__fadd_rn(__fadd_rn(1.0f, s), blob[d.stride]), 2.0f);  // NVQScorer.java:67
    if (METRIC == JV_METRIC_EUCLIDEAN) return __fdiv_rn(1.0f, __fadd_rn(1.0f, s));                       // :98
    nm = group_sum<32>(nm);
    const float cosine = __fdiv_rn(__fdiv_rn(s, blob[d.stride + 1]), __fsqrt_rn(nm));  // :129
    return __fdiv_rn(__fadd_rn(1.0f, cosine), 2.0f);
}

// ------------------------------------------------------------------------------------------------
// dispatch
// ------------------------------------------------------------------------------------------------
template <int KIND, int METRIC>
__device__ __forceinline__ float score_row(const DataDesc &d, const float *blob, int node, int lane_in_group)
{
    if (KIND == KIND_F32) return score_f32<METRIC>(d, blob, node, lane_in_group);
    if (KIND == KIND_PQ) return score_pq<METRIC>(d, blob, node, lane_in_group);
    if (KIND == KIND_BQ) return score_bq(d, blob, node, lane_in_group);
    return score_nvq<METRIC>(d, blob, node, lane_in_group);
}

// ------------------------------------------------------------------------------------------------
// node-vs-node ("diversity") scores: BuildScoreProvider.diversityProviderFor
//   f32: exact compare of two rows; PQ: codebook-vs-codebook (PQVectors.java:284-350); BQ: BQVectors.java:98-105
// ------------------------------------------------------------------------------------------------
template <int METRIC>
__device__ __forceinline__ float pair_f32(const DataDesc &d, int a, int b, int lane)
{
    const float4 *ra = reinterpret_cast<const float4 *>(d.rows + (size_t)a * d.stride);
    const float4 *rb = reinterpret_cast<const float4 *>(d.rows + (size_t)b * d.stride);
    const int n4 = d.stride >> 2;
    float s0 = 0.f, s1 = 0.f, aa = 0.f, bb = 0.f;
#pragma unroll 4
    for (int i = lane; i < n4; i += 32) {
        const float4 x = ldg_stream(ra + i), y = ldg_stream(rb + i);
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

template <int METRIC>
__device__ __forceinline__ float pair_pq(const DataDesc &d, int a, int b, int lane)
{
    const uint8_t *ca = d.codes + (size_t)a * d.code_stride, *cb = d.codes + (size_t)b * d.code_stride;
    float s = 0.f, n1 = 0.f, n2 = 0.f;
    for (int m = lane; m < d.M; m += 32) {
        const int sz = d.sub_sizes[m];
        const float *base = d.codebooks + (size_t)d.k * d.sub_offsets[m];
        const float *x = base + (size_t)ca[m] * sz, *y = base + (size_t)cb[m] * sz;
        float t = 0.f, tx = 0.f, ty = 0.f;
        for (int j = 0; j < sz; j++) {
            if (METRIC == JV_METRIC_EUCLIDEAN) {
                const float df = __fsub_rn(x[j], y[j]);
                t = fmaf(df, df, t);
            } else {
                t = fmaf(x[j], y[j], t);
                if (METRIC == JV_METRIC_COSINE) { tx = fmaf(x[j], x[j], tx); ty = fmaf(y[j], y[j], ty); }
            }
        }
        s = __fadd_rn(s, t); n1 = __fadd_rn(n1, tx); n2 = __fadd_rn(n2, ty);
    }
    s = group_sum<32>(s);
    if (METRIC == JV_METRIC_COSINE) {
        n1 = group_sum<32>(n1);
        n2 = group_sum<32>(n2);
        s = __fdiv_rn(s, __fsqrt_rn(__fmul_rn(n1, n2)));
    }
    return score_map(METRIC, s);
}

// assembleAndSumPQ (base:vector/DefaultVectorUtilSupport.java:321-336, native-c:src/jvector_simd_kernels.cpp:729-815) composed as
// ImmutablePQVectors.diversityFunctionFor does (base:quantization/ImmutablePQVectors.java:63-105): per sub-space one gather from the
// triangular centroid-vs-centroid table at (min(c1, c2), max(c1, c2)); cosine needs the two self sums as well.
__device__ __forceinline__ int tri_index(int a, int b, int k)
{
    const int r = min(a, b), c = max(a, b);
    return r * k - (r * (r - 1) / 2) + (c - r);
}

template <int METRIC>
__device__ __forceinline__ float pair_pq_table(const DataDesc &d, int a, int b, int lane)
{
    const uint8_t *ca = d.codes + (size_t)a * d.code_stride, *cb = d.codes + (size_t)b * d.code_stride;
    const float *T = d.pair_table[METRIC == JV_METRIC_EUCLIDEAN ? 0 : 1];
    const int k = d.k, block = k * (k + 1) / 2;
    float s = 0.f, n1 = 0.f, n2 = 0.f;
    for (int m = lane; m < d.M; m += 32) {
        const float *Tm = T + (size_t)m * block;
        const int x = ca[m], y = cb[m];
        s = __fadd_rn(s, __ldg(Tm + tri_index(x, y, k)));
        if (METRIC == JV_METRIC_COSINE) {
            n1 = __fadd_rn(n1, __ldg(Tm + tri_index(x, x, k)));
            n2 = __fadd_rn(n2, __ldg(Tm + tri_index(y, y, k)));
        }
    }
    s = group_sum<32>(s);
    if (METRIC == JV_METRIC_COSINE) {
        n1 = group_sum<32>(n1);
        n2 = group_sum<32>(n2);
        s = __fdiv_rn(s, __fsqrt_rn(__fmul_rn(n1, n2)));
    }
    return score_map(METRIC, s);
}

__device__ __forceinline__ float pair_bq(const DataDesc &d, int a, int b, int lane)
{
    const unsigned long long *x = d.words + (size_t)a * d.W, *y = d.words + (size_t)b * d.W;
    int hd = 0;
    for (int i = lane; i < d.W; i += 32) hd += __popcll(__ldg(x + i) ^ __ldg(y + i));
    hd = group_sum_int<32>(hd);
    return bq_score_from_hd(hd, d.dim);
}

}  // namespace jv
