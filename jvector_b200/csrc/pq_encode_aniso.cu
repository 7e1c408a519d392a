// pq_encode_aniso.cu — ProductQuantization.encodeAnisotropic on the device (base:quantization/ProductQuantization.java:269-420).
//
// One definition, restated bit for bit by tests/pq_aniso_model.py. For a row v (minus the global centroid), with every dot product
// accumulated in order in fp32 (round to nearest, no FMA):
//   inv = (float)(1 / sqrt((double)|v|^2)), |v|^2 over the whole row;
//   per sub-space m and centroid c: dot = c.x, R = fl(fl(|c|^2 - fl(2 dot)) + |x|^2), P = fl(fl(e * e) * inv), e = fl(dot - |x|^2);
//   start: per sub-space the first minimum R (code 0 when no R is below +inf), S = sum over m in order of P(start);
//   up to 10 sweeps over m = 0..M-1: for every candidate c != code[m] in index order S' = fl(fl(S - P_old) + P_c),
//   dP = fl(fl(S' S') - fl(S S)); skip when dP > 0; cost = fl(fl(pcm dP) + fl(fl(R_c - R_old) - dP)); the strictly least cost < 0
//   moves code[m] and sets S = S'. A sweep that moves nothing ends the row.
// A zero row has inv = +inf, so every P is NaN, no cost is below 0 and the row keeps its start, as in the reference.
//
// Shape: a CTA owns ENC_TILE rows (one warp walks ENC_ROWS of them) and the sub-spaces in lockstep. Per sub-space the codebook,
// transposed to [size_m][k] so that the lanes' candidates are consecutive floats, and its |c|^2 are staged in shared memory once for
// the tile; each (row, sub-space) recomputes its (R, P) for all k candidates (lane l takes c = l, l + 32, ...) and takes one
// descent step with an arg-min shuffle (ties to the lower index). Nothing per (row, candidate) is stored: the whole table would be
// M * k * 8 bytes per row.
#include "kernels.h"

namespace jv {
namespace {

constexpr int ENC_ROWS = 8;                     // rows per warp
constexpr int ENC_TILE = 8 * ENC_ROWS;          // rows per CTA (8 warps)
constexpr int ENC_REG = 16;                     // sub-vectors up to this size stay in registers
constexpr int ENC_SWEEPS = 10;                  // MAX_ITERATIONS of encodeAnisotropic
constexpr size_t ENC_SMEM_MAX = 96 * 1024;      // a codebook above this is read from global memory instead of shared memory

// the transposed codebooks ([size_m][k] at k * offset_m) and |c|^2 [M][k], accumulated in order; one thread per (m, c)
__global__ void pq_encode_aniso_prep_kernel(DataDesc pq, float *__restrict__ cbT, float *__restrict__ cn)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= pq.M * pq.k) return;
    const int m = idx / pq.k, c = idx - m * pq.k, k = pq.k;
    const int sz = pq.sub_sizes[m], off = pq.sub_offsets[m];
    const float *src = pq.codebooks + (size_t)k * off + (size_t)c * sz;
    float s = 0.f;
    for (int t = 0; t < sz; t++) {
        const float v = src[t];
        cbT[(size_t)k * off + (size_t)t * k + c] = v;
        s = __fadd_rn(s, __fmul_rn(v, v));
    }
    cn[idx] = s;
}

// c.x accumulated in order: x from registers (REG) or from the row (minus the centroid) in global memory
template <bool REG>
__device__ __forceinline__ float cdot(const float *cb, int k, int c, int sz, const float *xr, const float *v, const float *cv)
{
    float s = 0.f;
    if (REG) {
#pragma unroll
        for (int t = 0; t < ENC_REG; t++)
            if (t < sz) s = __fadd_rn(s, __fmul_rn(cb[t * k + c], xr[t]));
    } else {
        for (int t = 0; t < sz; t++) {
            float x = v[t];
            if (cv) x = __fsub_rn(x, cv[t]);
            s = __fadd_rn(s, __fmul_rn(cb[t * k + c], x));
        }
    }
    return s;
}

template <bool REG>
__global__ void __launch_bounds__(256) pq_encode_aniso_kernel(DataDesc pq, const float *__restrict__ rows, long long n, int stride,
                                                              const float *__restrict__ cbT, const float *__restrict__ cn, float pcm, bool staged,
                                                              uint8_t *__restrict__ codes, unsigned long long *__restrict__ stats)
{
    extern __shared__ float s_cb[];
    __shared__ float s_S[ENC_TILE], s_inv[ENC_TILE];
    __shared__ int s_active[ENC_TILE], s_changed[ENC_TILE], s_moves[ENC_TILE], s_sweeps[ENC_TILE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int dim = pq.dim, M = pq.M, k = pq.k;
    const float *cen = pq.centroid;
    const long long row0 = (long long)blockIdx.x * ENC_TILE;
    if (threadIdx.x < ENC_TILE) {
        const int t = threadIdx.x;
        const long long r = row0 + t;
        s_S[t] = 0.f;
        s_changed[t] = s_moves[t] = s_sweeps[t] = 0;
        s_active[t] = r < n;
        if (r < n) {
            const float *v = rows + r * stride;
            float s = 0.f;
            for (int d = 0; d < dim; d++) {
                float x = v[d];
                if (cen) x = __fsub_rn(x, cen[d]);
                s = __fadd_rn(s, __fmul_rn(x, x));
            }
            s_inv[t] = __double2float_rn(__ddiv_rn(1.0, __dsqrt_rn((double)s)));
        }
    }
    __syncthreads();
    for (int pass = 0; pass <= ENC_SWEEPS; pass++) {
        if (pass > 0 && !__syncthreads_or(threadIdx.x < ENC_TILE && s_active[threadIdx.x])) break;
        for (int m = 0; m < M; m++) {
            const int sz = pq.sub_sizes[m], off = pq.sub_offsets[m];
            const float *cb = cbT + (size_t)k * off, *nm = cn + (size_t)m * k;
            if (staged) {
                __syncthreads();
                for (int q = threadIdx.x; q < k * sz; q += blockDim.x) s_cb[q] = cb[q];
                for (int q = threadIdx.x; q < k; q += blockDim.x) s_cb[k * sz + q] = nm[q];
                __syncthreads();
                cb = s_cb;
                nm = s_cb + k * sz;
            }
            for (int rr = 0; rr < ENC_ROWS; rr++) {
                const int t = warp * ENC_ROWS + rr;
                const long long r = row0 + t;
                if (r >= n || !s_active[t]) continue;
                const float *v = rows + r * stride + off;
                const float *cv = cen ? cen + off : nullptr;
                float xr[REG ? ENC_REG : 1];
                float xx = 0.f;
                if (REG) {
#pragma unroll
                    for (int u = 0; u < ENC_REG; u++) {
                        float x = 0.f;
                        if (u < sz) {
                            x = v[u];
                            if (cv) x = __fsub_rn(x, cv[u]);
                            xx = __fadd_rn(xx, __fmul_rn(x, x));
                        }
                        xr[u] = x;
                    }
                } else
                    for (int u = 0; u < sz; u++) {
                        float x = v[u];
                        if (cv) x = __fsub_rn(x, cv[u]);
                        xx = __fadd_rn(xx, __fmul_rn(x, x));
                    }
                const float inv = s_inv[t];
                uint8_t *code = codes + r * M + m;
                if (pass == 0) {
                    // the first minimum residual, and its parallel component
                    float bR = __int_as_float(0x7f800000), bP = 0.f, p0 = 0.f;
                    int bI = 0x7fffffff;
                    for (int c = lane; c < k; c += 32) {
                        const float d = cdot<REG>(cb, k, c, sz, xr, v, cv);
                        const float R = __fadd_rn(__fsub_rn(nm[c], __fmul_rn(2.f, d)), xx);
                        const float e = __fsub_rn(d, xx);
                        const float P = __fmul_rn(__fmul_rn(e, e), inv);
                        if (c == lane) p0 = P;
                        if (R < bR) { bR = R; bI = c; bP = P; }
                    }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        const float oR = __shfl_xor_sync(FULL, bR, o), oP = __shfl_xor_sync(FULL, bP, o);
                        const int oI = __shfl_xor_sync(FULL, bI, o);
                        if (oR < bR || (oR == bR && oI < bI)) { bR = oR; bI = oI; bP = oP; }
                    }
                    const float P0 = __shfl_sync(FULL, p0, 0);
                    if (lane == 0) {
                        *code = (uint8_t)(bI == 0x7fffffff ? 0 : bI);
                        s_S[t] = __fadd_rn(s_S[t], bI == 0x7fffffff ? P0 : bP);
                    }
                } else {
                    // one coordinate-descent step (optimizeSingleSubspace)
                    const int old = *code;
                    const float dold = cdot<REG>(cb, k, old, sz, xr, v, cv);
                    const float Rold = __fadd_rn(__fsub_rn(nm[old], __fmul_rn(2.f, dold)), xx);
                    const float eold = __fsub_rn(dold, xx);
                    const float Pold = __fmul_rn(__fmul_rn(eold, eold), inv);
                    const float S = s_S[t], S2 = __fmul_rn(S, S);
                    float bC = 0.f, bS = 0.f;
                    int bI = 0x7fffffff;
                    for (int c = lane; c < k; c += 32) {
                        if (c == old) continue;
                        const float d = cdot<REG>(cb, k, c, sz, xr, v, cv);
                        const float R = __fadd_rn(__fsub_rn(nm[c], __fmul_rn(2.f, d)), xx);
                        const float e = __fsub_rn(d, xx);
                        const float P = __fmul_rn(__fmul_rn(e, e), inv);
                        const float Sn = __fadd_rn(__fsub_rn(S, Pold), P);
                        const float dP = __fsub_rn(__fmul_rn(Sn, Sn), S2);
                        if (dP > 0.f) continue;
                        const float cost = __fadd_rn(__fmul_rn(pcm, dP), __fsub_rn(__fsub_rn(R, Rold), dP));
                        if (cost < bC) { bC = cost; bI = c; bS = Sn; }
                    }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        const float oC = __shfl_xor_sync(FULL, bC, o), oS = __shfl_xor_sync(FULL, bS, o);
                        const int oI = __shfl_xor_sync(FULL, bI, o);
                        if (oC < bC || (oC == bC && oI < bI)) { bC = oC; bI = oI; bS = oS; }
                    }
                    if (lane == 0 && bI != 0x7fffffff) {
                        *code = (uint8_t)bI;
                        s_S[t] = bS;
                        s_changed[t] = 1;
                        s_moves[t]++;
                    }
                }
                __syncwarp();
            }
        }
        __syncthreads();
        if (pass > 0 && threadIdx.x < ENC_TILE && s_active[threadIdx.x]) {
            const int t = threadIdx.x;
            s_sweeps[t]++;
            if (!s_changed[t]) s_active[t] = 0;
            s_changed[t] = 0;
        }
    }
    __syncthreads();
    if (threadIdx.x < ENC_TILE && row0 + threadIdx.x < n) {
        const int t = threadIdx.x;
        if (s_moves[t]) {
            atomicAdd(stats, 1ull);
            atomicAdd(stats + 1, (unsigned long long)s_moves[t]);
        }
        atomicMax(stats + 2, (unsigned long long)s_sweeps[t]);
    }
}

template <bool REG>
cudaError_t launch(const DataDesc &pq, const float *rows, long long n, int stride, const float *cbT, const float *cn, float pcm, uint8_t *codes,
                   unsigned long long *stats, size_t smem, cudaStream_t s)
{
    auto kern = pq_encode_aniso_kernel<REG>;
    const bool staged = smem <= ENC_SMEM_MAX;
    if (staged) {
        const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    kern<<<(unsigned)((n + ENC_TILE - 1) / ENC_TILE), 256, staged ? smem : 0, s>>>(pq, rows, n, stride, cbT, cn, pcm, staged, codes, stats);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace

size_t pq_encode_aniso_scratch(int dim, int M, int k)
{
    Carver c(nullptr);
    c.take<float>((size_t)k * dim);
    c.take<float>((size_t)M * k);
    return c.bytes;
}

cudaError_t launch_pq_encode_aniso(const DataDesc &pq, const float *rows_dev, long long n, int row_stride, float pcm, void *scratch,
                                   unsigned long long *stats_dev, uint8_t *codes_dev, cudaStream_t s)
{
    const int dim = pq.dim, M = pq.M, k = pq.k;
    Carver c(scratch);
    float *cbT = c.take<float>((size_t)k * dim), *cn = c.take<float>((size_t)M * k);
    cudaError_t e = cudaMemsetAsync(stats_dev, 0, 3 * sizeof(unsigned long long), s);
    if (e != cudaSuccess || n <= 0) return e;
    if ((n + ENC_TILE - 1) / ENC_TILE > 0x7fffffffLL) return cudaErrorInvalidValue;
    pq_encode_aniso_prep_kernel<<<(M * k + 255) / 256, 256, 0, s>>>(pq, cbT, cn);
    g_launches++;
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    const int szmax = (dim + M - 1) / M;
    const size_t smem = ((size_t)k * szmax + k) * 4;
    if (szmax <= ENC_REG) return launch<true>(pq, rows_dev, n, row_stride, cbT, cn, pcm, codes_dev, stats_dev, smem, s);
    return launch<false>(pq, rows_dev, n, row_stride, cbT, cn, pcm, codes_dev, stats_dev, smem, s);
}

}  // namespace jv
