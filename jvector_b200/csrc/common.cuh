// common.cuh — shared device helpers for the sm_90a scoring kernels.
// Compiled with -fmad=false: every fused multiply-add in this library is an explicit fmaf()/__fmaf_rn(), so the
// NVQ bit tricks and the similarity->score maps round exactly like the reference's scalar code.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define JV_METRIC_EUCLIDEAN 0
#define JV_METRIC_DOT 1
#define JV_METRIC_COSINE 2

namespace jv {

constexpr unsigned FULL = 0xffffffffu;

// base:vector/VectorSimilarityFunction.java:37-69 — similarity -> score, fused into every kernel epilogue
__device__ __forceinline__ float score_map(int metric, float raw)
{
    if (metric == JV_METRIC_EUCLIDEAN) return __fdiv_rn(1.0f, __fadd_rn(1.0f, raw));
    return __fdiv_rn(__fadd_rn(1.0f, raw), 2.0f);
}

// base:util/NumericUtils.java:63-65 + base:graph/NodeQueue.java:125-137
__device__ __forceinline__ int32_t float_to_sortable(float f)
{
    int32_t b = __float_as_int(f);
    return b ^ ((b >> 31) & 0x7fffffff);
}
__device__ __forceinline__ long long topk_key(float score, int32_t node)
{
    return (long long)(((unsigned long long)(uint32_t)float_to_sortable(score) << 32) | (unsigned long long)(uint32_t)(~node));
}
__device__ __forceinline__ float key_score(long long key)
{
    int32_t s = (int32_t)(key >> 32);
    return __int_as_float(s ^ ((s >> 31) & 0x7fffffff));
}
__device__ __forceinline__ int32_t key_node(long long key) { return (int32_t)~(uint32_t)((unsigned long long)key & 0xffffffffull); }

constexpr long long KEY_MIN = (long long)0x8000000000000000ull;

// lanes of the calling thread's WIDTH-wide group (groups never straddle a warp; blocks are 1-D, multiple of 32).
// Sub-warp groups of one warp may sit in different loop iterations, so shuffles name only their own group.
template <int WIDTH>
__device__ __forceinline__ unsigned group_mask()
{
    if (WIDTH == 32) return FULL;
    return ((1u << WIDTH) - 1u) << ((threadIdx.x & 31u) & ~(unsigned)(WIDTH - 1));
}
template <int WIDTH>
__device__ __forceinline__ float group_sum(float v)
{
    const unsigned m = group_mask<WIDTH>();
#pragma unroll
    for (int o = WIDTH / 2; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(m, v, o, WIDTH));
    return v;
}
template <int WIDTH>
__device__ __forceinline__ int group_sum_int(int v)
{
    const unsigned m = group_mask<WIDTH>();
#pragma unroll
    for (int o = WIDTH / 2; o > 0; o >>= 1) v += __shfl_xor_sync(m, v, o, WIDTH);
    return v;
}

// 128-bit streaming load that bypasses L1 allocation (rows are touched once per query)
__device__ __forceinline__ float4 ldg_stream(const float4 *p)
{
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint2 ldg_stream_u2(const uint2 *p)
{
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ uint4 ldg_stream_u4(const uint4 *p)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// bulk DRAM -> L2 prefetch of `bytes` (multiple of 16) at a 16-byte aligned address: cp.async.bulk.prefetch.L2, SASS UBLKPF. The
// bytes are in flight without occupying a register or a byte of shared memory; the demand loads that follow hit L2.
__device__ __forceinline__ void bulk_prefetch_l2(const void *p, unsigned bytes)
{
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

// ---- TMA-style bulk async copy global -> shared with an mbarrier (cp.async.bulk; SASS UBLKCP) ----
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, unsigned bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, unsigned phase)
{
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(phase)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned phase)
{
    while (!mbar_try_wait(bar, phase)) {
    }
}
// generic-proxy shared-memory stores -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- warpgroup MMA (wgmma) plumbing shared by every wgmma kernel; the instruction-shape wrappers stay with their callers ----
// shared-memory matrix descriptor, K-major, SWIZZLE_128B: rows 128 B apart inside an 8-row atom, atoms SBO = 1024 B apart
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3ffff) >> 4);  // start address, bits [0,14)
    d |= (uint64_t)1 << 16;                       // leading byte offset (unused by swizzled K-major layouts), bits [16,30)
    d |= (uint64_t)(1024 >> 4) << 32;             // stride byte offset, bits [32,46)
    d |= (uint64_t)1 << 62;                       // layout type SWIZZLE_128B, bits [62,64)
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R>
__device__ __forceinline__ void acc_fence(uint32_t (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+r"(d[i])::"memory");
}

// block-wide bitonic sort of keys[0..n_pow2) (shared memory, n_pow2 a power of two), descending; ends on a barrier
__device__ __forceinline__ void bitonic_sort_desc(long long *keys, int n_pow2)
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

// smallest power of two >= v (1 for v <= 1)
__host__ __device__ __forceinline__ int next_pow2(int v)
{
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}

// The library's counter-based generator: a pure function of (seed, a, b, c), so a draw does not depend on thread order.
// Callers: the removal's random fallback (seed, level, node, attempt), PQ training (pq_train.cu) and the compaction's retraining
// sample (seed, TAG_COMPACT_SAMPLE, source, chunk).
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x)
{
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
__host__ __device__ __forceinline__ uint64_t counter_random(uint64_t seed, int a, int b, int c)
{
    return mix64(mix64(mix64(seed ^ (uint64_t)(uint32_t)a) ^ (uint64_t)(uint32_t)b) ^ (uint64_t)(uint32_t)c);
}
// first counter of the compaction's chunk shuffle (PQRetrainer.sampleBalanced): no PQ-training draw uses it (those take a
// sub-space < 2^29, sub-space | 0x20000000 or | 0x40000000, or 0x7fffffff) and the removal's fallback takes a level
constexpr int TAG_COMPACT_SAMPLE = 0x7ffffffe;

// -ln(u) for u in (0, 1] as a fixed sequence of round-to-nearest fp32 operations (no log intrinsic, no FMA), so a host model
// repeats it bit for bit: u = m 2^e with m in [sqrt(1/2), sqrt(2)], ln m = 2 s (1 + z/3 + z^2/5 + z^3/7 + z^4/9) with
// s = (m - 1) / (m + 1), z = s^2 (|s| <= 0.172: the truncated series is below 1e-9 relative). ln(1) gives +0.
__device__ __forceinline__ float neg_ln_unit(float u)
{
    const int bits = __float_as_int(u);
    int e = ((bits >> 23) & 0xff) - 127;
    float m = __int_as_float((bits & 0x7fffff) | 0x3f800000);
    if (m > __int_as_float(0x3fb504f3)) {  // fp32 sqrt(2)
        m = __fmul_rn(m, 0.5f);
        e += 1;
    }
    const float s = __fdiv_rn(__fsub_rn(m, 1.0f), __fadd_rn(m, 1.0f));
    const float z = __fmul_rn(s, s);
    float p = __int_as_float(0x3de38e39);                              // 1/9
    p = __fadd_rn(__fmul_rn(p, z), __int_as_float(0x3e124925));        // 1/7
    p = __fadd_rn(__fmul_rn(p, z), __int_as_float(0x3e4ccccd));        // 1/5
    p = __fadd_rn(__fmul_rn(p, z), __int_as_float(0x3eaaaaab));        // 1/3
    p = __fadd_rn(__fmul_rn(p, z), 1.0f);
    const float ln_m = __fmul_rn(__fmul_rn(2.0f, s), p);
    const float ln_u = __fadd_rn(__fmul_rn((float)e, __int_as_float(0x3f317218)), ln_m);  // fp32 ln(2)
    return __fsub_rn(0.0f, ln_u);
}

}  // namespace jv
