// bq_umma.cu — the FILTER pass of the BQ Hamming top-k (see bq_imma.cu for the whole pipeline) on Hopper's warpgroup tensor-core
// instructions: wgmma.mma_async kind u8 x u8 -> s32 (exact), operands in shared memory in the canonical K-major SWIZZLE_128B
// layout, accumulators in the registers of the two consumer warpgroups, producer and consumers connected by mbarriers.
//
//   D[128 rows][256 queries] += A[128][K] * B[256][K]^T,  A bytes in {0, 2^s}, B bytes in {0, 2^(7-s)} expanded from bit words
//   (D = 128 * popcount(row & query), exact in s32), K = dim rounded to 128
//
// Why a second kernel next to the IMMA one: the mma.sync path re-expands both operands in every warp tile; here the row tile is
// expanded ONCE per CTA tile into shared memory by the producer warpgroup, and the query tile arrives as a pre-expanded,
// pre-swizzled 32 KB image by one bulk copy.
//
// Roles (384 threads): warpgroup 0 = producers (one thread per row: 128 bits -> 128 bytes per stage, swizzled 16-byte stores,
// fence.proxy.async, arrive; thread 0 also issues the cp.async.bulk of the query image chunk), warpgroups 1 and 2 = consumers,
// each owning 64 rows of the tile: 4 x wgmma m64n256k32 per stage into 128 s32 registers per thread, then the epilogue on those
// registers. Pipeline: full[s] / empty[s] over 4 operand stages of 48 KB; a consumer keeps one wgmma group in flight and hands a
// stage back when the group that read it has completed. Epilogue: thresholds of the query tile sit in shared memory; a column
// costs IADD + ISETP; the rare survivors (about 0.3 %) append their keys with one atomic each. Row popcounts come from the
// producers. Every spin-wait is bounded and traps: a wrong barrier count aborts the launch instead of hanging the device.
#include <limits.h>

#include "kernels.h"

namespace jv {

namespace {

constexpr int UM = 128;           // rows per tile (two consumer warpgroups x wgmma M = 64)
constexpr int UN = 256;           // queries per tile (wgmma N)
constexpr int UKC = 128;          // K bytes per stage (one 128-byte swizzle atom wide)
constexpr int USTAGES = 4;
constexpr int UTHREADS = 384;
constexpr int A_STAGE_BYTES = UM * UKC;  // 16 KB
constexpr int B_STAGE_BYTES = UN * UKC;  // 32 KB
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int NPAR = 8;  // ring of row-popcount buffers: the producers run at most USTAGES stages (= tiles when K is one chunk) ahead

__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait_bounded(uint64_t *bar, unsigned phase)
{
    for (unsigned spins = 0; !mbar_try_wait(bar, phase); ++spins)
        if (spins > (1u << 28)) __trap();  // a pipeline bug must abort the launch, not hang the device
}

// D[64][256] (+)= A[64][32] * B[256][32]^T, u8 x u8 -> s32. Accumulator fragment: register 4 j + 2 h + e holds row
// 16 (warp % 4) + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e.
__device__ __forceinline__ void wgmma_u8_m64n256k32(uint32_t (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k32.s32.u8.u8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p;\n\t"
        "}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]), "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]), "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]), "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]), "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// the query tile as shared-memory images: [qtile][kchunk][UN rows x 128 B], swizzled exactly as the MMA reads it
__global__ void __launch_bounds__(256) bq_query_image_kernel(const uint32_t *__restrict__ qbits, int nq_pad, int W32, int kchunks, uint8_t *__restrict__ images)
{
    // one thread per (query, 16-byte chunk): 16 bits -> 16 bytes
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)nq_pad * kchunks * 8;
    if (idx >= total) return;
    const int j = (int)(idx & 7);
    const long long t = idx >> 3;
    const int kc = (int)(t % kchunks), q = (int)(t / kchunks);
    const uint32_t w = qbits[(size_t)q * W32 + kc * 4 + (j >> 1)];
    // K order inside a 32-bit word: output word s holds bits s, s + 8, s + 16, s + 24 (one per byte). The row side stores such a
    // bit as the byte value 2^s (a single AND with a shifted mask), the query side as 2^(7 - s): every matching bit pair
    // contributes exactly 128 to the s32 accumulator, so D = 128 * popcount(row & query).
    const int sb = (j & 1) * 4;
    uint4 v;
    v.x = ((w >> (sb + 0)) & 0x01010101u) << (7 - (sb + 0));
    v.y = ((w >> (sb + 1)) & 0x01010101u) << (7 - (sb + 1));
    v.z = ((w >> (sb + 2)) & 0x01010101u) << (7 - (sb + 2));
    v.w = ((w >> (sb + 3)) & 0x01010101u) << (7 - (sb + 3));
    const int qt = q / UN, r = q % UN;
    uint8_t *img = images + ((size_t)qt * kchunks + kc) * B_STAGE_BYTES;
    *reinterpret_cast<uint4 *>(img + (r >> 3) * 1024 + (r & 7) * 128 + ((j ^ (r & 7)) << 4)) = v;
}

struct UmmaParams {
    const uint32_t *rows;  // [n][W32]
    long long n;
    int W32, dim, kchunks;
    const uint8_t *images;  // [qtiles][kchunks][32 KB]
    int qtiles, nq;
    const int *t2, *pb;
    long long *buf;
    int *cnt;
    int cap;
    long long id_base;
};

__global__ void __launch_bounds__(UTHREADS, 1) bq_wgmma_filter_kernel(UmmaParams P)
{
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *stage0 = smem;  // USTAGES x (A 16 KB | B 32 KB), 1024-byte aligned
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + USTAGES * STAGE_BYTES);
    uint64_t *empty = full + USTAGES;
    int *s_t2 = reinterpret_cast<int *>(smem + USTAGES * STAGE_BYTES + 256);  // [UN] thresholds of the current query tile
    int *s_par = s_t2 + UN;                                                     // [NPAR tiles][UM] row popcounts from the producers

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long row_tiles = (P.n + UM - 1) / UM;
    const long long tiles = row_tiles * P.qtiles;

    if (tid == 0) {
        for (int s = 0; s < USTAGES; s++) {
            mbar_init(&full[s], UM + 1);  // 128 row producers + the bulk copy's arrive.expect_tx
            mbar_init(&empty[s], 8);      // one arrive per consumer warp
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===== producers: thread r expands row r of the tile; thread 0 also brings in the query image chunk =====
        const int r = tid;
        int stage = 0, tbuf = 0;
        unsigned phase = 0;
        for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
            const int qt = (int)(tile / row_tiles);
            const long long rr = (tile % row_tiles) * UM + r;
            const bool live = rr < P.n;
            const uint4 *rp = reinterpret_cast<const uint4 *>(P.rows + (size_t)(live ? rr : 0) * P.W32);
            uint4 w = make_uint4(0u, 0u, 0u, 0u);
            if (live) w = __ldg(rp);
            int pc = 0;
            for (int kc = 0; kc < P.kchunks; kc++) {
                uint4 wn = make_uint4(0u, 0u, 0u, 0u);
                if (live && kc + 1 < P.kchunks) wn = __ldg(rp + kc + 1);  // the next chunk's words are in flight during this one
                mbar_wait_bounded(&empty[stage], phase ^ 1);
                if (r == 0) {
                    mbar_expect_tx(&full[stage], B_STAGE_BYTES);
                    bulk_g2s(stage0 + stage * STAGE_BYTES + A_STAGE_BYTES, P.images + ((size_t)qt * P.kchunks + kc) * B_STAGE_BYTES, B_STAGE_BYTES, &full[stage]);
                }
                unsigned char *dst = stage0 + stage * STAGE_BYTES + (r >> 3) * 1024 + (r & 7) * 128;
                const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const int sb = (j & 1) * 4;
                    const uint32_t word = ws[j >> 1];
                    uint4 v;  // bit (8 b + s) of the word -> byte b of output word s, value 2^s: one AND per output word
                    v.x = word & (0x01010101u << (sb + 0));
                    v.y = word & (0x01010101u << (sb + 1));
                    v.z = word & (0x01010101u << (sb + 2));
                    v.w = word & (0x01010101u << (sb + 3));
                    *reinterpret_cast<uint4 *>(dst + ((j ^ (r & 7)) << 4)) = v;
                }
                pc += __popc(w.x) + __popc(w.y) + __popc(w.z) + __popc(w.w);
                if (kc + 1 == P.kchunks) s_par[tbuf * UM + r] = pc;  // this row's popcount, for the epilogue
                fence_proxy_async();  // generic-proxy stores -> visible to the tensor core's async-proxy reads
                mbar_arrive(&full[stage]);
                if (++stage == USTAGES) { stage = 0; phase ^= 1; }
                w = wn;
            }
            tbuf = (tbuf + 1) & (NPAR - 1);
        }
    } else {
        // ===== consumers: warpgroup cw owns rows [64 cw, 64 cw + 64) of every tile =====
        const int cw = (warp >> 2) - 1, ctid = tid - 128;
        const int rbase = 64 * cw + 16 * (warp & 3) + (lane >> 2);  // fragment rows rbase and rbase + 8
        const int cbase = 2 * (lane & 3);                           // fragment columns 8 j + cbase (+ 1)
        uint32_t d[128];
#pragma unroll
        for (int i = 0; i < 128; i++) d[i] = 0u;
        int stage = 0, cur_qt = -1, it = 0;
        unsigned phase = 0;
        for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x, it++) {
            const int qt = (int)(tile / row_tiles), tbuf = it & (NPAR - 1);
            const long long row0 = (tile % row_tiles) * UM;
            if (qt != cur_qt) {  // the thresholds of this query tile (padding queries never pass)
                asm volatile("bar.sync 1, 256;" ::: "memory");
                for (int c = ctid; c < UN; c += 256) {
                    const int q = qt * UN + c;
                    s_t2[c] = q < P.nq ? 128 * __ldg(P.t2 + q) : INT_MIN;  // the accumulators hold 128 * dot
                }
                cur_qt = qt;
                asm volatile("bar.sync 1, 256;" ::: "memory");
            }
            int prev = -1;
            for (int kc = 0; kc < P.kchunks; kc++) {
                mbar_wait_bounded(&full[stage], phase);
                const uint32_t a_addr = smem_u32(stage0 + stage * STAGE_BYTES) + cw * (64 / 8) * 1024, b_addr = smem_u32(stage0 + stage * STAGE_BYTES) + A_STAGE_BYTES;
                acc_fence(d);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < UKC / 32; k++) wgmma_u8_m64n256k32(d, wgmma_desc(a_addr + 32 * k), wgmma_desc(b_addr + 32 * k), (kc | k) != 0 ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<1>();  // the group of the previous stage has read its operands
                if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
                prev = stage;
                if (++stage == USTAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            acc_fence(d);
            // the row popcounts were written before the producers' arrive on the last stage (ordered through full[] -> here);
            // read them before that stage goes back to the producers
            int par[2], par128[2];
            long long rr[2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
                rr[h] = row0 + rbase + 8 * h;
                par[h] = s_par[tbuf * UM + rbase + 8 * h];
                par128[h] = rr[h] < P.n ? par[h] << 7 : INT_MAX;  // rows past the end never pass
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[prev]);
            // hd - pb = par - 2 dot <= t2  <=>  2 (128 dot) + 128 t2 >= 128 par
#pragma unroll
            for (int j = 0; j < UN / 8; j++) {
                const int2 t = *reinterpret_cast<const int2 *>(s_t2 + 8 * j + cbase);
#pragma unroll
                for (int h = 0; h < 2; h++) {
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const int v = (int)d[4 * j + 2 * h + e];
                        if (2 * v + (e ? t.y : t.x) >= par128[h]) {
                            const int q = qt * UN + 8 * j + cbase + e;
                            const int hd = par[h] - (v >> 6) + __ldg(P.pb + q);
                            const long long key = topk_key(bq_score_from_hd(hd, P.dim), (int32_t)(rr[h] + P.id_base));
                            const int pos = atomicAdd(&P.cnt[q], 1);
                            if (pos < P.cap) P.buf[(size_t)q * P.cap + pos] = key;
                        }
                    }
                }
            }
        }
    }
}

}  // namespace

size_t bq_umma_image_bytes(int nq, int W)
{
    const int qtiles = (nq + UN - 1) / UN, kchunks = (2 * W) / 4;
    return (size_t)qtiles * kchunks * B_STAGE_BYTES + 1024;
}

bool bq_umma_supported(const DataDesc &d)
{
    return d.kind == KIND_BQ && (d.W % 2) == 0 && d.W <= 32;
}

// the filter pass over queries [0, nq) (identity list): pairs with hd <= thr[q] append their keys to buf / cnt
cudaError_t launch_bq_umma_filter(const DataDesc &d, const uint32_t *qbits_dev, int nq, int nq_pad, const int *t2_dev, const int *pb_dev, long long *buf_dev,
                                  int *cnt_dev, int cap, long long id_base, uint8_t *images_dev, int sm_count, cudaStream_t s)
{
    const int W32 = 2 * d.W, kchunks = W32 / 4, qtiles = (nq + UN - 1) / UN;
    cudaError_t e;
    // padding queries of the last tile need defined (zero) bits: qbits rows [nq, nq_pad) are zero; rows past nq_pad are not read
    const int q_img = qtiles * UN;
    if (q_img > nq_pad) return cudaErrorInvalidValue;  // callers pad nq_pad to a multiple of 256
    {
        const long long total = (long long)q_img * kchunks * 8;
        bq_query_image_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(qbits_dev, q_img, W32, kchunks, images_dev);
        g_launches++;
    }
    UmmaParams P;
    P.rows = reinterpret_cast<const uint32_t *>(d.words);
    P.n = d.n; P.W32 = W32; P.dim = d.dim; P.kchunks = kchunks; P.images = images_dev; P.qtiles = qtiles; P.nq = nq; P.t2 = t2_dev; P.pb = pb_dev;
    P.buf = buf_dev; P.cnt = cnt_dev; P.cap = cap; P.id_base = id_base;
    const size_t smem = (size_t)USTAGES * STAGE_BYTES + 256 + UN * sizeof(int) + NPAR * UM * sizeof(int);
    if ((e = cudaFuncSetAttribute(bq_wgmma_filter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
    const long long tiles = ((d.n + UM - 1) / UM) * qtiles;
    const int grid = (int)(tiles < sm_count ? tiles : sm_count);
    bq_wgmma_filter_kernel<<<grid, UTHREADS, smem, s>>>(P);
    g_launches++;
    return cudaGetLastError();
}

}  // namespace jv
