// search.cu — GraphSearcher.search, device resident: one CTA walks one query through the whole traversal
// (base:graph/GraphSearcher.java:263-282 internalSearch, :334-353 initializeInternal, :355-370 stopSearch,
//  :406-457 searchOneLayer, :471-507 reranking; neighbour loop base:graph/OnHeapGraphIndex.java:475-483).
//
// State per query, all in shared memory (the kernel's own header comment, further down, has the exactness argument):
//   * ONE list sorted by the reference's 64-bit key holding the nodes SEEN so far that can still matter, each with an
//     "expanded" and an "accepted" flag; its unexpanded entries are the reference's candidate max-heap in pop order;
//   * a shadow copy of the reference's bounded result heap (same array, same sift procedures): stopSearch's strict <, the
//     "tie with the worst result is expanded but not added" rule and NodeQueue.rerank's array order come from it;
//   * upper levels run with a 1-entry result heap over the same list; moving down a level clears the expanded flags
//     (setEntryPointsFromPreviousLayer);
//   * visited = an exact set of node ids, never cleared between levels (GraphSearcher keeps `visited` across levels):
//     16-bit region-tagged slots in shared memory (visited_insert_smem), or — for graphs / beams the shared-memory table
//     does not take, and for the re-run of a query that outgrew it — an open-addressing table of 32-bit ids in a per-CTA slice
//     of global scratch (visited_insert).
// Every hop is: read one adjacency row (FusedPQ: one record) -> filter through visited, requesting every new row from DRAM
// with one bulk L2 prefetch (not for fp32 batches that fill the GPU, see launch_search) -> score the survivors with the row
// scorers of scorers.cuh -> parallel rank-merge into the list.
#include <limits.h>
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>

#include "kernels.h"

namespace jv {

struct SearchParams {
    GraphDesc g;
    DataDesc approx;
    DataDesc rerank;
    int has_rerank;
    int metric;
    const float *queries;
    int query_stride;
    int nq, topK, rerankK;
    int list_cap;    // entries the candidate list retains (>= rerankK; the slack holds the tie tail)
    int list_alloc;  // entries per list buffer (>= list_cap and >= sort_pow2)
    int sort_pow2;   // next power of two >= rerankK (bitonic sort of the result heap)
    int visited_cap;
    int visited_shift;
    int32_t *visited_tables;
    int *work_counter;
    int32_t *nodes_out;
    float *scores_out;
    SearchCounters *counters;
    uint8_t *overflow;
    const int32_t *query_index;
    int blobA_floats, blobR_floats, smemA_floats;  // smemA_floats: what the walking scorer's prepared query takes of shared memory
    float *blob_global;  // PQ: per-CTA slices of global scratch (L2 resident) hold the LUT rows of the sub-spaces >= pq_smem_m
    int pq_smem_m;       // PQ: sub-spaces [0, pq_smem_m) keep their LUT rows in shared memory (multiple of 4; M = all, 0 = none)
    // acceptOrds / threshold / rerankFloor of GraphSearcher.search(sp, topK, rerankK, threshold, rerankFloor, acceptOrds)
    const uint32_t *accept_bits;  // bit (node & 31) of word (node >> 5); nullptr = Bits.ALL
    long long accept_stride;      // words between two queries' bitsets (0 = one bitset shared by the batch)
    float threshold, rerank_floor;
    int filtered;                 // accept_bits != nullptr || threshold > 0 || exclude_ids != nullptr
    const int *arrived;           // nullptr, or: query i may be read only once *arrived > i (the H2D copy is still running)
    int lenient;                  // insert searches of the builder: a full visited table ends the walk with what it has, a tie tail
                                  // that does not fit is dropped — counted in counters->overflowed, never an error (build.cu)
    // visited set in shared memory (plan_search decides): 2^vis_slots_log 16-bit slots split into 2^(vis_bits-15) regions; 0 = the
    // per-CTA global table
    int vis_slots_log, vis_rlog;
    unsigned vis_idmask;
    int early_pf;      // request the adjacency / FusedPQ record of a new candidate that lands among the next two pops at score time
    int pq_rows;       // PQ walk: lane = candidate, warp = partial sum (score_pq_partial) instead of an 8-lane group per candidate
    int row_prefetch;  // fp32 / NVQ walks: 1 = a bulk L2 prefetch of every newly visited row is issued by the thread that discovered it
                       // (fp32: only for a batch that does not fill the GPU)
    unsigned long long *dbg;  // JV_SEARCH_PROFILE builds only: per-phase cycle totals
    const int32_t *exclude_ids;  // [nq]: query qi never accepts node exclude_ids[qi] (SearchFilter::exclude_ids, the EXCL instantiations)
    // SEG instantiations: the walked segments' descriptors; nq counts (segment, query) items, seg_nq the queries per segment
    const SegmentDesc *segs;
    int seg_nq;
};

__device__ __forceinline__ bool visited_insert(int32_t *t, unsigned mask, int shift, int32_t v)
{
    unsigned h = ((unsigned)v * 2654435761u) >> shift;
    for (unsigned probes = 0; probes <= mask; ++probes) {
        const int old = atomicCAS(&t[h], -1, v);
        if (old == -1) return true;
        if (old == v) return false;
        h = (h + 1) & mask;
    }
    return false;
}

// The same set in shared memory, 16 bits per slot. x = id * odd mod 2^bits is a bijection on [0, 2^bits) (bits = ceil(log2 n) >= 15);
// its top (bits - 15) bits choose a REGION of the table, its low 15 bits are the tag stored there (bit 15 = occupied), and a probe
// sequence never leaves its region — so (region, tag) identifies the id exactly and the set has no false positives. A full region
// reports through *fail (the query is re-run on the global table, like any visited-table overflow).
__device__ __forceinline__ bool visited_insert_smem(unsigned short *t, unsigned idmask, int rlog, int32_t v, int *fail)
{
    const unsigned x = ((unsigned)v * 0x9E3779B1u) & idmask;
    const unsigned tag = x & 0x7fffu;
    const unsigned short val = (unsigned short)(tag | 0x8000u);
    const unsigned rmask = (1u << rlog) - 1u;
    unsigned short *base = t + ((size_t)(x >> 15) << rlog);
    unsigned h = (tag * 0x9E3779B1u) >> (32 - rlog);
    for (unsigned probes = 0; probes <= rmask; ++probes) {
#ifdef JV_VIS_CAS_GENERIC
        const unsigned short old = atomicCAS(&base[h], (unsigned short)0, val);
#else
        // explicit .shared state space: a 16-bit CAS is an LDS + 32-bit ATOMS.CAS loop on the containing word; through a generic
        // pointer (atomicCAS on unsigned short *) the compiler emits the slower generic ATOM.E.CAS
        unsigned short old;
        asm volatile("atom.shared.cas.b16 %0, [%1], %2, %3;" : "=h"(old) : "r"(smem_u32(base + h)), "h"((unsigned short)0), "h"(val) : "memory");
#endif
        if (old == 0) return true;
        if (old == val) return false;
        h = (h + 1) & rmask;
    }
    *fail = 1;
    return false;
}

// number of keys in the descending-sorted array a[0..n) that are greater than k
__device__ __forceinline__ int count_greater_desc(const long long *a, int n, long long k)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] > k) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// The reference's result queue is a BoundedLongHeap (min-heap of keys, 1-based array): its ARRAY ORDER decides which of two
// equal exact scores survives NodeQueue.rerank, so the device keeps the same array with the same sift procedures
// (base:util/AbstractLongHeap.java:158-187 upHeap / downHeap, base:util/BoundedLongHeap.java:60-70,100-104 push / updateTop).
__device__ __forceinline__ void heap_up(long long *h, int pos)
{
    int i = pos;
    const long long v = h[i];
    int j = i >> 1;
    while (j > 0 && v < h[j]) {
        h[i] = h[j];
        i = j;
        j >>= 1;
    }
    h[i] = v;
}
__device__ __forceinline__ void heap_down(long long *h, int size, int pos)
{
    int i = pos;
    const long long v = h[i];
    int j = i << 1, k = j + 1;
    if (k <= size && h[k] < h[j]) j = k;
    while (j <= size && h[j] < v) {
        h[i] = h[j];
        i = j;
        j = i << 1;
        k = j + 1;
        if (k <= size && h[k] < h[j]) j = k;
    }
    h[i] = v;
}

#ifndef JV_SEARCH_THREADS
#define JV_SEARCH_THREADS 256
#endif
#ifndef JV_SEARCH_MINB
#define JV_SEARCH_MINB 5
#endif
#ifndef JV_SEARCH_MINB_PQ
#define JV_SEARCH_MINB_PQ 6
#endif
// CTA width per walking scorer. fp32 / NVQ rows are scored a warp per row and, with every new row already on its way to L2
// (bulk prefetch), the walk gains from MORE queries in flight rather than more warps per query: 128 threads, 10 CTAs per SM
// (c2: 14.7 -> 14.2 ms). PQ / BQ score a hop's ~28 candidates in one pass over 8 warps (PQ: one warp per partial sum): 256 threads.
#ifndef JV_SEARCH_THREADS_ROWS
#define JV_SEARCH_THREADS_ROWS 128
#endif
template <int KIND>
struct SearchThreads {
    static constexpr int value = (KIND == KIND_F32 || KIND == KIND_NVQ) ? JV_SEARCH_THREADS_ROWS : JV_SEARCH_THREADS;
};
static int search_threads_of(int kind) { return (kind == KIND_F32 || kind == KIND_NVQ) ? JV_SEARCH_THREADS_ROWS : JV_SEARCH_THREADS; }

// optional phase timers (tools/: build with JV_NVCC_EXTRA=-DJV_SEARCH_PROFILE); compiled out of the product build
#ifdef JV_SEARCH_PROFILE
#define JV_T(var) const long long var = clock64()
#define JV_ACC(slot, a, b) do { if (threadIdx.x == 0) dbg_local[slot] += (unsigned long long)((b) - (a)); } while (0)
#else
#define JV_T(var)
#define JV_ACC(slot, a, b)
#endif

// optional drop statistics of the fp32 DOT walk (tools/row_bound_stats.py: build with -DJV_ROW_BOUND_STATS); compiled out of the
// product build. [0] level-0 rows scored, [1] of them dropped by JV_EMIT against a full list; plus a 1-in-64 sample of the drops
// as {query, row, key of the list's last entry}, and a 1-in-64 sample of every row scored against a full list (the rows a sketched
// walk bounds on their edge record, then routes or bounds on their sketch) as {query, row, last key, the row's exact key}
#ifdef JV_ROW_BOUND_STATS
constexpr int RBS_CAP = 1 << 20;
struct RbsSample { int32_t q, row; long long last_key; };
struct RbsRow { int32_t q, row; long long last_key, key; };
__device__ unsigned long long g_rbs_count[4];  // scored, dropped, drop samples taken, row samples taken
__device__ RbsSample g_rbs_sample[RBS_CAP];
__device__ RbsRow g_rbs_row[RBS_CAP];
#define JV_RBS_ROW(k_, f_)                                                                                                    \
    do {                                                                                                                      \
        if (KIND == KIND_F32 && METRIC == JV_METRIC_DOT && lvl == 0 && size == LC &&                                          \
            (((unsigned)(f_) * 2246822519u) ^ ((unsigned)qi * 3266489917u)) % 64u == 0u) {                                    \
            const unsigned long long k_r = atomicAdd(&g_rbs_count[3], 1ull);                                                  \
            if (k_r < RBS_CAP) g_rbs_row[k_r] = RbsRow{qi, (f_), cur[LC - 1], (k_)};                                          \
        }                                                                                                                     \
    } while (0)
#define JV_RBS_SCORED(n_) do { if (KIND == KIND_F32 && METRIC == JV_METRIC_DOT && lvl == 0) atomicAdd(&g_rbs_count[0], (unsigned long long)(n_)); } while (0)
#define JV_RBS_DROP(f_)                                                                                                       \
    do {                                                                                                                      \
        if (KIND == KIND_F32 && METRIC == JV_METRIC_DOT && lvl == 0) {                                                        \
            atomicAdd(&g_rbs_count[1], 1ull);                                                                                 \
            if ((((unsigned)(f_) * 2654435761u) ^ ((unsigned)qi * 40503u)) % 64u == 0u) {                                     \
                const unsigned long long k_ = atomicAdd(&g_rbs_count[2], 1ull);                                               \
                if (k_ < RBS_CAP) g_rbs_sample[k_] = RbsSample{qi, (f_), cur[LC - 1]};                                        \
            }                                                                                                                 \
        }                                                                                                                     \
    } while (0)
#else
#define JV_RBS_SCORED(n_)
#define JV_RBS_DROP(f_)
#define JV_RBS_ROW(k_, f_)
#endif

// Edge tier (DESIGN §4.1): a new neighbour that its edge bound does not settle is routed direct to its full row, skipping its sketch,
// when the bound's point estimate scores more than this above the list's last entry. Only bytes depend on it, never results: a wrong
// route reads 3 072 - 784 B more at d = 768, a missed one 784 B more, so it leans towards the sketch (tools/row_bound_stats.py).
constexpr float EDGE_DIRECT_MARGIN = 0.002f;

// flags of a list entry
constexpr uint8_t F_EXPANDED = 1;  // popped from the candidate queue at this level
constexpr uint8_t F_ACCEPTED = 2;  // acceptOrds.get(node) && score >= threshold (what addTopCandidate requires at level 0)

// State per query (see the file header). The traversal is EXACTLY the reference's, ties included:
//   candidates  = the unexpanded entries of ONE list sorted by the reference key (pop order = the max-heap's pop order);
//   results     = `heap`, the reference's BoundedLongHeap of the best rerankK (1 on upper levels) popped nodes, same array order;
//   stopSearch  = results full && score(best candidate) < score(worst result)  (GraphSearcher.java:355-361, strict);
//   addTopCandidate = push while not full, replace the worst when strictly better, otherwise (tie with the worst) expand the
//                 node without adding it (GraphSearcher.java:520-530);
//   a list entry may be dropped when at least rerankK accepted entries score STRICTLY higher (it can never be popped before
//   stopSearch fires); the list keeps `list_cap` >= rerankK entries so a tie tail survives, and a query whose tail does not fit
//   is re-run by the host with a larger list (overflow code 2), never answered approximately;
//   upper levels: a node refused by addTopCandidate is neither a result nor evicted, so it is removed from the list at once
//   (setEntryPointsFromPreviousLayer re-queues results + evicted only, GraphSearcher.java:316-323).
// MINB: resident CTAs per SM the register allocation is capped for. PQ is compiled twice: 6 (40 registers; the L2-LUT mode, where
// nothing else limits residency) and 4 (64 registers; the modes whose shared-memory LUT part allows at most 4-5 CTAs anyway).
// VSM: the visited set lives in shared memory (a template parameter, not a run-time flag: the two forms must not cost each other
// registers — the fp32 walk lost 15 % when they shared one instantiation).
// EDGE: the fp32 DOT walk over a graph with edge records (P.g.edge_rec, launch_search), a separate instantiation for the same reason
// EXCL: the walks of a refine, which never accept their query's own node (P.exclude_ids); separate so that the other walks compile
// exactly as they do without it
// SEG: the walks of a multi-segment search (jv_segments_search_batch): work item w (or P.query_index[w]) is the pair
// (segment s, query q) = (w / P.seg_nq, w % P.seg_nq), and each item reads its segment's graph, data sets, bitset, counters and
// output rows from P.segs[s] instead of P; separate for the same reason as EXCL
template <int KIND, int METRIC, int MINB, bool VSM, bool EDGE = false, bool EXCL = false, bool SEG = false>
__global__ void __launch_bounds__(SearchThreads<KIND>::value, MINB) graph_search_kernel(SearchParams P)
{
    constexpr int SEARCH_THREADS = SearchThreads<KIND>::value;
    constexpr int HEAP_TID = SEARCH_THREADS - 32;  // the thread that maintains the result heap (lane 0 of the last warp)
    constexpr int G = GroupOf<KIND>::value;
    constexpr int NG = SEARCH_THREADS / G;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // prepared query of the walking scorer. PQ: the LUT may be split, rows of sub-spaces < pq_smem_m in shared memory (blobA), the
    // others in this CTA's global slice (blobH); every other kind: all of it in shared memory
    float *blobA = reinterpret_cast<float *>(smem_raw);
    float *blobH = P.blob_global ? P.blob_global + (size_t)blockIdx.x * P.blobA_floats : blobA;
    const int splitm = (KIND == KIND_PQ && P.blob_global) ? P.pq_smem_m : (1 << 30);
    float *blobR = reinterpret_cast<float *>(smem_raw) + P.smemA_floats;
    long long *keys0 = reinterpret_cast<long long *>(blobR + P.blobR_floats);
    long long *keys1 = keys0 + P.list_alloc;
    long long *cand_keys = keys1 + P.list_alloc;
    long long *heap = cand_keys + MAX_DEGREE;  // 1-based, rerankK entries
    int32_t *cand_ids = reinterpret_cast<int32_t *>(heap + ((P.rerankK + 2) & ~1));
    uint8_t *cand_acc = reinterpret_cast<uint8_t *>(cand_ids + MAX_DEGREE);
    uint8_t *cand_slot = cand_acc + MAX_DEGREE;  // fused PQ: position of the candidate inside the expanded node's record
    uint8_t *flags0 = cand_slot + MAX_DEGREE;
    uint8_t *flags1 = flags0 + P.list_alloc;
    unsigned short *vis = reinterpret_cast<unsigned short *>((reinterpret_cast<uintptr_t>(flags1 + P.list_alloc) + 15) & ~(uintptr_t)15);
    constexpr bool vsm = VSM;  // visited set in shared memory (16-bit slots) instead of the per-CTA global table
    uint32_t *pq_stage = reinterpret_cast<uint32_t *>(vis + (VSM ? (1 << P.vis_slots_log) : 0));  // PQ row mode: the hop's code rows
    float *pq_part = reinterpret_cast<float *>(pq_stage + P.g.degree * ((P.approx.code_stride >> 2) + 1));  // and its partial sums
    __shared__ int s_vfail;
    __shared__ long long s_nk;  // key of the second unexpanded entry behind the one being expanded (see JV_EMIT)
    __shared__ float red[36];
    __shared__ int s_q, s_n, s_m, s_hsize, s_cnt;
    __shared__ int s_settled;  // new neighbours of this hop settled on their edge record (counted as visited, never candidates)
    __shared__ unsigned long long s_settled_total;  // over this CTA's queries (thread 0 only), added to counters->settled at exit
    __shared__ int s_nd;  // new neighbours of this hop routed direct (edge tier): cand_ids[MAX_DEGREE - 1 - j], j < s_nd
    __shared__ unsigned long long s_direct_total[2];  // over this CTA's queries: routed direct, of them dropped by JV_EMIT
    __shared__ float s_lr[LR_QUERY];  // the query's low-rank terms (prepare_lowrank)
    __shared__ int s_drop[2];  // best sortable score that fell off the list, double-buffered like s_posv
    __shared__ int s_posv[2];
    // the descriptor of the work item's segment (SEG); every other walk reads P's own through the same names (macros, not
    // references: a reference to P compiles the other walks differently)
    __shared__ __align__(16) SegmentDesc s_seg;
#define PG (SEG ? s_seg.g : P.g)
#define PA (SEG ? s_seg.approx : P.approx)
#define PR (SEG ? s_seg.rerank : P.rerank)
#define PC (SEG ? P.counters + s_seg.slot : P.counters)

    const int tid = threadIdx.x;
    const int group = tid / G, lane = tid % G;
    const int L = P.rerankK, LC = P.list_cap;
    const unsigned vmask = (unsigned)P.visited_cap - 1u;
    const int vis_limit = 3 << (P.vis_slots_log > 2 ? P.vis_slots_log - 2 : 0);  // shared-memory table: at most 3/4 full
    int32_t *table = P.visited_tables + (size_t)blockIdx.x * P.visited_cap;
    int degree = P.g.degree;
    if (EDGE && tid == 0) { s_settled_total = 0; s_direct_total[0] = 0; s_direct_total[1] = 0; }

    for (;;) {
        if (tid == 0) {
            const int w = atomicAdd(P.work_counter, 1);
            if (P.arrived && w < P.nq) {
                // the batch is still being copied in (api.cu jv_graph_search_batch_ex): wait until the watermark has passed this query
                const int need = P.query_index ? P.query_index[w] : w;
                // (bounded: ~10 s of waiting for a copy that takes milliseconds means the copy stream died — trap, never hang the GPU)
                unsigned spins = 0;
                while (*reinterpret_cast<const volatile int *>(P.arrived) <= need) {
                    __nanosleep(200);
                    if (++spins > 50000000u) __trap();
                }
            }
            s_q = w;
        }
        __syncthreads();
        const int wq = s_q;
        if (wq >= P.nq) {
            if (EDGE && !SEG && tid == 0) {
                if (s_settled_total) atomicAdd(&P.counters->settled, s_settled_total);
                if (s_direct_total[0]) atomicAdd(&P.counters->direct, s_direct_total[0]);
                if (s_direct_total[1]) atomicAdd(&P.counters->direct_dropped, s_direct_total[1]);
            }
            break;
        }
        int qi = P.query_index ? P.query_index[wq] : wq;
        const float *q = P.queries + (size_t)qi * P.query_stride;
        const uint32_t *acc = P.accept_bits ? P.accept_bits + (size_t)qi * P.accept_stride : nullptr;
        if constexpr (SEG) {
            // item = (segment sg, query qq): load the segment's descriptor; qi becomes the query's output row (and overflow code)
            const int sg = qi / P.seg_nq, qq = qi - sg * P.seg_nq;
            const int *src = reinterpret_cast<const int *>(P.segs + sg);
            for (int i = tid; i < (int)(sizeof(SegmentDesc) / 4); i += SEARCH_THREADS) reinterpret_cast<int *>(&s_seg)[i] = __ldg(src + i);
            __syncthreads();
            degree = s_seg.g.degree;
            q = P.queries + (size_t)qq * P.query_stride;
            acc = s_seg.accept_bits;
            qi = s_seg.slot * P.seg_nq + qq;
        }
#ifdef JV_SEARCH_PROFILE
        unsigned long long dbg_local[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#endif
        JV_T(t_q0);
        prepare_blob<SEARCH_THREADS>(PA, P.metric, q, blobA, red, blobH, splitm);
        if (P.has_rerank) prepare_blob<SEARCH_THREADS>(PR, P.metric, q, blobR, red);
        if (EDGE) prepare_lowrank<SEARCH_THREADS>(PA.lr_basis, PA.stride, blobA, s_lr);
        if (vsm) {
            int4 *t4 = reinterpret_cast<int4 *>(vis);
            const int4 z = make_int4(0, 0, 0, 0);
            for (int i = tid; i < (1 << (P.vis_slots_log - 3)); i += SEARCH_THREADS) t4[i] = z;
            if (tid == 0) s_vfail = 0;
        } else {
            int4 *t4 = reinterpret_cast<int4 *>(table);
            const int4 m1 = make_int4(-1, -1, -1, -1);
            for (int i = tid; i < (P.visited_cap >> 2); i += SEARCH_THREADS) t4[i] = m1;
        }
        __syncthreads();
        JV_T(t_q1);
        JV_ACC(0, t_q0, t_q1);

        long long *cur = keys0, *nxt = keys1;
        uint8_t *fcur = flags0, *fnxt = flags1;
        // initializeInternal: score the entry node, mark it visited (GraphSearcher.java:346-348)
        if (group == 0) {
            const float sc = KIND == KIND_PQ ? score_pq<METRIC>(PA, blobA, PG.entry_node, lane, blobH, splitm) : score_row<KIND, METRIC>(PA, blobA, PG.entry_node, lane);
            if (lane == 0) {
                const int32_t en = PG.entry_node;
                cur[0] = topk_key(sc, en);
                fcur[0] = ((!acc || ((acc[en >> 5] >> (en & 31)) & 1u)) && sc >= P.threshold && !(EXCL && P.exclude_ids[qi] == en)) ? F_ACCEPTED : 0;
                if (vsm) visited_insert_smem(vis, P.vis_idmask, P.vis_rlog, en, &s_vfail);
                else visited_insert(table, vmask, P.visited_shift, en);
            }
        }
        int size = 1;
        int table_cnt = 1;
        unsigned visited = 0, expanded = 0, expanded_base = 0;
        int failed = 0;  // 1: visited table full, 2: candidate list too short for a tie tail
        bool truncated = false, inexact = false;  // lenient mode: the walk was cut short / a tie tail was dropped
        __syncthreads();

        for (int lvl = PG.entry_level; lvl >= 0 && !failed && !truncated; --lvl) {
            const int K = lvl > 0 ? 1 : L;
            // a new level: results + evicted are candidates again (setEntryPointsFromPreviousLayer), the result heap is empty
            for (int i = tid; i < size; i += SEARCH_THREADS) fcur[i] &= F_ACCEPTED;
            int sel = 0;
            // (the list is empty when every node an upper level expanded was refused: no entry point, nothing to walk)
            if (tid == 0) { s_posv[0] = size > 0 ? 0 : INT_MAX; s_posv[1] = INT_MAX; s_n = 0; s_m = 0; s_hsize = 0; s_drop[0] = INT_MIN; s_drop[1] = INT_MIN; s_cnt = 0; }
            if (EDGE && tid == 0) { s_settled = 0; s_nd = 0; }
            __syncthreads();
            for (;;) {
                const int p = s_posv[sel];  // first unexpanded entry = the top of the candidate queue
                if (p == INT_MAX) break;    // candidates.size() == 0
                JV_T(t_i0);
                const long long ckey = cur[p];
                const int hs = s_hsize;
                const float csc = key_score(ckey);
                const float wsc = hs > 0 ? key_score(heap[1]) : 0.f;
                if (hs >= K && csc < wsc) break;  // stopSearch (strict <: a tie with the worst result is still expanded)
                const int node = key_node(ckey);
                // addTopCandidate: 1 push, 2 replace the worst, 3 tie with the worst: not added, 0 not acceptable. searchOneLayer admits
                // a node only if score >= threshold: at level 0 with acceptOrds and the caller's threshold (F_ACCEPTED), on upper levels
                // with Bits.ALL and threshold 0, which refuses a DOT_PRODUCT score (1 + q.x) / 2 below 0 (GraphSearcher.java:273-278, 429)
                int action = 0;
                if (lvl > 0 ? csc >= 0.f : (fcur[p] & F_ACCEPTED) != 0) action = hs < K ? 1 : (csc > wsc ? 2 : 3);
                const int dead = (lvl > 0 && (action == 3 || action == 0)) ? p : -1;
                if (tid == 0) { fcur[p] |= F_EXPANDED; s_posv[sel ^ 1] = INT_MAX; s_m = 0; }
                expanded++;
                if (lvl == 0) expanded_base++;
                const int32_t *nb;
                if (lvl == 0) nb = PG.adj0 + (size_t)node * degree;
                else {
                    const int32_t row = PG.upper_row[(size_t)(lvl - 1) * PG.n + node];
                    nb = row >= 0 ? PG.upper_adj + ((size_t)PG.upper_off[lvl - 1] + row) * degree : nullptr;
                }
                // FusedPQ (OnDiskGraphIndex.java:639-651, "useEdgeLoading && level == 0"): ids and the neighbours' codes come from the
                // expanded node's own record
                const bool fused = KIND == KIND_PQ && lvl == 0 && PG.fused != nullptr;
                const uint8_t *rec = fused ? PG.fused + (size_t)node * PG.fused_rec : nullptr;
                if (fused) {
                    nb = reinterpret_cast<const int32_t *>(rec);
                    if (P.pq_rows) {
                        // the record's code rows do not depend on which neighbours turn out to be new: the warps that have no
                        // neighbour to test copy ALL of them (degree x code_stride contiguous bytes) into shared memory while
                        // warp 0 runs visited.add(); the scoring phase then finds candidate i's codes at slot cand_slot[i]
                        const int cw = PA.code_stride >> 2, cws = cw + 1;
                        const uint32_t *src = reinterpret_cast<const uint32_t *>(rec + 4 * degree);
                        for (int t = tid - 64; t >= 0 && t < degree * cw; t += SEARCH_THREADS - 64) {
                            const int i = t / cw;
                            pq_stage[i * cws + (t - i * cw)] = __ldg(src + t);
                        }
                    } else if (tid >= 64) {
                        // the code rows of this record are needed one barrier from now: pull the whole record towards L2 at once
                        const int o = (tid - 64) * 128;
                        if (o < PG.fused_rec) prefetch_l2(rec + o);
                    }
                }
                // sketched DOT walk over a graph with edge records (the condition of `sketched` below): a new neighbour whose low-rank
                // bound (lowrank_bound), read from slot t of the expanded node's record together with its id, falls under the list's
                // last key would be dropped by the scoring phase whatever its exact score. It is settled here: its bound goes into
                // s_drop (>= the exact score, like the sketch bound), it is counted as visited and takes no candidate slot.
                const bool edge_tier = EDGE && lvl == 0 && size == LC;
                // processNeighbors: score a neighbour only if visited.add() says it is new (OnHeapGraphIndex.java:478)
                if (nb)
                    for (int t = tid; t < degree; t += SEARCH_THREADS) {
                        const int32_t f = __ldg(nb + t);
                        if (f >= 0 && (vsm ? visited_insert_smem(vis, P.vis_idmask, P.vis_rlog, f, &s_vfail) : visited_insert(table, vmask, P.visited_shift, f))) {
                            if (edge_tier) {
                                // (the record was requested towards L2 with the adjacency row, by the speculation below one or more hops ago)
                                const uint4 *e = reinterpret_cast<const uint4 *>(PG.edge_rec + ((size_t)node * degree + t) * LR_SLOT);
                                float est;
                                const float ub = lowrank_bound(PA, blobA, s_lr, __ldg(e), __ldg(e + 1), __ldg(reinterpret_cast<const float4 *>(e + 2)), est);
                                const long long last = cur[LC - 1];
                                if (topk_key(ub, f) < last) {
                                    atomicAdd(&s_settled, 1);
                                    atomicMax(&s_drop[sel], float_to_sortable(ub));
                                    continue;
                                }
                                if (est > key_score(last) + EDGE_DIRECT_MARGIN) {
                                    // a likely list entrant, whose sketch bound would not settle it: routed direct to its full row
                                    const int j = atomicAdd(&s_nd, 1);
                                    cand_ids[MAX_DEGREE - 1 - j] = f;
                                    bulk_prefetch_l2(PA.rows + (size_t)f * PA.stride, (unsigned)PA.stride * 4u);
                                    continue;
                                }
                            }
                            const int slot = atomicAdd(&s_n, 1);
                            cand_ids[slot] = f;
                            if (KIND == KIND_PQ) cand_slot[slot] = (uint8_t)t;
                            // the row is needed one barrier from now: start the DRAM -> L2 transfer of all of it at once (one
                            // UBLKPF per row; bytes in flight that occupy no registers and no shared memory)
                            if (KIND == KIND_F32 && P.row_prefetch == 1) bulk_prefetch_l2(PA.rows + (size_t)f * PA.stride, (unsigned)PA.stride * 4u);
                            // a sketched walk (the condition of `sketched` below) reads this row's sketch and {s, r} first, one barrier
                            // from now: request them (768 + 8 B at d = 768) so that the bound waits on L2, not DRAM. The full rows are
                            // not prefetched: only the ~17 % the bound does not settle read them, and they would not fit in L2.
                            if (KIND == KIND_F32 && METRIC == JV_METRIC_DOT && lvl == 0 && size == LC && PA.sketch != nullptr) {
                                const char *sk = reinterpret_cast<const char *>(PA.sketch) + (size_t)f * PA.sketch_stride;
                                for (int o = 0; o < PA.sketch_stride; o += 128) prefetch_l2(sk + o);
                                prefetch_l2(sk + PA.sketch_stride - 1);
                                prefetch_l2(PA.sketch_meta + f);
                            }
                            if (KIND == KIND_NVQ && P.row_prefetch == 1) {
                                bulk_prefetch_l2(PA.bytes + (size_t)f * PA.byte_stride, (unsigned)PA.byte_stride);
                                prefetch_l2(PA.params + (size_t)f * 4 * PA.nsub);  // {min, max, growthRate, midpoint} per sub-vector
                            }
                        }
                    }
                // Speculation by the otherwise idle warps (PQ / BQ only: their traversal is a latency chain and HBM is idle, while
                // the fp32 / NVQ paths are bandwidth-bound and must not waste it): the entries right behind p are the likeliest to
                // be expanded next, so touch their adjacency rows and prefetch their neighbours' code rows into L2.
                // Reads only; results unchanged.
                if (lvl == 0 && (KIND == KIND_F32 || KIND == KIND_NVQ)) {
                    // bandwidth-bound kinds speculate on the ADJACENCY rows only (128 B each, nothing next to the 3 KB rows): the next
                    // pops are most likely the unexpanded entries right behind p, and their rows then come from L2 instead of DRAM
                    if (tid >= 32 && tid < 36) {
                        const int pp = p + (tid - 31);
                        if (pp < size && !(fcur[pp] & F_EXPANDED)) {
                            prefetch_l2(PG.adj0 + (size_t)key_node(cur[pp]) * degree);
                            // and their edge records (degree x 48 B), so that a hop's record reads wait on L2 like its adjacency row
                            if (edge_tier) bulk_prefetch_l2(PG.edge_rec + (size_t)key_node(cur[pp]) * degree * LR_SLOT, (unsigned)(degree * LR_SLOT));
                        }
                    }
                }
                if (lvl == 0 && P.early_pf && tid == 36) {
                    // the next pop is the best of {unexpanded old entries, this hop's new candidates}: a new candidate that beats the
                    // SECOND unexpanded old entry is among the next two pops, so its adjacency (or FusedPQ record) is requested the
                    // moment its score is known (JV_EMIT) instead of after the merge
                    int found = 0;
                    const int end = min(size, p + 17);
                    long long nk = end > p + 1 ? cur[end - 1] : KEY_MIN;
                    for (int i = p + 1; i < end; i++)
                        if (!(fcur[i] & F_EXPANDED) && ++found == 2) { nk = cur[i]; break; }
                    if (found < 2 && end == size) nk = KEY_MIN;
                    s_nk = nk;
                }
                if (lvl == 0 && (KIND == KIND_PQ || KIND == KIND_BQ)) {
                    const int w = tid >> 5;
                    if (w >= 1 && w <= 3) {
                        const int pp = p + w;
                        if (pp < size && !(fcur[pp] & F_EXPANDED) && KIND == KIND_PQ && PG.fused) {
                            // one record = ids + codes: pull its lines towards L2 (25 x 128 B at degree 32, M = 96)
                            const char *r2 = reinterpret_cast<const char *>(PG.fused + (size_t)key_node(cur[pp]) * PG.fused_rec);
                            for (int o = (tid & 31) * 128; o < PG.fused_rec; o += 32 * 128) prefetch_l2(r2 + o);
                        } else if (pp < size && !(fcur[pp] & F_EXPANDED)) {
                            const int32_t *nb2 = PG.adj0 + (size_t)key_node(cur[pp]) * degree;
                            for (int t = tid & 31; t < degree; t += 32) {
                                const int32_t f = __ldg(nb2 + t);
                                if (KIND == KIND_PQ && f >= 0) {
                                    const char *a = reinterpret_cast<const char *>(PA.codes + (size_t)f * PA.code_stride);
                                    prefetch_l2(a);
                                    prefetch_l2(a + PA.M - 1);
                                } else if (KIND == KIND_BQ && f >= 0) {
                                    const char *a = reinterpret_cast<const char *>(PA.words + (size_t)f * PA.W);
                                    for (int o = 0; o < PA.W * 8; o += 128) prefetch_l2(a + o);
                                    prefetch_l2(a + PA.W * 8 - 1);
                                }
                            }
                        }
                    }
                }
                __syncthreads();
                JV_T(t_i1);
                JV_ACC(1, t_i0, t_i1);
                // every thread has read the heap top by now: apply addTopCandidate to the result heap
                if (tid == HEAP_TID) {
                    if (action == 1) {
                        heap[hs + 1] = ckey;
                        heap_up(heap, hs + 1);
                        s_hsize = hs + 1;
                    } else if (action == 2) {
                        heap[1] = ckey;
                        heap_down(heap, hs, 1);
                    }
                }
                if (tid == 0) { s_drop[sel ^ 1] = INT_MIN; s_cnt = 0; }
                const int nd = EDGE ? s_nd : 0;  // routed direct, counted in n
                const int n = s_n + nd;
                table_cnt += n;
                if (EDGE) {
                    const int ns = s_settled;
                    table_cnt += ns;
                    visited += ns;
                    if (tid == 0) { s_settled_total += (unsigned)ns; s_direct_total[0] += (unsigned)nd; }
                }
                if (vsm ? (table_cnt > vis_limit || s_vfail) : (table_cnt * 2 > P.visited_cap)) {
                    if (P.lenient) truncated = true;
                    else failed = 1;
                    break;
                }
                // A candidate that scores under the last entry of a FULL list is dropped by the merge whatever the other candidates do, so
                // it is dropped here and the merge only ranks the survivors (late in a walk that is most of them).
                // (the list's last key is re-read from shared memory by the one lane that needs it: nothing extra lives in registers
                // across the scoring loop)
#define JV_EMIT(sc_, f_)                                                                                                            \
    do {                                                                                                                            \
        const long long key_ = topk_key((sc_), (f_));                                                                               \
        JV_RBS_ROW(key_, f_);                                                                                                       \
        if (lvl == 0 && P.early_pf && key_ > s_nk) {                                                                                \
            if (KIND == KIND_PQ && PG.fused) bulk_prefetch_l2(PG.fused + (size_t)(f_) * PG.fused_rec, (unsigned)PG.fused_rec);  \
            else prefetch_l2(PG.adj0 + (size_t)(f_) * degree);                                                                     \
        }                                                                                                                           \
        if (dead < 0 && size == LC && key_ < cur[LC - 1]) {                                                                         \
            JV_RBS_DROP(f_);                                                                                                        \
            atomicMax(&s_drop[sel], float_to_sortable(sc_));                                                                        \
        } else {                                                                                                                    \
            const int m_ = atomicAdd(&s_m, 1);                                                                                      \
            cand_keys[m_] = key_;                                                                                                   \
            if (P.filtered) cand_acc[m_] = ((!acc || ((acc[(f_) >> 5] >> ((f_) & 31)) & 1u)) && (sc_) >= P.threshold &&              \
                                            !(EXCL && P.exclude_ids[qi] == (f_))) ? F_ACCEPTED : 0;                               \
        }                                                                                                                           \
    } while (0)
                if (KIND == KIND_F32) {
                    // DOT walk with a full list and a row sketch (launch_search): a row whose score's upper bound from its sketch
                    // (half the bytes) already falls under the list's last key would be dropped by JV_EMIT whatever its exact score,
                    // so it is dropped on the bound, which also stands in for its score in s_drop (>= the exact one: the check after
                    // the merge stays conservative). Only the others read their full rows, scored exactly as below.
                    const bool sketched = METRIC == JV_METRIC_DOT && lvl == 0 && size == LC && PA.sketch != nullptr;
                    // two rows per warp at a time: twice the loads in flight, query fragment read once. EDGE: one flat pair index
                    // over both classes, so that the warps share them evenly: pairs [0, ps) read sketches first (rows i and i + ps of
                    // cand_ids), pairs [ps, ps + pd) are the rows routed direct (from the top of cand_ids), scored exactly at once
                    const int ns = n - nd, ps = (ns + 1) >> 1, pd = (nd + 1) >> 1;
                    for (int i = group; i < (EDGE ? ps + pd : n); i += (EDGE ? NG : 2 * NG)) {
                        const bool direct = EDGE && i >= ps;
                        int32_t fa, fb;
                        bool two;
                        if (!EDGE) {
                            fa = cand_ids[i];
                            two = i + NG < n;
                            fb = two ? cand_ids[i + NG] : fa;
                        } else if (!direct) {
                            fa = cand_ids[i];
                            two = i + ps < ns;
                            fb = two ? cand_ids[i + ps] : fa;
                        } else {
                            const int j = MAX_DEGREE - 1 - (i - ps);
                            fa = cand_ids[j];
                            two = i - ps + pd < nd;
                            fb = two ? cand_ids[j - pd] : fa;
                        }
                        bool xa = true, xb = two;  // exact score needed
                        if (sketched && !direct) {
                            float ua, ub;
                            sketch_bound_pair(PA, blobA, fa, fb, lane, ua, ub);
                            const long long last = cur[LC - 1];
                            xa = !(topk_key(ua, fa) < last);
                            xb = two && !(topk_key(ub, fb) < last);
                            if (lane == 0) {
                                if (!xa) atomicMax(&s_drop[sel], float_to_sortable(ua));
                                if (two && !xb) atomicMax(&s_drop[sel], float_to_sortable(ub));
                            }
                            if (!xa && !xb) continue;
                            if (!xa || !xb) {
                                const int32_t f = xa ? fa : fb;
                                const float sc = score_f32<METRIC>(PA, blobA, f, lane);
                                if (lane == 0) JV_EMIT(sc, f);
                                continue;
                            }
                        }
                        float sa, sb;
                        score_f32_pair<METRIC>(PA, blobA, fa, fb, lane, sa, sb);
                        if (lane == 0) {
                            JV_RBS_SCORED(two ? 2 : 1);
                            if (direct) {
                                // a wrong route: the row JV_EMIT drops below (its exact score, <= its sketch bound, goes into s_drop)
                                const long long last = cur[LC - 1];
                                const int dr = (topk_key(sa, fa) < last ? 1 : 0) + (two && topk_key(sb, fb) < last ? 1 : 0);
                                if (dr) atomicAdd(&s_direct_total[1], (unsigned long long)dr);
                            }
                            JV_EMIT(sa, fa);
                            if (two) JV_EMIT(sb, fb);
                        }
                    }
                } else if (KIND == KIND_PQ && P.pq_rows) {
                    // lane = candidate, warp = one of the 8 partial sums of the ADC score (score_pq_partial): the code rows of the
                    // hop are staged in shared memory by one coalesced pass, then every gather instruction of a warp reads ONE LUT row
                    const int cw = PA.code_stride >> 2, cws = cw + 1;  // odd word stride: no bank conflicts across candidates
                    if (!fused) {
                        for (int t = tid; t < n * cw; t += SEARCH_THREADS) {
                            const int i = t / cw, wd = t - i * cw;
                            pq_stage[i * cws + wd] = __ldg(reinterpret_cast<const uint32_t *>(PA.codes + (size_t)cand_ids[i] * PA.code_stride) + wd);
                        }
                        __syncthreads();
                    }
                    const int pstride = (degree + 31) & ~31;
                    for (int g = tid >> 5; g < 8; g += SEARCH_THREADS / 32)
                        for (int i = tid & 31; i < n; i += 32) {
                            float ps, pa;
                            score_pq_partial<METRIC>(PA, blobA, blobH, splitm, reinterpret_cast<const uint8_t *>(pq_stage + (fused ? (int)cand_slot[i] : i) * cws), g, ps, pa);
                            pq_part[g * pstride + i] = ps;
                            if (METRIC == JV_METRIC_COSINE) pq_part[(8 + g) * pstride + i] = pa;
                        }
                    __syncthreads();
                    for (int i = tid; i < n; i += SEARCH_THREADS) {
                        float sraw = pq_fold8(pq_part + i, pstride);
                        if (METRIC == JV_METRIC_COSINE)
                            sraw = __fdiv_rn(sraw, __fsqrt_rn(__fmul_rn(pq_fold8(pq_part + 8 * pstride + i, pstride), blobH[PA.M * PA.k])));
                        const float sc = score_map(METRIC, sraw);
                        const int32_t f = cand_ids[i];
                        JV_EMIT(sc, f);
                    }
                } else if (KIND == KIND_PQ && fused) {
                    // FusedPQDecoder.similarityToNeighbor (FusedPQDecoder.java:107-114): the code row sits inside the record just read
                    const uint8_t *codes0 = rec + 4 * degree;
                    for (int i = group; i < n; i += NG) {
                        const int32_t f = cand_ids[i];
                        const float sc = score_pq_codes<METRIC>(PA, blobA, codes0 + (size_t)cand_slot[i] * PG.fused_code_stride, lane, blobH, splitm);
                        if (lane == 0) JV_EMIT(sc, f);
                    }
                } else {
                    for (int i = group; i < n; i += NG) {
                        const int32_t f = cand_ids[i];
                        const float sc = KIND == KIND_PQ ? score_pq<METRIC>(PA, blobA, f, lane, blobH, splitm) : score_row<KIND, METRIC>(PA, blobA, f, lane);
                        if (lane == 0) JV_EMIT(sc, f);
                    }
                }
#undef JV_EMIT
                __syncthreads();
                JV_T(t_i2);
                JV_ACC(2, t_i1, t_i2);
                visited += n;
                const int nm = s_m;  // candidates that survived the pre-filter
                // rank-merge (old list is sorted; candidates are few): every element computes its slot directly and the
                // first unexpanded slot of the next list falls out of the same pass. The entry at `dead` (refused on an
                // upper level) leaves the list.
                const int live = size - (dead >= 0 ? 1 : 0);
                const int newsize = min(LC, live + nm);
                const long long dead_key = dead >= 0 ? cur[dead] : KEY_MIN;
                int mypos = INT_MAX, mydrop = INT_MIN;
                // one work item per thread: items [0, size) are old entries, [size, size + n) the new candidates, so the
                // two kinds run on different warps instead of back to back on warp 0
                for (int it = tid; it < size + nm; it += SEARCH_THREADS) {
                    if (it < size) {
                        if (it == dead) continue;
                        const long long k = cur[it];
                        int c = 0;
#pragma unroll 8
                        for (int j = 0; j < nm; j++) c += (cand_keys[j] > k);
                        const int np = it + c - ((dead >= 0 && it > dead) ? 1 : 0);
                        const uint8_t fl = fcur[it];
                        if (np < LC) {
                            nxt[np] = k;
                            fnxt[np] = fl;
                            if (!(fl & F_EXPANDED)) mypos = min(mypos, np);
                        } else if (!(fl & F_EXPANDED) || lvl > 0) mydrop = max(mydrop, float_to_sortable(key_score(k)));
                    } else {
                        const long long k = cand_keys[it - size];
                        int c = count_greater_desc(cur, size, k) - ((dead >= 0 && dead_key > k) ? 1 : 0);
#pragma unroll 8
                        for (int jj = 0; jj < nm; jj++) c += (cand_keys[jj] > k);
                        if (c < LC) {
                            nxt[c] = k;
                            // unfiltered (threshold 0, no acceptOrds): only a score below 0 is refused, and the key carries the score
                            fnxt[c] = P.filtered ? cand_acc[it - size] : (key_score(k) >= 0.f ? F_ACCEPTED : 0);
                            mypos = min(mypos, c);
                            // a new candidate that lands at the very front is the likeliest next expansion: start pulling
                            // its adjacency row towards L2 now (128 B; reads only)
                            if (c < 2 && lvl == 0) {
                                if (KIND == KIND_PQ && PG.fused) prefetch_l2(PG.fused + (size_t)key_node(k) * PG.fused_rec);
                                else prefetch_l2(PG.adj0 + (size_t)key_node(k) * degree);
                                if (EDGE && size == LC)
                                    bulk_prefetch_l2(PG.edge_rec + (size_t)key_node(k) * degree * LR_SLOT, (unsigned)(degree * LR_SLOT));
                            }
                        } else mydrop = max(mydrop, float_to_sortable(key_score(k)));
                    }
                }
                if (mypos != INT_MAX) atomicMin(&s_posv[sel ^ 1], mypos);
                if (mydrop != INT_MIN) atomicMax(&s_drop[sel], mydrop);
                if (tid == 0) {
                    s_n = 0;
                    if (EDGE) { s_settled = 0; s_nd = 0; }
                }
                __syncthreads();
                JV_T(t_i3);
                JV_ACC(3, t_i2, t_i3);
#ifdef JV_SEARCH_PROFILE
                if (tid == 0) { dbg_local[5] += 1; dbg_local[6] += (unsigned long long)n; }
#endif
                // something fell off the end of the list: that is exact only if at least rerankK accepted entries score strictly
                // higher than everything dropped (then none of it can be popped before stopSearch fires)
                const int dm = s_drop[sel];
                if (dm != INT_MIN) {
                    bool ok;
                    // unfiltered, the list is sorted by score: when its L-th entry scores >= 0 all L are accepted (newsize == LC >= L)
                    const float sl = key_score(nxt[L - 1]);
                    if (!P.filtered && sl >= 0.f) ok = float_to_sortable(sl) > dm;
                    else {
                        int c = 0;
                        for (int i = tid; i < newsize; i += SEARCH_THREADS)
                            c += ((fnxt[i] & F_ACCEPTED) && float_to_sortable(key_score(nxt[i])) > dm) ? 1 : 0;
                        if (c) atomicAdd(&s_cnt, c);
                        __syncthreads();
                        ok = s_cnt >= L;
                    }
                    if (!ok) {
                        if (P.lenient) inexact = true;  // keep walking: only the exactness of tie handling is lost
                        else { failed = 2; break; }
                    }
                }
                { long long *t = cur; cur = nxt; nxt = t; }
                { uint8_t *t = fcur; fcur = fnxt; fnxt = t; }
                size = newsize;
                sel ^= 1;
            }
            __syncthreads();
        }

        JV_T(t_r0);
        int32_t *no = P.nodes_out + (size_t)qi * P.topK;
        float *so = P.scores_out + (size_t)qi * P.topK;
        unsigned reranked = 0;
        if (failed) {
            for (int i = tid; i < P.topK; i += SEARCH_THREADS) { no[i] = -1; so[i] = 0.f; }
            if (tid == 0) { P.overflow[qi] = (uint8_t)failed; atomicAdd(&PC->overflowed, 1ull); }
        } else {
            if (tid == 0) {
                P.overflow[qi] = 0;
                if (truncated || inexact) atomicAdd(&PC->overflowed, 1ull);
            }
            const int hs = s_hsize;  // the results: heap[1 .. hs]
            if (P.has_rerank) {
                // NodeQueue.rerank (NodeQueue.java:168-230): rescore, in HEAP-ARRAY order, the results whose approximate score
                // is >= rerankFloor (or the single best one if none is), keep the topK best exact scores; on an exact-score
                // tie at the topK boundary the entry met first in array order stays.
                constexpr int NGR = SEARCH_THREADS / 32;
                const int wgroup = tid >> 5, wlane = tid & 31;
                if (tid == 0) s_cnt = 0;
                __syncthreads();
                {
                    int c = 0;
                    for (int i = tid; i < hs; i += SEARCH_THREADS) {
                        const bool above = key_score(heap[1 + i]) >= P.rerank_floor;
                        fcur[i] = above ? 1 : 0;
                        c += above ? 1 : 0;
                    }
                    if (c) atomicAdd(&s_cnt, c);
                }
                __syncthreads();
                int nrr = s_cnt;
                if (nrr == 0 && hs > 0) {
                    // nothing above the floor: the best approximate score is reranked alone (first maximum in array order)
                    if (tid == 0) {
                        int bi = 0;
                        float bs = key_score(heap[1]);
                        for (int i = 1; i < hs; i++) {
                            const float s = key_score(heap[1 + i]);
                            if (s > bs) { bs = s; bi = i; }
                        }
                        fcur[bi] = 1;
                    }
                    nrr = 1;
                    __syncthreads();
                }
                if (KIND == KIND_PQ || KIND == KIND_BQ) {
                    // the approximate walk left HBM idle: pull every survivor's exact row towards L2 before the rescoring loop
                    const int lines = PR.kind == KIND_F32 ? (PR.stride * 4 + 127) / 128 : (PR.byte_stride + 127) / 128;
                    for (int t = tid; t < hs * lines; t += SEARCH_THREADS) {
                        const int i = t / lines, l = t - i * lines;
                        if (!fcur[i]) continue;
                        const int32_t f = key_node(heap[1 + i]);
                        const char *a = PR.kind == KIND_F32 ? reinterpret_cast<const char *>(PR.rows + (size_t)f * PR.stride)
                                                                  : reinterpret_cast<const char *>(PR.bytes + (size_t)f * PR.byte_stride);
                        prefetch_l2(a + (size_t)l * 128);
                    }
                }
                // exact keys in array order -> cur[0 .. hs) (KEY_MIN = not reranked)
                if (PR.kind == KIND_F32) {
                    for (int i = wgroup; i < hs; i += 2 * NGR) {
                        const int32_t fa = key_node(heap[1 + i]);
                        const bool two = i + NGR < hs;
                        const int32_t fb = two ? key_node(heap[1 + i + NGR]) : fa;
                        const bool da = fcur[i] != 0, db = two && fcur[i + NGR] != 0;
                        float sa = 0.f, sb = 0.f;
                        if (da || db) score_f32_pair<METRIC>(PR, blobR, da ? fa : fb, db ? fb : fa, wlane, sa, sb);
                        if (wlane == 0) {
                            cur[i] = da ? topk_key(sa, fa) : KEY_MIN;
                            if (two) cur[i + NGR] = db ? topk_key(sb, fb) : KEY_MIN;
                        }
                    }
                } else {
                    for (int i = wgroup; i < hs; i += NGR) {
                        const int32_t f = key_node(heap[1 + i]);
                        float sc = 0.f;
                        const bool d = fcur[i] != 0;
                        if (d) sc = score_row<KIND_NVQ, METRIC>(PR, blobR, f, wlane);
                        if (wlane == 0) cur[i] = d ? topk_key(sc, f) : KEY_MIN;
                    }
                }
                __syncthreads();
                for (int i = tid; i < P.sort_pow2; i += SEARCH_THREADS) nxt[i] = i < hs ? cur[i] : KEY_MIN;
                __syncthreads();
                bitonic_sort_desc(nxt, P.sort_pow2);
                reranked = (unsigned)nrr;
                const bool boundary_tie = nrr > P.topK && key_score(nxt[P.topK - 1]) == key_score(nxt[P.topK]);
                if (!boundary_tie) {
                    for (int i = tid; i < P.topK; i += SEARCH_THREADS) {
                        if (i < nrr) { no[i] = key_node(nxt[i]); so[i] = key_score(nxt[i]); }
                        else { no[i] = -1; so[i] = 0.f; }
                    }
                } else if (tid == 0) {
                    // replay the reference loop (NodeQueue.java:199-215) over the array order; `heap` is free to be reused
                    long long *rh = heap;
                    int rs = 0;
                    for (int i = 0; i < hs; i++) {
                        const long long v = cur[i];
                        if (v == KEY_MIN) continue;
                        if (rs < P.topK) { rh[++rs] = v; heap_up(rh, rs); }
                        else if (key_score(v) > key_score(rh[1])) { rh[1] = v; heap_down(rh, rs, 1); }
                    }
                    for (int i = rs - 1; i >= 0; i--) {  // pop: worst first
                        const long long v = rh[1];
                        rh[1] = rh[rs--];
                        if (rs > 0) heap_down(rh, rs, 1);
                        no[i] = key_node(v);
                        so[i] = key_score(v);
                    }
                }
            } else {
                // no reranker: the best topK of the results by approximate key (GraphSearcher.java:478-486, :494-500)
                for (int i = tid; i < P.sort_pow2; i += SEARCH_THREADS) nxt[i] = i < hs ? heap[1 + i] : KEY_MIN;
                __syncthreads();
                bitonic_sort_desc(nxt, P.sort_pow2);
                for (int i = tid; i < P.topK; i += SEARCH_THREADS) {
                    if (i < hs) { no[i] = key_node(nxt[i]); so[i] = key_score(nxt[i]); }
                    else { no[i] = -1; so[i] = 0.f; }
                }
            }
            if (tid == 0) {
                atomicAdd(&PC->visited, (unsigned long long)visited);
                atomicAdd(&PC->expanded, (unsigned long long)expanded);
                atomicAdd(&PC->expanded_base, (unsigned long long)expanded_base);
                atomicAdd(&PC->reranked, (unsigned long long)reranked);
            }
        }
        if constexpr (SEG && EDGE) {
            // the next item may belong to another segment: this one's edge-tier totals go to its own counters now
            if (tid == 0) {
                if (s_settled_total) atomicAdd(&PC->settled, s_settled_total);
                if (s_direct_total[0]) atomicAdd(&PC->direct, s_direct_total[0]);
                if (s_direct_total[1]) atomicAdd(&PC->direct_dropped, s_direct_total[1]);
                s_settled_total = 0; s_direct_total[0] = 0; s_direct_total[1] = 0;
            }
        }
        __syncthreads();
#ifdef JV_SEARCH_PROFILE
        {
            JV_T(t_r1);
            JV_ACC(4, t_r0, t_r1);
            JV_ACC(7, t_q0, t_r1);
            if (tid == 0 && P.dbg)
                for (int i = 0; i < 8; i++) atomicAdd(&P.dbg[i], dbg_local[i]);
        }
#endif
    }
#undef PC
#undef PR
#undef PA
#undef PG
}

// shared-memory floats of the walking scorer's prepared query: everything, except for a PQ LUT of which only the rows of the
// first pq_smem_m sub-spaces stay in shared memory
static int search_smemA_floats(const DataDesc &approx, int pq_smem_m)
{
    if (approx.kind != KIND_PQ || pq_smem_m >= approx.M) return blob_floats(approx);
    return (pq_smem_m * approx.k + 3) & ~3;
}

static size_t search_smem_bytes(const DataDesc &approx, const DataDesc *rerank, int rerankK, int list_alloc, int pq_smem_m, int vis_slots_log = 0, int pq_rows_degree = 0)
{
    size_t b = (size_t)search_smemA_floats(approx, pq_smem_m) * 4;
    if (rerank) b += (size_t)blob_floats(*rerank) * 4;
    b += (size_t)list_alloc * 8 * 2;                  // the two list buffers
    b += (size_t)MAX_DEGREE * 8;                      // candidate keys of one hop
    b += (size_t)((rerankK + 2) & ~1) * 8;            // result heap (1-based)
    b += (size_t)MAX_DEGREE * 4 + (size_t)MAX_DEGREE * 2; // candidate ids + accept flags + record slots
    b += (size_t)list_alloc * 2;                      // entry flags of the two buffers
    b = (b + 15) & ~(size_t)15;
    if (vis_slots_log) b += (size_t)2 << vis_slots_log;  // visited set, 16 bits per slot
    if (pq_rows_degree) b += (size_t)pq_rows_degree * ((approx.code_stride >> 2) + 1) * 4 + (size_t)16 * ((pq_rows_degree + 31) & ~31) * 4;  // staged codes + partial sums
    return (b + 15) & ~(size_t)15;
}

#ifndef JV_VISITED_SMEM_DEFAULT
#define JV_VISITED_SMEM_DEFAULT true
#endif
#ifndef JV_PQ_ROWS_DEFAULT
#define JV_PQ_ROWS_DEFAULT 1
#endif
#ifndef JV_SEARCH_MINB_PQ_WIDE
#define JV_SEARCH_MINB_PQ_WIDE 4
#endif
#ifndef JV_ROW_PREFETCH_DEFAULT
#define JV_ROW_PREFETCH_DEFAULT 1
#endif
#ifndef JV_SEARCH_MINB_ROWS
#define JV_SEARCH_MINB_ROWS 9
#endif
#ifndef JV_SEARCH_MINB_ROWS_WIDE
#define JV_SEARCH_MINB_ROWS_WIDE 8
#endif
constexpr int MINB_DEFAULT = JV_SEARCH_MINB, MINB_PQ_LITE = JV_SEARCH_MINB_PQ, MINB_PQ_WIDE = JV_SEARCH_MINB_PQ_WIDE;
constexpr int MINB_ROWS = JV_SEARCH_MINB_ROWS, MINB_ROWS_WIDE = JV_SEARCH_MINB_ROWS_WIDE;  // fp32 / NVQ walks (56 registers at 128 threads, 9 CTAs per SM)

template <int KIND, int METRIC, int MINB, bool VSM>
static cudaError_t occupancy_of(size_t smem, int *blocks_per_sm)
{
    cudaError_t e = cudaFuncSetAttribute(graph_search_kernel<KIND, METRIC, MINB, VSM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, graph_search_kernel<KIND, METRIC, MINB, VSM>, SearchThreads<KIND>::value, smem);
}

// the fp32, PQ and BQ walks; any other kind runs OTHER
#define JV_SEARCH_DISPATCH_FPB_V(kind, metric, pq_wide, V, CALL, OTHER)                                            \
    do {                                                                                        \
        if ((kind) == KIND_F32 && (pq_wide)) {                                                  \
            if ((metric) == JV_METRIC_EUCLIDEAN) { CALL(KIND_F32, JV_METRIC_EUCLIDEAN, MINB_ROWS_WIDE, V); } \
            else if ((metric) == JV_METRIC_DOT) { CALL(KIND_F32, JV_METRIC_DOT, MINB_ROWS_WIDE, V); } \
            else { CALL(KIND_F32, JV_METRIC_COSINE, MINB_ROWS_WIDE, V); }                            \
        } else if ((kind) == KIND_F32) {                                                        \
            if ((metric) == JV_METRIC_EUCLIDEAN) { CALL(KIND_F32, JV_METRIC_EUCLIDEAN, MINB_ROWS, V); }       \
            else if ((metric) == JV_METRIC_DOT) { CALL(KIND_F32, JV_METRIC_DOT, MINB_ROWS, V); }              \
            else { CALL(KIND_F32, JV_METRIC_COSINE, MINB_ROWS, V); }                                          \
        } else if ((kind) == KIND_PQ && (pq_wide)) {                                            \
            if ((metric) == JV_METRIC_EUCLIDEAN) { CALL(KIND_PQ, JV_METRIC_EUCLIDEAN, MINB_PQ_WIDE, V); } \
            else if ((metric) == JV_METRIC_DOT) { CALL(KIND_PQ, JV_METRIC_DOT, MINB_PQ_WIDE, V); } \
            else { CALL(KIND_PQ, JV_METRIC_COSINE, MINB_PQ_WIDE, V); }                             \
        } else if ((kind) == KIND_PQ) {                                                         \
            if ((metric) == JV_METRIC_EUCLIDEAN) { CALL(KIND_PQ, JV_METRIC_EUCLIDEAN, MINB_PQ_LITE, V); } \
            else if ((metric) == JV_METRIC_DOT) { CALL(KIND_PQ, JV_METRIC_DOT, MINB_PQ_LITE, V); } \
            else { CALL(KIND_PQ, JV_METRIC_COSINE, MINB_PQ_LITE, V); }                             \
        } else if ((kind) == KIND_BQ) {                                                         \
            if ((metric) == JV_METRIC_EUCLIDEAN) { CALL(KIND_BQ, JV_METRIC_EUCLIDEAN, MINB_DEFAULT, V); }        \
            else if ((metric) == JV_METRIC_DOT) { CALL(KIND_BQ, JV_METRIC_DOT, MINB_DEFAULT, V); }               \
            else { CALL(KIND_BQ, JV_METRIC_COSINE, MINB_DEFAULT, V); }                                           \
        } else {                                                                                \
            OTHER;                                                                              \
        }                                                                                       \
    } while (0)
#define JV_SEARCH_DISPATCH_NVQ_V(metric, V, CALL)                                               \
    do {                                                                                        \
        if ((metric) == JV_METRIC_EUCLIDEAN) { CALL(KIND_NVQ, JV_METRIC_EUCLIDEAN, MINB_ROWS, V); }           \
        else if ((metric) == JV_METRIC_DOT) { CALL(KIND_NVQ, JV_METRIC_DOT, MINB_ROWS, V); }                  \
        else { CALL(KIND_NVQ, JV_METRIC_COSINE, MINB_ROWS, V); }                                              \
    } while (0)
#define JV_SEARCH_DISPATCH_V(kind, metric, pq_wide, V, CALL) \
    JV_SEARCH_DISPATCH_FPB_V(kind, metric, pq_wide, V, CALL, JV_SEARCH_DISPATCH_NVQ_V(metric, V, CALL))
#define JV_SEARCH_DISPATCH(kind, metric, pq_wide, vsm, CALL)                    \
    do {                                                                       \
        if (vsm) JV_SEARCH_DISPATCH_V(kind, metric, pq_wide, true, CALL);      \
        else JV_SEARCH_DISPATCH_V(kind, metric, pq_wide, false, CALL);         \
    } while (0)

cudaError_t plan_search(const DataDesc &approx, const DataDesc *rerank, const GraphDesc &g, int topK, int rerankK, int nq,
                        int visited_cap_hint, int list_cap_hint, int sm_count, SearchPlan *plan)
{
    if (g.degree > MAX_DEGREE || rerankK < 1 || topK < 1 || topK > rerankK) return cudaErrorInvalidValue;
    plan->threads = search_threads_of(approx.kind);
    plan->sort_pow2 = next_pow2(rerankK);
    // The list keeps rerankK entries plus a tie tail (see the kernel header). Continuous scores tie rarely: the slack that
    // rounds rerankK up to a multiple of 32 is enough; BQ scores take at most dim + 1 values, so whole groups tie at the
    // boundary. A query whose tail does not fit reports overflow code 2 and is re-run with list_cap_hint = 4x.
    int cap = list_cap_hint > 0 ? list_cap_hint : (approx.kind == KIND_BQ ? 2 * rerankK + 64 : rerankK + 28);
    if (cap < rerankK) cap = rerankK;
    cap = (cap + 3) & ~3;
    if (cap > MAX_LIST_CAP) cap = MAX_LIST_CAP;
    if (cap < rerankK) return cudaErrorInvalidValue;
    plan->list_cap = cap;
    plan->list_alloc = cap > plan->sort_pow2 ? cap : plan->sort_pow2;
    // PQ: a LUT of M*k fp32 (96 KB at M=96) in shared memory limits residency to 2 CTAs per SM, and the walk is a latency chain.
    // When five LUTs do not fit an SM's shared memory the LUT lives in an L2-resident
    // global slice per CTA instead: residency becomes register-limited (5 CTAs per SM) and the gathers are served by L2.
    // JV_PQ_LUT=smem|l2 overrides.
    // Round 2: the LUT may be SPLIT — rows of the first pq_smem_m sub-spaces in shared memory, the rest in the L2 slice — which
    // trades L2 gather traffic against residency continuously (JV_PQ_LUT=smem|l2 or JV_PQ_LUT_SMEM_M=<sub-spaces> override).
    plan->blob_in_global = 0;
    plan->pq_smem_m = approx.kind == KIND_PQ ? approx.M : 0;
    if (approx.kind == KIND_PQ) {
        const char *mode = getenv("JV_PQ_LUT");
        const char *msub = getenv("JV_PQ_LUT_SMEM_M");
        if (msub) plan->pq_smem_m = std::max(0, std::min(approx.M, atoi(msub))) & ~3;
        else if (mode && mode[0] == 'l') plan->pq_smem_m = 0;
        else if (mode && mode[0] == 's') plan->pq_smem_m = approx.M;
        else plan->pq_smem_m = (size_t)blob_floats(approx) * 4 * 5 > 200 * 1024 ? 0 : approx.M;
        plan->blob_in_global = plan->pq_smem_m < approx.M ? 1 : 0;
    }
    plan->blob_floats = blob_floats(approx);
    // PQ scoring layout of a hop: JV_PQ_SCORE=rows (lane = candidate, warp = partial sum) | group (8 lanes per candidate)
    plan->pq_rows = 0;
    if (approx.kind == KIND_PQ) {
        const char *pt = getenv("JV_PQ_SCORE");
        plan->pq_rows = pt ? (pt[0] == 'r') : JV_PQ_ROWS_DEFAULT;
    }
    const int prd = plan->pq_rows ? g.degree : 0;
    plan->smem_bytes = search_smem_bytes(approx, rerank, rerankK, plan->list_alloc, plan->pq_smem_m, 0, prd);
    if (plan->smem_bytes > 227 * 1024 && approx.kind == KIND_PQ && plan->pq_smem_m > 0) {
        plan->pq_smem_m = 0;  // a long list next to a LUT: keep the list in shared memory, move the whole LUT to L2
        plan->blob_in_global = 1;
        plan->smem_bytes = search_smem_bytes(approx, rerank, rerankK, plan->list_alloc, 0, 0, prd);
    }
    if (plan->smem_bytes > 227 * 1024) return cudaErrorInvalidValue;
    int vcap = visited_cap_hint > 0 ? visited_cap_hint : next_pow2(4 * rerankK * (g.degree > 16 ? g.degree : 16));
    if (vcap < 2048) vcap = 2048;
    if (vcap > (1 << 22)) vcap = 1 << 22;
    plan->visited_cap = next_pow2(vcap);
    // Visited set in shared memory (16-bit slots, see visited_insert_smem): no L2 round trip per neighbour, no 64 KB table to clear
    // per query, nothing of it in L2. Taken on the first attempt when the table a walk of this effort needs fits 32 KB and every
    // region keeps at least 32 slots; a query that outgrows it (or fills one region) is re-run on the global table
    // (visited_cap_hint > 0).
    // JV_VISITED=global|smem overrides, JV_VISITED_SMEM_SLOTS sets the slot count.
    plan->vis_slots_log = 0;
    plan->vis_rlog = 0;
    plan->vis_idmask = 0;
    {
        const char *vm = getenv("JV_VISITED");
        const char *vs = getenv("JV_VISITED_SMEM_SLOTS");
        int bits = 15;
        while ((1ll << bits) < g.n) bits++;
        int slots = vs ? next_pow2(atoi(vs)) : plan->visited_cap / 2;
        int slog = 0;
        while ((1 << slog) < slots) slog++;
        // many regions (large n) want more slots each: grow the table up to 32 KB (10M nodes: 512 regions of 32 slots, ~6 expected
        // entries each for a 3 200-node walk)
        while (!vs && slog - (bits - 15) < 7 && slog < 14) slog++;
        const int rlog = slog - (bits - 15);
        const bool want = vm ? vm[0] == 's' : JV_VISITED_SMEM_DEFAULT;
        if (want && visited_cap_hint <= 0 && slog >= 10 && slog <= 14 && rlog >= 5) {
            const size_t sb = search_smem_bytes(approx, rerank, rerankK, plan->list_alloc, plan->pq_smem_m, slog, prd);
            if (sb <= 227 * 1024) {
                plan->vis_slots_log = slog;
                plan->vis_rlog = rlog;
                plan->vis_idmask = (unsigned)((1ull << bits) - 1ull);
                plan->smem_bytes = sb;
            }
        }
    }
    // JV_ROW_PREFETCH=0|1|2: L2 prefetch of the newly visited rows (fp32 / NVQ walks)
    {
        const char *rp = getenv("JV_ROW_PREFETCH");
        plan->row_prefetch = rp ? atoi(rp) : JV_ROW_PREFETCH_DEFAULT;
        if (approx.kind == KIND_NVQ && ((approx.byte_stride & 15) || plan->row_prefetch != 1)) plan->row_prefetch = 0;
        if (approx.kind != KIND_F32 && approx.kind != KIND_NVQ) plan->row_prefetch = 0;
    }
    int bps = 0;
    cudaError_t e = cudaSuccess;
    const int metric_for_occ = JV_METRIC_DOT;
#define CALL(K, M, B, V) e = occupancy_of<K, M, B, V>(plan->smem_bytes, &bps)
    JV_SEARCH_DISPATCH(approx.kind, metric_for_occ, false, plan->vis_slots_log != 0, CALL);
    plan->pq_wide = 0;
    if (e == cudaSuccess && approx.kind == KIND_PQ) {
        // the 64-register build wherever shared memory (not registers) is what limits residency
        int bw = 0;
        const int lite = bps;
        JV_SEARCH_DISPATCH(approx.kind, metric_for_occ, true, plan->vis_slots_log != 0, CALL);
        bw = bps;
        const char *pw = getenv("JV_PQ_WIDE");  // 0 | 1: force the register build (tuning)
        if (e == cudaSuccess && (pw ? pw[0] == '1' : bw >= lite)) plan->pq_wide = 1;
        else bps = lite;
    }
    if (e == cudaSuccess && approx.kind == KIND_F32) {
        // JV_SEARCH_WIDE=1: the 64-register build of the fp32 walk (4 resident CTAs per SM instead of 5, no spills) — a tuning knob
        const char *w = getenv("JV_SEARCH_WIDE");
        if (w && w[0] == '1') {
            plan->pq_wide = 1;
            JV_SEARCH_DISPATCH(approx.kind, metric_for_occ, true, plan->vis_slots_log != 0, CALL);
        }
    }
#undef CALL
    if (e != cudaSuccess) return e;
    if (bps < 1) return cudaErrorInvalidValue;
    long long ctas = (long long)bps * sm_count;
    if (ctas > nq) ctas = nq;
    if (ctas < 1) ctas = 1;
    plan->ctas = (int)ctas;
    return cudaSuccess;
}

// launch_search's device scratch, carved from `base` (nullptr: only measured): the per-CTA visited tables (unused when the visited
// set lives in shared memory), then the per-CTA L2 slices of the LUT when plan.blob_in_global
struct SearchScratch {
    int32_t *visited_tables;
    float *blob_global;
    size_t bytes;
    SearchScratch(const SearchPlan &p, void *base)
    {
        Carver c(base);
        visited_tables = c.take<int32_t>(p.vis_slots_log ? 1 : (size_t)p.ctas * p.visited_cap);
        blob_global = p.blob_in_global ? c.take<float>((size_t)p.ctas * p.blob_floats) : nullptr;
        bytes = c.bytes;
    }
};

size_t search_scratch_bytes(const SearchPlan &p) { return SearchScratch(p, nullptr).bytes; }

// a batch with more queries than resident CTAs fills the GPU: bandwidth bound rather than latency bound
static bool fills_gpu(const SearchPlan &plan, int nq) { return nq > plan.ctas; }

// fp32 DOT walks of such batches drop hopeless neighbours on the bound of their row sketch (sketch_bound_pair): HBM bound, a quarter
// of the bytes per dropped row, the sketch requested at gather time. A latency-bound batch reads the rows it prefetched anyway.
bool search_uses_sketch(const DataDesc &approx, int metric, const SearchPlan &plan, int nq)
{
    return approx.kind == KIND_F32 && metric == JV_METRIC_DOT && fills_gpu(plan, nq);
}

int sketch_stride(int stride) { return (stride + 7) & ~7; }

void search_walk_descs(GraphDesc &g, DataDesc &approx, int metric, bool sketch)
{
    if (!(approx.kind == KIND_PQ && g.fused && g.fused_codes_of == approx.codes && g.fused_code_stride == approx.code_stride)) g.fused = nullptr;
    {
        const char *fe = getenv("JV_FUSED_PQ");
        if (fe && fe[0] == '0') g.fused = nullptr;
    }
    if (!sketch) {
        approx.sketch = nullptr;
        approx.sketch_meta = nullptr;
    }
#ifdef JV_ROW_BOUND_STATS
    approx.sketch = nullptr;  // the drop statistics describe the walk that reads every row
#endif
    if (!approx.sketch || !approx.lr_basis || approx.kind != KIND_F32 || metric != JV_METRIC_DOT) g.edge_rec = nullptr;
}

cudaError_t launch_search(const GraphDesc &g, const DataDesc &approx, const DataDesc *rerank, int metric, const float *queries_dev,
                          int nq, int topK, int rerankK, const SearchPlan &plan, void *scratch_dev, int *work_counter_dev,
                          int32_t *nodes_out_dev, float *scores_out_dev, SearchCounters *counters_dev, uint8_t *overflow_flags_dev,
                          const int32_t *query_index_dev, int query_stride, const SearchFilter *filter, cudaStream_t s,
                          const SegmentGroup *segments)
{
    if (nq <= 0) return cudaSuccess;
    SearchParams P;
    P.accept_bits = filter ? filter->accept_bits : nullptr;
    P.accept_stride = filter ? filter->accept_stride_words : 0;
    P.threshold = filter ? filter->threshold : 0.f;
    P.rerank_floor = filter ? filter->rerank_floor : 0.f;
    P.exclude_ids = filter ? filter->exclude_ids : nullptr;
    P.filtered = (P.accept_bits != nullptr || P.threshold > 0.f || P.exclude_ids != nullptr) ? 1 : 0;
    P.lenient = filter ? filter->lenient : 0;
    P.arrived = filter ? filter->arrived : nullptr;
    P.query_stride = query_stride > 0 ? query_stride : approx.dim;
    // SEG walks (segments != nullptr): g and approx stand for the group (its largest degree, the first segment's data set), each
    // item reads its own segment's from segments->descs_dev
    P.g = g;
    P.approx = approx;
    P.segs = segments ? segments->descs_dev : nullptr;
    P.seg_nq = segments ? segments->nq : 0;
    P.has_rerank = rerank ? 1 : 0;
    P.rerank = rerank ? *rerank : approx;
    P.metric = metric;
    P.queries = queries_dev;
    P.nq = nq;
    P.topK = topK;
    P.rerankK = rerankK;
    P.list_cap = plan.list_cap;
    P.list_alloc = plan.list_alloc;
    P.sort_pow2 = plan.sort_pow2;
    P.visited_cap = plan.visited_cap;
    int lg = 0;
    while ((1 << lg) < plan.visited_cap) lg++;
    P.visited_shift = 32 - lg;
    const SearchScratch scratch(plan, scratch_dev);
    P.visited_tables = scratch.visited_tables;
    P.blob_global = scratch.blob_global;
    P.work_counter = work_counter_dev;
    P.nodes_out = nodes_out_dev;
    P.scores_out = scores_out_dev;
    P.counters = counters_dev;
    P.overflow = overflow_flags_dev;
    P.query_index = query_index_dev;
    P.blobA_floats = blob_floats(approx);
    P.pq_smem_m = plan.pq_smem_m;
    P.smemA_floats = search_smemA_floats(approx, plan.pq_smem_m);
    P.blobR_floats = rerank ? blob_floats(*rerank) : 0;
    P.vis_slots_log = plan.vis_slots_log;
    P.vis_rlog = plan.vis_rlog;
    P.vis_idmask = plan.vis_idmask;
    // fp32: only a batch that does not fill the GPU (latency bound, L2 to spare) prefetches its rows. A full batch would keep up to
    // 9 CTAs x 28 rows x 3 KB per SM waiting in L2, twice an H100 SM's ~380 KB share: rows were evicted before their demand load and
    // read from DRAM twice (c2: 35.2 ms with the prefetch, 30.7 ms without)
    P.row_prefetch = (approx.kind == KIND_F32 && fills_gpu(plan, nq)) ? 0 : plan.row_prefetch;
    // the same batches, when they are DOT walks, use the row sketch where the caller passes one
    // (SEG walks: the caller decided for the whole call and prepared every segment's descriptor so, search_walk_descs included)
    if (!segments) search_walk_descs(P.g, P.approx, metric, search_uses_sketch(approx, metric, plan, nq));
    P.pq_rows = plan.pq_rows;
    {
        // on for the latency-bound walks (PQ / BQ: c3 12.0 -> 11.5 ms); off where HBM is already saturated and a wasted adjacency
        // line costs more than an early one saves (fp32 / NVQ: c2 13.8 vs 14.0 ms). JV_EARLY_PREFETCH=0|1 overrides.
        const char *ep = getenv("JV_EARLY_PREFETCH");
        // (a batch that does not fill the GPU is latency bound whatever the scorer: on as well)
        P.early_pf = ep ? atoi(ep) : ((approx.kind == KIND_PQ || approx.kind == KIND_BQ || !fills_gpu(plan, nq)) ? 1 : 0);
    }
    P.dbg = nullptr;
#ifdef JV_SEARCH_PROFILE
    static unsigned long long *dbg_dev = nullptr;
    if (!dbg_dev) cudaMalloc(&dbg_dev, 8 * sizeof(unsigned long long));
    cudaMemsetAsync(dbg_dev, 0, 8 * sizeof(unsigned long long), s);
    P.dbg = dbg_dev;
#endif
#ifdef JV_ROW_BOUND_STATS
    {
        const unsigned long long z[4] = {0, 0, 0, 0};
        cudaMemcpyToSymbolAsync(g_rbs_count, z, sizeof(z), 0, cudaMemcpyHostToDevice, s);
    }
#endif
    cudaError_t e = cudaMemsetAsync(work_counter_dev, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
#define CALL(K, M, B, V)                                                                                                            \
    do {                                                                                                                              \
        e = cudaFuncSetAttribute(graph_search_kernel<K, M, B, V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem_bytes); \
        if (e == cudaSuccess) graph_search_kernel<K, M, B, V><<<plan.ctas, SearchThreads<K>::value, plan.smem_bytes, s>>>(P);               \
    } while (0)
#define CALL_EDGE(B, V)                                                                                                                \
    do {                                                                                                                              \
        e = cudaFuncSetAttribute(graph_search_kernel<KIND_F32, JV_METRIC_DOT, B, V, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem_bytes); \
        if (e == cudaSuccess) graph_search_kernel<KIND_F32, JV_METRIC_DOT, B, V, true><<<plan.ctas, SearchThreads<KIND_F32>::value, plan.smem_bytes, s>>>(P); \
    } while (0)
    // a refine's walks, over fp32, PQ or BQ rows (no NVQ data set is refined); the edge records are off for them, with the same answers
#define CALL_EXCL(K, M, B, V)                                                                                                       \
    do {                                                                                                                              \
        e = cudaFuncSetAttribute(graph_search_kernel<K, M, B, V, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem_bytes); \
        if (e == cudaSuccess) graph_search_kernel<K, M, B, V, false, true><<<plan.ctas, SearchThreads<K>::value, plan.smem_bytes, s>>>(P); \
    } while (0)
#define CALL_SEG(K, M, B, V)                                                                                                        \
    do {                                                                                                                              \
        e = cudaFuncSetAttribute(graph_search_kernel<K, M, B, V, false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem_bytes); \
        if (e == cudaSuccess) graph_search_kernel<K, M, B, V, false, false, true><<<plan.ctas, SearchThreads<K>::value, plan.smem_bytes, s>>>(P); \
    } while (0)
#define CALL_EDGE_SEG(B, V)                                                                                                            \
    do {                                                                                                                              \
        e = cudaFuncSetAttribute(graph_search_kernel<KIND_F32, JV_METRIC_DOT, B, V, true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)plan.smem_bytes); \
        if (e == cudaSuccess) graph_search_kernel<KIND_F32, JV_METRIC_DOT, B, V, true, false, true><<<plan.ctas, SearchThreads<KIND_F32>::value, plan.smem_bytes, s>>>(P); \
    } while (0)
    if (segments) {
        if (P.exclude_ids) e = cudaErrorInvalidValue;
        else if (P.g.edge_rec) {
            if (plan.vis_slots_log != 0) {
                if (plan.pq_wide) CALL_EDGE_SEG(MINB_ROWS_WIDE, true);
                else CALL_EDGE_SEG(MINB_ROWS, true);
            } else if (plan.pq_wide) CALL_EDGE_SEG(MINB_ROWS_WIDE, false);
            else CALL_EDGE_SEG(MINB_ROWS, false);
        } else JV_SEARCH_DISPATCH(approx.kind, metric, plan.pq_wide != 0, plan.vis_slots_log != 0, CALL_SEG);
    } else if (P.exclude_ids) {
        P.g.edge_rec = nullptr;
        if (plan.vis_slots_log != 0) JV_SEARCH_DISPATCH_FPB_V(approx.kind, metric, plan.pq_wide != 0, true, CALL_EXCL, e = cudaErrorInvalidValue);
        else JV_SEARCH_DISPATCH_FPB_V(approx.kind, metric, plan.pq_wide != 0, false, CALL_EXCL, e = cudaErrorInvalidValue);
    } else if (P.g.edge_rec) {
        if (plan.vis_slots_log != 0) {
            if (plan.pq_wide) CALL_EDGE(MINB_ROWS_WIDE, true);
            else CALL_EDGE(MINB_ROWS, true);
        } else if (plan.pq_wide) CALL_EDGE(MINB_ROWS_WIDE, false);
        else CALL_EDGE(MINB_ROWS, false);
    } else JV_SEARCH_DISPATCH(approx.kind, metric, plan.pq_wide != 0, plan.vis_slots_log != 0, CALL);
#undef CALL_EDGE_SEG
#undef CALL_SEG
#undef CALL_EXCL
#undef CALL_EDGE
#undef CALL
    if (e != cudaSuccess) return e;
    g_launches++;
#ifdef JV_SEARCH_PROFILE
    {
        unsigned long long h[8];
        cudaStreamSynchronize(s);
        cudaMemcpy(h, P.dbg, sizeof(h), cudaMemcpyDeviceToHost);
        const double it = h[5] ? (double)h[5] : 1.0, nqd = (double)nq;
        fprintf(stderr, "[search profile] kind=%d nq=%d iterations/q=%.1f scored/it=%.1f cycles/it: gather=%.0f score=%.0f merge=%.0f | per query: prepare+clear=%.0f rerank+out=%.0f total=%.0f\n",
                approx.kind, nq, it / nqd, (double)h[6] / it, (double)h[1] / it, (double)h[2] / it, (double)h[3] / it, (double)h[0] / nqd, (double)h[4] / nqd, (double)h[7] / nqd);
    }
#endif
#ifdef JV_ROW_BOUND_STATS
    // one record per launch appended to $JV_ROW_BOUND_STATS_OUT: u64 scored, dropped, drop samples, row samples; then the drop
    // samples (16 B each), then the row samples (24 B each)
    if (const char *out = getenv("JV_ROW_BOUND_STATS_OUT")) {
        unsigned long long c[4];
        cudaStreamSynchronize(s);
        cudaMemcpyFromSymbol(c, g_rbs_count, sizeof(c));
        if (c[2] > (unsigned long long)RBS_CAP) c[2] = RBS_CAP;
        if (c[3] > (unsigned long long)RBS_CAP) c[3] = RBS_CAP;
        RbsSample *h = (RbsSample *)malloc(sizeof(RbsSample) * (c[2] ? c[2] : 1));
        RbsRow *hr = (RbsRow *)malloc(sizeof(RbsRow) * (c[3] ? c[3] : 1));
        cudaMemcpyFromSymbol(h, g_rbs_sample, sizeof(RbsSample) * c[2]);
        cudaMemcpyFromSymbol(hr, g_rbs_row, sizeof(RbsRow) * c[3]);
        if (FILE *f = fopen(out, "ab")) {
            fwrite(c, sizeof(c), 1, f);
            fwrite(h, sizeof(RbsSample), c[2], f);
            fwrite(hr, sizeof(RbsRow), c[3], f);
            fclose(f);
        }
        free(h);
        free(hr);
    }
#endif
    return cudaGetLastError();
}

}  // namespace jv
