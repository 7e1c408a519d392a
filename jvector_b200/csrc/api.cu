// api.cu — the C ABI of include/jvector_b200.h, batched GPU group: handle management, host<->HBM staging, launches.
// No CPU fallback lives here: without an sm_90 device every entry point returns JV_ERR_NO_DEVICE.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <memory>
#include <mutex>
#include <thread>
#include <string>
#include <vector>

#include "../../include/jvector_b200.h"
#include "host_mem.h"
#include "kernels.h"

using namespace jv;

namespace {

thread_local std::string t_err;
std::mutex g_mu;
constexpr int MAX_DEVICES = 16;
// One process may drive several GPUs (the reference host is one JVM, all parallelism is threads: base:vector/
// VectorizationProvider.java:79-177, base:graph/GraphIndexBuilder.java:440-444): every handle remembers the device it lives on,
// every caller thread owns one context (stream + staging buffers) per device.
unsigned g_mask = 0;                 // devices bound by jv_gpu_init / jv_gpu_init_mask
int g_default_device = -1;           // first device bound
int g_sm_counts[MAX_DEVICES] = {0};
thread_local int t_device = -1;      // device new data sets / graphs of this thread are created on (jv_gpu_set_device); -1 = default
thread_local int t_active = 0;       // device of the call in progress

int fail(int code, const std::string &msg)
{
    t_err = msg;
    return code;
}
int cuda_fail(cudaError_t e, const char *what)
{
    t_err = std::string(what) + ": " + cudaGetErrorString(e);
    return e == cudaErrorMemoryAllocation ? JV_ERR_OOM : JV_ERR_CUDA;
}
#define CK(x, what)                                      \
    do {                                                 \
        cudaError_t e_ = (x);                            \
        if (e_ != cudaSuccess) return cuda_fail(e_, what); \
    } while (0)
// enter a call that creates something: the thread's target device
#define NEED_INIT()                                                                            \
    do {                                                                                       \
        const int d0_ = t_device >= 0 ? t_device : g_default_device;                           \
        if (d0_ < 0) return fail(JV_ERR_NO_DEVICE, "jv_gpu_init() has not succeeded");         \
        t_active = d0_;                                                                        \
        cudaError_t e0_ = cudaSetDevice(d0_);                                                  \
        if (e0_ != cudaSuccess) return cuda_fail(e0_, "cudaSetDevice");                        \
    } while (0)
// enter a call on an existing handle: the handle's device
#define ON_DEVICE_OF(h)                                                                        \
    do {                                                                                       \
        if (g_default_device < 0) return fail(JV_ERR_NO_DEVICE, "jv_gpu_init() has not succeeded"); \
        if (!(h)) return fail(JV_ERR_INVALID, "null handle");                                  \
        t_active = (h)->device;                                                                \
        cudaError_t e0_ = cudaSetDevice(t_active);                                             \
        if (e0_ != cudaSuccess) return cuda_fail(e0_, "cudaSetDevice");                        \
    } while (0)
#define g_sm_count (g_sm_counts[t_active])

// per-thread, per-device stream + growable staging buffers (callers are ForkJoinPool workers: no global locks on the score
// path); released when the thread exits. Each buffer has one role. A buffer whose contents outlive the call that filled it (the
// async top-k scratch, the copy stream's watermark) is used by nothing else.
struct ThreadCtx {
    int device = -1;
    cudaStream_t stream = nullptr;
    DeviceBuffer input;         // host queries / rows / points of the call
    DeviceBuffer aux;           // small per-call inputs: ids, offsets, centroids, codebooks, sub-vector layouts
    DeviceBuffer blobs;         // prepared queries
    DeviceBuffer output;        // what the call downloads: scores, keys, codes, assignments, search nodes + scores
    DeviceBuffer topk_scratch;  // generic top-k: the launcher's scratch
    DeviceBuffer bq_scratch;    // synchronous BQ top-k: the launcher's scratch + status word
    DeviceBuffer flag;          // synchronous top-k: overflow flag / unresolved count, read back before the call returns
    DeviceBuffer bq_async;      // jv_topk_bruteforce_device_async: still read on the caller's stream after the call returns
    DeviceBuffer search_scratch, search_aux;  // the search kernel's scratch; its counters and per-query overflow codes
    DeviceBuffer accept_bits;   // host-pointer searches: the uploaded acceptOrds bitsets
    DeviceBuffer accept_lists;  // filtered top-k: accepted counts, accepted-row lists, the sampled tier's query list
    DeviceBuffer rerank;        // exhaustive search: candidate keys, the reranker's prepared queries, taken ids, exact scores
    DeviceBuffer watermark;     // host-pointer searches: the arrival watermark the copy stream writes
    DeviceBuffer segments;      // multi-segment search: queries, bitsets, segment descriptors, per-segment answers and counters, merged answers
    StreamTimer timer;
    // host-pointer searches: a second stream carries the query chunks while the search kernel already runs (arrival watermark)
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_copy = nullptr;
    PinnedBuffer marks;  // the watermark values the copy stream writes behind each chunk
    static constexpr int MARKS = 16;
    int init_copy()
    {
        if (copy_stream) return JV_OK;
        CK(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking), "cudaStreamCreate(copy)");
        CK(cudaEventCreateWithFlags(&ev_copy, cudaEventDisableTiming), "cudaEventCreate(copy)");
        CK(marks.grow(MARKS * sizeof(int)), "cudaHostAlloc(marks)");
        return JV_OK;
    }
    int init()
    {
        if (stream) return JV_OK;
        device = t_active;
        CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking), "cudaStreamCreate");
        return JV_OK;
    }
    template <typename F>
    void each_owner(F f)
    {
        for (DeviceBuffer *b : {&input, &aux, &blobs, &output, &topk_scratch, &bq_scratch, &flag, &bq_async, &search_scratch, &search_aux, &accept_bits, &accept_lists, &rerank, &watermark, &segments})
            f(*b);
        f(marks);
        f(timer);
    }
    ~ThreadCtx()
    {
        if (!stream) return;
        int cur = -1;
        if (cudaGetDevice(&cur) != cudaSuccess || cudaSetDevice(device) != cudaSuccess) {
            each_owner([](auto &o) { o.abandon(); });  // runtime already torn down at process exit: nothing left to free
            return;
        }
        cudaStreamSynchronize(stream);
        if (copy_stream) cudaStreamSynchronize(copy_stream);
        each_owner([](auto &o) { o.reset(); });
        cudaStreamDestroy(stream);
        if (copy_stream) {
            cudaStreamDestroy(copy_stream);
            cudaEventDestroy(ev_copy);
        }
        if (cur >= 0) cudaSetDevice(cur);
    }
};
thread_local ThreadCtx t_ctxs[MAX_DEVICES];
thread_local ThreadCtx *t_ctx_override = nullptr;  // worker threads of the multi-device entry points run on the shard's own context
#define t_ctx (*(t_ctx_override ? t_ctx_override : &t_ctxs[t_active]))
thread_local BuildStats t_build_stats = {0, 0, 0, 0, 0};

int round4(int v) { return (v + 3) & ~3; }

int grow(DeviceBuffer &b, size_t bytes)
{
    CK(b.grow(bytes), "cudaMalloc(staging)");
    return JV_OK;
}

// the sub-vector split of `dim` into M parts (base:quantization/ProductQuantization.java:535-550; NVQuantization.java:236-251
// uses the same), enqueued on `s` into layout_dev: sizes [M], then offsets [M]
cudaError_t upload_layout(int dim, int M, int *layout_dev, cudaStream_t s)
{
    std::vector<int> h(2 * (size_t)M);
    int base = dim / M, rem = dim % M, off = 0;
    for (int m = 0; m < M; m++) {
        h[m] = base + (m < rem ? 1 : 0);
        h[M + m] = off;
        off += h[m];
    }
    return cudaMemcpyAsync(layout_dev, h.data(), h.size() * 4, cudaMemcpyHostToDevice, s);
}

// n host rows of row_bytes into device rows of stride_bytes, the padding zeroed
cudaError_t upload_padded(void *dev, const void *host, size_t n, size_t row_bytes, size_t stride_bytes)
{
    if (stride_bytes == row_bytes) return cudaMemcpy(dev, host, n * row_bytes, cudaMemcpyHostToDevice);
    cudaError_t e = cudaMemset(dev, 0, n * stride_bytes);
    if (e == cudaSuccess) e = cudaMemcpy2D(dev, stride_bytes, host, row_bytes, row_bytes, n, cudaMemcpyHostToDevice);
    return e;
}

}  // namespace

struct jv_dataset_s {
    int device = t_active;
    bool borrowed_rows = false;  // jv_dataset_adopt_f32_device: rows belong to the caller
    DataDesc d;
    std::vector<DeviceBuffer> allocs;
    size_t bytes = 0;
    // fp32 row sketch (row_sketch_kernel): built by the first search that can use it (search_device), freed with the data set.
    // Not part of `d`: only the search kernel's fp32 DOT walks read it, the builder and the batch scorers never see it
    DeviceBuffer sketch, sketch_meta;
    bool sketch_failed = false;  // the allocation failed once: walk without it from then on
    // low-rank rows (lowrank_rows_kernel) and their basis, built with the sketch (ensure_lowrank); lr_id names this build for the
    // graphs' edge records (0: none). lr_off: the data set does not get them (too wide, too far from a rank-LR_K subspace, or out of memory)
    DeviceBuffer lr_basis, lr_rows;
    uint64_t lr_id = 0;
    bool lr_off = false;
    std::mutex sketch_mu;
    // PQ: guards the lazily built centroid-pair tables (d.pair_table, jv_dataset_pq_pair_table), whose allocation also grows
    // `allocs` and `bytes`: callers on several threads build each table once
    std::mutex pair_mu;
    // an empty data set of n rows of `kind` on the active device: every other field of `d` is zero
    jv_dataset_s(int kind, long long n, int dim)
    {
        memset(&d, 0, sizeof(DataDesc));
        d.kind = kind;
        d.dim = dim;
        d.n = n;
    }
    template <typename T>
    int alloc(T **p, size_t n)
    {
        CK(alloc_owned(allocs, *p, n ? n : 16), "cudaMalloc(dataset)");
        bytes += n;
        return JV_OK;
    }
    // the fp32 row layout (DataDesc::rows): every row zero padded to a multiple of 4 floats
    static int f32_stride(int dim) { return round4(dim); }
    // fp32 rows [n][f32_stride(dim)], d.rows pointing at them, for the caller to fill (padding included)
    int alloc_rows(float **rows)
    {
        d.stride = f32_stride(d.dim);
        const int rc = alloc(rows, (size_t)d.n * d.stride * sizeof(float));
        d.rows = *rows;
        return rc;
    }
};

struct jv_query_s {
    int device = 0;
    jv_dataset ds;
    int metric;
    DeviceBuffer blob;
};

// the upper levels of a graph, level l >= 1 at [l - 1]: its members (node ids), or their rows ([members][degree] node ids, -1 = empty)
using Levels = std::vector<std::vector<int32_t>>;

// Only create, set_levels and jv_graph_fuse_pq write `g`.
struct jv_graph_s {
    int device = t_active;
    GraphDesc g;
    DeviceBuffer fused;  // FusedPQ records
    DeviceBuffer adj0, upper_row, upper_adj, upper_off;
    Levels level_ids, level_adj;  // host copies of the upper levels
    std::vector<uint32_t> removed;  // ids taken out by jv_graph_remove_deleted (holes), bit (id & 31) of word (id >> 5); empty = none
    // edge records of the low-rank bound (launch_edge_records) for the data set whose lr_id is edge_rec_of; built by the first
    // sketched search over that data set, freed with the graph
    // (shared: a search holds its records until its kernels are done, so a concurrent search over another data set that replaces
    // them cannot free them under it)
    std::shared_ptr<DeviceBuffer> edge_rec;
    uint64_t edge_rec_of = 0;
    std::mutex edge_mu;
    // a graph of n nodes with `degree` neighbour slots each on the active device, into `out`: adj0 allocated for the caller to
    // fill, level 0 only and no entry until set_levels
    static int create(int32_t n, int degree, std::unique_ptr<jv_graph_s> &out)
    {
        std::unique_ptr<jv_graph_s> h(new jv_graph_s());
        memset(&h->g, 0, sizeof(GraphDesc));
        h->g.n = n; h->g.degree = degree; h->g.levels = 1; h->g.entry_level = 0; h->g.entry_node = -1;
        CK(h->adj0.alloc((size_t)n * degree * 4), "cudaMalloc(adjacency)");
        h->g.adj0 = h->adj0.get<int32_t>();
        out = std::move(h);
        return JV_OK;
    }
    int set_levels(Levels ids, Levels adj, int32_t entry);
};

struct jv_multi_s {
    int kind = 0, dim = 0;
    int64_t n = 0;
    std::vector<int> devices;
    std::vector<int64_t> lo;        // shard i holds rows [lo[i], lo[i + 1])
    std::vector<jv_dataset> shards;
    std::vector<ThreadCtx *> ctx;   // one persistent context per shard (worker threads come and go)
    DeviceBuffer gathered;          // on the first shard's device: the shards' top-k keys [parts][nq][k], then the merged [nq][k]
};

static void shard_ranges(int64_t n, int parts, std::vector<int64_t> &lo)
{
    lo.resize(parts + 1);
    const int64_t base = n / parts, rem = n % parts;
    for (int i = 0; i <= parts; i++) lo[i] = i * base + std::min<int64_t>(i, rem);
}

static int multi_devices(std::vector<int> &devs)
{
    devs.clear();
    for (int d = 0; d < MAX_DEVICES; d++)
        if (g_mask & (1u << d)) devs.push_back(d);
    if (devs.empty()) return fail(JV_ERR_NO_DEVICE, "jv_gpu_init_mask() has not succeeded");
    return JV_OK;
}

template <typename F>
static int multi_register(jv_multi m, F reg)
{
    int rc = multi_devices(m->devices);
    if (rc) return rc;
    const int parts = (int)std::min<int64_t>((int64_t)m->devices.size(), m->n);
    m->devices.resize(parts);
    shard_ranges(m->n, parts, m->lo);
    const int saved = t_device;
    for (int i = 0; i < parts; i++) {
        t_device = m->devices[i];
        jv_dataset ds = nullptr;
        rc = reg(i, m->lo[i], m->lo[i + 1] - m->lo[i], &ds);
        if (rc) break;
        m->shards.push_back(ds);
        m->ctx.push_back(new ThreadCtx());
    }
    t_device = saved;
    return rc;
}

extern "C" {

int jv_gpu_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

static int bind_device(int device)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) return fail(JV_ERR_NO_DEVICE, std::string("no CUDA device: ") + cudaGetErrorString(e));
    if (device < 0 || device >= n || device >= MAX_DEVICES) return fail(JV_ERR_INVALID, "device index out of range");
    cudaDeviceProp p;
    CK(cudaGetDeviceProperties(&p, device), "cudaGetDeviceProperties");
    if (p.major != 9 || p.minor != 0) return fail(JV_ERR_NO_DEVICE, "device is not sm_90 (this library carries sm_90a code only)");
    CK(cudaSetDevice(device), "cudaSetDevice");
    g_sm_counts[device] = p.multiProcessorCount;
    g_mask |= 1u << device;
    if (g_default_device < 0) g_default_device = device;
    return JV_OK;
}

int jv_gpu_init(int device)
{
    std::lock_guard<std::mutex> lk(g_mu);
    int rc = bind_device(device);
    if (rc) return rc;
    t_device = device;  // the calling thread creates its data sets here; handles remember their device, so a later
    return JV_OK;       // jv_gpu_init(other) never invalidates them
}

int jv_gpu_init_mask(uint32_t device_mask)
{
    std::lock_guard<std::mutex> lk(g_mu);
    if (device_mask == 0) return fail(JV_ERR_INVALID, "gpu_init_mask: empty mask");
    for (int d = 0; d < MAX_DEVICES; d++)
        if (device_mask & (1u << d)) {
            int rc = bind_device(d);
            if (rc) return rc;
        }
    // peer access between every pair (NVLink / NVSwitch): the multi-device entry points copy shard results device to device
    for (int a = 0; a < MAX_DEVICES; a++)
        for (int b = 0; b < MAX_DEVICES; b++)
            if (a != b && (g_mask & (1u << a)) && (g_mask & (1u << b))) {
                int can = 0;
                if (cudaDeviceCanAccessPeer(&can, a, b) == cudaSuccess && can) {
                    cudaSetDevice(a);
                    cudaError_t e = cudaDeviceEnablePeerAccess(b, 0);
                    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return cuda_fail(e, "cudaDeviceEnablePeerAccess");
                    cudaGetLastError();
                }
            }
    cudaSetDevice(g_default_device);
    return JV_OK;
}

int jv_gpu_set_device(int device)
{
    if (device < 0 || device >= MAX_DEVICES || !(g_mask & (1u << device))) return fail(JV_ERR_INVALID, "gpu_set_device: device was not bound by jv_gpu_init / jv_gpu_init_mask");
    t_device = device;
    return JV_OK;
}

uint32_t jv_gpu_bound_mask(void) { return g_mask; }

const char *jv_last_error(void) { return t_err.c_str(); }
const char *jv_version(void) { return "jvector-b200 0.1 (sm_90a)"; }
int jv_gpu_sm_count(void) { return g_default_device >= 0 ? g_sm_counts[t_device >= 0 ? t_device : g_default_device] : 0; }
int64_t jv_kernel_launch_count(void) { return (int64_t)g_launches.load(); }

// ------------------------------------------------------------------------------------------------ data sets
int jv_dataset_register_f32(const float *rows, int64_t n, int dim, jv_dataset *out)
{
    NEED_INIT();
    if (!rows || !out || n <= 0 || dim <= 0 || n > 0x7fffffffLL) return fail(JV_ERR_INVALID, "register_f32: bad arguments");
    std::unique_ptr<jv_dataset_s> ds(new jv_dataset_s(KIND_F32, n, dim));
    float *dev = nullptr;
    int rc = ds->alloc_rows(&dev);
    if (rc) return rc;
    CK(upload_padded(dev, rows, (size_t)n, (size_t)dim * 4, (size_t)ds->d.stride * 4), "upload rows");
    *out = ds.release();
    return JV_OK;
}

// a new PQ data set of n rows on the current device: code rows [n][code_stride] allocated for the caller to fill, codebooks,
// centroid (host, or NULL) and the sub-space layout uploaded and the self magnitudes computed on `s`
static int pq_dataset(int64_t n, int dim, int M, int k, const float *codebooks, const float *centroid, cudaStream_t s,
                      std::unique_ptr<jv_dataset_s> &ds, uint8_t **codes_dev)
{
    ds.reset(new jv_dataset_s(KIND_PQ, n, dim));
    DataDesc &d = ds->d;
    d.M = M; d.k = k; d.code_stride = round4(M);
    float *dcb = nullptr, *dcen = nullptr, *dmag = nullptr;
    int *dlay = nullptr;
    int rc;
    if ((rc = ds->alloc(codes_dev, (size_t)n * d.code_stride)) || (rc = ds->alloc(&dcb, (size_t)k * dim * 4)) || (rc = ds->alloc(&dlay, (size_t)M * 8)) ||
        (rc = ds->alloc(&dmag, (size_t)M * k * 4)) || (centroid && (rc = ds->alloc(&dcen, (size_t)dim * 4))))
        return rc;
    cudaError_t e = cudaMemcpyAsync(dcb, codebooks, (size_t)k * dim * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = upload_layout(dim, M, dlay, s);
    if (e == cudaSuccess && centroid) e = cudaMemcpyAsync(dcen, centroid, (size_t)dim * 4, cudaMemcpyHostToDevice, s);
    CK(e, "upload pq");
    d.codes = *codes_dev; d.codebooks = dcb; d.sub_sizes = dlay; d.sub_offsets = dlay + M; d.centroid = dcen; d.mag = dmag;
    CK(launch_pq_self_magnitudes(d, dmag, s), "pq self magnitudes");
    return JV_OK;
}

int jv_dataset_register_pq(const uint8_t *codes, int64_t n, int dim, int M, int k, const float *codebooks, const float *centroid, jv_dataset *out)
{
    NEED_INIT();
    if (!codes || !codebooks || !out || n <= 0 || dim <= 0 || M <= 0 || M > dim || k <= 0 || k > 256 || n > 0x7fffffffLL)
        return fail(JV_ERR_INVALID, "register_pq: bad arguments");
    std::unique_ptr<jv_dataset_s> ds;
    uint8_t *dcodes = nullptr;
    int rc = pq_dataset(n, dim, M, k, codebooks, centroid, 0, ds, &dcodes);
    cudaError_t e = rc ? cudaSuccess : upload_padded(dcodes, codes, (size_t)n, (size_t)M, (size_t)ds->d.code_stride);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (rc) return rc;
    CK(e, "upload pq");
    *out = ds.release();
    return JV_OK;
}

int jv_dataset_pq_download(jv_dataset pq, uint8_t *codes_out, float *codebooks_out, float *centroid_out)
{
    ON_DEVICE_OF(pq);
    if (pq->d.kind != KIND_PQ) return fail(JV_ERR_INVALID, "dataset_pq_download: not a PQ data set");
    if (centroid_out && !pq->d.centroid) return fail(JV_ERR_INVALID, "dataset_pq_download: the data set has no centroid");
    const DataDesc &d = pq->d;
    cudaError_t e = cudaSuccess;
    if (codes_out) e = cudaMemcpy2D(codes_out, (size_t)d.M, d.codes, (size_t)d.code_stride, (size_t)d.M, (size_t)d.n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && codebooks_out) e = cudaMemcpy(codebooks_out, d.codebooks, (size_t)d.k * d.dim * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && centroid_out) e = cudaMemcpy(centroid_out, d.centroid, (size_t)d.dim * 4, cudaMemcpyDeviceToHost);
    CK(e, "D2H pq");
    return JV_OK;
}

int jv_dataset_register_bq(const uint64_t *words, int64_t n, int dim, jv_dataset *out)
{
    NEED_INIT();
    if (!words || !out || n <= 0 || dim <= 0 || n > 0x7fffffffLL) return fail(JV_ERR_INVALID, "register_bq: bad arguments");
    std::unique_ptr<jv_dataset_s> ds(new jv_dataset_s(KIND_BQ, n, dim));
    ds->d.W = (dim + 63) / 64;
    unsigned long long *dw = nullptr;
    int rc = ds->alloc(&dw, (size_t)n * ds->d.W * 8);
    if (rc) return rc;
    CK(cudaMemcpy(dw, words, (size_t)n * ds->d.W * 8, cudaMemcpyHostToDevice), "upload bq");
    ds->d.words = dw;
    *out = ds.release();
    return JV_OK;
}

// a new NVQ data set of n rows on the current device: bytes and params allocated for the caller to fill, the zero-padded mean
// and the sub-vector layout enqueued on `s`
static int nvq_dataset(int64_t n, int dim, int nsub, const float *mean, cudaStream_t s, std::unique_ptr<jv_dataset_s> &ds, uint8_t **bytes_dev,
                       float **params_dev)
{
    ds.reset(new jv_dataset_s(KIND_NVQ, n, dim));
    DataDesc &d = ds->d;
    d.nsub = nsub; d.stride = round4(dim); d.byte_stride = round4(dim);
    float *dm = nullptr;
    int *dlay = nullptr;
    int rc;
    if ((rc = ds->alloc(bytes_dev, (size_t)n * d.byte_stride)) || (rc = ds->alloc(params_dev, (size_t)n * nsub * 16)) ||
        (rc = ds->alloc(&dm, (size_t)d.stride * 4)) || (rc = ds->alloc(&dlay, (size_t)nsub * 8)))
        return rc;
    cudaError_t e = cudaMemsetAsync(dm, 0, (size_t)d.stride * 4, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(dm, mean, (size_t)dim * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = upload_layout(dim, nsub, dlay, s);
    CK(e, "upload nvq");
    d.bytes = *bytes_dev; d.params = *params_dev; d.mean = dm; d.sub_sizes = dlay; d.sub_offsets = dlay + nsub;
    return JV_OK;
}

int jv_dataset_register_nvq(const uint8_t *bytes, const float *params, int64_t n, int dim, int nsub, const float *mean, jv_dataset *out)
{
    NEED_INIT();
    if (!bytes || !params || !mean || !out || n <= 0 || dim <= 0 || nsub <= 0 || nsub > dim || n > 0x7fffffffLL)
        return fail(JV_ERR_INVALID, "register_nvq: bad arguments");
    std::unique_ptr<jv_dataset_s> ds;
    uint8_t *db;
    float *dp;
    int rc;
    if ((rc = t_ctx.init()) || (rc = nvq_dataset(n, dim, nsub, mean, t_ctx.stream, ds, &db, &dp))) return rc;
    cudaError_t e = upload_padded(db, bytes, (size_t)n, (size_t)dim, (size_t)ds->d.byte_stride);
    if (e == cudaSuccess) e = cudaMemcpy(dp, params, (size_t)n * nsub * 16, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaStreamSynchronize(t_ctx.stream);
    CK(e, "upload nvq");
    *out = ds.release();
    return JV_OK;
}

static int check_metric(const DataDesc &d, int metric);

int jv_dataset_pq_pair_table(jv_dataset pq, int metric)
{
    ON_DEVICE_OF(pq);
    if (pq->d.kind != KIND_PQ) return fail(JV_ERR_INVALID, "pq_pair_table: not a PQ data set");
    int rc = check_metric(pq->d, metric);
    if (rc) return rc;
    const int which = metric == JV_METRIC_EUCLIDEAN ? 0 : 1;  // cosine sums the dot-product table (ImmutablePQVectors.java:78-92)
    std::lock_guard<std::mutex> lk(pq->pair_mu);
    if (pq->d.pair_table[which]) return JV_OK;
    if ((rc = t_ctx.init())) return rc;
    float *t = nullptr;
    const size_t entries = (size_t)pq->d.M * ((size_t)pq->d.k * (pq->d.k + 1) / 2);
    if ((rc = pq->alloc((void **)&t, entries * 4))) return rc;
    CK(launch_pq_pair_table(pq->d, which == 0, t, t_ctx.stream), "pq_pair_table");
    CK(cudaStreamSynchronize(t_ctx.stream), "pq_pair_table");
    pq->d.pair_table[which] = t;
    return JV_OK;
}

int jv_dataset_pq_pair_table_download(jv_dataset pq, int metric, float *table_out)
{
    ON_DEVICE_OF(pq);
    const int which = metric == JV_METRIC_EUCLIDEAN ? 0 : 1;
    std::lock_guard<std::mutex> lk(pq->pair_mu);
    if (pq->d.kind != KIND_PQ || !pq->d.pair_table[which] || !table_out) return fail(JV_ERR_INVALID, "pq_pair_table_download: no table for this metric");
    const size_t entries = (size_t)pq->d.M * ((size_t)pq->d.k * (pq->d.k + 1) / 2);
    CK(cudaMemcpy(table_out, pq->d.pair_table[which], entries * 4, cudaMemcpyDeviceToHost), "D2H pair table");
    return JV_OK;
}

int jv_kmeans_assign_batch(const float *points, int64_t n, int dim, const float *centroids, int k, int32_t *assignments_out)
{
    NEED_INIT();
    if (!points || !centroids || !assignments_out || n <= 0 || dim <= 0 || k <= 0) return fail(JV_ERR_INVALID, "kmeans_assign: bad arguments");
    int rc;
    if ((rc = t_ctx.init()) || (rc = grow(t_ctx.input, (size_t)n * dim * 4)) || (rc = grow(t_ctx.output, (size_t)n * 4)) || (rc = grow(t_ctx.aux, (size_t)k * dim * 4)))
        return rc;
    cudaStream_t s = t_ctx.stream;
    float *dpoints = t_ctx.input.get<float>(), *dcen = t_ctx.aux.get<float>();
    int32_t *dassign = t_ctx.output.get<int32_t>();
    CK(cudaMemcpyAsync(dpoints, points, (size_t)n * dim * 4, cudaMemcpyHostToDevice, s), "H2D points");
    CK(cudaMemcpyAsync(dcen, centroids, (size_t)k * dim * 4, cudaMemcpyHostToDevice, s), "H2D centroids");
    CK(launch_kmeans_assign(dpoints, n, dim, dim, dcen, k, dassign, s), "kmeans_assign");
    CK(cudaMemcpyAsync(assignments_out, dassign, (size_t)n * 4, cudaMemcpyDeviceToHost, s), "D2H assignments");
    CK(cudaStreamSynchronize(s), "sync");
    return JV_OK;
}

int jv_dataset_adopt_f32_device(const float *rows_device, int64_t n, int dim, int row_stride, jv_dataset *out)
{
    NEED_INIT();
    if (!rows_device || !out || n <= 0 || dim <= 0 || n > 0x7fffffffLL || row_stride < dim || (row_stride & 3) || ((uintptr_t)rows_device & 15))
        return fail(JV_ERR_INVALID, "adopt_f32_device: need 16-byte aligned rows and a row stride that is a multiple of 4 floats >= dim");
    if (row_stride != jv_dataset_s::f32_stride(dim)) return fail(JV_ERR_INVALID, "adopt_f32_device: row_stride must equal dim rounded up to 4 (padding floats must be zero)");
    jv_dataset ds = new jv_dataset_s(KIND_F32, n, dim);
    ds->borrowed_rows = true;
    ds->d.stride = row_stride;
    ds->d.rows = rows_device;
    *out = ds;
    return JV_OK;
}

int jv_dataset_device(jv_dataset ds) { return ds ? ds->device : -1; }

int jv_dataset_free(jv_dataset ds)
{
    if (!ds) return JV_OK;
    cudaSetDevice(ds->device);
    cudaDeviceSynchronize();
    delete ds;
    return JV_OK;
}
int64_t jv_dataset_size(jv_dataset ds) { return ds ? ds->d.n : 0; }
int jv_dataset_dim(jv_dataset ds) { return ds ? ds->d.dim : 0; }
int64_t jv_dataset_device_bytes(jv_dataset ds) { return ds ? (int64_t)ds->bytes : 0; }

// ------------------------------------------------------------------------------------------------ one query
static int check_metric(const DataDesc &d, int metric)
{
    if (metric < 0 || metric > 2) return fail(JV_ERR_INVALID, "unknown similarity function");
    (void)d;
    return JV_OK;
}

int jv_query_begin(jv_dataset ds, const float *q, int metric, jv_query *out)
{
    ON_DEVICE_OF(ds);
    if (!ds || !q || !out) return fail(JV_ERR_INVALID, "query_begin: null argument");
    int rc = check_metric(ds->d, metric);
    if (rc) return rc;
    if ((rc = t_ctx.init())) return rc;
    std::unique_ptr<jv_query_s> h(new jv_query_s());
    h->ds = ds;
    h->device = ds->device;
    h->metric = metric;
    CK(h->blob.alloc((size_t)blob_floats(ds->d) * 4), "cudaMalloc(query)");
    if ((rc = grow(t_ctx.input, (size_t)ds->d.dim * 4))) return rc;
    cudaStream_t s = t_ctx.stream;
    cudaError_t e = cudaMemcpyAsync(t_ctx.input.get(), q, (size_t)ds->d.dim * 4, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = launch_prepare(ds->d, metric, t_ctx.input.get<float>(), 1, h->blob.get<float>(), s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    CK(e, "prepare query");
    *out = h.release();
    return JV_OK;
}

int jv_score_batch(jv_query q, const int32_t *ids, int n, float *scores_out)
{
    ON_DEVICE_OF(q);
    if (!q || (n > 0 && (!ids || !scores_out)) || n < 0) return fail(JV_ERR_INVALID, "score_batch: bad arguments");
    if (n == 0) return JV_OK;
    int rc;
    if ((rc = t_ctx.init()) || (rc = grow(t_ctx.aux, (size_t)n * 4)) || (rc = grow(t_ctx.output, (size_t)n * 4))) return rc;
    cudaStream_t s = t_ctx.stream;
    int32_t *dids = t_ctx.aux.get<int32_t>();
    float *dscores = t_ctx.output.get<float>();
    CK(cudaMemcpyAsync(dids, ids, (size_t)n * 4, cudaMemcpyHostToDevice, s), "H2D ids");
    CK(launch_score_ragged(q->ds->d, q->metric, q->blob.get<float>(), 1, dids, nullptr, n, n, dscores, s), "score_ragged");
    CK(cudaMemcpyAsync(scores_out, dscores, (size_t)n * 4, cudaMemcpyDeviceToHost, s), "D2H scores");
    CK(cudaStreamSynchronize(s), "sync");
    return JV_OK;
}

int jv_query_get_lut(jv_query q, float *lut_out)
{
    ON_DEVICE_OF(q);
    if (!q || !lut_out || q->ds->d.kind != KIND_PQ) return fail(JV_ERR_INVALID, "get_lut: not a PQ query");
    CK(cudaMemcpy(lut_out, q->blob.get(), (size_t)q->ds->d.M * q->ds->d.k * 4, cudaMemcpyDeviceToHost), "D2H lut");
    return JV_OK;
}

int jv_query_end(jv_query q)
{
    if (!q) return JV_OK;
    cudaSetDevice(q->device);
    delete q;
    return JV_OK;
}

int jv_score_multi(jv_dataset ds, int metric, const float *queries, int nq, const int32_t *ids, const int32_t *offsets, float *scores_out)
{
    ON_DEVICE_OF(ds);
    if (!ds || !queries || !ids || !offsets || !scores_out || nq <= 0) return fail(JV_ERR_INVALID, "score_multi: bad arguments");
    if (nq > 65535) return fail(JV_ERR_INVALID, "score_multi: at most 65535 queries per call");
    int rc = check_metric(ds->d, metric);
    if (rc) return rc;
    const int total = offsets[nq];
    int maxc = 0;
    for (int i = 0; i < nq; i++) {
        if (offsets[i + 1] < offsets[i]) return fail(JV_ERR_INVALID, "score_multi: offsets not monotone");
        maxc = std::max(maxc, offsets[i + 1] - offsets[i]);
    }
    if (total == 0) return JV_OK;
    const size_t bf = (size_t)blob_floats(ds->d);
    int32_t *dids, *doff;
    auto carve = [&](void *base) {
        Carver c(base);
        dids = c.take<int32_t>(total);
        doff = c.take<int32_t>(nq + 1);
        return c.bytes;
    };
    if ((rc = t_ctx.init()) || (rc = grow(t_ctx.input, (size_t)nq * ds->d.dim * 4)) || (rc = grow(t_ctx.aux, carve(nullptr))) ||
        (rc = grow(t_ctx.output, (size_t)total * 4)) || (rc = grow(t_ctx.blobs, (size_t)nq * bf * 4)))
        return rc;
    carve(t_ctx.aux.get());
    cudaStream_t s = t_ctx.stream;
    float *dq = t_ctx.input.get<float>(), *dblobs = t_ctx.blobs.get<float>(), *dscores = t_ctx.output.get<float>();
    CK(cudaMemcpyAsync(dq, queries, (size_t)nq * ds->d.dim * 4, cudaMemcpyHostToDevice, s), "H2D queries");
    CK(cudaMemcpyAsync(dids, ids, (size_t)total * 4, cudaMemcpyHostToDevice, s), "H2D ids");
    CK(cudaMemcpyAsync(doff, offsets, (size_t)(nq + 1) * 4, cudaMemcpyHostToDevice, s), "H2D offsets");
    CK(launch_prepare(ds->d, metric, dq, nq, dblobs, s), "prepare");
    CK(launch_score_ragged(ds->d, metric, dblobs, nq, dids, doff, 0, maxc, dscores, s), "score_ragged");
    CK(cudaMemcpyAsync(scores_out, dscores, (size_t)total * 4, cudaMemcpyDeviceToHost, s), "D2H scores");
    CK(cudaStreamSynchronize(s), "sync");
    return JV_OK;
}

int jv_score_pairs(jv_dataset ds, int metric, const int32_t *a, const int32_t *b, int n, float *scores_out)
{
    ON_DEVICE_OF(ds);
    if (!ds || n < 0 || (n > 0 && (!a || !b || !scores_out))) return fail(JV_ERR_INVALID, "score_pairs: bad arguments");
    if (ds->d.kind == KIND_NVQ) return fail(JV_ERR_UNSUPPORTED, "score_pairs: NVQ has no node-vs-node scorer in the reference");
    if (n == 0) return JV_OK;
    for (int i = 0; i < n; i++)
        if (a[i] < 0 || a[i] >= ds->d.n || b[i] < 0 || b[i] >= ds->d.n) return fail(JV_ERR_INVALID, "score_pairs: node id out of range");
    int rc = check_metric(ds->d, metric);
    if (rc) return rc;
    if ((rc = t_ctx.init()) || (rc = grow(t_ctx.aux, (size_t)n * 8)) || (rc = grow(t_ctx.output, (size_t)n * 4))) return rc;
    cudaStream_t s = t_ctx.stream;
    int32_t *da = t_ctx.aux.get<int32_t>(), *db = da + n;
    float *dscores = t_ctx.output.get<float>();
    CK(cudaMemcpyAsync(da, a, (size_t)n * 4, cudaMemcpyHostToDevice, s), "H2D a");
    CK(cudaMemcpyAsync(db, b, (size_t)n * 4, cudaMemcpyHostToDevice, s), "H2D b");
    CK(launch_score_pairs(ds->d, metric, da, db, n, dscores, s), "score_pairs");
    CK(cudaMemcpyAsync(scores_out, dscores, (size_t)n * 4, cudaMemcpyDeviceToHost, s), "D2H scores");
    CK(cudaStreamSynchronize(s), "sync");
    return JV_OK;
}

// generic exhaustive top-k (any storage kind): sample -> key threshold -> filtered pass -> per-query selection, with a host
// decision between passes (kernels_batch.cu). Queries and keys in HBM; id_base is added to every node id.
static int topk_device_generic(jv_dataset ds, int metric, const float *queries_dev, int nq, int k, int64_t id_base, long long *keys_dev)
{
    cudaStream_t s = t_ctx.stream;
    int rc;
    const size_t bf = (size_t)blob_floats(ds->d);
    const int chunk_max = (int)std::max<size_t>(1, std::min<size_t>(4096, ((size_t)512 << 20) / (bf * 4)));
    for (int q0 = 0; q0 < nq; q0 += chunk_max) {
        const int cq = std::min(chunk_max, nq - q0);
        if ((rc = grow(t_ctx.blobs, (size_t)cq * bf * 4)) || (rc = grow(t_ctx.topk_scratch, topk_scratch_bytes(ds->d, cq, k))) || (rc = grow(t_ctx.flag, 64)))
            return rc;
        int *dflag = t_ctx.flag.get<int>();
        float *dblobs = t_ctx.blobs.get<float>();
        CK(cudaMemsetAsync(dflag, 0, sizeof(int), s), "memset flag");
        CK(launch_prepare(ds->d, metric, queries_dev + (size_t)q0 * ds->d.dim, cq, dblobs, s), "prepare");
        CK(launch_topk_bruteforce(ds->d, metric, dblobs, cq, k, t_ctx.topk_scratch.get(), keys_dev + (size_t)q0 * k, dflag, s), "topk");
        if (id_base) CK(launch_key_rebase(keys_dev + (size_t)q0 * k, (long long)cq * k, (long long)id_base, s), "rebase");
        int flag = 0;
        CK(cudaMemcpyAsync(&flag, dflag, sizeof(int), cudaMemcpyDeviceToHost, s), "D2H flag");
        CK(cudaStreamSynchronize(s), "sync");
        if (flag) return fail(JV_ERR_OVERFLOW, "topk_bruteforce: candidate buffer overflow (adversarial score distribution)");
    }
    return JV_OK;
}

constexpr int IMMA_QUERY_CHUNK = 4096;  // queries per bq_imma launch sequence (bounds the capture buffers: 64 KB per query)

// BQ: the tensor-core contraction (bq_imma.cu), enqueued on `s` without any host synchronisation. status_dev receives the number of
// queries the integer-threshold path left unresolved (0 in the normal case). `buf` is in use until `s` has passed this work.
static int topk_bq_imma_enqueue(jv_dataset ds, const float *queries_dev, int nq, int k, int64_t id_base, long long *keys_dev, int *status_dev,
                                DeviceBuffer &buf, cudaStream_t s)
{
    int rc;
    const int chunk = std::min(nq, IMMA_QUERY_CHUNK);
    // the launcher's scratch, then the status word of the chunks after the first (carved over nullptr: the buffer's size)
    void *scratch;
    int *tmp;
    auto carve = [&](void *base) {
        Carver c(base);
        scratch = c.take<char>(bq_imma_scratch_bytes(ds->d.n, chunk, ds->d.W));
        tmp = c.take<int>(1);
        return c.bytes;
    };
    if ((rc = grow(buf, carve(nullptr)))) return rc;
    carve(buf.get());
    for (int q0 = 0; q0 < nq; q0 += chunk) {
        const int cq = std::min(chunk, nq - q0);
        // one status word per call: chunks after the first accumulate through a scratch word
        int *st = q0 == 0 ? status_dev : tmp;
        CK(launch_bq_topk_imma(ds->d, queries_dev + (size_t)q0 * ds->d.dim, cq, k, (long long)id_base, scratch, keys_dev + (size_t)q0 * k, st, g_sm_count, s), "bq_topk_imma");
        if (q0 > 0) CK(launch_add_int(status_dev, tmp, s), "status");
    }
    return JV_OK;
}

static int topk_device(jv_dataset ds, int metric, const float *queries_dev, int nq, int k, int64_t id_base, long long *keys_dev)
{
    const char *force = getenv("JV_BQ_BRUTEFORCE");  // "popc": keep the round-1 popcount kernels (A/B timing, fallback tests)
    if (bq_imma_supported(ds->d, k) && !(force && force[0] == 'p')) {
        int rc;
        if ((rc = grow(t_ctx.flag, 64))) return rc;
        int *dflag = t_ctx.flag.get<int>();
        if ((rc = topk_bq_imma_enqueue(ds, queries_dev, nq, k, id_base, keys_dev, dflag, t_ctx.bq_scratch, t_ctx.stream))) return rc;
        int unresolved = 0;
        CK(cudaMemcpyAsync(&unresolved, dflag, sizeof(int), cudaMemcpyDeviceToHost, t_ctx.stream), "D2H status");
        CK(cudaStreamSynchronize(t_ctx.stream), "sync");
        if (unresolved == 0) return JV_OK;
        // a Hamming bin wider than the capture buffer (very low dimension, or adversarial duplicates): the key-threshold path decides
    }
    return topk_device_generic(ds, metric, queries_dev, nq, k, id_base, keys_dev);
}

int jv_topk_bruteforce(jv_dataset ds, int metric, const float *queries, int nq, int k, int64_t *keys_out)
{
    ON_DEVICE_OF(ds);
    if (!ds || !queries || !keys_out || nq <= 0 || k <= 0) return fail(JV_ERR_INVALID, "topk_bruteforce: bad arguments");
    if (k > 2048) return fail(JV_ERR_INVALID, "topk_bruteforce: k <= 2048");
    int rc = check_metric(ds->d, metric);
    if (rc) return rc;
    if ((rc = t_ctx.init()) || (rc = grow(t_ctx.input, (size_t)nq * ds->d.dim * 4)) || (rc = grow(t_ctx.output, (size_t)nq * k * 8))) return rc;
    cudaStream_t s = t_ctx.stream;
    CK(cudaMemcpyAsync(t_ctx.input.get(), queries, (size_t)nq * ds->d.dim * 4, cudaMemcpyHostToDevice, s), "H2D queries");
    if ((rc = topk_device(ds, metric, t_ctx.input.get<float>(), nq, k, 0, t_ctx.output.get<long long>()))) return rc;
    CK(cudaMemcpyAsync(keys_out, t_ctx.output.get(), (size_t)nq * k * 8, cudaMemcpyDeviceToHost, s), "D2H keys");
    CK(cudaStreamSynchronize(s), "sync");
    return JV_OK;
}

int jv_topk_bruteforce_device(jv_dataset ds, int metric, const float *queries_device, int nq, int k, int64_t id_base, int64_t *keys_out_device)
{
    ON_DEVICE_OF(ds);
    if (!ds || !queries_device || !keys_out_device || nq <= 0 || k <= 0 || k > 2048 || id_base < 0) return fail(JV_ERR_INVALID, "topk_bruteforce_device: bad arguments");
    int rc = check_metric(ds->d, metric);
    if (rc) return rc;
    if ((rc = t_ctx.init())) return rc;
    return topk_device(ds, metric, queries_device, nq, k, id_base, (long long *)keys_out_device);
}

int jv_topk_merge_device(const int64_t *keys_in_device, int nq, int parts, int k, int64_t *keys_out_device)
{
    NEED_INIT();
    if (!keys_in_device || !keys_out_device || nq <= 0 || parts <= 0 || k <= 0 || (long long)parts * k > 16384) return fail(JV_ERR_INVALID, "topk_merge: bad arguments");
    int rc;
    if ((rc = t_ctx.init())) return rc;
    CK(launch_topk_merge((const long long *)keys_in_device, nq, parts, k, (long long *)keys_out_device, t_ctx.stream), "topk_merge");
    CK(cudaStreamSynchronize(t_ctx.stream), "sync");
    return JV_OK;
}

int jv_topk_bruteforce_device_async(jv_dataset ds, int metric, const float *queries_device, int nq, int k, int64_t id_base, int64_t *keys_out_device,
                                    int32_t *status_device, void *cuda_stream)
{
    ON_DEVICE_OF(ds);
    if (!queries_device || !keys_out_device || !status_device || nq <= 0 || k <= 0 || id_base < 0) return fail(JV_ERR_INVALID, "topk_bruteforce_device_async: bad arguments");
    (void)metric;
    if (!bq_imma_supported(ds->d, k)) return fail(JV_ERR_UNSUPPORTED, "topk_bruteforce_device_async: BQ data sets (even word count, n >= 4096) only; use jv_topk_bruteforce_device");
    int rc;
    if ((rc = t_ctx.init())) return rc;
    return topk_bq_imma_enqueue(ds, queries_device, nq, k, id_base, (long long *)keys_out_device, status_device, t_ctx.bq_async, (cudaStream_t)cuda_stream);
}

int jv_topk_merge_device_async(const int64_t *keys_in_device, int nq, int parts, int k, int64_t *keys_out_device, void *cuda_stream)
{
    NEED_INIT();
    if (!keys_in_device || !keys_out_device || nq <= 0 || parts <= 0 || k <= 0 || (long long)parts * k > 16384) return fail(JV_ERR_INVALID, "topk_merge: bad arguments");
    CK(launch_topk_merge_strided((const long long *)keys_in_device, nq, parts, k, (long long *)keys_out_device, (cudaStream_t)cuda_stream), "topk_merge");
    return JV_OK;
}

// ------------------------------------------------------------------------------------------------ filtered exhaustive top-k
// the acceptOrds / threshold fields of jv_search_options over a data set of n rows (the graph search's checks and wording)
static int check_accept_options(const jv_search_options *opts, long long n, const char *who)
{
    if (!opts) return JV_OK;
    if (opts->threshold < 0.f || opts->rerank_floor < 0.f || opts->accept_stride_words < 0)
        return fail(JV_ERR_INVALID, std::string(who) + ": negative threshold / rerankFloor / stride");
    const long long words = (n + 31) / 32;
    if (opts->accept_bits && opts->accept_stride_words != 0 && opts->accept_stride_words < words)
        return fail(JV_ERR_INVALID, std::string(who) + ": accept_stride_words shorter than one bitset");
    return JV_OK;
}

// the lowest top-k key whose score passes `score >= threshold` (threshold > 0): every key below it scores less
static long long threshold_key(float threshold)
{
    if (!(threshold > 0.f)) return KEY_MIN;
    int32_t b;
    memcpy(&b, &threshold, 4);
    b ^= (b >> 31) & 0x7fffffff;
    return (long long)((unsigned long long)(uint32_t)b << 32);
}

// Keys of the k best rows each query accepts (opts->accept_bits: host bitsets, NULL = every row; opts->threshold), queries in HBM.
// The bitsets are compacted on the device (a shared one once, per-query ones chunk by chunk with the queries) and each query goes
// to the whole or the sampled tier on its accepted count (launch_topk_accepted). *visited += the accepted rows of every query.
static int topk_accepted_device(jv_dataset ds, int metric, const float *queries_dev, int nq, int k, const jv_search_options *opts, long long *keys_dev,
                                int64_t *visited)
{
    cudaStream_t s = t_ctx.stream;
    int rc;
    const long long n = ds->d.n;
    const size_t words = (size_t)((n + 31) / 32);
    const int S = accept_sample_size(n);
    const bool per_query = opts->accept_bits && opts->accept_stride_words != 0;
    const long long stride = per_query ? opts->accept_stride_words : 0;
    const size_t bf = (size_t)blob_floats(ds->d);
    const int chunk_max = (int)std::max<size_t>(1, std::min<size_t>(4096, ((size_t)512 << 20) / (bf * 4)));
    const int chunk = std::min(nq, chunk_max);
    const int nsets = per_query ? chunk : 1;
    const size_t bit_words = per_query ? (size_t)stride * (size_t)(chunk - 1) + words : words;
    int *dcnt, *dsampled;
    int32_t *dids;
    auto carve = [&](void *base) {
        Carver c(base);
        dcnt = c.take<int>(nsets);
        dids = c.take<int32_t>((size_t)nsets * S);
        dsampled = c.take<int>(chunk);
        return c.bytes;
    };
    if ((rc = grow(t_ctx.accept_bits, bit_words * 4)) || (rc = grow(t_ctx.accept_lists, carve(nullptr))) || (rc = grow(t_ctx.blobs, (size_t)chunk * bf * 4)) ||
        (rc = grow(t_ctx.topk_scratch, topk_scratch_bytes(ds->d, chunk, k))) || (rc = grow(t_ctx.flag, 64)))
        return rc;
    carve(t_ctx.accept_lists.get());
    uint32_t *dbits = t_ctx.accept_bits.get<uint32_t>();
    std::vector<int> cnt(nsets), sampled;
    if (!per_query) {
        if (opts->accept_bits) CK(cudaMemcpyAsync(dbits, opts->accept_bits, words * 4, cudaMemcpyHostToDevice, s), "H2D accept bits");
        else CK(cudaMemsetAsync(dbits, 0xff, words * 4, s), "memset accept bits");  // a threshold alone: every row is accepted
        CK(launch_accept_compact(dbits, 0, 1, n, dcnt, dids, s), "accept_compact");
        CK(cudaMemcpyAsync(cnt.data(), dcnt, sizeof(int), cudaMemcpyDeviceToHost, s), "D2H accepted count");
        CK(cudaStreamSynchronize(s), "sync");
    }
    const long long floor_key = threshold_key(opts->threshold);
    for (int q0 = 0; q0 < nq; q0 += chunk) {
        const int cq = std::min(chunk, nq - q0);
        if (per_query) {
            CK(cudaMemcpyAsync(dbits, opts->accept_bits + (size_t)q0 * stride, ((size_t)stride * (cq - 1) + words) * 4, cudaMemcpyHostToDevice, s), "H2D accept bits");
            CK(launch_accept_compact(dbits, stride, cq, n, dcnt, dids, s), "accept_compact");
            CK(cudaMemcpyAsync(cnt.data(), dcnt, (size_t)cq * sizeof(int), cudaMemcpyDeviceToHost, s), "D2H accepted counts");
            CK(cudaStreamSynchronize(s), "sync");
        }
        AcceptLists acc{dbits, stride, per_query, dcnt, dids, 0, dsampled, 0};
        sampled.clear();
        for (int i = 0; i < cq; i++) {
            const int c = cnt[per_query ? i : 0];
            acc.max_listed = std::max(acc.max_listed, std::min(c, S));
            if (c > S) sampled.push_back(i);
            *visited += c;
        }
        acc.n_sampled = (int)sampled.size();
        if (acc.n_sampled) CK(cudaMemcpyAsync(dsampled, sampled.data(), sampled.size() * sizeof(int), cudaMemcpyHostToDevice, s), "H2D sampled queries");
        int *dflag = t_ctx.flag.get<int>();
        CK(cudaMemsetAsync(dflag, 0, sizeof(int), s), "memset flag");
        CK(launch_prepare(ds->d, metric, queries_dev + (size_t)q0 * ds->d.dim, cq, t_ctx.blobs.get<float>(), s), "prepare");
        CK(launch_topk_accepted(ds->d, metric, t_ctx.blobs.get<float>(), cq, k, acc, floor_key, t_ctx.topk_scratch.get(), keys_dev + (size_t)q0 * k, dflag, s),
           "topk_accepted");
        int flag = 0;
        CK(cudaMemcpyAsync(&flag, dflag, sizeof(int), cudaMemcpyDeviceToHost, s), "D2H flag");
        CK(cudaStreamSynchronize(s), "sync");
        if (flag) return fail(JV_ERR_OVERFLOW, "topk_bruteforce_ex: candidate buffer overflow (adversarial score distribution)");
    }
    return JV_OK;
}

int jv_topk_bruteforce_ex(jv_dataset ds, int metric, const float *queries, int nq, int k, const jv_search_options *opts, int64_t *keys_out)
{
    ON_DEVICE_OF(ds);
    if (!queries || !keys_out || nq <= 0 || k <= 0) return fail(JV_ERR_INVALID, "topk_bruteforce_ex: bad arguments");
    if (k > 2048) return fail(JV_ERR_INVALID, "topk_bruteforce_ex: k <= 2048");
    int rc = check_accept_options(opts, ds->d.n, "topk_bruteforce_ex");
    if (rc) return rc;
    if (opts && opts->rerank_floor != 0.f) return fail(JV_ERR_INVALID, "topk_bruteforce_ex: rerank_floor must be 0 (nothing is reranked)");
    if (!opts || (!opts->accept_bits && !(opts->threshold > 0.f))) return jv_topk_bruteforce(ds, metric, queries, nq, k, keys_out);
    if ((rc = check_metric(ds->d, metric))) return rc;
    if ((rc = t_ctx.init()) || (rc = grow(t_ctx.input, (size_t)nq * ds->d.dim * 4)) || (rc = grow(t_ctx.output, (size_t)nq * k * 8))) return rc;
    cudaStream_t s = t_ctx.stream;
    CK(cudaMemcpyAsync(t_ctx.input.get(), queries, (size_t)nq * ds->d.dim * 4, cudaMemcpyHostToDevice, s), "H2D queries");
    int64_t visited = 0;
    if ((rc = topk_accepted_device(ds, metric, t_ctx.input.get<float>(), nq, k, opts, t_ctx.output.get<long long>(), &visited))) return rc;
    CK(cudaMemcpyAsync(keys_out, t_ctx.output.get(), (size_t)nq * k * 8, cudaMemcpyDeviceToHost, s), "D2H keys");
    CK(cudaStreamSynchronize(s), "sync");
    return JV_OK;
}

constexpr int EXHAUSTIVE_QUERY_CHUNK = 4096;  // queries per candidate / rerank step (bounds the candidate keys and rerank scratch)

// jv_exhaustive_search_batch's checks of its arguments (rerankK's bound excepted)
static int exhaustive_check(jv_dataset approx, jv_dataset reranker, int metric, int topK, int rerankK, const jv_search_options *opts)
{
    if (topK < 1 || rerankK < topK) return fail(JV_ERR_INVALID, "exhaustive_search: need 1 <= topK <= rerankK");
    if (reranker && reranker->device != approx->device) return fail(JV_ERR_INVALID, "exhaustive_search: data sets live on different devices");
    if (reranker && (reranker->d.n != approx->d.n || reranker->d.dim != approx->d.dim)) return fail(JV_ERR_INVALID, "exhaustive_search: reranker shape mismatch");
    if (reranker && reranker->d.kind != KIND_F32 && reranker->d.kind != KIND_NVQ)
        return fail(JV_ERR_UNSUPPORTED, "exhaustive_search: the reranker must be fp32 or NVQ (OnDiskGraphIndex.java:705-713)");
    int rc = check_accept_options(opts, approx->d.n, "exhaustive_search");
    if (rc || (rc = check_metric(approx->d, metric))) return rc;
    return JV_OK;
}

// jv_exhaustive_search_batch's device work: the queries' answers [nq][topK] from the nq queries in HBM (queries_dev; nullptr: copied
// chunk by chunk from the host `queries` into the thread's input buffer) into nodes_dev / scores_dev (nullptr: each chunk is
// downloaded to the host nodes_out / scores_out); *visited += the rows scored, *taken = the candidates reranked. Asynchronous on the
// thread's stream, which the host must synchronise before it reads what the call downloads, *taken included.
static int exhaustive_device(jv_dataset approx, jv_dataset reranker, int metric, const float *queries, const float *queries_dev, int nq, int topK,
                             int rerankK, const jv_search_options *opts, int32_t *nodes_out, float *scores_out, int32_t *nodes_dev, float *scores_dev,
                             int64_t *visited, unsigned long long *taken)
{
    const bool filtered = opts && (opts->accept_bits || opts->threshold > 0.f);
    const float floor = opts ? opts->rerank_floor : 0.f;
    const int R = rerankK, chunk = std::min(nq, EXHAUSTIVE_QUERY_CHUNK);
    const size_t rbf = reranker ? (size_t)blob_floats(reranker->d) : 0;
    long long *dcand;
    int32_t *dnodes, *dids, *doffsets;
    float *dscores, *drblobs, *dexact;
    unsigned long long *dtaken;
    auto carve = [&](void *base) {
        Carver c(base);
        dcand = c.take<long long>((size_t)chunk * R);
        dnodes = c.take<int32_t>(nodes_dev ? 0 : (size_t)chunk * topK);
        dscores = c.take<float>(nodes_dev ? 0 : (size_t)chunk * topK);
        dtaken = c.take<unsigned long long>(1);
        drblobs = c.take<float>(reranker ? (size_t)chunk * rbf : 0);
        dids = c.take<int32_t>(reranker ? (size_t)chunk * R : 0);
        doffsets = c.take<int32_t>(reranker ? (size_t)chunk + 1 : 0);
        dexact = c.take<float>(reranker ? (size_t)chunk * R : 0);
        return c.bytes;
    };
    int rc;
    if ((rc = t_ctx.init()) || (!queries_dev && (rc = grow(t_ctx.input, (size_t)chunk * approx->d.dim * 4))) || (rc = grow(t_ctx.rerank, carve(nullptr)))) return rc;
    carve(t_ctx.rerank.get());
    cudaStream_t s = t_ctx.stream;
    CK(cudaMemsetAsync(dtaken, 0, sizeof(unsigned long long), s), "memset taken");
    for (int q0 = 0; q0 < nq; q0 += chunk) {
        const int cq = std::min(chunk, nq - q0);
        const float *dq;
        if (queries_dev) dq = queries_dev + (size_t)q0 * approx->d.dim;
        else {
            CK(cudaMemcpyAsync(t_ctx.input.get(), queries + (size_t)q0 * approx->d.dim, (size_t)cq * approx->d.dim * 4, cudaMemcpyHostToDevice, s), "H2D queries");
            dq = t_ctx.input.get<float>();
        }
        if (filtered) {
            jv_search_options o = *opts;
            if (o.accept_bits && o.accept_stride_words) o.accept_bits += (size_t)q0 * o.accept_stride_words;
            if ((rc = topk_accepted_device(approx, metric, dq, cq, R, &o, dcand, visited))) return rc;
        } else {
            if ((rc = topk_device(approx, metric, dq, cq, R, 0, dcand))) return rc;
            *visited += (int64_t)cq * approx->d.n;
        }
        int32_t *on = nodes_dev ? nodes_dev + (size_t)q0 * topK : dnodes;
        float *os = nodes_dev ? scores_dev + (size_t)q0 * topK : dscores;
        if (reranker) CK(launch_prepare(reranker->d, metric, dq, cq, drblobs, s), "prepare reranker");
        CK(launch_rerank_accepted(reranker ? &reranker->d : nullptr, metric, drblobs, cq, R, topK, floor, dcand, dids, doffsets, dexact, dtaken, on, os, s),
           "rerank");
        if (!nodes_dev) {
            CK(cudaMemcpyAsync(nodes_out + (size_t)q0 * topK, dnodes, (size_t)cq * topK * 4, cudaMemcpyDeviceToHost, s), "D2H nodes");
            CK(cudaMemcpyAsync(scores_out + (size_t)q0 * topK, dscores, (size_t)cq * topK * 4, cudaMemcpyDeviceToHost, s), "D2H scores");
        }
    }
    CK(cudaMemcpyAsync(taken, dtaken, sizeof(*taken), cudaMemcpyDeviceToHost, s), "D2H taken");
    return JV_OK;
}

int jv_exhaustive_search_batch(jv_dataset approx, jv_dataset reranker, int metric, const float *queries, int nq, int topK, int rerankK,
                               const jv_search_options *opts, int32_t *nodes_out, float *scores_out, jv_search_stats *stats)
{
    ON_DEVICE_OF(approx);
    if (!queries || !nodes_out || !scores_out || nq <= 0) return fail(JV_ERR_INVALID, "exhaustive_search: bad arguments");
    if (topK < 1 || rerankK < topK) return fail(JV_ERR_INVALID, "exhaustive_search: need 1 <= topK <= rerankK");
    if (rerankK > 2048) return fail(JV_ERR_INVALID, "exhaustive_search: rerankK <= 2048");
    int rc = exhaustive_check(approx, reranker, metric, topK, rerankK, opts);
    if (rc) return rc;
    if ((rc = t_ctx.init())) return rc;
    cudaStream_t s = t_ctx.stream;
    int64_t visited = 0;
    unsigned long long taken = 0;
    CK(t_ctx.timer.start(s), "event");
    if ((rc = exhaustive_device(approx, reranker, metric, queries, nullptr, nq, topK, rerankK, opts, nodes_out, scores_out, nullptr, nullptr, &visited, &taken)))
        return rc;
    CK(t_ctx.timer.stop(s), "event");
    CK(cudaStreamSynchronize(s), "sync");
    if (stats) {
        memset(stats, 0, sizeof(*stats));
        stats->visited = visited;
        stats->reranked = (int64_t)taken;
        stats->device_ms = t_ctx.timer.ms();
    }
    return JV_OK;
}

// ------------------------------------------------------------------------------------------------ encoders
static int bq_encode_impl(const float *rows_host, const float *rows_dev, int row_stride, int64_t n, int dim, uint64_t *words_out)
{
    int rc;
    const int W = (dim + 63) / 64;
    if ((rc = t_ctx.init()) || (rows_host && (rc = grow(t_ctx.input, (size_t)n * dim * 4))) || (rc = grow(t_ctx.output, (size_t)n * W * 8))) return rc;
    cudaStream_t s = t_ctx.stream;
    if (rows_host) {
        CK(cudaMemcpyAsync(t_ctx.input.get(), rows_host, (size_t)n * dim * 4, cudaMemcpyHostToDevice, s), "H2D rows");
        rows_dev = t_ctx.input.get<float>();
        row_stride = dim;
    }
    CK(launch_bq_encode(rows_dev, n, dim, row_stride, t_ctx.output.get<unsigned long long>(), s), "bq_encode");
    CK(cudaMemcpyAsync(words_out, t_ctx.output.get(), (size_t)n * W * 8, cudaMemcpyDeviceToHost, s), "D2H words");
    CK(cudaStreamSynchronize(s), "sync");
    return JV_OK;
}

int jv_bq_encode_batch(const float *rows, int64_t n, int dim, uint64_t *words_out)
{
    NEED_INIT();
    if (!rows || !words_out || n <= 0 || dim <= 0) return fail(JV_ERR_INVALID, "bq_encode: bad arguments");
    return bq_encode_impl(rows, nullptr, 0, n, dim, words_out);
}

int jv_bq_encode_dataset(jv_dataset f32, uint64_t *words_out)
{
    ON_DEVICE_OF(f32);
    if (!f32 || f32->d.kind != KIND_F32 || !words_out) return fail(JV_ERR_INVALID, "bq_encode_dataset: needs an fp32 data set");
    return bq_encode_impl(nullptr, f32->d.rows, f32->d.stride, f32->d.n, f32->d.dim, words_out);
}

// ProductQuantization.anisotropicThreshold: UNWEIGHTED (-1) <= T < 1, not NaN (KMeansPlusPlusClusterer.java:86-92)
static bool bad_threshold(float t) { return !(t >= -1.f && t < 1.f); }

// threshold > -1: the anisotropic encoder (ProductQuantization.encodeAnisotropic); stats (optional) also times the stream's work
static int pq_encode_impl(const float *rows, const float *rows_dev, int row_stride, int64_t n, int dim, int M, int k, const float *codebooks,
                          const float *centroid, uint8_t *codes_out, float threshold = -1.f, jv_pq_encode_stats *stats = nullptr)
{
    int rc;
    const bool aniso = threshold > -1.f;
    float *dcb, *dcen;
    int *dlay;
    unsigned long long *dstats;
    void *dscratch;
    auto carve = [&](void *base) {
        Carver c(base);
        dcb = c.take<float>((size_t)k * dim);
        dcen = c.take<float>(dim);
        dlay = c.take<int>(2 * (size_t)M);
        dstats = c.take<unsigned long long>(aniso ? 3 : 0);
        dscratch = c.take<char>(aniso ? pq_encode_aniso_scratch(dim, M, k) : 0);
        return c.bytes;
    };
    if ((rc = t_ctx.init()) || (rows && (rc = grow(t_ctx.input, (size_t)n * dim * 4))) || (rc = grow(t_ctx.output, (size_t)n * M)) ||
        (rc = grow(t_ctx.aux, carve(nullptr))))
        return rc;
    carve(t_ctx.aux.get());
    cudaStream_t s = t_ctx.stream;
    StreamTimer timer;
    if (stats) CK(timer.start(s), "timer");
    if (rows) {
        CK(cudaMemcpyAsync(t_ctx.input.get(), rows, (size_t)n * dim * 4, cudaMemcpyHostToDevice, s), "H2D rows");
        rows_dev = t_ctx.input.get<float>();
        row_stride = dim;
    }
    CK(cudaMemcpyAsync(dcb, codebooks, (size_t)k * dim * 4, cudaMemcpyHostToDevice, s), "H2D codebooks");
    if (centroid) CK(cudaMemcpyAsync(dcen, centroid, (size_t)dim * 4, cudaMemcpyHostToDevice, s), "H2D centroid");
    CK(upload_layout(dim, M, dlay, s), "H2D layout");
    DataDesc d;
    memset(&d, 0, sizeof(d));
    d.kind = KIND_PQ; d.dim = dim; d.n = n; d.M = M; d.k = k; d.codebooks = dcb; d.sub_sizes = dlay; d.sub_offsets = dlay + M; d.centroid = centroid ? dcen : nullptr;
    if (aniso)
        CK(launch_pq_encode_aniso(d, rows_dev, n, row_stride, pq_parallel_cost_multiplier(threshold, dim), dscratch, dstats, t_ctx.output.get<uint8_t>(), s),
           "pq_encode_aniso");
    else
        CK(launch_pq_encode(d, rows_dev, n, row_stride, t_ctx.output.get<uint8_t>(), s), "pq_encode");
    CK(cudaMemcpyAsync(codes_out, t_ctx.output.get(), (size_t)n * M, cudaMemcpyDeviceToHost, s), "D2H codes");
    unsigned long long counters[3] = {0, 0, 0};
    if (stats && aniso) CK(cudaMemcpyAsync(counters, dstats, sizeof(counters), cudaMemcpyDeviceToHost, s), "D2H stats");
    if (stats) CK(timer.stop(s), "timer");
    CK(cudaStreamSynchronize(s), "sync");
    if (stats) {
        stats->rows_moved = (int64_t)counters[0];
        stats->moves = (int64_t)counters[1];
        stats->max_sweeps = (int32_t)counters[2];
        stats->device_ms = timer.ms();
    }
    return JV_OK;
}

static int pq_encode_batch_entry(const float *rows, int64_t n, int dim, int M, int k, const float *codebooks, const float *centroid, uint8_t *codes_out,
                                 float threshold, jv_pq_encode_stats *stats)
{
    NEED_INIT();
    if (!rows || !codebooks || !codes_out || n <= 0 || dim <= 0 || M <= 0 || M > dim || k <= 0 || k > 256) return fail(JV_ERR_INVALID, "pq_encode: bad arguments");
    if (bad_threshold(threshold)) return fail(JV_ERR_INVALID, "pq_encode: anisotropic threshold outside [-1, 1)");
    return pq_encode_impl(rows, nullptr, 0, n, dim, M, k, codebooks, centroid, codes_out, threshold, stats);
}

static int pq_encode_dataset_entry(jv_dataset f32, int M, int k, const float *codebooks, const float *centroid, uint8_t *codes_out, float threshold,
                                   jv_pq_encode_stats *stats)
{
    ON_DEVICE_OF(f32);
    if (!f32 || f32->d.kind != KIND_F32 || !codebooks || !codes_out || M <= 0 || M > f32->d.dim || k <= 0 || k > 256)
        return fail(JV_ERR_INVALID, "pq_encode_dataset: bad arguments");
    if (bad_threshold(threshold)) return fail(JV_ERR_INVALID, "pq_encode_dataset: anisotropic threshold outside [-1, 1)");
    return pq_encode_impl(nullptr, f32->d.rows, f32->d.stride, f32->d.n, f32->d.dim, M, k, codebooks, centroid, codes_out, threshold, stats);
}

int jv_pq_encode_batch(const float *rows, int64_t n, int dim, int M, int k, const float *codebooks, const float *centroid, uint8_t *codes_out)
{
    return pq_encode_batch_entry(rows, n, dim, M, k, codebooks, centroid, codes_out, -1.f, nullptr);
}

int jv_pq_encode_dataset(jv_dataset f32, int M, int k, const float *codebooks, const float *centroid, uint8_t *codes_out)
{
    return pq_encode_dataset_entry(f32, M, k, codebooks, centroid, codes_out, -1.f, nullptr);
}

int jv_pq_encode_batch_anisotropic(const float *rows, int64_t n, int dim, int M, int k, const float *codebooks, const float *centroid,
                                   float anisotropic_threshold, uint8_t *codes_out, jv_pq_encode_stats *stats)
{
    return pq_encode_batch_entry(rows, n, dim, M, k, codebooks, centroid, codes_out, anisotropic_threshold, stats);
}

int jv_pq_encode_dataset_anisotropic(jv_dataset f32, int M, int k, const float *codebooks, const float *centroid, float anisotropic_threshold,
                                     uint8_t *codes_out, jv_pq_encode_stats *stats)
{
    return pq_encode_dataset_entry(f32, M, k, codebooks, centroid, codes_out, anisotropic_threshold, stats);
}

// the resident rows of f32 encoded (ProductQuantization.encodeAll) into a new resident PQ data set on `s`, no host round trip
// (returns once the stream has drained):
// pq_encode_kernel writes packed [n][M] rows, copied into the data set's [n][code_stride] rows when M is not a multiple of 4
static int pq_encode_resident(jv_dataset f32, int M, int k, const float *codebooks, const float *centroid, cudaStream_t s,
                              std::unique_ptr<jv_dataset_s> &ds)
{
    const int64_t n = f32->d.n;
    uint8_t *codes;
    int rc = pq_dataset(n, f32->d.dim, M, k, codebooks, centroid, s, ds, &codes);
    if (rc) return rc;
    const int stride = ds->d.code_stride;
    DeviceBuffer packed;
    if (stride != M) {
        CK(packed.alloc((size_t)n * M), "cudaMalloc(packed codes)");
        CK(cudaMemsetAsync(codes, 0, (size_t)n * stride, s), "memset codes");
    }
    CK(launch_pq_encode(ds->d, f32->d.rows, n, f32->d.stride, stride != M ? packed.get<uint8_t>() : codes, s), "pq_encode");
    if (stride != M) CK(cudaMemcpy2DAsync(codes, stride, packed.get(), M, M, n, cudaMemcpyDeviceToDevice, s), "pad codes");
    CK(cudaStreamSynchronize(s), "pq_encode_resident");  // `packed` goes on return
    return JV_OK;
}

int jv_pq_encode_dataset_resident(jv_dataset f32, int M, int k, const float *codebooks, const float *centroid, jv_dataset *out)
{
    ON_DEVICE_OF(f32);
    if (f32->d.kind != KIND_F32 || !codebooks || !out || M <= 0 || M > f32->d.dim || k <= 0 || k > 256)
        return fail(JV_ERR_INVALID, "pq_encode_dataset_resident: bad arguments");
    int rc;
    std::unique_ptr<jv_dataset_s> ds;
    if ((rc = t_ctx.init()) || (rc = pq_encode_resident(f32, M, k, codebooks, centroid, t_ctx.stream, ds))) return rc;
    *out = ds.release();
    return JV_OK;
}

// ------------------------------------------------------------------------------------------------ PQ training
constexpr int64_t MAX_PQ_TRAINING_SET_SIZE = 128000;  // ProductQuantization.java:64

// threshold > -1 adds the anisotropic rounds: lloyd_iterations of them after compute's Lloyd, or in place of refine's
static int pq_train_impl(jv_dataset f32, const jv_pq_train_params *p, const float *codebooks, const float *centroid, float *codebooks_out,
                         float *centroid_out, jv_pq_train_stats *stats, float threshold = -1.f, jv_pq_anisotropic_stats *astats = nullptr)
{
    if (f32->d.kind != KIND_F32) return fail(JV_ERR_INVALID, "pq_train: needs an fp32 data set");
    if (!p || !codebooks_out) return fail(JV_ERR_INVALID, "pq_train: null argument");
    if (p->M < 1 || p->M > f32->d.dim) return fail(JV_ERR_INVALID, "pq_train: M must be in 1..dim");
    if (p->k < 1 || p->k > 256) return fail(JV_ERR_INVALID, "pq_train: k must be in 1..256");
    if (p->lloyd_iterations < 0 || p->max_train_rows < 0) return fail(JV_ERR_INVALID, "pq_train: negative iteration count or row cap");
    const int64_t cap = p->max_train_rows ? p->max_train_rows : MAX_PQ_TRAINING_SET_SIZE;
    if (std::min<int64_t>(f32->d.n, cap) < p->k) return fail(JV_ERR_INVALID, "pq_train: fewer training rows than clusters");
    const bool aniso = threshold > -1.f;
    if (aniso && (f32->d.dim + p->M - 1) / p->M > 64) return fail(JV_ERR_UNSUPPORTED, "pq_train: anisotropic sub-spaces above 64 floats");
    int rc;
    if ((rc = t_ctx.init())) return rc;
    const int lloyd = aniso && codebooks ? 0 : p->lloyd_iterations;  // refine: anisotropic rounds only (ProductQuantization.refine)
    const PqTrainArgs a = {p->M, p->k, p->globally_center, lloyd, (long long)cap, p->seed, aniso ? p->lloyd_iterations : 0, threshold};
    PqTrainStats st;
    CK(pq_train(f32->d, a, codebooks, centroid, codebooks_out, centroid_out, &st, t_ctx.stream), "pq_train");
    if (stats) {
        stats->train_rows = st.train_rows;
        stats->max_lloyd_updates = st.max_lloyd_updates;
        stats->changed_last = st.changed_last;
        stats->empty_reseeds = st.empty_reseeds;
        stats->seeding_fallbacks = st.seeding_fallbacks;
        stats->device_ms = st.device_ms;
    }
    if (astats) {
        astats->max_anisotropic_updates = st.aniso_updates;
        astats->changed_last_anisotropic = st.aniso_changed_last;
        astats->anisotropic_reseeds = st.aniso_reseeds;
    }
    return JV_OK;
}

int jv_pq_train(jv_dataset f32, const jv_pq_train_params *p, float *codebooks_out, float *centroid_out, jv_pq_train_stats *stats)
{
    ON_DEVICE_OF(f32);
    if (p && p->globally_center && !centroid_out) return fail(JV_ERR_INVALID, "pq_train: globally_center needs centroid_out");
    return pq_train_impl(f32, p, nullptr, nullptr, codebooks_out, centroid_out, stats);
}

int jv_pq_refine(jv_dataset f32, const jv_pq_train_params *p, const float *codebooks, const float *centroid, float *codebooks_out, jv_pq_train_stats *stats)
{
    ON_DEVICE_OF(f32);
    if (!codebooks) return fail(JV_ERR_INVALID, "pq_refine: null codebooks");
    return pq_train_impl(f32, p, codebooks, centroid, codebooks_out, nullptr, stats);
}

static void unweighted_stats(jv_pq_anisotropic_stats *stats, const jv_pq_train_stats &st)
{
    stats->lloyd = st;
    stats->max_anisotropic_updates = 0;
    stats->changed_last_anisotropic = 0;
    stats->anisotropic_reseeds = 0;
}

int jv_pq_train_anisotropic(jv_dataset f32, const jv_pq_train_params *p, float anisotropic_threshold, float *codebooks_out, float *centroid_out,
                            jv_pq_anisotropic_stats *stats)
{
    ON_DEVICE_OF(f32);
    if (bad_threshold(anisotropic_threshold)) return fail(JV_ERR_INVALID, "pq_train: anisotropic threshold outside [-1, 1)");
    jv_pq_train_stats st;
    if (anisotropic_threshold == -1.f) {
        const int rc = jv_pq_train(f32, p, codebooks_out, centroid_out, stats ? &st : nullptr);
        if (rc == JV_OK && stats) unweighted_stats(stats, st);
        return rc;
    }
    if (p && p->globally_center && !centroid_out) return fail(JV_ERR_INVALID, "pq_train: globally_center needs centroid_out");
    return pq_train_impl(f32, p, nullptr, nullptr, codebooks_out, centroid_out, stats ? &stats->lloyd : nullptr, anisotropic_threshold, stats);
}

int jv_pq_refine_anisotropic(jv_dataset f32, const jv_pq_train_params *p, float anisotropic_threshold, const float *codebooks, const float *centroid,
                             float *codebooks_out, jv_pq_anisotropic_stats *stats)
{
    ON_DEVICE_OF(f32);
    if (bad_threshold(anisotropic_threshold)) return fail(JV_ERR_INVALID, "pq_refine: anisotropic threshold outside [-1, 1)");
    jv_pq_train_stats st;
    if (anisotropic_threshold == -1.f) {
        const int rc = jv_pq_refine(f32, p, codebooks, centroid, codebooks_out, stats ? &st : nullptr);
        if (rc == JV_OK && stats) unweighted_stats(stats, st);
        return rc;
    }
    if (!codebooks) return fail(JV_ERR_INVALID, "pq_refine: null codebooks");
    return pq_train_impl(f32, p, codebooks, centroid, codebooks_out, nullptr, stats ? &stats->lloyd : nullptr, anisotropic_threshold, stats);
}

static int nvq_encode_impl(const float *rows, const float *rows_dev, int row_stride, int64_t n, int dim, int nsub, const float *mean, int learn,
                           float *params_out, uint8_t *bytes_out)
{
    int rc;
    float *dmean, *dparams;
    int *dlay;
    uint8_t *dbytes;
    auto carve_aux = [&](void *base) {
        Carver c(base);
        dmean = c.take<float>(dim);
        dlay = c.take<int>(2 * (size_t)nsub);
        return c.bytes;
    };
    auto carve_out = [&](void *base) {
        Carver c(base);
        dbytes = c.take<uint8_t>((size_t)n * dim);
        dparams = c.take<float>((size_t)n * nsub * 4);
        return c.bytes;
    };
    if ((rc = t_ctx.init()) || (rows && (rc = grow(t_ctx.input, (size_t)n * dim * 4))) || (rc = grow(t_ctx.aux, carve_aux(nullptr))) ||
        (rc = grow(t_ctx.output, carve_out(nullptr))))
        return rc;
    carve_aux(t_ctx.aux.get());
    carve_out(t_ctx.output.get());
    cudaStream_t s = t_ctx.stream;
    if (rows) {
        CK(cudaMemcpyAsync(t_ctx.input.get(), rows, (size_t)n * dim * 4, cudaMemcpyHostToDevice, s), "H2D rows");
        rows_dev = t_ctx.input.get<float>();
        row_stride = dim;
    }
    CK(cudaMemcpyAsync(dmean, mean, (size_t)dim * 4, cudaMemcpyHostToDevice, s), "H2D mean");
    CK(upload_layout(dim, nsub, dlay, s), "H2D layout");
    CK(launch_nvq_encode(rows_dev, n, row_stride, nsub, dlay, dlay + nsub, dmean, learn, dparams, dbytes, dim, s), "nvq_encode");
    CK(cudaMemcpyAsync(params_out, dparams, (size_t)n * nsub * 16, cudaMemcpyDeviceToHost, s), "D2H params");
    CK(cudaMemcpyAsync(bytes_out, dbytes, (size_t)n * dim, cudaMemcpyDeviceToHost, s), "D2H bytes");
    CK(cudaStreamSynchronize(s), "sync");
    return JV_OK;
}

int jv_nvq_encode_batch(const float *rows, int64_t n, int dim, int nsub, const float *mean, int learn, float *params_out, uint8_t *bytes_out)
{
    NEED_INIT();
    if (!rows || !mean || !params_out || !bytes_out || n <= 0 || dim <= 0 || nsub <= 0 || nsub > dim) return fail(JV_ERR_INVALID, "nvq_encode: bad arguments");
    return nvq_encode_impl(rows, nullptr, 0, n, dim, nsub, mean, learn, params_out, bytes_out);
}

int jv_nvq_encode_dataset(jv_dataset f32, int nsub, const float *mean, int learn, float *params_out, uint8_t *bytes_out)
{
    ON_DEVICE_OF(f32);
    if (!f32 || f32->d.kind != KIND_F32 || !mean || !params_out || !bytes_out || nsub <= 0 || nsub > f32->d.dim)
        return fail(JV_ERR_INVALID, "nvq_encode_dataset: bad arguments");
    return nvq_encode_impl(nullptr, f32->d.rows, f32->d.stride, f32->d.n, f32->d.dim, nsub, mean, learn, params_out, bytes_out);
}

// NVQ "inline vectors" without a host round trip: encode the resident fp32 rows into a new resident NVQ data set
int jv_nvq_encode_dataset_resident(jv_dataset f32, int nsub, const float *mean, int learn, jv_dataset *out)
{
    ON_DEVICE_OF(f32);
    if (f32->d.kind != KIND_F32 || !mean || !out || nsub <= 0 || nsub > f32->d.dim) return fail(JV_ERR_INVALID, "nvq_encode_dataset_resident: bad arguments");
    std::unique_ptr<jv_dataset_s> ds;
    uint8_t *db;
    float *dp;
    int rc;
    if ((rc = t_ctx.init()) || (rc = nvq_dataset(f32->d.n, f32->d.dim, nsub, mean, t_ctx.stream, ds, &db, &dp))) return rc;
    cudaStream_t s = t_ctx.stream;
    cudaError_t e = ds->d.byte_stride != ds->d.dim ? cudaMemsetAsync(db, 0, (size_t)ds->d.n * ds->d.byte_stride, s) : cudaSuccess;
    if (e == cudaSuccess) e = launch_nvq_encode(f32->d.rows, ds->d.n, f32->d.stride, nsub, ds->d.sub_sizes, ds->d.sub_offsets, ds->d.mean, learn, dp, db, ds->d.byte_stride, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    CK(e, "nvq_encode_dataset_resident");
    *out = ds.release();
    return JV_OK;
}

// ------------------------------------------------------------------------------------------------ graph
int jv_graph_create(int32_t n, int degree, const int32_t *adj0, int32_t entry_node, jv_graph *out)
{
    NEED_INIT();
    if (!adj0 || !out || n <= 0 || degree <= 0 || degree > MAX_DEGREE || entry_node < 0 || entry_node >= n)
        return fail(JV_ERR_INVALID, "graph_create: bad arguments");
    // one pass over data that is copied anyway: a neighbour id outside [-1, n) would be an illegal address inside the search kernel
    for (size_t i = 0, tot = (size_t)n * degree; i < tot; i++)
        if (adj0[i] < -1 || adj0[i] >= n) return fail(JV_ERR_INVALID, "graph_create: neighbour id out of range");
    std::unique_ptr<jv_graph_s> g;
    int rc = jv_graph_s::create(n, degree, g);
    if (rc) return rc;
    CK(cudaMemcpy(g->adj0.get(), adj0, (size_t)n * degree * 4, cudaMemcpyHostToDevice), "upload adjacency");
    if ((rc = g->set_levels({}, {}, entry_node))) return rc;
    *out = g.release();
    return JV_OK;
}

// the whole hierarchy: the upper levels (none: level 0 only) on the host and on the device, and the entry node, which belongs to the
// top level. The device copies are made before anything is replaced, so a failure leaves the graph as it was.
int jv_graph_s::set_levels(Levels ids, Levels adj, int32_t entry)
{
    const int L = (int)ids.size(), n = g.n;
    DeviceBuffer row, cat, off;  // upper_row, upper_adj, upper_off to be
    if (L > 0) {
        std::vector<int32_t> rows((size_t)L * n, -1), adjs;
        std::vector<long long> offs(L);
        long long o = 0;
        for (int l = 0; l < L; l++) {
            offs[l] = o;
            for (size_t i = 0; i < ids[l].size(); i++) rows[(size_t)l * n + ids[l][i]] = (int32_t)i;
            adjs.insert(adjs.end(), adj[l].begin(), adj[l].end());
            o += (long long)ids[l].size();
        }
        CK(row.alloc(rows.size() * 4), "cudaMalloc(upper_row)");
        CK(cat.alloc(std::max<size_t>(adjs.size(), 1) * 4), "cudaMalloc(upper_adj)");
        CK(off.alloc((size_t)L * 8), "cudaMalloc(upper_off)");
        CK(cudaMemcpy(row.get(), rows.data(), rows.size() * 4, cudaMemcpyHostToDevice), "H2D upper_row");
        CK(cudaMemcpy(cat.get(), adjs.data(), adjs.size() * 4, cudaMemcpyHostToDevice), "H2D upper_adj");
        CK(cudaMemcpy(off.get(), offs.data(), (size_t)L * 8, cudaMemcpyHostToDevice), "H2D upper_off");
    }
    // the old device copies go with the locals
    std::swap(upper_row, row); std::swap(upper_adj, cat); std::swap(upper_off, off);
    level_ids = std::move(ids);
    level_adj = std::move(adj);
    g.levels = L + 1; g.entry_level = L; g.entry_node = entry;
    g.upper_row = upper_row.get<int32_t>(); g.upper_adj = upper_adj.get<int32_t>(); g.upper_off = upper_off.get<long long>();
    return JV_OK;
}

int jv_graph_add_level(jv_graph g, int32_t count, const int32_t *node_ids, const int32_t *adj)
{
    ON_DEVICE_OF(g);
    if (!g || count <= 0 || !node_ids || !adj) return fail(JV_ERR_INVALID, "graph_add_level: bad arguments");
    for (size_t i = 0, tot = (size_t)count * g->g.degree; i < tot; i++)
        if (adj[i] < -1 || adj[i] >= g->g.n) return fail(JV_ERR_INVALID, "graph_add_level: neighbour id out of range");
    bool has_entry = false;
    for (int i = 0; i < count; i++) {
        if (node_ids[i] < 0 || node_ids[i] >= g->g.n) return fail(JV_ERR_INVALID, "graph_add_level: node id out of range");
        if (node_ids[i] == g->g.entry_node) has_entry = true;
    }
    if (!has_entry) return fail(JV_ERR_INVALID, "graph_add_level: the entry node must belong to every level");
    Levels ids = g->level_ids, rows = g->level_adj;
    ids.emplace_back(node_ids, node_ids + count);
    rows.emplace_back(adj, adj + (size_t)count * g->g.degree);
    return g->set_levels(std::move(ids), std::move(rows), g->g.entry_node);
}

// g's FusedPQ records packed from pq, enqueued on `s` (the caller synchronises before g is searched)
static int fuse_pq(jv_graph g, jv_dataset pq, cudaStream_t s)
{
    const int rec = (g->g.degree * (4 + pq->d.code_stride) + 15) & ~15;
    g->g.fused = nullptr;
    CK(g->fused.alloc((size_t)g->g.n * rec), "cudaMalloc(fused records)");
    CK(launch_fuse_pq(g->g, pq->d, g->fused.get<uint8_t>(), rec, s), "fuse_pq");
    g->g.fused = g->fused.get<uint8_t>();
    g->g.fused_codes_of = pq->d.codes;
    g->g.fused_rec = rec;
    g->g.fused_code_stride = pq->d.code_stride;
    return JV_OK;
}

int jv_graph_fuse_pq(jv_graph g, jv_dataset pq)
{
    ON_DEVICE_OF(g);
    if (!pq || pq->d.kind != KIND_PQ) return fail(JV_ERR_INVALID, "graph_fuse_pq: needs a PQ data set");
    if (pq->device != g->device || pq->d.n != g->g.n) return fail(JV_ERR_INVALID, "graph_fuse_pq: data set and graph differ in device or size");
    int rc;
    if ((rc = t_ctx.init()) || (rc = fuse_pq(g, pq, t_ctx.stream))) return rc;
    CK(cudaStreamSynchronize(t_ctx.stream), "fuse_pq");
    return JV_OK;
}

int jv_graph_fused_download(jv_graph g, uint8_t *records_out, int *record_bytes)
{
    ON_DEVICE_OF(g);
    if (!g->fused.get()) return fail(JV_ERR_INVALID, "graph_fused_download: jv_graph_fuse_pq has not been called");
    if (record_bytes) *record_bytes = g->g.fused_rec;
    if (records_out) CK(cudaMemcpy(records_out, g->fused.get(), (size_t)g->g.n * g->g.fused_rec, cudaMemcpyDeviceToHost), "D2H fused records");
    return JV_OK;
}

int jv_graph_free(jv_graph g)
{
    if (!g) return JV_OK;
    cudaSetDevice(g->device);
    cudaDeviceSynchronize();
    delete g;
    return JV_OK;
}

int jv_graph_info(jv_graph g, int32_t *n, int *degree, int *levels, int32_t *entry_node)
{
    if (!g) return fail(JV_ERR_INVALID, "graph_info: null graph");
    if (n) *n = g->g.n;
    if (degree) *degree = g->g.degree;
    if (levels) *levels = g->g.levels;
    if (entry_node) *entry_node = g->g.entry_node;
    return JV_OK;
}

int jv_graph_download(jv_graph g, int level, int32_t *node_ids_out, int32_t *adj_out, int32_t *count_out)
{
    ON_DEVICE_OF(g);
    if (!g || level < 0 || level >= g->g.levels) return fail(JV_ERR_INVALID, "graph_download: bad level");
    if (level == 0) {
        if (count_out) *count_out = g->g.n;
        if (node_ids_out)
            for (int i = 0; i < g->g.n; i++) node_ids_out[i] = i;
        if (adj_out) CK(cudaMemcpy(adj_out, g->adj0.get(), (size_t)g->g.n * g->g.degree * 4, cudaMemcpyDeviceToHost), "D2H adjacency");
        return JV_OK;
    }
    const auto &ids = g->level_ids[level - 1];
    if (count_out) *count_out = (int32_t)ids.size();
    if (node_ids_out) memcpy(node_ids_out, ids.data(), ids.size() * 4);
    if (adj_out) memcpy(adj_out, g->level_adj[level - 1].data(), g->level_adj[level - 1].size() * 4);
    return JV_OK;
}

int jv_dataset_row_sketch_download(jv_dataset f32, int8_t *codes_out, float *meta_out, int *sketch_stride_out)
{
    ON_DEVICE_OF(f32);
    if (f32->d.kind != KIND_F32) return fail(JV_ERR_INVALID, "row_sketch_download: not an fp32 data set");
    const int ss = sketch_stride(f32->d.stride);
    if (sketch_stride_out) *sketch_stride_out = ss;
    std::lock_guard<std::mutex> lk(f32->sketch_mu);
    if (!f32->sketch.get()) return fail(JV_ERR_INVALID, "row_sketch_download: no row sketch");
    if (codes_out) CK(cudaMemcpy(codes_out, f32->sketch.get(), (size_t)f32->d.n * ss, cudaMemcpyDeviceToHost), "D2H row sketch");
    if (meta_out) CK(cudaMemcpy(meta_out, f32->sketch_meta.get(), (size_t)f32->d.n * sizeof(float2), cudaMemcpyDeviceToHost), "D2H row sketch meta");
    return JV_OK;
}

static thread_local int64_t t_last_settled = 0;
int64_t jv_search_last_settled(void) { return t_last_settled; }
static thread_local int64_t t_last_direct[2] = {0, 0};
void jv_search_last_direct(int64_t *routed, int64_t *routed_dropped)
{
    if (routed) *routed = t_last_direct[0];
    if (routed_dropped) *routed_dropped = t_last_direct[1];
}

int jv_lowrank_bound_pairs(const float *basis, int dim, const float *rows, const float *queries, int64_t n, uint8_t *records_out, float *bounds_out)
{
    if (!basis || !rows || !queries || dim <= 0 || n <= 0 || !bounds_out) return fail(JV_ERR_INVALID, "lowrank_bound_pairs: bad arguments");
    int rc = t_ctx.init();
    if (rc) return rc;
    cudaStream_t s = t_ctx.stream;
    const int stride = (dim + 3) & ~3;
    if (lowrank_warps(stride) == 0) return fail(JV_ERR_UNSUPPORTED, "lowrank_bound_pairs: rows too wide");
    DeviceBuffer B, X, Q, R, O;
    CK(B.alloc((size_t)LR_K * stride * 4), "cudaMalloc");
    CK(X.alloc((size_t)n * stride * 4), "cudaMalloc");
    CK(Q.alloc((size_t)n * stride * 4), "cudaMalloc");
    CK(R.alloc((size_t)n * LR_SLOT), "cudaMalloc");
    CK(O.alloc((size_t)n * 4), "cudaMalloc");
    // basis: [dim][LR_K] row-major on the host (column j = basis vector j), stored [LR_K][stride] on the device
    std::vector<float> bt((size_t)LR_K * stride, 0.f);
    for (int i = 0; i < dim; i++)
        for (int j = 0; j < LR_K; j++) bt[(size_t)j * stride + i] = basis[(size_t)i * LR_K + j];
    CK(cudaMemsetAsync(X.get(), 0, (size_t)n * stride * 4, s), "memset");
    CK(cudaMemsetAsync(Q.get(), 0, (size_t)n * stride * 4, s), "memset");
    CK(cudaMemcpyAsync(B.get(), bt.data(), bt.size() * 4, cudaMemcpyHostToDevice, s), "H2D basis");
    CK(cudaMemcpy2DAsync(X.get(), (size_t)stride * 4, rows, (size_t)dim * 4, (size_t)dim * 4, n, cudaMemcpyHostToDevice, s), "H2D rows");
    CK(cudaMemcpy2DAsync(Q.get(), (size_t)stride * 4, queries, (size_t)dim * 4, (size_t)dim * 4, n, cudaMemcpyHostToDevice, s), "H2D queries");
    CK(launch_lowrank_rows(X.get<float>(), n, stride, B.get<float>(), R.get<uint8_t>(), s), "lowrank_rows");
    CK(launch_lowrank_bound_pairs(B.get<float>(), dim, stride, Q.get<float>(), R.get<uint8_t>(), n, O.get<float>(), s), "lowrank_bound_pairs");
    if (records_out) CK(cudaMemcpyAsync(records_out, R.get(), (size_t)n * LR_SLOT, cudaMemcpyDeviceToHost, s), "D2H records");
    CK(cudaMemcpyAsync(bounds_out, O.get(), (size_t)n * 4, cudaMemcpyDeviceToHost, s), "D2H bounds");
    CK(cudaStreamSynchronize(s), "lowrank_bound_pairs");
    return JV_OK;
}

int jv_dataset_lowrank_download(jv_dataset f32, float *basis_out, uint8_t *rows_out, int *rank_out)
{
    ON_DEVICE_OF(f32);
    if (f32->d.kind != KIND_F32) return fail(JV_ERR_INVALID, "lowrank_download: not an fp32 data set");
    if (rank_out) *rank_out = LR_K;
    std::lock_guard<std::mutex> lk(f32->sketch_mu);
    if (!f32->lr_rows.get()) return fail(JV_ERR_INVALID, f32->lr_off ? "lowrank_download: the data set has no low-rank rows" : "lowrank_download: no sketched search has run");
    if (basis_out) CK(cudaMemcpy(basis_out, f32->lr_basis.get(), (size_t)LR_K * f32->d.stride * 4, cudaMemcpyDeviceToHost), "D2H low-rank basis");
    if (rows_out) CK(cudaMemcpy(rows_out, f32->lr_rows.get(), (size_t)f32->d.n * LR_SLOT, cudaMemcpyDeviceToHost), "D2H low-rank rows");
    return JV_OK;
}

int jv_graph_edge_records_download(jv_graph g, uint8_t *out)
{
    ON_DEVICE_OF(g);
    std::lock_guard<std::mutex> lk(g->edge_mu);
    if (!g->edge_rec) return fail(JV_ERR_INVALID, "edge_records_download: no edge records");
    if (out) CK(cudaMemcpy(out, g->edge_rec->get(), (size_t)g->g.n * g->g.degree * LR_SLOT, cudaMemcpyDeviceToHost), "D2H edge records");
    return JV_OK;
}

// modified Gram-Schmidt over the LR_K columns (rows of v, `stride` apart) in double; a column that vanishes becomes 0
static void orthonormalise(std::vector<double> &v, int stride)
{
    for (int j = 0; j < LR_K; j++) {
        double *vj = v.data() + (size_t)j * stride;
        for (int i = 0; i < j; i++) {
            const double *vi = v.data() + (size_t)i * stride;
            double d = 0.0;
            for (int x = 0; x < stride; x++) d += vi[x] * vj[x];
            for (int x = 0; x < stride; x++) vj[x] -= d * vi[x];
        }
        double nn = 0.0;
        for (int x = 0; x < stride; x++) nn += vj[x] * vj[x];
        nn = std::sqrt(nn);
        for (int x = 0; x < stride; x++) vj[x] = nn > 1e-300 ? vj[x] / nn : 0.0;
    }
}

// The low-rank rows of a data set (scorers.cuh lowrank_bound), caller holds sketch_mu. The basis: LR_BASIS_ITERS steps of subspace
// iteration over LR_BASIS_ROWS evenly spaced rows, started from the first LR_K of them. The bound only pays where the rows lie close
// to a rank-LR_K subspace: if the median rho / ||x|| over the sampled rows exceeds LR_MAX_RESIDUAL the data set gets none (an
// isotropic data set would read the edge records and settle almost nothing on them).
constexpr int LR_BASIS_ROWS = 4096, LR_BASIS_ITERS = 4;
constexpr double LR_MAX_RESIDUAL = 0.5;
static int ensure_lowrank(jv_dataset ds, cudaStream_t s)
{
    static std::atomic<uint64_t> next_id{1};
    const int stride = ds->d.stride;
    const long long n = ds->d.n;
    const int S = (int)std::min<long long>(n, LR_BASIS_ROWS);
    const long long step = std::max<long long>(1, n / LR_BASIS_ROWS);
    DeviceBuffer V, Z, Y, B, rows;
    if (n < LR_K || lowrank_warps(stride) == 0 || V.alloc((size_t)LR_K * stride * 8) != cudaSuccess || Y.alloc((size_t)LR_K * stride * 8) != cudaSuccess ||
        Z.alloc((size_t)S * LR_K * 8) != cudaSuccess || B.alloc((size_t)LR_K * stride * 4) != cudaSuccess || rows.alloc((size_t)n * LR_SLOT) != cudaSuccess) {
        cudaGetLastError();  // out of memory (or too few rows): the walk keeps the sketch alone
        ds->lr_off = true;
        return JV_OK;
    }
    // every copy and kernel below runs on `s` (a non-blocking stream: the legacy default stream would not order against it), and the
    // host waits for `s` before it reads or rewrites a host buffer the stream uses
    std::vector<float> x0((size_t)LR_K * stride);
    CK(cudaMemcpy2DAsync(x0.data(), (size_t)stride * 4, ds->d.rows, (size_t)step * stride * 4, (size_t)stride * 4, LR_K, cudaMemcpyDeviceToHost, s), "D2H basis rows");
    CK(cudaStreamSynchronize(s), "D2H basis rows");
    std::vector<double> v(x0.begin(), x0.end());
    orthonormalise(v, stride);
    for (int it = 0; it < LR_BASIS_ITERS; it++) {
        CK(cudaMemcpyAsync(V.get(), v.data(), v.size() * 8, cudaMemcpyHostToDevice, s), "H2D basis");
        CK(launch_lowrank_iteration(ds->d.rows, stride, step, S, V.get<double>(), Z.get<double>(), Y.get<double>(), s), "lowrank_iteration");
        CK(cudaMemcpyAsync(v.data(), Y.get(), v.size() * 8, cudaMemcpyDeviceToHost, s), "D2H basis");
        CK(cudaStreamSynchronize(s), "lowrank_iteration");
        orthonormalise(v, stride);
    }
    std::vector<float> bf(v.begin(), v.end());
    CK(cudaMemcpyAsync(B.get(), bf.data(), bf.size() * 4, cudaMemcpyHostToDevice, s), "H2D basis");
    cudaError_t e = launch_lowrank_rows(ds->d.rows, n, stride, B.get<float>(), rows.get<uint8_t>(), s);
    std::vector<float4> meta(S);
    if (e == cudaSuccess) e = cudaMemcpy2DAsync(meta.data(), 16, rows.get<uint8_t>() + LR_K, (size_t)step * LR_SLOT, 16, S, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    CK(e, "lowrank_rows");
    std::vector<double> ratio;
    for (const float4 &m : meta)
        if (m.w > 0.f) ratio.push_back((double)m.y / m.w);
    if (ratio.empty()) {
        ds->lr_off = true;
        return JV_OK;
    }
    std::nth_element(ratio.begin(), ratio.begin() + ratio.size() / 2, ratio.end());
    if (ratio[ratio.size() / 2] > LR_MAX_RESIDUAL) {
        ds->lr_off = true;
        return JV_OK;
    }
    ds->lr_basis = std::move(B);
    ds->lr_rows = std::move(rows);
    ds->lr_id = next_id++;
    return JV_OK;
}

// the edge records of graph g for data set ds's low-rank rows, built once per (graph, data set build). *out: the records (empty when
// there are none), which the caller holds until its kernels have finished
static int ensure_edge_records(jv_graph g, jv_dataset ds, cudaStream_t s, std::shared_ptr<DeviceBuffer> *out)
{
    out->reset();
    uint64_t id;
    const uint8_t *lr;
    {
        std::lock_guard<std::mutex> lk(ds->sketch_mu);
        id = ds->lr_id;
        lr = ds->lr_rows.get<uint8_t>();
    }
    if (!id || g->g.n <= 0) return JV_OK;
    std::lock_guard<std::mutex> lk(g->edge_mu);
    if (g->edge_rec_of != id) {
        g->edge_rec.reset();  // freed here unless a running search still holds it (then when that search ends)
        g->edge_rec_of = 0;
        auto rec = std::make_shared<DeviceBuffer>();
        if (rec->alloc((size_t)g->g.n * g->g.degree * LR_SLOT) != cudaSuccess) {
            cudaGetLastError();  // out of memory: the walk keeps the sketch alone
            return JV_OK;
        }
        cudaError_t e = launch_edge_records(g->g.adj0, g->g.n, g->g.degree, lr, rec->get<uint8_t>(), s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        CK(e, "edge_records");
        g->edge_rec = std::move(rec);
        g->edge_rec_of = id;
    }
    *out = g->edge_rec;
    return JV_OK;
}

// the fp32 row sketch of a data set (row_sketch_kernel), built once, and its low-rank rows (ensure_lowrank). Complete when this
// returns: another thread's stream may read them
static int ensure_sketch(jv_dataset ds, cudaStream_t s)
{
    std::lock_guard<std::mutex> lk(ds->sketch_mu);
    if (ds->sketch.get() || ds->sketch_failed) return JV_OK;
    const int ss = sketch_stride(ds->d.stride);
    DeviceBuffer sk, meta;
    if (sk.alloc((size_t)ds->d.n * ss) != cudaSuccess || meta.alloc((size_t)ds->d.n * sizeof(float2)) != cudaSuccess) {
        cudaGetLastError();  // out of memory: not an error of the search, which walks without the sketch
        ds->sketch_failed = true;
        return JV_OK;
    }
    cudaError_t e = launch_row_sketch(ds->d.rows, ds->d.n, ds->d.stride, ss, sk.get<int8_t>(), meta.get<float2>(), s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    CK(e, "row_sketch");
    ds->sketch = std::move(sk);
    ds->sketch_meta = std::move(meta);
    return ensure_lowrank(ds, s);
}

// query_stride: floats between two queries (0: dim)
static int search_device(jv_graph g, jv_dataset approx, jv_dataset reranker, int metric, const float *queries_dev, int nq, int topK, int rerankK,
                         const SearchFilter *filter, int32_t *nodes_dev, float *scores_dev, jv_search_stats *stats, int query_stride = 0)
{
    if (!g || !approx || !queries_dev || !nodes_dev || !scores_dev || nq <= 0) return fail(JV_ERR_INVALID, "graph_search: bad arguments");
    if (topK < 1 || rerankK < topK) return fail(JV_ERR_INVALID, "graph_search: need 1 <= topK <= rerankK");
    if (rerankK > 4096) return fail(JV_ERR_INVALID, "graph_search: rerankK <= 4096");
    if (approx->d.n != g->g.n) return fail(JV_ERR_INVALID, "graph_search: data set and graph sizes differ");
    if (approx->device != g->device || (reranker && reranker->device != g->device)) return fail(JV_ERR_INVALID, "graph_search: graph and data sets live on different devices");
    if (reranker && (reranker->d.n != g->g.n || reranker->d.dim != approx->d.dim)) return fail(JV_ERR_INVALID, "graph_search: reranker shape mismatch");
    if (reranker && reranker->d.kind != KIND_F32 && reranker->d.kind != KIND_NVQ)
        return fail(JV_ERR_UNSUPPORTED, "graph_search: the reranker must be fp32 or NVQ (OnDiskGraphIndex.java:705-713)");
    int rc = check_metric(approx->d, metric);
    if (rc) return rc;
    if ((rc = t_ctx.init())) return rc;
    cudaStream_t s = t_ctx.stream;
    if (g->g.entry_node < 0) {
        // every node was removed (jv_graph_remove_deleted): no entry point, nothing to walk
        CK(cudaMemsetAsync(nodes_dev, 0xff, (size_t)nq * topK * 4, s), "memset nodes");
        CK(cudaMemsetAsync(scores_dev, 0, (size_t)nq * topK * 4, s), "memset scores");
        CK(cudaStreamSynchronize(s), "sync");
        if (stats) memset(stats, 0, sizeof(*stats));
        return JV_OK;
    }
    const DataDesc *rr = reranker ? &reranker->d : nullptr;
    SearchPlan plan;
    // JV_VISITED_CAP / JV_LIST_CAP: first visited-table / candidate-list sizes (testing and tuning knobs; queries that outgrow
    // either are re-run below with 4x)
    const char *cap_env = getenv("JV_VISITED_CAP");
    const char *lcap_env = getenv("JV_LIST_CAP");
    const int cap_hint = cap_env ? atoi(cap_env) : 0, lcap_hint = lcap_env ? atoi(lcap_env) : 0;
    CK(plan_search(approx->d, rr, g->g, topK, rerankK, nq, cap_hint > 0 ? cap_hint : 0, lcap_hint > 0 ? lcap_hint : 0, g_sm_count, &plan), "plan_search");
    // A walk that drops hopeless neighbours on a bound from the row sketch (launch_search): the first such batch builds the sketch.
    // Without it (the allocation failed) the walk reads every full row, with the same answers.
    DataDesc ad = approx->d;
    if (search_uses_sketch(ad, metric, plan, nq) && (rc = ensure_sketch(approx, s))) return rc;
    if (ad.kind == KIND_F32) {
        std::lock_guard<std::mutex> lk(approx->sketch_mu);
        ad.sketch = approx->sketch.get<int8_t>();
        ad.sketch_meta = approx->sketch_meta.get<float2>();
        ad.sketch_stride = sketch_stride(ad.stride);
        ad.lr_basis = approx->lr_basis.get<float>();
    }
    // a sketched walk over a data set with low-rank rows settles most hopeless neighbours at gather time on the graph's edge records
    GraphDesc gd = g->g;
    std::shared_ptr<DeviceBuffer> edge_rec;  // held until this function returns: every path out of it has synchronised `s`
    if (ad.sketch && ad.lr_basis && search_uses_sketch(ad, metric, plan, nq) && (rc = ensure_edge_records(g, approx, s, &edge_rec))) return rc;
    gd.edge_rec = edge_rec ? edge_rec->get<uint8_t>() : nullptr;
    // counters, work counter, per-query overflow codes, retry index (carved over nullptr: the block's size)
    SearchCounters *dcnt;
    int *dwork;
    uint8_t *dover;
    int32_t *dindex;
    auto carve = [&](void *base) {
        Carver c(base);
        dcnt = c.take<SearchCounters>(1);
        dwork = c.take<int>(1);
        dover = c.take<uint8_t>(nq);
        dindex = c.take<int32_t>(nq);
        return c.bytes;
    };
    if ((rc = grow(t_ctx.search_aux, carve(nullptr)))) return rc;
    carve(t_ctx.search_aux.get());
    CK(cudaMemsetAsync(dcnt, 0, sizeof(SearchCounters), s), "memset counters");
    SearchCounters hc;
    float ms = 0.f;
    long long retried = 0;
    int cap = plan.visited_cap, lcap = plan.list_cap;
    std::vector<int32_t> idx;  // the queries an attempt after the first re-runs
    for (int attempt = 0;; attempt++) {
        const int cnt = attempt ? (int)idx.size() : nq;
        if (attempt) {
            CK(plan_search(approx->d, rr, g->g, topK, rerankK, cnt, cap, lcap, g_sm_count, &plan), "plan_search(retry)");
            CK(cudaMemcpyAsync(dindex, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, s), "H2D retry index");
            unsigned long long zero = 0;
            CK(cudaMemcpyAsync(&dcnt->overflowed, &zero, sizeof(zero), cudaMemcpyHostToDevice, s), "reset overflow");
        }
        if ((rc = grow(t_ctx.search_scratch, search_scratch_bytes(plan)))) return rc;
        CK(t_ctx.timer.start(s), "event");
        CK(launch_search(gd, ad, rr, metric, queries_dev, cnt, topK, rerankK, plan, t_ctx.search_scratch.get(), dwork, nodes_dev, scores_dev, dcnt, dover,
                         attempt ? dindex : nullptr, query_stride, filter, s),
           "launch_search");
        CK(t_ctx.timer.stop(s), "event");
        CK(cudaMemcpyAsync(&hc, dcnt, sizeof(hc), cudaMemcpyDeviceToHost, s), "D2H counters");
        CK(cudaStreamSynchronize(s), "search kernel");
        ms += t_ctx.timer.ms();
        if (hc.overflowed == 0 || attempt == 6) break;
        // queries whose visited table filled up (code 1) or whose candidate list could not hold a tie tail (code 2) are re-run with a
        // 4x larger table / list: the result does not depend on either size, only whether the run completes does
        std::vector<uint8_t> hover(nq);
        CK(cudaMemcpy(hover.data(), dover, (size_t)nq, cudaMemcpyDeviceToHost), "D2H overflow flags");
        idx.clear();
        bool need_table = false, need_list = false;
        for (int i = 0; i < nq; i++)
            if (hover[i]) {
                idx.push_back(i);
                if (hover[i] == 1) need_table = true;
                else need_list = true;
            }
        if (idx.empty()) break;
        retried += (long long)idx.size();
        if (need_table) cap *= 4;
        if (need_list) {
            if (lcap >= MAX_LIST_CAP) return fail(JV_ERR_OVERFLOW, "graph_search: more equal-score (or filtered-out) candidates than the longest candidate list holds");
            lcap = std::min(MAX_LIST_CAP, lcap * 4);
        }
    }
    if (hc.overflowed > 0) return fail(JV_ERR_OVERFLOW, "graph_search: visited table / candidate list overflow after retries");
    if (stats) {
        stats->visited = (int64_t)hc.visited;
        stats->expanded = (int64_t)hc.expanded;
        stats->expanded_base = (int64_t)hc.expanded_base;
        stats->reranked = (int64_t)hc.reranked;
    }
    t_last_settled = (int64_t)hc.settled;
    t_last_direct[0] = (int64_t)hc.direct;
    t_last_direct[1] = (int64_t)hc.direct_dropped;
    if (stats) {
        stats->retried = retried;
        stats->device_ms = ms;
    }
    return JV_OK;
}

// jv_search_options -> device-side SearchFilter (the bitset is uploaded when it is a host pointer)
static int make_filter(const jv_search_options *opts, jv_graph g, int nq, bool bits_on_device, SearchFilter *f, bool *use)
{
    *use = false;
    memset(f, 0, sizeof(*f));
    if (!opts) return JV_OK;
    if (opts->threshold < 0.f || opts->rerank_floor < 0.f || opts->accept_stride_words < 0) return fail(JV_ERR_INVALID, "graph_search: negative threshold / rerankFloor / stride");
    f->threshold = opts->threshold;
    f->rerank_floor = opts->rerank_floor;
    f->lenient = 0;
    f->accept_stride_words = opts->accept_stride_words;
    if (opts->accept_bits) {
        const size_t words = ((size_t)g->g.n + 31) / 32;
        if (opts->accept_stride_words != 0 && (size_t)opts->accept_stride_words < words) return fail(JV_ERR_INVALID, "graph_search: accept_stride_words shorter than one bitset");
        if (bits_on_device) f->accept_bits = opts->accept_bits;
        else {
            const size_t total = opts->accept_stride_words ? (size_t)opts->accept_stride_words * (size_t)(nq - 1) + words : words;
            int rc = grow(t_ctx.accept_bits, total * 4);
            if (rc) return rc;
            CK(cudaMemcpyAsync(t_ctx.accept_bits.get(), opts->accept_bits, total * 4, cudaMemcpyHostToDevice, t_ctx.stream), "H2D accept bits");
            f->accept_bits = t_ctx.accept_bits.get<uint32_t>();
        }
    }
    *use = f->accept_bits != nullptr || f->threshold > 0.f || f->rerank_floor > 0.f;
    return JV_OK;
}

int jv_graph_search_batch_device_ex(jv_graph g, jv_dataset approx, jv_dataset reranker, int metric, const float *queries_device, int nq, int topK,
                                    int rerankK, const jv_search_options *opts_device_bits, int32_t *nodes_out_device, float *scores_out_device,
                                    jv_search_stats *stats)
{
    ON_DEVICE_OF(g);
    if (!g || nq <= 0) return fail(JV_ERR_INVALID, "graph_search: bad arguments");
    int rc;
    if ((rc = t_ctx.init())) return rc;
    SearchFilter f;
    bool use;
    if ((rc = make_filter(opts_device_bits, g, nq, true, &f, &use))) return rc;
    return search_device(g, approx, reranker, metric, queries_device, nq, topK, rerankK, use ? &f : nullptr, nodes_out_device, scores_out_device, stats);
}

int jv_graph_search_batch_device(jv_graph g, jv_dataset approx, jv_dataset reranker, int metric, const float *queries_device, int nq, int topK,
                                 int rerankK, int32_t *nodes_out_device, float *scores_out_device, jv_search_stats *stats)
{
    return jv_graph_search_batch_device_ex(g, approx, reranker, metric, queries_device, nq, topK, rerankK, nullptr, nodes_out_device, scores_out_device, stats);
}

int jv_graph_search_batch_ex(jv_graph g, jv_dataset approx, jv_dataset reranker, int metric, const float *queries, int nq, int topK, int rerankK,
                             const jv_search_options *opts, int32_t *nodes_out, float *scores_out, jv_search_stats *stats)
{
    ON_DEVICE_OF(g);
    if (!g || !approx || !queries || !nodes_out || !scores_out || nq <= 0 || topK < 1) return fail(JV_ERR_INVALID, "graph_search: bad arguments");
    int rc;
    const size_t qb = (size_t)nq * approx->d.dim * 4, ob = (size_t)nq * topK * 4;
    int32_t *dnodes;
    float *dscores;
    auto carve = [&](void *base) {
        Carver c(base);
        dnodes = c.take<int32_t>((size_t)nq * topK);
        dscores = c.take<float>((size_t)nq * topK);
        return c.bytes;
    };
    if ((rc = t_ctx.init()) || (rc = grow(t_ctx.input, qb)) || (rc = grow(t_ctx.output, carve(nullptr)))) return rc;
    carve(t_ctx.output.get());
    char *dq = t_ctx.input.get<char>();
    cudaStream_t s = t_ctx.stream;
    SearchFilter f;
    bool use;
    if ((rc = make_filter(opts, g, nq, false, &f, &use))) return rc;
    // Large batches: the queries travel in chunks on a second stream, each followed by a 4-byte watermark ("queries [0, w) have
    // arrived"), and the search kernel — launched at once — takes query i only when the watermark has passed it. The H2D copy
    // (30 MB at c2) hides behind the first wave of queries instead of preceding the kernel. JV_SEARCH_OVERLAP=0 disables.
    const char *ov = getenv("JV_SEARCH_OVERLAP");
    const bool overlap = qb >= ((size_t)1 << 20) && nq >= 64 && !(ov && ov[0] == '0');
    if (overlap) {
        if ((rc = t_ctx.init_copy()) || (rc = grow(t_ctx.watermark, sizeof(int)))) return rc;
        int *arrived = t_ctx.watermark.get<int>();
        CK(cudaMemsetAsync(arrived, 0, sizeof(int), s), "memset watermark");
        CK(cudaEventRecord(t_ctx.ev_copy, s), "event");
        cudaStream_t s2 = t_ctx.copy_stream;
        CK(cudaStreamSynchronize(s2), "copy stream");  // the pinned watermark values of the previous call are free again
        CK(cudaStreamWaitEvent(s2, t_ctx.ev_copy, 0), "wait");
        const int chunks = ThreadCtx::MARKS;
        const size_t row = (size_t)approx->d.dim * 4;
        for (int c = 0; c < chunks; c++) {
            // first chunk small (one kernel wave starts as early as possible), the rest equal. Boundaries are multiples of 32 queries:
            // 32 rows of 4 * dim bytes end on a 128-byte line, so no cache line holds queries of two chunks (a kernel that has read
            // the last query of a chunk can never hold a stale L1 copy of the first bytes of the next one)
            auto bound = [&](int c_) -> long long {
                if (c_ <= 0) return 0;
                if (c_ >= chunks) return nq;
                const long long rest = nq > 2048 ? nq - 2048 : 0;
                const long long b = 2048 + rest * (c_ - 1) / (chunks - 1);
                return std::min<long long>(nq, b & ~31ll);
            };
            const long long lo = bound(c), hi = bound(c + 1);
            if (hi <= lo) continue;
            CK(cudaMemcpyAsync(dq + (size_t)lo * row, (const char *)queries + (size_t)lo * row, (size_t)(hi - lo) * row, cudaMemcpyHostToDevice, s2), "H2D queries");
            int *mark = t_ctx.marks.get<int>() + c;
            *mark = (int)hi;
            CK(cudaMemcpyAsync(arrived, mark, sizeof(int), cudaMemcpyHostToDevice, s2), "H2D watermark");
        }
        f.arrived = arrived;
        rc = search_device(g, approx, reranker, metric, (const float *)dq, nq, topK, rerankK, &f, dnodes, dscores, stats);
    } else {
        CK(cudaMemcpyAsync(dq, queries, qb, cudaMemcpyHostToDevice, s), "H2D queries");
        rc = search_device(g, approx, reranker, metric, (const float *)dq, nq, topK, rerankK, use ? &f : nullptr, dnodes, dscores, stats);
    }
    if (rc) return rc;
    CK(cudaMemcpyAsync(nodes_out, dnodes, ob, cudaMemcpyDeviceToHost, s), "D2H nodes");
    CK(cudaMemcpyAsync(scores_out, dscores, ob, cudaMemcpyDeviceToHost, s), "D2H scores");
    CK(cudaStreamSynchronize(s), "sync");
    return JV_OK;
}

int jv_graph_search_batch(jv_graph g, jv_dataset approx, jv_dataset reranker, int metric, const float *queries, int nq, int topK, int rerankK,
                          int32_t *nodes_out, float *scores_out, jv_search_stats *stats)
{
    return jv_graph_search_batch_ex(g, approx, reranker, metric, queries, nq, topK, rerankK, nullptr, nodes_out, scores_out, stats);
}

// ------------------------------------------------------------------------------------------------ segments
constexpr int MAX_SEGMENTS = 1024;  // the merge key holds the segment in 10 bits (and the list position in 12)

int jv_segments_search_batch(const jv_search_segment *segments, int nsegments, int metric, const float *queries, int nq, int topK, int rerankK,
                             float threshold, float rerank_floor, int32_t *segments_out, int32_t *nodes_out, float *scores_out, jv_search_stats *stats,
                             jv_search_stats *segment_stats)
{
    if (!segments || !queries || !segments_out || !nodes_out || !scores_out) return fail(JV_ERR_INVALID, "segments_search: bad arguments");
    if (nsegments < 1 || nq <= 0 || topK < 1 || rerankK < topK) return fail(JV_ERR_INVALID, "segments_search: need nsegments >= 1, nq >= 1 and 1 <= topK <= rerankK");
    const int S = nsegments;
    for (int i = 0; i < S; i++)
        if (!segments[i].approx) return fail(JV_ERR_INVALID, "segments_search: segment " + std::to_string(i) + " has no data set");
    ON_DEVICE_OF(segments[0].approx);
    // ---- every check before any device work
    const jv_dataset a0 = segments[0].approx, r0 = segments[0].reranker;
    bool exhaustive = false;
    for (int i = 0; i < S; i++) {
        const jv_search_segment &sg = segments[i];
        const std::string who = "segments_search: segment " + std::to_string(i);
        const jv_dataset a = sg.approx, r = sg.reranker;
        if (a->device != a0->device || (sg.graph && sg.graph->device != a0->device) || (r && r->device != a0->device))
            return fail(JV_ERR_INVALID, who + " lives on another device");
        if (sg.graph && sg.graph->g.n != a->d.n) return fail(JV_ERR_INVALID, who + ": data set and graph sizes differ");
        if (a->d.kind != a0->d.kind || a->d.dim != a0->d.dim) return fail(JV_ERR_INVALID, who + ": data sets of different kinds or dims");
        if ((a->d.kind == KIND_PQ && (a->d.M != a0->d.M || a->d.k != a0->d.k)) || (a->d.kind == KIND_NVQ && a->d.nsub != a0->d.nsub))
            return fail(JV_ERR_INVALID, who + ": PQ data sets of different M or k, or NVQ data sets of different sub-vectors");
        if ((r == nullptr) != (r0 == nullptr) || (r && (r->d.kind != r0->d.kind || (r->d.kind == KIND_NVQ && r->d.nsub != r0->d.nsub))))
            return fail(JV_ERR_INVALID, who + ": rerankers mixed or of different kinds");
        if (!sg.graph) exhaustive = true;
    }
    int rc = check_metric(a0->d, metric);
    if (rc) return rc;
    if (!(threshold >= 0.f) || !(rerank_floor >= 0.f)) return fail(JV_ERR_INVALID, "segments_search: negative threshold / rerankFloor");
    if (S > MAX_SEGMENTS) return fail(JV_ERR_UNSUPPORTED, "segments_search: nsegments <= 1024");
    if ((long long)S * topK > SEGMENT_MERGE_MAX_KEYS) return fail(JV_ERR_UNSUPPORTED, "segments_search: nsegments * topK <= 16384 (the merge sorts them in shared memory)");
    if (rerankK > 4096 || (exhaustive && rerankK > 2048))
        return fail(JV_ERR_UNSUPPORTED, "segments_search: rerankK <= 4096, and <= 2048 with a segment without graph");
    std::vector<int> walked;  // the segments with a graph that has an entry, in segment order
    GraphDesc gmax;           // what the plan sizes for: the largest n and degree among them
    memset(&gmax, 0, sizeof(gmax));
    for (int i = 0; i < S; i++) {
        const jv_search_segment &sg = segments[i];
        const jv_dataset a = sg.approx, r = sg.reranker;
        jv_search_options o = {sg.accept_bits, 0, threshold, rerank_floor};
        if (!sg.graph) {
            if ((rc = exhaustive_check(a, r, metric, topK, rerankK, &o))) return rc;
            continue;
        }
        if (r && (r->d.n != a->d.n || r->d.dim != a->d.dim)) return fail(JV_ERR_INVALID, "segments_search: segment " + std::to_string(i) + ": reranker shape mismatch");
        if (r && r->d.kind != KIND_F32 && r->d.kind != KIND_NVQ)
            return fail(JV_ERR_UNSUPPORTED, "segments_search: the reranker must be fp32 or NVQ (OnDiskGraphIndex.java:705-713)");
        if (sg.graph->g.entry_node < 0) continue;  // every node removed: nothing to walk
        walked.push_back(i);
        gmax.n = std::max(gmax.n, sg.graph->g.n);
        gmax.degree = std::max(gmax.degree, sg.graph->g.degree);
    }
    const int W = (int)walked.size();
    const DataDesc *rr0 = r0 ? &r0->d : nullptr;
    const char *cap_env = getenv("JV_VISITED_CAP");
    const char *lcap_env = getenv("JV_LIST_CAP");
    const int cap_hint = cap_env ? std::max(0, atoi(cap_env)) : 0, lcap_hint = lcap_env ? std::max(0, atoi(lcap_env)) : 0;
    SearchPlan plan;
    if (W && (plan_search(a0->d, rr0, gmax, topK, rerankK, W * nq, cap_hint, lcap_hint, g_sm_count, &plan) != cudaSuccess ||
              plan.smem_bytes + sizeof(SegmentDesc) > 227 * 1024)) {
        cudaGetLastError();
        return fail(JV_ERR_UNSUPPORTED, "segments_search: no walk of these segments fits an SM (degree, rerankK or codebook too large)");
    }

    // ---- device buffers: queries, the walked segments' bitsets, descriptors, answers [S][nq][topK], overflow codes [S][nq],
    // counters [S], retry index, merged answers [nq][topK]
    std::vector<size_t> bits_off(S, 0);
    size_t bit_words = 0;
    for (int i : walked)
        if (segments[i].accept_bits) {
            bits_off[i] = bit_words;
            bit_words += ((size_t)segments[i].approx->d.n + 31) / 32;
        }
    const size_t rows = (size_t)S * nq, dim = (size_t)a0->d.dim;
    float *dq, *dscores, *mscores;
    uint32_t *dbits;
    SegmentDesc *ddesc;
    int32_t *dnodes, *dindex, *mseg, *mnodes;
    uint8_t *dover;
    SearchCounters *dcnt;
    int *dwork;
    auto carve = [&](void *base) {
        Carver c(base);
        dq = c.take<float>((size_t)nq * dim);
        dbits = c.take<uint32_t>(bit_words);
        ddesc = c.take<SegmentDesc>(W);
        dnodes = c.take<int32_t>(rows * topK);
        dscores = c.take<float>(rows * topK);
        dover = c.take<uint8_t>(rows);
        dcnt = c.take<SearchCounters>(S);
        dwork = c.take<int>(1);
        dindex = c.take<int32_t>(rows);
        mseg = c.take<int32_t>((size_t)nq * topK);
        mnodes = c.take<int32_t>((size_t)nq * topK);
        mscores = c.take<float>((size_t)nq * topK);
        return c.bytes;
    };
    if ((rc = t_ctx.init()) || (rc = grow(t_ctx.segments, carve(nullptr)))) return rc;
    carve(t_ctx.segments.get());
    cudaStream_t s = t_ctx.stream;
    CK(t_ctx.timer.start(s), "event");
    CK(cudaMemcpyAsync(dq, queries, (size_t)nq * dim * 4, cudaMemcpyHostToDevice, s), "H2D queries");
    if (bit_words) {
        std::vector<uint32_t> hb(bit_words);
        for (int i : walked)
            if (segments[i].accept_bits) memcpy(hb.data() + bits_off[i], segments[i].accept_bits, (((size_t)segments[i].approx->d.n + 31) / 32) * 4);
        CK(cudaMemcpyAsync(dbits, hb.data(), bit_words * 4, cudaMemcpyHostToDevice, s), "H2D accept bits");
        CK(cudaStreamSynchronize(s), "H2D accept bits");  // hb is a pageable host vector
    }
    CK(cudaMemsetAsync(dcnt, 0, sizeof(SearchCounters) * S, s), "memset counters");
    for (int i = 0; i < S; i++)
        if (segments[i].graph && segments[i].graph->g.entry_node < 0) {
            // every node removed: the segment answers nothing
            CK(cudaMemsetAsync(dnodes + (size_t)i * nq * topK, 0xff, (size_t)nq * topK * 4, s), "memset nodes");
            CK(cudaMemsetAsync(dscores + (size_t)i * nq * topK, 0, (size_t)nq * topK * 4, s), "memset scores");
        }

    // ---- the walks: one launch per group of segments prepared alike (with edge records, without), as search_device prepares one
    std::vector<long long> retried(S, 0);
    std::vector<SearchCounters> hc(S);
    memset(hc.data(), 0, sizeof(SearchCounters) * S);
    if (W) {
        const bool sketch = search_uses_sketch(a0->d, metric, plan, W * nq);
        std::vector<std::shared_ptr<DeviceBuffer>> edge_recs(W);  // held until the call returns: every path out of it synchronises `s`
        std::vector<SegmentDesc> desc(W);
        for (int l = 0; l < W; l++) {
            const int i = walked[l];
            const jv_dataset a = segments[i].approx;
            if (sketch && (rc = ensure_sketch(a, s))) return rc;
            SegmentDesc &d = desc[l];
            memset(&d, 0, sizeof(d));
            d.approx = a->d;
            if (d.approx.kind == KIND_F32) {
                std::lock_guard<std::mutex> lk(a->sketch_mu);
                d.approx.sketch = a->sketch.get<int8_t>();
                d.approx.sketch_meta = a->sketch_meta.get<float2>();
                d.approx.sketch_stride = sketch_stride(d.approx.stride);
                d.approx.lr_basis = a->lr_basis.get<float>();
            }
            d.g = segments[i].graph->g;
            if (d.approx.sketch && d.approx.lr_basis && sketch && (rc = ensure_edge_records(segments[i].graph, a, s, &edge_recs[l]))) return rc;
            d.g.edge_rec = edge_recs[l] ? edge_recs[l]->get<uint8_t>() : nullptr;
            search_walk_descs(d.g, d.approx, metric, sketch);
            d.rerank = r0 ? segments[i].reranker->d : d.approx;
            d.accept_bits = segments[i].accept_bits ? dbits + bits_off[i] : nullptr;
            d.slot = i;
        }
        // groups: the segments with edge records first, then the others (a stable partition keeps segment order inside each)
        std::vector<int> order(W);
        for (int l = 0; l < W; l++) order[l] = l;
        std::stable_partition(order.begin(), order.end(), [&](int l) { return desc[l].g.edge_rec != nullptr; });
        std::vector<SegmentDesc> sorted(W);
        for (int l = 0; l < W; l++) sorted[l] = desc[order[l]];
        CK(cudaMemcpyAsync(ddesc, sorted.data(), sizeof(SegmentDesc) * W, cudaMemcpyHostToDevice, s), "H2D segment descriptors");
        const int nedge = (int)std::count_if(sorted.begin(), sorted.end(), [](const SegmentDesc &d) { return d.g.edge_rec != nullptr; });
        struct Group { int first, count; std::vector<int32_t> idx; };
        std::vector<Group> groups;
        if (nedge) groups.push_back({0, nedge, {}});
        if (W > nedge) groups.push_back({nedge, W - nedge, {}});
        SearchFilter f;
        memset(&f, 0, sizeof(f));
        f.threshold = threshold;
        f.rerank_floor = rerank_floor;
        f.accept_bits = bit_words ? dbits : nullptr;  // marks the walk filtered: each segment reads its own bitset from its descriptor
        int cap = plan.visited_cap, lcap = plan.list_cap;
        for (int attempt = 0;; attempt++) {
            for (const Group &gr : groups) {
                const int cnt = attempt ? (int)gr.idx.size() : gr.count * nq;
                if (cnt == 0) continue;
                SearchPlan pl = plan;
                if (attempt) CK(plan_search(a0->d, rr0, gmax, topK, rerankK, cnt, cap, lcap, g_sm_count, &pl), "plan_search(retry)");
                else pl.ctas = (int)std::min<long long>((long long)plan.ctas, cnt);
                if ((rc = grow(t_ctx.search_scratch, search_scratch_bytes(pl)))) return rc;
                int32_t *gidx = dindex + (size_t)gr.first * nq;
                if (attempt) CK(cudaMemcpyAsync(gidx, gr.idx.data(), gr.idx.size() * 4, cudaMemcpyHostToDevice, s), "H2D retry index");
                GraphDesc gg = sorted[gr.first].g;  // the group's walk: its kind of walk, sized for the largest degree
                gg.n = gmax.n;
                gg.degree = gmax.degree;
                const SegmentGroup sgp{ddesc + gr.first, gr.count, nq};
                CK(launch_search(gg, sorted[gr.first].approx, r0 ? &sorted[gr.first].rerank : nullptr, metric, dq, cnt, topK, rerankK, pl,
                                 t_ctx.search_scratch.get(), dwork, dnodes, dscores, dcnt, dover, attempt ? gidx : nullptr, 0, &f, s, &sgp),
                   "launch_search(segments)");
                if (attempt) CK(cudaStreamSynchronize(s), "segments search");  // gr.idx is read by the copy above
            }
            CK(cudaMemcpyAsync(hc.data(), dcnt, sizeof(SearchCounters) * S, cudaMemcpyDeviceToHost, s), "D2H counters");
            CK(cudaStreamSynchronize(s), "segments search");
            bool over = false;
            for (int i : walked) over = over || hc[i].overflowed > 0;
            if (!over || attempt == 6) break;
            // pairs whose visited table filled up (code 1) or whose list could not hold a tie tail (code 2) are re-run with 4x, as
            // search_device re-runs queries
            std::vector<uint8_t> hover(rows);
            CK(cudaMemcpy(hover.data(), dover, rows, cudaMemcpyDeviceToHost), "D2H overflow flags");
            bool need_table = false, need_list = false;
            for (Group &gr : groups) {
                gr.idx.clear();
                for (int l = 0; l < gr.count; l++) {
                    const int slot = sorted[gr.first + l].slot;
                    if (!hc[slot].overflowed) continue;
                    for (int q = 0; q < nq; q++) {
                        const uint8_t o = hover[(size_t)slot * nq + q];
                        if (!o) continue;
                        gr.idx.push_back(l * nq + q);
                        retried[slot]++;
                        if (o == 1) need_table = true;
                        else need_list = true;
                    }
                    CK(cudaMemsetAsync(&dcnt[slot].overflowed, 0, sizeof(unsigned long long), s), "reset overflow");
                }
            }
            if (need_table) cap *= 4;
            if (need_list) {
                if (lcap >= MAX_LIST_CAP)
                    for (int i : walked)
                        if (hc[i].overflowed)
                            return fail(JV_ERR_OVERFLOW, "segments_search: segment " + std::to_string(i) +
                                                             ": more equal-score (or filtered-out) candidates than the longest candidate list holds");
                lcap = std::min(MAX_LIST_CAP, lcap * 4);
            }
        }
        for (int i : walked)
            if (hc[i].overflowed > 0) return fail(JV_ERR_OVERFLOW, "segments_search: segment " + std::to_string(i) + ": visited table / candidate list overflow after retries");
    }

    // ---- segments without a graph: jv_exhaustive_search_batch's device work into their rows of the same answers
    std::vector<int64_t> ex_visited(S, 0);
    std::vector<unsigned long long> ex_taken(S, 0);
    for (int i = 0; i < S; i++) {
        if (segments[i].graph) continue;
        const jv_search_options o = {segments[i].accept_bits, 0, threshold, rerank_floor};
        if ((rc = exhaustive_device(segments[i].approx, segments[i].reranker, metric, nullptr, dq, nq, topK, rerankK, &o, nullptr, nullptr,
                                    dnodes + (size_t)i * nq * topK, dscores + (size_t)i * nq * topK, &ex_visited[i], &ex_taken[i])))
            return rc;
    }

    // ---- the merge, and the answers back
    CK(launch_segment_merge(dnodes, dscores, nq, S, topK, mseg, mnodes, mscores, s), "segment_merge");
    CK(cudaMemcpyAsync(segments_out, mseg, (size_t)nq * topK * 4, cudaMemcpyDeviceToHost, s), "D2H segments");
    CK(cudaMemcpyAsync(nodes_out, mnodes, (size_t)nq * topK * 4, cudaMemcpyDeviceToHost, s), "D2H nodes");
    CK(cudaMemcpyAsync(scores_out, mscores, (size_t)nq * topK * 4, cudaMemcpyDeviceToHost, s), "D2H scores");
    CK(t_ctx.timer.stop(s), "event");
    CK(cudaStreamSynchronize(s), "sync");
    const double ms = t_ctx.timer.ms();
    t_last_settled = t_last_direct[0] = t_last_direct[1] = 0;
    for (int i : walked) {
        t_last_settled += (int64_t)hc[i].settled;
        t_last_direct[0] += (int64_t)hc[i].direct;
        t_last_direct[1] += (int64_t)hc[i].direct_dropped;
    }
    jv_search_stats total;
    memset(&total, 0, sizeof(total));
    for (int i = 0; i < S; i++) {
        jv_search_stats st;
        memset(&st, 0, sizeof(st));
        if (segments[i].graph) {
            st.visited = (int64_t)hc[i].visited;
            st.expanded = (int64_t)hc[i].expanded;
            st.expanded_base = (int64_t)hc[i].expanded_base;
            st.reranked = (int64_t)hc[i].reranked;
        } else {
            st.visited = ex_visited[i];
            st.reranked = (int64_t)ex_taken[i];
        }
        st.retried = retried[i];
        st.device_ms = ms;
        total.visited += st.visited;
        total.expanded += st.expanded;
        total.expanded_base += st.expanded_base;
        total.reranked += st.reranked;
        total.retried += st.retried;
        if (segment_stats) segment_stats[i] = st;
    }
    total.device_ms = ms;
    if (stats) *stats = total;
    return JV_OK;
}

int jv_graph_search_exclude(jv_graph g, jv_dataset approx, int metric, const float *queries, int nq, int topK, int rerankK,
                            const int32_t *exclude_ids, int32_t *nodes_out, float *scores_out, int64_t *counters_out)
{
    ON_DEVICE_OF(g);
    if (!approx || !queries || !exclude_ids || !nodes_out || !scores_out || nq <= 0 || topK < 1) return fail(JV_ERR_INVALID, "search_exclude: bad arguments");
    for (int i = 0; i < nq; i++)
        if (exclude_ids[i] < -1 || exclude_ids[i] >= g->g.n) return fail(JV_ERR_INVALID, "search_exclude: excluded id out of range");
    int rc;
    int32_t *dnodes, *dex;
    float *dscores;
    auto carve = [&](void *base) {
        Carver c(base);
        dnodes = c.take<int32_t>((size_t)nq * topK);
        dscores = c.take<float>((size_t)nq * topK);
        dex = c.take<int32_t>(nq);
        return c.bytes;
    };
    if ((rc = t_ctx.init()) || (rc = grow(t_ctx.input, (size_t)nq * approx->d.dim * 4)) || (rc = grow(t_ctx.output, carve(nullptr)))) return rc;
    carve(t_ctx.output.get());
    cudaStream_t s = t_ctx.stream;
    CK(cudaMemcpyAsync(t_ctx.input.get(), queries, (size_t)nq * approx->d.dim * 4, cudaMemcpyHostToDevice, s), "H2D queries");
    CK(cudaMemcpyAsync(dex, exclude_ids, (size_t)nq * 4, cudaMemcpyHostToDevice, s), "H2D excluded ids");
    SearchFilter f;
    memset(&f, 0, sizeof(f));
    f.exclude_ids = dex;
    jv_search_stats st;
    if ((rc = search_device(g, approx, nullptr, metric, t_ctx.input.get<float>(), nq, topK, rerankK, &f, dnodes, dscores, &st))) return rc;
    CK(cudaMemcpyAsync(nodes_out, dnodes, (size_t)nq * topK * 4, cudaMemcpyDeviceToHost, s), "D2H nodes");
    CK(cudaMemcpyAsync(scores_out, dscores, (size_t)nq * topK * 4, cudaMemcpyDeviceToHost, s), "D2H scores");
    CK(cudaStreamSynchronize(s), "sync");
    if (counters_out) {
        counters_out[0] = st.visited;
        counters_out[1] = st.expanded;
        counters_out[2] = st.expanded_base;
        counters_out[3] = st.reranked;
    }
    return JV_OK;
}

static int build_params_check(const jv_build_params *params, BuildParams *bp)
{
    if (params->degree < 1 || params->degree > 64 || params->beam_width < 1 || params->beam_width > 256 || params->overflow < 1.0f || params->alpha < 1.0f)
        return fail(JV_ERR_INVALID, "graph_build: need 1 <= degree <= 64, 1 <= beam <= 256, overflow >= 1, alpha >= 1");
    // the prune holds at most 256 candidates: a wider beam + window would silently lose the last window peers
    if (params->concurrent_window >= 0 && params->beam_width + params->concurrent_window > 256)
        return fail(JV_ERR_INVALID, "graph_build: need beam + concurrent_window <= 256");
    bp->degree = params->degree; bp->beam = params->beam_width; bp->overflow = params->overflow; bp->alpha = params->alpha;
    bp->max_batch = params->max_batch; bp->window = params->concurrent_window;
    return JV_OK;
}

// HNSW-style levels (GraphIndexBuilder.java:562-575): level(node) = floor(-ln(U) / ln(M)), node i takes draw i of the generator
static std::vector<int> draw_levels(int n, int degree, uint64_t seed)
{
    uint64_t st = seed ? seed : 0x9E3779B97F4A7C15ull;
    auto next_u = [&st]() {
        st ^= st << 13; st ^= st >> 7; st ^= st << 17;
        return ((st >> 11) + 1) * (1.0 / 9007199254740993.0);
    };
    const double ml = degree == 1 ? 1.0 : 1.0 / log((double)degree);
    std::vector<int> level(n);
    for (int i = 0; i < n; i++) level[i] = (int)(-log(next_u()) * ml);
    return level;
}

// the members of every level >= 1 (ascending ids) and the entry node (the first node of the top level)
static void assign_levels(int n, int degree, uint64_t seed, std::vector<std::vector<int32_t>> &members, int *entry)
{
    const std::vector<int> level = draw_levels(n, degree, seed);
    int maxl = 0;
    for (int i = 0; i < n; i++) maxl = std::max(maxl, level[i]);
    *entry = 0;
    for (int i = 0; i < n; i++)
        if (level[i] == maxl) { *entry = i; break; }
    members.assign(maxl, {});
    for (int i = 0; i < n; i++)
        for (int l = 1; l <= level[i]; l++) members[l - 1].push_back(i);
}

// one upper level: a Vamana graph over its members ids (local row r = node ids[r]), built by the device builder on the members'
// rows (one gather kernel), from nothing or from `seed` (local rows). ladj: [ids.size()][degree] in node ids. Synchronises `s`.
// A PQ data set (jv_graph_build_pq) gives the level its members' code rows; codebooks, centroid, magnitudes and pair tables are shared.
// A BQ data set (jv_graph_build_bq) gives it their word rows.
// the members ids of a level as a data set of their own, local row r = node ids[r] (one gather kernel on `s`): their fp32 rows, code
// rows or word rows in `rows`, the ids in `dids`; codebooks, centroid, magnitudes and pair tables are shared with ds
static cudaError_t gather_level(jv_dataset ds, const std::vector<int32_t> &ids, DeviceBuffer &rows, DeviceBuffer &dids, DataDesc *sub, cudaStream_t s)
{
    const int cnt = (int)ids.size();
    const bool codes = ds->d.kind == KIND_PQ || ds->d.kind == KIND_BQ;
    memset(sub, 0, sizeof(DataDesc));
    if (codes) *sub = ds->d;
    sub->kind = ds->d.kind; sub->dim = ds->d.dim; sub->stride = ds->d.stride; sub->n = cnt;
    cudaError_t e = rows.alloc(codes ? (size_t)cnt * code_row_bytes(*sub) : (size_t)cnt * sub->stride * 4);
    if (e == cudaSuccess) e = dids.alloc((size_t)cnt * 4);
    if (e == cudaSuccess) e = cudaMemcpyAsync(dids.get(), ids.data(), (size_t)cnt * 4, cudaMemcpyHostToDevice, s);
    if (codes) {
        if (e == cudaSuccess) e = launch_gather_codes(ds->d, dids.get<int32_t>(), cnt, rows.get(), s);
        if (sub->kind == KIND_BQ) sub->words = rows.get<unsigned long long>();
        else sub->codes = rows.get<uint8_t>();
    } else {
        if (e == cudaSuccess) e = launch_gather_rows(ds->d, dids.get<int32_t>(), cnt, rows.get<float>(), s);
        sub->rows = rows.get<float>();
    }
    return e;
}

static int build_level(jv_dataset ds, int metric, const BuildParams &bp, const std::vector<int32_t> &ids, const BuilderSeed *seed,
                       std::vector<int32_t> &ladj, cudaStream_t s)
{
    const int cnt = (int)ids.size(), degree = bp.degree;
    ladj.assign((size_t)cnt * degree, -1);
    if (cnt <= 1) return JV_OK;
    DataDesc sub;
    DeviceBuffer rows, adj, dids;  // the members' rows (fp32 rows, code rows or word rows), their adjacency, their ids
    cudaError_t e = gather_level(ds, ids, rows, dids, &sub, s);
    if (e == cudaSuccess) e = adj.alloc((size_t)cnt * degree * 4);
    BuildStats bs2;
    if (e == cudaSuccess) e = build_graph_flat(sub, metric, bp, adj.get<int32_t>(), g_sm_count, &bs2, s, seed);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ladj.data(), adj.get(), ladj.size() * 4, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return cuda_fail(e, "build upper level");
    for (auto &x : ladj)
        if (x >= 0) x = ids[x];
    return JV_OK;
}

// the hierarchy of a build: every upper level is a Vamana graph over its members, built by the same device builder on the members'
// rows. Without one (hierarchy false, or a single node) the build's entry is node 0.
static int build_upper_levels(jv_graph g, jv_dataset ds, int metric, const BuildParams &bp, bool hierarchy, uint64_t seed, cudaStream_t s)
{
    const int n = (int)ds->d.n;
    Levels members, adj;
    int entry = 0;
    if (hierarchy && n > 1) assign_levels(n, bp.degree, seed, members, &entry);
    for (const std::vector<int32_t> &ids : members) {
        adj.emplace_back();
        const int rc = build_level(ds, metric, bp, ids, nullptr, adj.back(), s);
        if (rc) return rc;
    }
    return g->set_levels(std::move(members), std::move(adj), entry);
}

// the whole build over an fp32, a PQ or a BQ data set whose arguments have been checked: level 0, then the upper levels
static int graph_build(jv_dataset ds, int metric, const jv_build_params *params, const BuildParams &bp, jv_graph *out, double *device_ms)
{
    int rc;
    if ((rc = t_ctx.init())) return rc;
    cudaStream_t s = t_ctx.stream;
    std::unique_ptr<jv_graph_s> g;
    if ((rc = jv_graph_s::create((int32_t)ds->d.n, params->degree, g))) return rc;
    StreamTimer timer;
    CK(timer.start(s), "event");
    BuildStats bs;
    cudaError_t e = build_graph_flat(ds->d, metric, bp, g->adj0.get<int32_t>(), g_sm_count, &bs, s);
    t_build_stats = bs;
    rc = e == cudaSuccess ? JV_OK : cuda_fail(e, "build_graph_flat");
    if (!rc) rc = build_upper_levels(g.get(), ds, metric, bp, params->add_hierarchy, params->seed, s);
    cudaError_t e1 = timer.stop(s);  // the upper levels are part of the build and of its time
    cudaStreamSynchronize(s);
    if (rc) return rc;
    CK(e1, "event");
    if (device_ms) *device_ms = timer.ms();
    *out = g.release();
    return JV_OK;
}

// the requirements of a build, add or removal over a data set of `kind` (fp32 rows, PQ codes: pqBuildScoreProvider, BQ words:
// bqBuildScoreProvider), in this order: the kind; the metric (checked as every call checks it; no BQ score uses it); a row the
// builder and the prune handle (the graph's degree for an add or a removal, params->degree for a build over codes; an fp32 build
// leaves it to build_params_check); with params (build and add) the build parameters; over PQ a LUT the prune holds next to its
// candidates (the builder's, or with params == nullptr the removal's tier), then the metric's centroid-pair table, built and kept
// on the data set when it has none (as jv_dataset_pq_pair_table does); over BQ no bit set past dim. Every refusal comes before any
// device work except the BQ padding check, one reduction over the last word of every row (bq_padding_set).
static int provider_check(jv_graph g, jv_dataset ds, int kind, int metric, const jv_build_params *params, BuildParams *bp, const char *who)
{
    const std::string w(who);
    if (ds->d.kind != kind)
        return fail(JV_ERR_INVALID, w + (kind == KIND_PQ ? ": needs a PQ data set" : kind == KIND_BQ ? ": needs a BQ data set" : ": needs an fp32 data set"));
    int rc = check_metric(ds->d, metric);
    if (rc) return rc;
    const int degree = g ? g->g.degree : params->degree;
    if (degree > 64 && (g || kind != KIND_F32))
        return fail(JV_ERR_UNSUPPORTED, w + ": degree " + std::to_string(degree) + " > 64, the largest row the builder and the prune handle");
    if (params) {
        if (g && params->degree != degree) return fail(JV_ERR_INVALID, w + ": params->degree differs from the graph's degree");
        if ((rc = build_params_check(params, bp))) return rc;
    }
    if (kind == KIND_PQ) {
        if (!(params ? pq_prune_fits(ds->d) : pq_repair_fits(ds->d, degree)))
            return fail(JV_ERR_UNSUPPORTED, w + ": a LUT of M * k = " + std::to_string(ds->d.M * ds->d.k) +
                                                " entries does not fit the prune's shared memory next to its candidates (DESIGN §4.3c, §4.3e)");
        return jv_dataset_pq_pair_table(ds, metric);
    }
    if (kind == KIND_BQ) {
        // the walk re-encodes its query with the bits past dim clear while the prune's pair scores read the raw words, so the two
        // would disagree on Hamming distances. BinaryQuantization.encode and jv_bq_encode_* never set them.
        if ((rc = t_ctx.init())) return rc;
        bool set = false;
        CK(bq_padding_set(ds->d, &set, t_ctx.stream), "bq padding check");
        if (set) return fail(JV_ERR_INVALID, w + ": a row of the BQ data set has bits set past dim " + std::to_string(ds->d.dim));
    }
    return JV_OK;
}

// jv_graph_build (kind = KIND_F32), jv_graph_build_pq (KIND_PQ) and jv_graph_build_bq (KIND_BQ)
static int graph_build_of(jv_dataset ds, int kind, int metric, const jv_build_params *params, jv_graph *out, double *device_ms)
{
    ON_DEVICE_OF(ds);
    if (!params || !out) return fail(JV_ERR_INVALID, "graph_build: null argument");
    BuildParams bp;
    const int rc = provider_check(nullptr, ds, kind, metric, params, &bp, "graph_build");
    if (rc) return rc;
    return graph_build(ds, metric, params, bp, out, device_ms);
}

int jv_graph_build(jv_dataset f32, int metric, const jv_build_params *params, jv_graph *out, double *device_ms)
{
    return graph_build_of(f32, KIND_F32, metric, params, out, device_ms);
}

int jv_graph_build_pq(jv_dataset pq, int metric, const jv_build_params *params, jv_graph *out, double *device_ms)
{
    return graph_build_of(pq, KIND_PQ, metric, params, out, device_ms);
}

int jv_graph_build_bq(jv_dataset bq, int metric, const jv_build_params *params, jv_graph *out, double *device_ms)
{
    return graph_build_of(bq, KIND_BQ, metric, params, out, device_ms);
}

static inline bool bit_of(const std::vector<uint32_t> &bits, int v) { return (bits[(size_t)v >> 5] >> (v & 31)) & 1u; }

// ------------------------------------------------------------------------------------------------ addGraphNode for a batch
// Nodes [n0, n) of a data set go into a graph of n0 nodes (GraphIndexBuilder.addGraphNode, base:graph/GraphIndexBuilder.java:588-659,
// for each of them): level 0 through a builder seeded with g's rows, then every upper level that gains members through a builder
// seeded with that level's rows. GraphAdd is what the add keeps of g, so that g is no longer read once the builder exists.
struct GraphAdd {
    int32_t n0 = 0, entry = -1;
    Levels level_ids, level_adj;                            // g's upper levels
    std::vector<uint32_t> removed;                          // g's holes (jv_graph_remove_deleted)
    std::vector<uint32_t> marks;                            // deleted_bits over the n0 old nodes; empty = none marked
    DeviceBuffer upper_row;                                 // g's id -> row maps of its upper levels, [levels - 1][n0]
};

// the accept bits of an insert over `rows` builder rows: row r < nold is node ids[r] (ids == nullptr: node r) and is refused when
// marked, the rows past nold are new nodes. Empty when nothing is marked: the insert searches then run unfiltered, as a build's do.
static std::vector<uint32_t> add_accept_bits(const GraphAdd &A, const int32_t *ids, int nold, int rows)
{
    std::vector<uint32_t> bits;
    if (A.marks.empty()) return bits;
    bits.assign(((size_t)rows + 31) / 32, 0u);
    for (int r = 0; r < rows; r++)
        if (r >= nold || !bit_of(A.marks, ids ? ids[r] : r)) bits[(size_t)r >> 5] |= 1u << (r & 31);
    return bits;
}

// the checks of an add over a data set of `kind` (KIND_F32: jv_graph_add_nodes, KIND_PQ: jv_graph_add_nodes_pq, KIND_BQ:
// jv_graph_add_nodes_bq)
static int add_check(jv_graph g, jv_dataset ds, int kind, int metric, const jv_build_params *params, BuildParams *bp)
{
    if (!ds || !params) return fail(JV_ERR_INVALID, "add_nodes: null argument");
    if (ds->device != g->device) return fail(JV_ERR_INVALID, "add_nodes: data set and graph live on different devices");
    if (ds->d.n < g->g.n || ds->d.n > INT32_MAX) return fail(JV_ERR_INVALID, "add_nodes: the data set must hold the graph's nodes first");
    return provider_check(g, ds, kind, metric, params, bp, "add_nodes");
}

// g's state into A and the seed of a level-0 builder over n rows (accept: the storage of its bits). Enqueues a copy of g's
// upper_row and, through the seed, a read of g's adjacency on `s`.
static int add_prepare(jv_graph g, const uint32_t *deleted_bits, int n, GraphAdd &A, std::vector<uint32_t> &accept, BuilderSeed *seed, cudaStream_t s)
{
    const int n0 = g->g.n;
    A.n0 = n0; A.entry = g->g.entry_node; A.level_ids = g->level_ids; A.level_adj = g->level_adj; A.removed = g->removed;
    if (deleted_bits) {
        const size_t W0 = ((size_t)n0 + 31) / 32;
        A.marks.assign(deleted_bits, deleted_bits + W0);
        if (n0 & 31) A.marks[W0 - 1] &= (1u << (n0 & 31)) - 1u;
    }
    if (!A.level_ids.empty()) {
        const size_t bytes = A.level_ids.size() * (size_t)n0 * 4;
        CK(A.upper_row.alloc(bytes), "cudaMalloc(upper_row)");
        CK(cudaMemcpyAsync(A.upper_row.get(), g->upper_row.get(), bytes, cudaMemcpyDeviceToDevice, s), "copy upper_row");
    }
    accept = add_accept_bits(A, nullptr, n0, n);
    *seed = {g->adj0.get<int32_t>(), n0, g->g.degree, nullptr, A.entry, accept.empty() ? nullptr : accept.data()};
    return JV_OK;
}

// the upper levels after an add. New node i joins the levels its draw i of draw_levels(n, M, seed) reaches, so a node's level does
// not depend on when it was added. A level of g that gains members is extended by a builder seeded with its rows: local rows are the
// old members in the level's order, then the new members ascending; the old rows are mapped to local rows through g's upper_row on
// the device; the inserts start at the entry's row (the level's first row if the entry is not a member). A level above g's top is
// built over its members, all new, and its lowest id becomes the entry.
// Over a PQ data set build_level gathers the members' code rows instead of their fp32 rows; nothing else differs.
static int add_upper_levels(const GraphAdd &A, jv_dataset ds, int metric, const BuildParams &bp, uint64_t seed, Levels &level_ids, Levels &level_adj,
                            int32_t *entry, cudaStream_t s)
{
    const int n = (int)ds->d.n, n0 = A.n0, degree = bp.degree, L = (int)A.level_ids.size();
    const std::vector<int> level = draw_levels(n, degree, seed);
    int top = L;
    for (int i = n0; i < n; i++) top = std::max(top, level[i]);
    for (int l = 1; l <= top; l++) {
        std::vector<int32_t> ids = l <= L ? A.level_ids[l - 1] : std::vector<int32_t>();
        const int nold = (int)ids.size();
        for (int i = n0; i < n; i++)
            if (level[i] >= l) ids.push_back(i);
        std::vector<int32_t> ladj;
        int rc = JV_OK;
        if (l > L) {
            rc = build_level(ds, metric, bp, ids, nullptr, ladj, s);
        } else if ((int)ids.size() == nold) {
            ladj = A.level_adj[l - 1];
        } else {
            const std::vector<int32_t> &old = A.level_adj[l - 1];
            DeviceBuffer rows;
            cudaError_t e = rows.alloc(std::max<size_t>(old.size(), 1) * 4);
            if (e == cudaSuccess) e = cudaMemcpyAsync(rows.get(), old.data(), old.size() * 4, cudaMemcpyHostToDevice, s);
            if (e != cudaSuccess) return cuda_fail(e, "add_nodes: upper level rows");
            const int at = (int)(std::find(ids.begin(), ids.begin() + nold, A.entry) - ids.begin());
            const std::vector<uint32_t> accept = add_accept_bits(A, ids.data(), nold, (int)ids.size());
            const BuilderSeed sd = {rows.get<int32_t>(), nold, degree, A.upper_row.get<int32_t>() + (size_t)(l - 1) * n0, at < nold ? at : 0,
                                    accept.empty() ? nullptr : accept.data()};
            rc = build_level(ds, metric, bp, ids, &sd, ladj, s);
        }
        if (rc) return rc;
        level_ids.push_back(std::move(ids));
        level_adj.push_back(std::move(ladj));
    }
    if (top > L) *entry = level_ids[top - 1][0];
    return JV_OK;
}

// the new graph around its level-0 adjacency (already in ng->adj0, ng sized to the data set): holes widened to n, upper levels, entry
static int add_finish(jv_graph_s *ng, const GraphAdd &A, jv_dataset ds, int metric, const BuildParams &bp, uint64_t seed, cudaStream_t s)
{
    const int n = (int)ds->d.n;
    int32_t entry = A.entry >= 0 ? A.entry : n > A.n0 ? A.n0 : -1;  // an empty graph's first new node is its entry (build.cu)
    if (!A.removed.empty()) {
        ng->removed = A.removed;
        ng->removed.resize(((size_t)n + 31) / 32, 0u);
    }
    Levels ids, adj;
    if (!A.level_ids.empty()) {
        const int rc = add_upper_levels(A, ds, metric, bp, seed, ids, adj, &entry, s);
        if (rc) return rc;
    }
    return ng->set_levels(std::move(ids), std::move(adj), entry);
}

// jv_graph_add_nodes (kind = KIND_F32), jv_graph_add_nodes_pq (KIND_PQ) and jv_graph_add_nodes_bq (KIND_BQ): the builder scores
// whatever kind of rows it is given
static int graph_add_nodes(jv_graph g, jv_dataset ds, int kind, int metric, const jv_build_params *params, const uint32_t *deleted_bits, jv_graph *out,
                           double *device_ms)
{
    ON_DEVICE_OF(g);
    if (!out) return fail(JV_ERR_INVALID, "add_nodes: null argument");
    BuildParams bp;
    int rc = add_check(g, ds, kind, metric, params, &bp);
    if (rc) return rc;
    if ((rc = t_ctx.init())) return rc;
    cudaStream_t s = t_ctx.stream;
    const int n0 = g->g.n, n = (int)ds->d.n, degree = g->g.degree;
    StreamTimer timer;
    CK(timer.start(s), "event");
    std::unique_ptr<jv_graph_s> ng;
    if ((rc = jv_graph_s::create(n, degree, ng))) return rc;
    BuildStats bs = {0, 0, 0, 0, 0};
    if (n == n0) {
        // nothing to insert: a copy of g
        CK(cudaMemcpyAsync(ng->adj0.get(), g->adj0.get(), (size_t)n * degree * 4, cudaMemcpyDeviceToDevice, s), "copy adjacency");
        ng->removed = g->removed;
        rc = ng->set_levels(g->level_ids, g->level_adj, g->g.entry_node);
    } else {
        GraphAdd A;
        std::vector<uint32_t> accept;
        BuilderSeed seed;
        rc = add_prepare(g, deleted_bits, n, A, accept, &seed, s);
        if (!rc) {
            const cudaError_t e = build_graph_flat(ds->d, metric, bp, ng->adj0.get<int32_t>(), g_sm_count, &bs, s, &seed);
            rc = e == cudaSuccess ? JV_OK : cuda_fail(e, "graph_add_nodes");
        }
        if (!rc) rc = add_finish(ng.get(), A, ds, metric, bp, params->seed, s);
    }
    t_build_stats = bs;
    const cudaError_t e1 = timer.stop(s);
    cudaStreamSynchronize(s);
    if (rc) return rc;
    CK(e1, "event");
    if (device_ms) *device_ms = timer.ms();
    *out = ng.release();
    return JV_OK;
}

int jv_graph_add_nodes(jv_graph g, jv_dataset f32, int metric, const jv_build_params *params, const uint32_t *deleted_bits, jv_graph *out,
                       double *device_ms)
{
    return graph_add_nodes(g, f32, KIND_F32, metric, params, deleted_bits, out, device_ms);
}

int jv_graph_add_nodes_pq(jv_graph g, jv_dataset pq, int metric, const jv_build_params *params, const uint32_t *deleted_bits, jv_graph *out,
                          double *device_ms)
{
    return graph_add_nodes(g, pq, KIND_PQ, metric, params, deleted_bits, out, device_ms);
}

int jv_graph_add_nodes_bq(jv_graph g, jv_dataset bq, int metric, const jv_build_params *params, const uint32_t *deleted_bits, jv_graph *out,
                          double *device_ms)
{
    return graph_add_nodes(g, bq, KIND_BQ, metric, params, deleted_bits, out, device_ms);
}

// ---- the same build advanced batch by batch, for a build SHARDED over several GPUs (BASELINE config 5) ----------------------
// Every rank holds a replica of the rows and of the adjacency. Per batch: each rank searches + prunes ITS slice of the batch
// (jv_builder_insert_slice -> rows in a caller buffer), the slices are all-gathered by the caller (NCCL; jvector_b200/parallel.py),
// every rank applies the whole batch deterministically (jv_builder_apply_new), then the rows that passed overflow * M are
// re-pruned slice-wise and exchanged the same way. The device pointers are the caller's (e.g. torch tensors = the NCCL buffers).
struct jv_builder_s {
    int device = 0;
    jv_dataset data = nullptr;  // fp32 rows, PQ codes (jv_builder_create_pq) or BQ words (jv_builder_create_bq)
    int metric = 0;
    jv_build_params params;
    BuildParams bp;
    GraphBuilder *B = nullptr;
    cudaStream_t stream = nullptr;
    StreamTimer timer;  // jv_builder_create to jv_builder_finish
    std::unique_ptr<GraphAdd> add;  // jv_builder_create_from_graph: the graph the builder extends
    ~jv_builder_s() { builder_destroy(B); }
};

// jv_builder_create (kind = KIND_F32), jv_builder_create_pq (KIND_PQ) and jv_builder_create_bq (KIND_BQ)
static int builder_of(jv_dataset ds, int kind, int metric, const jv_build_params *params, void *cuda_stream, jv_builder *out)
{
    ON_DEVICE_OF(ds);
    if (!params || !out) return fail(JV_ERR_INVALID, "builder_create: null argument");
    std::unique_ptr<jv_builder_s> b(new jv_builder_s());
    const int rc = provider_check(nullptr, ds, kind, metric, params, &b->bp, "builder_create");
    if (rc) return rc;
    b->device = ds->device; b->data = ds; b->metric = metric; b->params = *params; b->stream = (cudaStream_t)cuda_stream;
    CK(b->timer.start(b->stream), "event");
    CK(builder_create(ds->d, metric, b->bp, g_sm_count, &b->B, b->stream), "builder_create");
    *out = b.release();
    return JV_OK;
}

int jv_builder_create(jv_dataset f32, int metric, const jv_build_params *params, void *cuda_stream, jv_builder *out)
{
    return builder_of(f32, KIND_F32, metric, params, cuda_stream, out);
}

int jv_builder_create_pq(jv_dataset pq, int metric, const jv_build_params *params, void *cuda_stream, jv_builder *out)
{
    return builder_of(pq, KIND_PQ, metric, params, cuda_stream, out);
}

int jv_builder_create_bq(jv_dataset bq, int metric, const jv_build_params *params, void *cuda_stream, jv_builder *out)
{
    return builder_of(bq, KIND_BQ, metric, params, cuda_stream, out);
}

static int builder_from_graph(jv_graph g, jv_dataset ds, int kind, int metric, const jv_build_params *params, const uint32_t *deleted_bits,
                              void *cuda_stream, jv_builder *out)
{
    ON_DEVICE_OF(g);
    if (!out) return fail(JV_ERR_INVALID, "builder_create_from_graph: null argument");
    BuildParams bp;
    int rc = add_check(g, ds, kind, metric, params, &bp);
    if (rc) return rc;
    std::unique_ptr<jv_builder_s> b(new jv_builder_s());
    b->device = g->device; b->data = ds; b->metric = metric; b->params = *params; b->bp = bp; b->stream = (cudaStream_t)cuda_stream;
    b->add.reset(new GraphAdd());
    CK(b->timer.start(b->stream), "event");
    std::vector<uint32_t> accept;
    BuilderSeed seed;
    if ((rc = add_prepare(g, deleted_bits, (int)ds->d.n, *b->add, accept, &seed, b->stream))) return rc;
    CK(builder_create(ds->d, metric, bp, g_sm_count, &b->B, b->stream, &seed), "builder_create");
    CK(cudaStreamSynchronize(b->stream), "builder_create_from_graph");  // g has been read: the caller may free it
    *out = b.release();
    return JV_OK;
}

int jv_builder_create_from_graph(jv_graph g, jv_dataset f32, int metric, const jv_build_params *params, const uint32_t *deleted_bits,
                                 void *cuda_stream, jv_builder *out)
{
    return builder_from_graph(g, f32, KIND_F32, metric, params, deleted_bits, cuda_stream, out);
}

int jv_builder_create_from_graph_pq(jv_graph g, jv_dataset pq, int metric, const jv_build_params *params, const uint32_t *deleted_bits,
                                    void *cuda_stream, jv_builder *out)
{
    return builder_from_graph(g, pq, KIND_PQ, metric, params, deleted_bits, cuda_stream, out);
}

int jv_builder_create_from_graph_bq(jv_graph g, jv_dataset bq, int metric, const jv_build_params *params, const uint32_t *deleted_bits,
                                    void *cuda_stream, jv_builder *out)
{
    return builder_from_graph(g, bq, KIND_BQ, metric, params, deleted_bits, cuda_stream, out);
}

int jv_builder_info(jv_builder b, int *degree, int *row_cap, int *max_batch)
{
    if (!b) return fail(JV_ERR_INVALID, "builder_info: null");
    if (degree) *degree = builder_degree(b->B);
    if (row_cap) *row_cap = builder_row_cap(b->B);
    if (max_batch) *max_batch = builder_max_batch(b->B);
    return JV_OK;
}

int jv_builder_next_batch(jv_builder b, int32_t *first, int32_t *count)
{
    if (!b || !first || !count) return fail(JV_ERR_INVALID, "builder_next_batch: null");
    int f = 0, c = 0;
    const bool more = builder_next_batch(b->B, &f, &c);
    *first = f;
    *count = more ? c : 0;
    return JV_OK;
}

int jv_builder_insert_slice(jv_builder b, int32_t first, int32_t count, int32_t lo, int32_t hi, int32_t *rows_out_device, int32_t *deg_out_device)
{
    ON_DEVICE_OF(b);
    if (lo < 0 || hi > count || !rows_out_device || !deg_out_device) return fail(JV_ERR_INVALID, "builder_insert_slice: bad arguments");
    CK(builder_insert_slice(b->B, first, count, lo, hi, rows_out_device, deg_out_device, b->stream), "builder_insert_slice");
    return JV_OK;
}

int jv_builder_apply_new(jv_builder b, int32_t first, int32_t count, const int32_t *rows_device, const int32_t *deg_device, int32_t *overflow_rows)
{
    ON_DEVICE_OF(b);
    if (!rows_device || !deg_device) return fail(JV_ERR_INVALID, "builder_apply_new: bad arguments");
    CK(builder_apply_new(b->B, first, count, rows_device, deg_device, b->stream), "builder_apply_new");
    if (overflow_rows) {
        int c = 0;
        CK(builder_list_count(b->B, &c, b->stream), "builder_list_count");
        *overflow_rows = c;
    }
    return JV_OK;
}

int jv_builder_reprune_slice(jv_builder b, int32_t lo, int32_t hi, int32_t *rows_out_device, int32_t *deg_out_device)
{
    ON_DEVICE_OF(b);
    if (!rows_out_device || !deg_out_device || lo < 0) return fail(JV_ERR_INVALID, "builder_reprune_slice: bad arguments");
    CK(builder_reprune_slice(b->B, lo, hi, rows_out_device, deg_out_device, b->stream), "builder_reprune_slice");
    return JV_OK;
}

int jv_builder_apply_repruned(jv_builder b, int32_t count, const int32_t *rows_device, const int32_t *deg_device)
{
    ON_DEVICE_OF(b);
    CK(builder_apply_repruned(b->B, count, rows_device, deg_device, b->stream), "builder_apply_repruned");
    return JV_OK;
}

int jv_builder_collect_over_degree(jv_builder b, int32_t *rows)
{
    ON_DEVICE_OF(b);
    CK(builder_collect_over_degree(b->B, b->stream), "builder_collect_over_degree");
    int c = 0;
    CK(builder_list_count(b->B, &c, b->stream), "builder_list_count");
    if (rows) *rows = c;
    return JV_OK;
}

// compacts the level-0 adjacency into a graph; the upper levels (3 % of the nodes at M = 32) are built by every replica itself
int jv_builder_finish(jv_builder b, jv_graph *out, double *device_ms)
{
    ON_DEVICE_OF(b);
    if (!out) return fail(JV_ERR_INVALID, "builder_finish: null");
    int rc;
    if ((rc = t_ctx.init())) return rc;
    std::unique_ptr<jv_graph_s> g;
    if ((rc = jv_graph_s::create((int32_t)b->data->d.n, b->bp.degree, g))) return rc;
    BuildStats bs;
    cudaError_t e = builder_finish(b->B, g->adj0.get<int32_t>(), &bs, b->stream);
    t_build_stats = bs;
    CK(e, "builder_finish");
    if (b->add) rc = add_finish(g.get(), *b->add, b->data, b->metric, b->bp, b->params.seed, b->stream);  // the hierarchy follows the graph
    else rc = build_upper_levels(g.get(), b->data, b->metric, b->bp, b->params.add_hierarchy, b->params.seed, b->stream);
    if (rc) return rc;
    CK(b->timer.stop(b->stream), "event");
    cudaStreamSynchronize(b->stream);
    if (device_ms) *device_ms = b->timer.ms();
    *out = g.release();
    return JV_OK;
}

int jv_builder_stats(jv_builder b, int64_t *batches, int64_t *truncated_searches, int64_t *dropped_backlinks)
{
    ON_DEVICE_OF(b);
    BuildStats bs;
    CK(builder_stats(b->B, &bs, b->stream), "builder_stats");
    if (batches) *batches = bs.batches;
    if (truncated_searches) *truncated_searches = bs.truncated_searches;
    if (dropped_backlinks) *dropped_backlinks = bs.dropped_backlinks;
    return JV_OK;
}

int jv_builder_free(jv_builder b)
{
    if (!b) return JV_OK;
    cudaSetDevice(b->device);
    if (b->stream) cudaStreamSynchronize(b->stream);
    else cudaDeviceSynchronize();
    delete b;
    return JV_OK;
}

int jv_graph_build_stats(int64_t *scored_vectors, int64_t *batches, int64_t *dropped_backlinks)
{
    if (scored_vectors) *scored_vectors = t_build_stats.searched;
    if (batches) *batches = t_build_stats.batches;
    if (dropped_backlinks) *dropped_backlinks = t_build_stats.dropped_backlinks;
    return JV_OK;
}

// ------------------------------------------------------------------------------------------------ removeDeletedNodes

// one level of the repair on the device (repair_level, build.cu); level L >= 1 also hands back its repaired rows
static int remove_deleted_level(jv_graph g, jv_graph ng, jv_dataset ds, int metric, float alpha, uint64_t seed, int level, const std::vector<uint32_t> &dead,
                                const uint32_t *dead_dev, RepairStats *st, std::vector<int32_t> *adj_out, cudaStream_t s)
{
    const int n = g->g.n, degree = g->g.degree;
    const std::vector<int32_t> *ids = level ? &g->level_ids[level - 1] : nullptr;
    const int rows = level ? (int)ids->size() : n;
    std::vector<int32_t> members;
    for (int r = 0; r < rows; r++) {
        const int v = ids ? (*ids)[r] : r;
        if (!bit_of(dead, v)) members.push_back(v);
    }
    std::sort(members.begin(), members.end());
    // level 0: g's adjacency is copied into ng's and repaired there; an upper level: its host rows are uploaded as old and new rows
    DeviceBuffer dmem, dids, old_rows, new_rows;
    int32_t *dold = g->adj0.get<int32_t>(), *dnew = ng->adj0.get<int32_t>();
    cudaError_t e = dmem.alloc(std::max<size_t>(members.size(), 1) * 4);
    if (e == cudaSuccess && !members.empty()) e = cudaMemcpyAsync(dmem.get(), members.data(), members.size() * 4, cudaMemcpyHostToDevice, s);
    if (level == 0) {
        if (e == cudaSuccess) e = cudaMemcpyAsync(dnew, dold, (size_t)n * degree * 4, cudaMemcpyDeviceToDevice, s);
    } else {
        const std::vector<int32_t> &adj = g->level_adj[level - 1];
        if (e == cudaSuccess) e = dids.alloc((size_t)rows * 4);
        if (e == cudaSuccess) e = old_rows.alloc(adj.size() * 4);
        if (e == cudaSuccess) e = new_rows.alloc(adj.size() * 4);
        dold = old_rows.get<int32_t>();
        dnew = new_rows.get<int32_t>();
        if (e == cudaSuccess) e = cudaMemcpyAsync(dids.get(), ids->data(), (size_t)rows * 4, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dold, adj.data(), adj.size() * 4, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dnew, adj.data(), adj.size() * 4, cudaMemcpyHostToDevice, s);
    }
    const int32_t *rowmap = level ? g->upper_row.get<int32_t>() + (size_t)(level - 1) * n : nullptr;
    if (e == cudaSuccess)
        e = repair_level(ds->d, metric, alpha, degree, rows, dold, dnew, dids.get<int32_t>(), rowmap, dead_dev, dmem.get<int32_t>(), (int)members.size(), seed,
                         level, g_sm_count, st, s);
    if (e == cudaSuccess && level == 0) e = launch_clear_dead_rows(dnew, n, degree, dead_dev, s);
    if (e == cudaSuccess && level > 0) {
        adj_out->resize((size_t)rows * degree);
        e = cudaMemcpyAsync(adj_out->data(), dnew, adj_out->size() * 4, cudaMemcpyDeviceToHost, s);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    else cudaStreamSynchronize(s);  // the buffers above are freed on return
    return e == cudaSuccess ? JV_OK : cuda_fail(e, "graph_remove_deleted");
}

// jv_graph_remove_deleted (kind = KIND_F32), jv_graph_remove_deleted_pq (KIND_PQ) and jv_graph_remove_deleted_bq (KIND_BQ): repair_level
// dispatches its prune by kind. Every check comes before any device work, so a refused call has done none of it.
static int graph_remove_deleted(jv_graph g, jv_dataset ds, int kind, int metric, float alpha, uint64_t seed, const uint32_t *deleted_bits, jv_graph *out,
                                jv_remove_stats *stats)
{
    ON_DEVICE_OF(g);
    if (!ds || !deleted_bits || !out || !stats) return fail(JV_ERR_INVALID, "graph_remove_deleted: null argument");
    if (ds->d.n != g->g.n || ds->device != g->device) return fail(JV_ERR_INVALID, "graph_remove_deleted: data set and graph differ in size or device");
    if (!(alpha >= 1.0f)) return fail(JV_ERR_INVALID, "graph_remove_deleted: need alpha >= 1");
    int rc = provider_check(g, ds, kind, metric, nullptr, nullptr, "graph_remove_deleted");
    if (rc || (rc = t_ctx.init())) return rc;
    cudaStream_t s = t_ctx.stream;
    const int n = g->g.n, degree = g->g.degree;
    const size_t W = ((size_t)n + 31) / 32;
    // deleted now or removed earlier: both are gone from the new graph
    std::vector<uint32_t> dead(deleted_bits, deleted_bits + W);
    if (n & 31) dead[W - 1] &= (1u << (n & 31)) - 1u;
    long long holes = 0, gone = 0;
    for (size_t w = 0; w < W; w++) {
        const uint32_t h = g->removed.empty() ? 0u : g->removed[w];
        holes += __builtin_popcount(h);
        dead[w] |= h;
        gone += __builtin_popcount(dead[w]);
    }
    DeviceBuffer dead_buf;
    RepairStats st;
    memset(&st, 0, sizeof(st));
    StreamTimer timer;
    CK(timer.start(s), "event");
    std::unique_ptr<jv_graph_s> ng;
    if ((rc = jv_graph_s::create(n, degree, ng))) return rc;
    ng->removed = dead;
    cudaError_t e = dead_buf.alloc(W * 4);
    if (e == cudaSuccess) e = cudaMemcpyAsync(dead_buf.get(), dead.data(), W * 4, cudaMemcpyHostToDevice, s);
    rc = e == cudaSuccess ? JV_OK : cuda_fail(e, "graph_remove_deleted: allocation");
    const uint32_t *dead_dev = dead_buf.get<uint32_t>();
    if (!rc) rc = remove_deleted_level(g, ng.get(), ds, metric, alpha, seed, 0, dead, dead_dev, &st, nullptr, s);
    // upper levels: repaired on the device like level 0, then their deleted members are dropped from the host copies
    Levels level_ids, level_adj;
    for (int level = 1; !rc && level < g->g.levels; level++) {
        std::vector<int32_t> adj;
        rc = remove_deleted_level(g, ng.get(), ds, metric, alpha, seed, level, dead, dead_dev, &st, &adj, s);
        if (rc) break;
        const std::vector<int32_t> &ids = g->level_ids[level - 1];
        std::vector<int32_t> nids, nadj;
        for (size_t r = 0; r < ids.size(); r++) {
            if (bit_of(dead, ids[r])) continue;
            nids.push_back(ids[r]);
            nadj.insert(nadj.end(), adj.begin() + r * degree, adj.begin() + (r + 1) * degree);
        }
        level_ids.push_back(std::move(nids));
        level_adj.push_back(std::move(nadj));
    }
    if (!rc) {
        // entry (GraphIndexBuilder.java:769-786): kept while it lives; otherwise the lowest live id of the highest level that still has a
        // live member, with the emptied levels above it dropped (the entry must belong to the top level)
        int entry = g->g.entry_node;
        if (entry < 0 || bit_of(dead, entry)) {
            entry = -1;
            int top = (int)level_ids.size();
            while (top > 0 && level_ids[top - 1].empty()) top--;
            level_ids.resize(top);
            level_adj.resize(top);
            if (top > 0) entry = *std::min_element(level_ids[top - 1].begin(), level_ids[top - 1].end());
            else
                for (int v = 0; v < n; v++)
                    if (!bit_of(dead, v)) { entry = v; break; }
        }
        rc = ng->set_levels(std::move(level_ids), std::move(level_adj), entry);
    }
    timer.stop(s);
    cudaStreamSynchronize(s);
    if (rc) return rc;
    stats->live_nodes = (int32_t)(n - gone);
    stats->removed = (int32_t)(gone - holes);
    stats->repaired_rows = st.repaired_rows;
    stats->candidates = st.candidates;
    stats->max_candidates = st.max_candidates;
    stats->random_fallbacks = st.random_fallbacks;
    stats->device_ms = timer.ms();
    *out = ng.release();
    return JV_OK;
}

int jv_graph_remove_deleted(jv_graph g, jv_dataset f32, int metric, float alpha, uint64_t seed, const uint32_t *deleted_bits, jv_graph *out,
                            jv_remove_stats *stats)
{
    return graph_remove_deleted(g, f32, KIND_F32, metric, alpha, seed, deleted_bits, out, stats);
}

int jv_graph_remove_deleted_pq(jv_graph g, jv_dataset pq, int metric, float alpha, uint64_t seed, const uint32_t *deleted_bits, jv_graph *out,
                               jv_remove_stats *stats)
{
    return graph_remove_deleted(g, pq, KIND_PQ, metric, alpha, seed, deleted_bits, out, stats);
}

int jv_graph_remove_deleted_bq(jv_graph g, jv_dataset bq, int metric, float alpha, uint64_t seed, const uint32_t *deleted_bits, jv_graph *out,
                               jv_remove_stats *stats)
{
    return graph_remove_deleted(g, bq, KIND_BQ, metric, alpha, seed, deleted_bits, out, stats);
}

// ------------------------------------------------------------------------------------------------ OnDiskGraphIndexCompactor
// Merging S graphs into one (DESIGN §4.3h): per level, the live members of every source are the rows, source by source. Every other
// source t is searched once per level for all of them (the search kernel over t, or over t's sub-hierarchy from level L up), the
// assembly kernel writes each row's candidates under their new ids and the repair's ragged prune picks its neighbours.

// one source as the compaction sees it: the new id of every live node (-1: dead or a hole), and per level its live members in the
// level's order with their rows in the level's adjacency
struct CompactSource {
    jv_graph g;
    jv_dataset ds;
    jv_dataset pq = nullptr;  // the fused form (jv_graph_compact_pq): the source's codes, which its searches walk (ds reranks)
    std::vector<int32_t> map;
    std::vector<std::vector<int32_t>> live, live_row;
};

// source t's level L (>= 1) and everything above it as a graph of its own: node p is t's p-th member of level L, its rows are the
// members' rows (gathered on `s`) and, when t.pq is set, sp holds their code rows (t.pq's codebooks, centroid and magnitudes; the
// graph has no FusedPQ records); the search of it descends from t's entry exactly as a search of t would down to level L
static int compact_sub_hierarchy(const CompactSource &t, int L, std::unique_ptr<jv_graph_s> &sg, std::unique_ptr<jv_dataset_s> &sd,
                                 std::unique_ptr<jv_dataset_s> &sp, cudaStream_t s)
{
    const jv_graph_s &g = *t.g;
    const std::vector<int32_t> &ids = g.level_ids[L - 1];
    const int m = (int)ids.size(), degree = g.g.degree;
    std::vector<int32_t> pos(g.g.n, -1);
    for (int p = 0; p < m; p++) pos[ids[p]] = p;
    auto remap = [&](const std::vector<int32_t> &a) {
        std::vector<int32_t> r(a.size());
        for (size_t i = 0; i < a.size(); i++) r[i] = a[i] >= 0 ? pos[a[i]] : -1;
        return r;
    };
    sd.reset(new jv_dataset_s(KIND_F32, m, t.ds->d.dim));
    float *rows;
    int32_t *dids;
    int rc = sd->alloc_rows(&rows);
    if (rc || (rc = sd->alloc(&dids, (size_t)m * 4))) return rc;
    CK(cudaMemcpyAsync(dids, ids.data(), (size_t)m * 4, cudaMemcpyHostToDevice, s), "H2D members");
    CK(launch_gather_rows(t.ds->d, dids, m, rows, s), "gather member rows");
    if (t.pq) {
        sp.reset(new jv_dataset_s(KIND_PQ, m, t.pq->d.dim));
        sp->d = t.pq->d;
        sp->d.n = m;
        uint8_t *codes;
        if ((rc = sp->alloc(&codes, (size_t)m * code_row_bytes(sp->d)))) return rc;
        CK(launch_gather_codes(t.pq->d, dids, m, codes, s), "gather member codes");
        sp->d.codes = codes;
    }
    const std::vector<int32_t> adj = remap(g.level_adj[L - 1]);
    if ((rc = jv_graph_s::create(m, degree, sg))) return rc;
    CK(cudaMemcpy(sg->adj0.get(), adj.data(), adj.size() * 4, cudaMemcpyHostToDevice), "H2D sub-hierarchy");
    Levels up_ids, up_adj;
    for (size_t l = L; l < g.level_ids.size(); l++) {
        up_ids.push_back(remap(g.level_ids[l]));
        up_adj.push_back(remap(g.level_adj[l]));
    }
    return sg->set_levels(std::move(up_ids), std::move(up_adj), pos[g.g.entry_node]);
}

// the searchTopK best live members of source t at level `level` for every row of the level that belongs to another source, into
// res [queries][K] (t's node ids, or member positions above level 0). qids: the queries' new ids (their rows in `merged`). The
// search walks t's fp32 rows exactly, or, when t.pq is set, t's codes (its FusedPQ records at level 0) with an exact rerank of
// its K survivors over t's rows (OnDiskGraphIndexCompactor.buildCrossSourceScoreProvider)
static int compact_search(const CompactSource &t, int level, jv_dataset merged, int metric, int K, const std::vector<int32_t> &qids, int32_t *res,
                          jv_compact_stats *stats, cudaStream_t s)
{
    constexpr int QUERY_CHUNK = 1 << 18;  // queries per search call: bounds the search's scratch and the gathered query rows
    std::unique_ptr<jv_graph_s> sg;
    std::unique_ptr<jv_dataset_s> sd, sp;
    jv_graph g = t.g;
    jv_dataset ds = t.ds, pq = t.pq;
    int rc;
    if (level > 0) {
        if ((rc = compact_sub_hierarchy(t, level, sg, sd, sp, s))) return rc;
        g = sg.get();
        ds = sd.get();
        pq = sp.get();
    }
    // accept bits: the live nodes of the searched graph (acceptOrds = live_t)
    const int n = g->g.n;
    std::vector<uint32_t> bits(((size_t)n + 31) / 32, 0u);
    for (size_t p = 0; p < t.live_row[level].size(); p++) {
        const int v = t.live_row[level][p];
        bits[v >> 5] |= 1u << (v & 31);
    }
    const int nq = (int)qids.size(), chunk = std::min(nq, QUERY_CHUNK), stride = merged->d.stride;
    std::vector<DeviceBuffer> mem;
    uint32_t *dbits;
    int32_t *dq;
    float *qrows, *scores;
    CK(alloc_owned(mem, dbits, bits.size() * 4), "cudaMalloc(accept bits)");
    CK(alloc_owned(mem, dq, (size_t)nq * 4), "cudaMalloc(query ids)");
    CK(alloc_owned(mem, qrows, (size_t)chunk * stride * 4), "cudaMalloc(query rows)");
    CK(alloc_owned(mem, scores, (size_t)chunk * K * 4), "cudaMalloc(search scores)");
    CK(cudaMemcpyAsync(dbits, bits.data(), bits.size() * 4, cudaMemcpyHostToDevice, s), "H2D accept bits");
    CK(cudaMemcpyAsync(dq, qids.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, s), "H2D query ids");
    SearchFilter f;
    memset(&f, 0, sizeof(f));
    f.accept_bits = dbits;
    for (int q0 = 0; q0 < nq; q0 += chunk) {
        const int c = std::min(chunk, nq - q0);
        CK(launch_gather_rows(merged->d, dq + q0, c, qrows, s), "gather query rows");
        jv_search_stats st;
        if ((rc = search_device(g, pq ? pq : ds, pq ? ds : nullptr, metric, qrows, c, K, K, &f, res + (size_t)q0 * K, scores, &st, stride))) return rc;
        stats->searches += c;
        stats->visited += st.visited;
    }
    return JV_OK;
}

// one level of the merge: the rows of every source's live members, their candidates and their pruned neighbours. Level 0 scatters
// the rows into ng's adjacency; an upper level hands back its members (ascending new ids) and their rows.
static int compact_level(const std::vector<CompactSource> &src, int level, int K, jv_dataset merged, int metric, float alpha, jv_graph_s *ng,
                         const std::vector<const int32_t *> &maps_dev, std::vector<int32_t> *ids_out, std::vector<int32_t> *adj_out,
                         jv_compact_stats *stats, cudaStream_t s)
{
    const int S = (int)src.size(), degree = ng->g.degree;
    std::vector<long long> start(S + 1, 0);
    std::vector<int32_t> row_node;
    for (int i = 0; i < S; i++) {
        start[i + 1] = start[i] + (long long)src[i].live[level].size();
        for (int32_t v : src[i].live[level]) row_node.push_back(src[i].map[v]);
    }
    const int rows = (int)start[S];
    const int cand_stride = degree + (S - 1) * K;
    std::vector<DeviceBuffer> mem;  // the level's scratch: every return below comes after the stream has drained
    int32_t *drow_node, *cand, *out_rows;
    long long *cand_off;
    int *cand_cnt;
    CompactTarget *dtargets;
    cudaError_t e = alloc_owned(mem, drow_node, (size_t)rows * 4);
    if (e == cudaSuccess) e = alloc_owned(mem, cand, (size_t)rows * cand_stride * 4);
    if (e == cudaSuccess) e = alloc_owned(mem, cand_off, (size_t)rows * 8);
    if (e == cudaSuccess) e = alloc_owned(mem, cand_cnt, (size_t)rows * 4);
    if (e == cudaSuccess) e = alloc_owned(mem, out_rows, (size_t)rows * degree * 4);
    if (e == cudaSuccess) e = alloc_owned(mem, dtargets, (size_t)S * sizeof(CompactTarget));
    if (e == cudaSuccess) e = cudaMemcpyAsync(drow_node, row_node.data(), (size_t)rows * 4, cudaMemcpyHostToDevice, s);
    CK(e, "graph_compact: level scratch");
    // per other source: its search results for the rows of every other source, in source order, or its whole live membership
    std::vector<CompactTarget> target(S, CompactTarget{nullptr, nullptr, nullptr, 0});
    std::vector<const int32_t *> pos_map(S, nullptr);
    int rc = JV_OK;
    for (int t = 0; t < S && !rc; t++) {
        const long long cnt = start[t + 1] - start[t], nq = rows - cnt;
        if (src[t].g->g.levels <= level || nq == 0) continue;
        if (cnt <= K) {
            target[t].list = drow_node + start[t];
            target[t].count = (int)cnt;
            stats->exhaustive += nq;
            continue;
        }
        std::vector<int32_t> qids(row_node.begin(), row_node.begin() + start[t]);
        qids.insert(qids.end(), row_node.begin() + start[t + 1], row_node.end());
        int32_t *res, *map = nullptr;
        if ((e = alloc_owned(mem, res, (size_t)nq * K * 4)) != cudaSuccess) { rc = cuda_fail(e, "cudaMalloc(search results)"); break; }
        if (level == 0) map = const_cast<int32_t *>(maps_dev[t]);
        else {
            // member position -> new id (-1: dead)
            const std::vector<int32_t> &ids = src[t].g->level_ids[level - 1];
            std::vector<int32_t> hm(ids.size());
            for (size_t p = 0; p < ids.size(); p++) hm[p] = src[t].map[ids[p]];
            e = alloc_owned(mem, map, hm.size() * 4);
            if (e == cudaSuccess) e = cudaMemcpyAsync(map, hm.data(), hm.size() * 4, cudaMemcpyHostToDevice, s);
            if (e != cudaSuccess) { rc = cuda_fail(e, "graph_compact: member map"); break; }
        }
        rc = compact_search(src[t], level, merged, metric, K, qids, res, stats, s);
        target[t].res = res;
        target[t].map = map;
    }
    // the candidate segments, source block by source block
    for (int i = 0; i < S && !rc; i++) {
        const int cnt = (int)(start[i + 1] - start[i]);
        if (cnt == 0) continue;
        std::vector<CompactTarget> tg(S, CompactTarget{nullptr, nullptr, nullptr, 0});
        for (int t = 0; t < S; t++) {
            if (t == i) continue;
            tg[t] = target[t];
            if (tg[t].res) tg[t].res += (size_t)(start[i] - (i > t ? start[t + 1] - start[t] : 0)) * K;  // this block's first query of t
        }
        const jv_graph_s &g = *src[i].g;
        const int32_t *own_adj = g.adj0.get<int32_t>(), *own_row;
        int32_t *dadj, *drow;
        e = alloc_owned(mem, drow, (size_t)cnt * 4);
        if (e == cudaSuccess) e = cudaMemcpyAsync(drow, src[i].live_row[level].data(), (size_t)cnt * 4, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess && level > 0) {
            const std::vector<int32_t> &a = g.level_adj[level - 1];
            e = alloc_owned(mem, dadj, a.size() * 4);
            if (e == cudaSuccess) e = cudaMemcpyAsync(dadj, a.data(), a.size() * 4, cudaMemcpyHostToDevice, s);
            own_adj = dadj;
        }
        own_row = drow;
        // the targets' device copy is read by the launch below before the next block's copy is enqueued behind it on `s`
        if (e == cudaSuccess) e = cudaMemcpyAsync(dtargets, tg.data(), (size_t)S * sizeof(CompactTarget), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess)
            e = launch_compact_assemble(cnt, degree, K, own_adj, own_row, maps_dev[i], dtargets, S, start[i], cand_stride, cand, cand_off + start[i],
                                        cand_cnt + start[i], s);
        if (e != cudaSuccess) rc = cuda_fail(e, "graph_compact: candidates");
    }
    std::vector<int> hcnt(rows);
    if (!rc) {
        e = cudaMemcpyAsync(hcnt.data(), cand_cnt, (size_t)rows * 4, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e == cudaSuccess) e = prune_ragged_rows(merged->d, metric, alpha, degree, rows, cand, drow_node, cand_off, cand_cnt, hcnt, out_rows, g_sm_count, s);
        if (e == cudaSuccess && level == 0) e = launch_scatter_rows(ng->adj0.get<int32_t>(), degree, drow_node, rows, out_rows, s);
        std::vector<int32_t> hrows;
        if (e == cudaSuccess && level > 0) {
            hrows.resize((size_t)rows * degree);
            e = cudaMemcpyAsync(hrows.data(), out_rows, hrows.size() * 4, cudaMemcpyDeviceToHost, s);
        }
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) rc = cuda_fail(e, "graph_compact: prune");
        for (int a = 0; a < rows && !rc; a++) {
            stats->candidates += hcnt[a];
            stats->max_candidates = std::max(stats->max_candidates, hcnt[a]);
        }
        if (!rc && level > 0) {
            std::vector<int32_t> order(rows);
            for (int a = 0; a < rows; a++) order[a] = a;
            std::sort(order.begin(), order.end(), [&](int x, int y) { return row_node[x] < row_node[y]; });
            ids_out->resize(rows);
            adj_out->resize((size_t)rows * degree);
            for (int r = 0; r < rows; r++) {
                (*ids_out)[r] = row_node[order[r]];
                std::copy_n(hrows.begin() + (size_t)order[r] * degree, degree, adj_out->begin() + (size_t)r * degree);
            }
        }
    }
    cudaStreamSynchronize(s);  // the level's scratch goes on return
    return rc;
}

// jv_graph_compact's checks, all on the host: every refusal comes before any device work. Fills src (maps and live members per
// level), the live total, the level count and searchTopK.
static int compact_prepare(const jv_compact_source *sources, int nsources, int metric, float alpha, std::vector<CompactSource> &src, long long *total_out,
                           int *levels_out, int *K_out)
{
    for (int i = 0; i < nsources; i++)
        if (!sources[i].graph || !sources[i].rows || !sources[i].old_to_new) return fail(JV_ERR_INVALID, "graph_compact: null argument");
    ON_DEVICE_OF(sources[0].graph);
    const int S = nsources, degree = sources[0].graph->g.degree, dim = sources[0].rows->d.dim;
    for (int i = 0; i < S; i++) {
        const jv_compact_source &c = sources[i];
        if (c.rows->d.kind != KIND_F32) return fail(JV_ERR_INVALID, "graph_compact: the sources' rows must be fp32");
        if (c.rows->d.n != c.graph->g.n) return fail(JV_ERR_INVALID, "graph_compact: a source's rows and graph differ in size");
        if (c.rows->d.dim != dim || c.graph->g.degree != degree || c.graph->device != t_active || c.rows->device != t_active)
            return fail(JV_ERR_INVALID, "graph_compact: the sources differ in dim, degree or device");
    }
    int rc = check_metric(sources[0].rows->d, metric);
    if (rc) return rc;
    if (!(alpha >= 1.0f)) return fail(JV_ERR_INVALID, "graph_compact: need alpha >= 1");
    // the live nodes (holes are dead) and their new ids, which must be exactly [0, live nodes)
    src.assign(S, CompactSource());
    long long total = 0;
    int levels = 0;
    for (int i = 0; i < S; i++) {
        CompactSource &c = src[i];
        c.g = sources[i].graph;
        c.ds = sources[i].rows;
        const int n = c.g->g.n;
        c.map.assign(n, -1);
        for (int v = 0; v < n; v++) {
            const bool hole = !c.g->removed.empty() && bit_of(c.g->removed, v);
            const bool live = !hole && (!sources[i].live_bits || ((sources[i].live_bits[v >> 5] >> (v & 31)) & 1u));
            if (!live) continue;
            c.map[v] = sources[i].old_to_new[v];
            if (c.map[v] < 0) return fail(JV_ERR_INVALID, "graph_compact: a live node has a negative new id");
            total++;
        }
        levels = std::max(levels, c.g->g.levels);
    }
    if (total == 0 || total > 0x7fffffffLL) return fail(JV_ERR_INVALID, "graph_compact: no live node, or more than 2^31 - 1");
    std::vector<uint8_t> seen(total, 0);
    for (const CompactSource &c : src)
        for (int32_t x : c.map) {
            if (x < 0) continue;
            if (x >= total || seen[x]) return fail(JV_ERR_INVALID, "graph_compact: the new ids of the live nodes must be exactly [0, live nodes)");
            seen[x] = 1;
        }
    if (degree > 64) return fail(JV_ERR_UNSUPPORTED, "graph_compact: degree above 64");
    const int K = std::max(2, (degree + S - 1) / S * 4);
    // a row's candidates must fit the prune's largest tier (8192): true for every S up to 2033 at degree 64
    if (degree + (long long)(S - 1) * K > 8192) return fail(JV_ERR_UNSUPPORTED, "graph_compact: too many sources for one row's candidates");
    for (CompactSource &c : src) {
        c.live.resize(levels);  // a level the source does not have has no member
        c.live_row.resize(levels);
        for (int L = 0; L < c.g->g.levels; L++) {
            const int cnt = L ? (int)c.g->level_ids[L - 1].size() : c.g->g.n;
            for (int r = 0; r < cnt; r++) {
                const int v = L ? c.g->level_ids[L - 1][r] : r;
                if (c.map[v] < 0) continue;
                c.live[L].push_back(v);
                c.live_row[L].push_back(r);
            }
        }
    }
    *total_out = total;
    *levels_out = levels;
    *K_out = K;
    return JV_OK;
}

// the merge itself on the device, for the sources compact_prepare accepted: the new graph and its fp32 rows into ng / nd
static int compact_merge(const std::vector<CompactSource> &src, int metric, float alpha, long long total, int levels, int K,
                         std::unique_ptr<jv_graph_s> &ng, std::unique_ptr<jv_dataset_s> &nd, jv_compact_stats *stats)
{
    const int S = (int)src.size(), degree = src[0].g->g.degree, dim = src[0].ds->d.dim;
    int rc;
    if ((rc = t_ctx.init())) return rc;
    cudaStream_t s = t_ctx.stream;
    memset(stats, 0, sizeof(*stats));
    nd.reset(new jv_dataset_s(KIND_F32, total, dim));
    float *rows = nullptr;
    if ((rc = nd->alloc_rows(&rows))) return rc;
    if ((rc = jv_graph_s::create((int32_t)total, degree, ng))) return rc;
    StreamTimer timer;
    CK(timer.start(s), "event");
    // every source's old -> new map on the device, and its live rows scattered to their new ids
    std::vector<DeviceBuffer> mem;
    std::vector<const int32_t *> maps_dev(S);
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < S && e == cudaSuccess; i++) {
        const CompactSource &c = src[i];
        const size_t cnt = c.live[0].size();
        int32_t *dmap, *dold, *dnew;
        std::vector<int32_t> hnew(cnt);
        for (size_t j = 0; j < cnt; j++) hnew[j] = c.map[c.live[0][j]];
        e = alloc_owned(mem, dmap, c.map.size() * 4);
        if (e == cudaSuccess) e = alloc_owned(mem, dold, std::max<size_t>(cnt, 1) * 4);
        if (e == cudaSuccess) e = alloc_owned(mem, dnew, std::max<size_t>(cnt, 1) * 4);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dmap, c.map.data(), c.map.size() * 4, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dold, c.live[0].data(), cnt * 4, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(dnew, hnew.data(), cnt * 4, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = launch_gather_rows(c.ds->d, dold, (int)cnt, rows, s, dnew);
        maps_dev[i] = dmap;
    }
    if (e != cudaSuccess) rc = cuda_fail(e, "graph_compact: merged rows");
    stats->search_top_k = K;
    int nlev = 0;
    Levels level_ids, level_adj;
    for (int L = 0; L < levels && !rc; L++) {
        long long members = 0;
        for (const CompactSource &c : src) members += (long long)c.live[L].size();
        if (members == 0) break;  // levels without a live member are dropped, and every level above one is empty too
        if (L == 0) rc = compact_level(src, 0, K, nd.get(), metric, alpha, ng.get(), maps_dev, nullptr, nullptr, stats, s);
        else {
            level_ids.emplace_back();
            level_adj.emplace_back();
            rc = compact_level(src, L, K, nd.get(), metric, alpha, ng.get(), maps_dev, &level_ids.back(), &level_adj.back(), stats, s);
        }
        nlev = L + 1;
    }
    timer.stop(s);
    cudaStreamSynchronize(s);
    if (rc) return rc;
    // entry: the first source whose top level is the merged top level and whose entry is live, else the top level's lowest new id
    int32_t entry = -1;
    for (const CompactSource &c : src)
        if (c.g->g.levels == nlev && c.g->g.entry_node >= 0 && c.map[c.g->g.entry_node] >= 0) {
            entry = c.map[c.g->g.entry_node];
            break;
        }
    if (entry < 0) entry = nlev > 1 ? level_ids.back().front() : 0;
    if ((rc = ng->set_levels(std::move(level_ids), std::move(level_adj), entry))) return rc;
    stats->nodes = (int32_t)total;
    stats->levels = ng->g.levels;
    stats->device_ms = timer.ms();
    return JV_OK;
}

int jv_graph_compact(const jv_compact_source *sources, int nsources, int metric, float alpha, jv_graph *graph_out, jv_dataset *rows_out,
                     jv_compact_stats *stats)
{
    if (!sources || nsources < 1 || !graph_out || !rows_out || !stats) return fail(JV_ERR_INVALID, "graph_compact: null argument or no source");
    std::vector<CompactSource> src;
    long long total;
    int levels, K, rc;
    if ((rc = compact_prepare(sources, nsources, metric, alpha, src, &total, &levels, &K))) return rc;
    std::unique_ptr<jv_graph_s> ng;
    std::unique_ptr<jv_dataset_s> nd;
    if ((rc = compact_merge(src, metric, alpha, total, levels, K, ng, nd, stats))) return rc;
    *graph_out = ng.release();
    *rows_out = nd.release();
    return JV_OK;
}

// PQRetrainer.sampleBalanced (PQRetrainer.java:127-212) over the sources' live nodes, with counter_random in place of
// ThreadLocalRandom: per source its sampled node ids, ascending. Every live node when there are at most 128 000; otherwise each
// source's quota (at least min(1000, 128 000 / S), else its share of 128 000, normalised to 128 000 in total) is filled from its
// 32-node chunks in a Fisher-Yates order, each chunk's live nodes ascending. A source short of its quota gives what it has.
static std::vector<std::vector<int32_t>> retrain_sample(const std::vector<CompactSource> &src, uint64_t seed)
{
    constexpr long long MIN_SAMPLES_PER_SOURCE = 1000;
    constexpr int SAMPLE_CHUNK_SIZE = 32;
    const int S = (int)src.size();
    const long long cap = MAX_PQ_TRAINING_SET_SIZE;
    std::vector<std::vector<int32_t>> out(S);
    long long total = 0;
    for (const CompactSource &c : src) total += (long long)c.live[0].size();
    if (total <= cap) {
        for (int s = 0; s < S; s++) out[s] = src[s].live[0];  // level 0's live members, ascending
        return out;
    }
    const long long min_per = std::min(MIN_SAMPLES_PER_SOURCE, cap / S);
    std::vector<long long> quota(S);
    long long assigned = 0;
    for (int s = 0; s < S; s++) {
        quota[s] = std::max(min_per, cap * (long long)src[s].live[0].size() / total);
        assigned += quota[s];
    }
    while (assigned > cap)
        for (int s = 0; s < S && assigned > cap; s++)
            if (quota[s] > min_per) {
                quota[s]--;
                assigned--;
            }
    while (assigned < cap)
        for (int s = 0; s < S && assigned < cap; s++) {
            quota[s]++;
            assigned++;
        }
    for (int s = 0; s < S; s++) {
        const CompactSource &c = src[s];
        const int n = c.g->g.n, chunks = (n + SAMPLE_CHUNK_SIZE - 1) / SAMPLE_CHUNK_SIZE;
        std::vector<int> order(chunks);
        for (int i = 0; i < chunks; i++) order[i] = i;
        for (int i = chunks - 1; i > 0; i--) std::swap(order[i], order[counter_random(seed, TAG_COMPACT_SAMPLE, s, i) % (uint64_t)(i + 1)]);
        long long count = 0;
        for (int ci = 0; ci < chunks && count < quota[s]; ci++) {
            const int start = order[ci] * SAMPLE_CHUNK_SIZE, end = std::min(n, start + SAMPLE_CHUNK_SIZE);
            for (int v = start; v < end && count < quota[s]; v++)
                if (c.map[v] >= 0) {
                    out[s].push_back(v);
                    count++;
                }
        }
        std::sort(out[s].begin(), out[s].end());
    }
    return out;
}

int jv_graph_compact_pq(const jv_compact_source *sources, const jv_dataset *source_pq, int nsources, int metric, float alpha, uint64_t seed,
                        jv_graph *graph_out, jv_dataset *rows_out, jv_dataset *pq_out, float *codebooks_out, float *centroid_out,
                        int64_t *samples_per_source_out, jv_compact_pq_stats *stats)
{
    if (!sources || !source_pq || nsources < 1 || !graph_out || !rows_out || !pq_out || !codebooks_out || !stats)
        return fail(JV_ERR_INVALID, "graph_compact_pq: null argument or no source");
    for (int i = 0; i < nsources; i++)
        if (!source_pq[i]) return fail(JV_ERR_INVALID, "graph_compact_pq: null argument");
    std::vector<CompactSource> src;
    long long total;
    int levels, K, rc;
    if ((rc = compact_prepare(sources, nsources, metric, alpha, src, &total, &levels, &K))) return rc;
    const int S = nsources, dim = sources[0].rows->d.dim;
    // the form: every source's FusedPQ records packed from its own codes (fused), or no records at all (sidecar)
    int fused = 0, plain = 0;
    for (int i = 0; i < S; i++) {
        const jv_dataset pq = source_pq[i];
        const GraphDesc &g = sources[i].graph->g;
        if (pq->d.kind != KIND_PQ) return fail(JV_ERR_INVALID, "graph_compact_pq: source_pq must hold PQ codes");
        if (pq->d.n != g.n || pq->d.dim != dim || pq->device != t_active)
            return fail(JV_ERR_INVALID, "graph_compact_pq: a source's codes differ from its graph in size, dim or device");
        if (!g.fused) plain++;
        else if (g.fused_codes_of == pq->d.codes && g.fused_code_stride == pq->d.code_stride) fused++;
    }
    if (fused != S && plain != S)
        return fail(JV_ERR_INVALID, "graph_compact_pq: either every source carries FusedPQ records packed from its own codes, or none carries records");
    const DataDesc &p0 = source_pq[0]->d;
    if (p0.centroid && !centroid_out) return fail(JV_ERR_INVALID, "graph_compact_pq: source 0's PQ has a centroid: need centroid_out");
    const std::vector<std::vector<int32_t>> sample = retrain_sample(src, seed);
    long long train_rows = 0;
    for (const std::vector<int32_t> &x : sample) train_rows += (long long)x.size();
    if (train_rows < p0.k) return fail(JV_ERR_INVALID, "graph_compact_pq: fewer training rows than clusters");
    if (fused == S)
        for (int i = 0; i < S; i++) src[i].pq = source_pq[i];
    jv_compact_pq_stats st;
    memset(&st, 0, sizeof(st));
    st.fused = fused == S;
    st.train_rows = train_rows;
    std::unique_ptr<jv_graph_s> ng;
    std::unique_ptr<jv_dataset_s> nd, np, tr;
    if ((rc = compact_merge(src, metric, alpha, total, levels, K, ng, nd, &st.graph))) return rc;
    cudaStream_t s = t_ctx.stream;
    // retraining (PQRetrainer.retrain): source 0's codebooks refined by 6 unweighted Lloyd rounds over the sample, gathered source by
    // source into one fp32 data set in (source, node) order
    std::vector<float> cb0((size_t)p0.k * dim), cen0(p0.centroid ? dim : 0);
    CK(cudaMemcpy(cb0.data(), p0.codebooks, cb0.size() * 4, cudaMemcpyDeviceToHost), "D2H source 0's codebooks");
    if (p0.centroid) CK(cudaMemcpy(cen0.data(), p0.centroid, cen0.size() * 4, cudaMemcpyDeviceToHost), "D2H source 0's centroid");
    const float *cen = p0.centroid ? cen0.data() : nullptr;
    tr.reset(new jv_dataset_s(KIND_F32, train_rows, dim));
    float *trows;
    if ((rc = tr->alloc_rows(&trows))) return rc;
    std::vector<int32_t> ids;
    for (const std::vector<int32_t> &x : sample) ids.insert(ids.end(), x.begin(), x.end());
    DeviceBuffer dids;
    CK(dids.alloc(ids.size() * 4), "cudaMalloc(sample ids)");
    StreamTimer t_train, t_encode, t_fuse;
    CK(t_train.start(s), "event");
    CK(cudaMemcpyAsync(dids.get(), ids.data(), ids.size() * 4, cudaMemcpyHostToDevice, s), "H2D sample ids");
    for (int i = 0, off = 0; i < S; off += (int)sample[i].size(), i++)
        CK(launch_gather_rows(src[i].ds->d, dids.get<int32_t>() + off, (int)sample[i].size(), trows + (size_t)off * tr->d.stride, s), "gather sample");
    const jv_pq_train_params tp = {p0.M, p0.k, 0, 6 /* K_MEANS_ITERATIONS */, MAX_PQ_TRAINING_SET_SIZE, seed};
    rc = pq_train_impl(tr.get(), &tp, cb0.data(), cen, codebooks_out, nullptr, &st.train);
    CK(t_train.stop(s), "event");
    if (rc) return rc;
    // the merged rows encoded with the new codebooks, and (fused form) the merged graph's records packed from them
    CK(t_encode.start(s), "event");
    if ((rc = pq_encode_resident(nd.get(), p0.M, p0.k, codebooks_out, cen, s, np))) return rc;
    CK(t_encode.stop(s), "event");
    if (st.fused) {
        CK(t_fuse.start(s), "event");
        if ((rc = fuse_pq(ng.get(), np.get(), s))) return rc;
        CK(t_fuse.stop(s), "event");
    }
    CK(cudaStreamSynchronize(s), "graph_compact_pq");
    st.retrain_ms = t_train.ms();
    st.encode_ms = t_encode.ms();
    st.fuse_ms = st.fused ? t_fuse.ms() : 0.0;
    if (cen) std::copy(cen0.begin(), cen0.end(), centroid_out);
    if (samples_per_source_out)
        for (int i = 0; i < S; i++) samples_per_source_out[i] = (int64_t)sample[i].size();
    *stats = st;
    *graph_out = ng.release();
    *rows_out = nd.release();
    *pq_out = np.release();
    return JV_OK;
}

// ------------------------------------------------------------------------------------------------ refinement (DESIGN §4.3i)
// One level of jv_graph_refine through refine_level (build.cu). Level 0 reads g's adjacency and writes ng's; an upper level is a graph
// of its own over its members' rows (gather_level, as build_level builds it), its rows mapped to local ids and back, into *adj_out.
// nodes: the rows of the level to refine, ascending.
static int refine_graph_level(jv_graph g, jv_graph_s *ng, jv_dataset ds, int metric, const BuildParams &bp, int beam, bool compactor, int level,
                              const std::vector<int32_t> &nodes, RefineStats *st, std::vector<int32_t> *adj_out, cudaStream_t s)
{
    const int n = g->g.n, degree = g->g.degree;
    cudaError_t e;
    if (nodes.empty()) {  // nothing to refine: the level as it was
        if (level > 0) *adj_out = g->level_adj[level - 1];
        else CK(cudaMemcpyAsync(ng->adj0.get(), g->adj0.get(), (size_t)n * degree * 4, cudaMemcpyDeviceToDevice, s), "copy adjacency");
        return JV_OK;
    }
    if (level == 0) {
        e = refine_level(ds->d, metric, bp, beam, compactor, g->adj0.get<int32_t>(), degree, g->g.entry_node, nodes, ng->adj0.get<int32_t>(), g_sm_count, st, s);
        return e == cudaSuccess ? JV_OK : cuda_fail(e, "graph_refine");
    }
    const std::vector<int32_t> &ids = g->level_ids[level - 1];
    const int cnt = (int)ids.size();
    std::vector<int32_t> pos(n, -1);
    for (int r = 0; r < cnt; r++) pos[ids[r]] = r;
    std::vector<int32_t> local(g->level_adj[level - 1]);
    for (int32_t &x : local) x = x >= 0 ? pos[x] : -1;
    DataDesc sub;
    DeviceBuffer rows, dids, din, dout;
    e = gather_level(ds, ids, rows, dids, &sub, s);
    if (e == cudaSuccess) e = din.alloc(local.size() * 4);
    if (e == cudaSuccess) e = dout.alloc(local.size() * 4);
    if (e == cudaSuccess) e = cudaMemcpyAsync(din.get(), local.data(), local.size() * 4, cudaMemcpyHostToDevice, s);
    const int32_t entry = pos[g->g.entry_node] >= 0 ? pos[g->g.entry_node] : 0;
    if (e == cudaSuccess) e = refine_level(sub, metric, bp, beam, compactor, din.get<int32_t>(), degree, entry, nodes, dout.get<int32_t>(), g_sm_count, st, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(local.data(), dout.get(), local.size() * 4, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    else cudaStreamSynchronize(s);  // the buffers above are freed on return
    if (e != cudaSuccess) return cuda_fail(e, "graph_refine");
    adj_out->resize(local.size());
    for (size_t i = 0; i < local.size(); i++) (*adj_out)[i] = local[i] >= 0 ? ids[local[i]] : -1;
    return JV_OK;
}

int jv_graph_refine(jv_graph g, jv_dataset ds, int metric, const jv_build_params *params, int mode, jv_graph *out, jv_refine_stats *stats)
{
    ON_DEVICE_OF(g);
    if (!ds || !params || !out || !stats) return fail(JV_ERR_INVALID, "graph_refine: null argument");
    if (mode != JV_REFINE_BUILDER && mode != JV_REFINE_COMPACTOR) return fail(JV_ERR_INVALID, "graph_refine: unknown mode");
    if (ds->d.n != g->g.n || ds->device != g->device) return fail(JV_ERR_INVALID, "graph_refine: data set and graph differ in size or device");
    const bool compactor = mode == JV_REFINE_COMPACTOR;
    const int kind = ds->d.kind;
    if (compactor ? kind != KIND_F32 : (kind != KIND_F32 && kind != KIND_PQ && kind != KIND_BQ))
        return fail(JV_ERR_INVALID, compactor ? "graph_refine: the compactor form takes fp32 rows" : "graph_refine: needs fp32 rows, PQ codes or BQ codes");
    int rc = check_metric(ds->d, metric);
    if (rc) return rc;
    const int degree = g->g.degree;
    if (params->degree != degree) return fail(JV_ERR_INVALID, "graph_refine: params->degree differs from the graph's degree");
    if (degree > 64) return fail(JV_ERR_UNSUPPORTED, "graph_refine: degree above 64");
    BuildParams bp;
    if ((rc = build_params_check(params, &bp))) return rc;
    // the compactor's beam: 2 * max(M, max(2, 4 M)) (OnDiskGraphIndexCompactor)
    const int beam = compactor ? 8 * degree : bp.beam;
    const int row_cap = std::max(2 * degree, (int)(bp.overflow * degree) + 1);
    if (row_cap > MAX_DEGREE) return fail(JV_ERR_INVALID, "graph_refine: overflow * degree above the widest row");
    if (kind == KIND_PQ && !pq_ragged_fits(ds->d, row_cap + beam))
        return fail(JV_ERR_UNSUPPORTED, "graph_refine: the PQ LUT does not fit the prune's shared memory next to the candidates");
    if ((rc = provider_check(g, ds, kind, metric, params, &bp, "graph_refine"))) return rc;
    if ((rc = t_ctx.init())) return rc;
    cudaStream_t s = t_ctx.stream;
    const int n = g->g.n, levels = g->g.levels;
    memset(stats, 0, sizeof(*stats));
    RefineStats st;
    memset(&st, 0, sizeof(st));
    std::unique_ptr<jv_graph_s> ng;
    if ((rc = jv_graph_s::create(n, degree, ng))) return rc;
    ng->removed = g->removed;
    Levels level_adj = g->level_adj;
    // builder form: refined only when there are upper levels (maxLevel > 0); compactor form: level 0 whenever there is an entry
    const bool run = g->g.entry_node >= 0 && (compactor || levels > 1);
    if (!run) CK(cudaMemcpyAsync(ng->adj0.get(), g->adj0.get(), (size_t)n * degree * 4, cudaMemcpyDeviceToDevice, s), "copy adjacency");
    std::vector<int32_t> adj0;
    if (run && !compactor) {
        adj0.resize((size_t)n * degree);
        CK(cudaMemcpyAsync(adj0.data(), g->adj0.get(), adj0.size() * 4, cudaMemcpyDeviceToHost, s), "D2H adjacency");
        CK(cudaStreamSynchronize(s), "D2H adjacency");
    }
    auto empty_row = [&](const int32_t *row) { return std::all_of(row, row + degree, [](int32_t x) { return x < 0; }); };
    const int refined_levels = run ? (compactor ? 1 : levels) : 0;
    for (int L = 0; L < refined_levels && !rc; L++) {
        std::vector<int32_t> nodes;
        if (L == 0) {
            if (levels > 1) {
                for (int32_t v : g->level_ids[0])
                    if (compactor || !empty_row(adj0.data() + (size_t)v * degree)) nodes.push_back(v);
            } else {
                for (int v = 0; v < n; v++)
                    if (g->removed.empty() || !bit_of(g->removed, v)) nodes.push_back(v);
            }
            std::sort(nodes.begin(), nodes.end());
        } else {
            const std::vector<int32_t> &a = g->level_adj[L - 1];
            for (int r = 0; r < (int)g->level_ids[L - 1].size(); r++)
                if (!empty_row(a.data() + (size_t)r * degree)) nodes.push_back(r);
        }
        const long long before = st.nodes;
        rc = refine_graph_level(g, ng.get(), ds, metric, bp, beam, compactor, L, nodes, &st, L ? &level_adj[L - 1] : nullptr, s);
        stats->nodes_refined[std::min(L, JV_REFINE_MAX_LEVELS - 1)] += st.nodes - before;
    }
    if (!rc) rc = ng->set_levels(g->level_ids, std::move(level_adj), g->g.entry_node);
    cudaStreamSynchronize(s);
    if (rc) return rc;
    stats->levels = refined_levels;
    stats->candidates = st.candidates;
    stats->max_candidates = st.max_candidates;
    stats->rows_changed = st.rows_changed;
    stats->backlinks_added = st.backlinks_added;
    stats->backlinks_dropped = st.backlinks_dropped;
    stats->rows_repruned = st.rows_repruned;
    stats->device_ms = st.device_ms;
    *out = ng.release();
    return JV_OK;
}

// ------------------------------------------------------------------------------------------------ query batches (host-driven seam)
// north_star's literal form of the path: the host expands the frontier and sends each hop's candidate set as one launch. What
// makes that seam fast is what persists between calls: the prepared queries (LUTs / bit packs / shifted copies) stay in HBM for
// the life of the batch, and ids / offsets / scores travel through pinned, device-mapped staging that belongs to the batch.
struct jv_query_batch_s {
    int device = 0;
    jv_dataset ds = nullptr;
    int metric = 0, nq = 0;
    DeviceBuffer blobs;  // [nq][blob_floats]
    size_t blob_floats = 0;
    // staging, grown on demand: pinned copies for pageable caller buffers, and the device side
    PinnedBuffer h_ids, h_off, h_scores;
    DeviceBuffer d_ids, d_off, d_scores;
    cudaStream_t stream = nullptr;
    StreamTimer timer;
    // single-hop path: mapped pinned ids / scores / completion flag the kernel reads and writes directly, a device-side CTA counter
    PinnedBuffer hop_ids, hop_scores, hop_flag;
    DeviceBuffer hop_done;
    int hop_seq = 0;
    ~jv_query_batch_s()
    {
        cudaSetDevice(device);
        if (stream) {
            cudaStreamSynchronize(stream);
            cudaStreamDestroy(stream);
        }
    }
};

int jv_query_batch_begin(jv_dataset ds, int metric, const float *queries, int nq, jv_query_batch *out)
{
    ON_DEVICE_OF(ds);
    if (!queries || !out || nq <= 0 || nq > 65535) return fail(JV_ERR_INVALID, "query_batch_begin: 1 <= nq <= 65535");
    int rc = check_metric(ds->d, metric);
    if (rc) return rc;
    if ((rc = t_ctx.init()) || (rc = grow(t_ctx.input, (size_t)nq * ds->d.dim * 4))) return rc;
    std::unique_ptr<jv_query_batch_s> b(new jv_query_batch_s());
    b->device = ds->device; b->ds = ds; b->metric = metric; b->nq = nq; b->blob_floats = (size_t)blob_floats(ds->d);
    cudaError_t e = b->blobs.alloc((size_t)nq * b->blob_floats * 4);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMemcpyAsync(t_ctx.input.get(), queries, (size_t)nq * ds->d.dim * 4, cudaMemcpyHostToDevice, t_ctx.stream);
    if (e == cudaSuccess) e = launch_prepare(ds->d, metric, t_ctx.input.get<float>(), nq, b->blobs.get<float>(), t_ctx.stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(t_ctx.stream);
    CK(e, "query_batch_begin");
    *out = b.release();
    return JV_OK;
}

// one step of all the batch's searches: query i scores ids[offsets[i] .. offsets[i+1]); only ids + offsets go up, scores come down
int jv_query_batch_score(jv_query_batch b, const int32_t *ids, const int32_t *offsets, float *scores_out, double *device_ms)
{
    ON_DEVICE_OF(b);
    if (!ids || !offsets || !scores_out) return fail(JV_ERR_INVALID, "query_batch_score: null argument");
    const int nq = b->nq;
    const int total = offsets[nq];
    int maxc = 0;
    for (int i = 0; i < nq; i++) {
        if (offsets[i + 1] < offsets[i]) return fail(JV_ERR_INVALID, "query_batch_score: offsets not monotone");
        maxc = std::max(maxc, offsets[i + 1] - offsets[i]);
    }
    if (device_ms) *device_ms = 0.0;
    if (total <= 0) return JV_OK;
    const size_t ib = (size_t)total * 4, ob = ((size_t)nq + 1) * 4;
    CK(b->h_ids.grow(ib), "cudaHostAlloc(ids)");
    CK(b->h_scores.grow(ib), "cudaHostAlloc(scores)");
    CK(b->h_off.grow(ob), "cudaHostAlloc(offsets)");
    CK(b->d_ids.grow(ib), "cudaMalloc(ids)");
    CK(b->d_scores.grow(ib), "cudaMalloc(scores)");
    CK(b->d_off.grow(ob), "cudaMalloc(offsets)");
    // caller buffers that are already pinned (jv_host_register / cudaHostAlloc) are copied from / to directly; pageable ones go
    // through the batch's own pinned staging so that the copies stay asynchronous and full speed
    auto pinned = [](const void *p) {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
        return a.type == cudaMemoryTypeHost;
    };
    const bool ids_pinned = pinned(ids), out_pinned = pinned(scores_out);
    if (!ids_pinned) memcpy(b->h_ids.get(), ids, ib);
    memcpy(b->h_off.get(), offsets, ob);
    cudaStream_t s = b->stream;
    CK(cudaMemcpyAsync(b->d_ids.get(), ids_pinned ? ids : b->h_ids.get(), ib, cudaMemcpyHostToDevice, s), "H2D ids");
    CK(cudaMemcpyAsync(b->d_off.get(), b->h_off.get(), ob, cudaMemcpyHostToDevice, s), "H2D offsets");
    CK(b->timer.start(s), "event");
    CK(launch_score_ragged(b->ds->d, b->metric, b->blobs.get<float>(), nq, b->d_ids.get<int32_t>(), b->d_off.get<int32_t>(), 0, maxc, b->d_scores.get<float>(), s),
       "score_ragged");
    CK(b->timer.stop(s), "event");
    CK(cudaMemcpyAsync(out_pinned ? scores_out : b->h_scores.get(), b->d_scores.get(), ib, cudaMemcpyDeviceToHost, s), "D2H scores");
    CK(cudaStreamSynchronize(s), "sync");
    if (!out_pinned) memcpy(scores_out, b->h_scores.get(), ib);
    if (device_ms) *device_ms = b->timer.ms();
    return JV_OK;
}

// one hop of ONE search of the batch. Latency path: the kernel reads the ids from, and writes the scores and a completion
// sequence number to, mapped pinned memory; the host spins on that word instead of synchronising the stream (a blocking
// cudaStreamSynchronize costs more than the launch and the kernel together), and polls the stream only to notice a failed launch.
int jv_query_batch_score_one(jv_query_batch b, int query_index, const int32_t *ids, int n, float *scores_out)
{
    ON_DEVICE_OF(b);
    if (query_index < 0 || query_index >= b->nq || n < 0 || (n > 0 && (!ids || !scores_out))) return fail(JV_ERR_INVALID, "query_batch_score_one: bad arguments");
    if (n == 0) return JV_OK;
    if ((size_t)n * 4 > b->hop_ids.capacity()) {
        CK(cudaStreamSynchronize(b->stream), "sync");  // the previous hop's kernel is done with the blocks about to be replaced
        CK(b->hop_ids.grow((size_t)n * 4), "cudaHostAlloc(hop ids)");
        CK(b->hop_scores.grow((size_t)n * 4), "cudaHostAlloc(hop scores)");
    }
    if (!b->hop_flag.get()) {
        CK(b->hop_flag.grow(64), "cudaHostAlloc(hop flag)");
        *b->hop_flag.get<int>() = 0;
        CK(b->hop_done.alloc(64), "cudaMalloc(hop counter)");
        CK(cudaMemset(b->hop_done.get(), 0, 64), "memset");
    }
    const float *blob = b->blobs.get<float>() + (size_t)query_index * b->blob_floats;
    if (n <= HOP_MAX_IDS) {
        // ids in the kernel parameters, every score word pre-set to a pattern no score can have and polled until it is overwritten
        volatile uint32_t *sc = b->hop_scores.get<volatile uint32_t>();
        for (int i = 0; i < n; i++) sc[i] = 0xffffffffu;
        __atomic_thread_fence(__ATOMIC_SEQ_CST);
        CK(launch_score_hop(b->ds->d, b->metric, blob, ids, n, b->hop_scores.dev<float>(), b->stream), "score_hop");
        unsigned spins = 0;
        for (int i = 0; i < n; i++) {
            while (sc[i] == 0xffffffffu) {
                if ((++spins & 0x3fffu) == 0) {
                    const cudaError_t e = cudaStreamQuery(b->stream);
                    if (e == cudaSuccess) {
                        if (sc[i] != 0xffffffffu) break;
                        return fail(JV_ERR_CUDA, "query_batch_score_one: the kernel finished without writing its scores");
                    }
                    if (e != cudaErrorNotReady) return cuda_fail(e, "query_batch_score_one");
                }
#if defined(__x86_64__)
                __builtin_ia32_pause();
#endif
            }
        }
        __atomic_thread_fence(__ATOMIC_ACQUIRE);
        memcpy(scores_out, b->hop_scores.get(), (size_t)n * 4);
        return JV_OK;
    }
    memcpy(b->hop_ids.get(), ids, (size_t)n * 4);
    const int seq = ++b->hop_seq == 0 ? ++b->hop_seq : b->hop_seq;
    // one lane group per id and 4 ids per CTA: the hop's rows are fetched in one wave instead of one CTA walking them in turn
    CK(launch_score_ragged(b->ds->d, b->metric, blob, 1, b->hop_ids.dev<int32_t>(), nullptr, n, n, b->hop_scores.dev<float>(), b->stream, 4,
                           b->hop_done.get<int>(), b->hop_flag.dev<int>(), seq),
       "score_ragged");
    volatile int *flag = b->hop_flag.get<volatile int>();
    for (unsigned spins = 1; *flag != seq; spins++) {
        if ((spins & 0x3fffu) == 0) {
            const cudaError_t e = cudaStreamQuery(b->stream);
            if (e == cudaSuccess) {
                if (*flag == seq) break;
                return fail(JV_ERR_CUDA, "query_batch_score_one: the kernel finished without its completion signal");
            }
            if (e != cudaErrorNotReady) return cuda_fail(e, "query_batch_score_one");
        }
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
    }
    __atomic_thread_fence(__ATOMIC_ACQUIRE);
    memcpy(scores_out, b->hop_scores.get(), (size_t)n * 4);
    return JV_OK;
}

int jv_query_batch_end(jv_query_batch b)
{
    delete b;
    return JV_OK;
}

// ------------------------------------------------------------------------------------------------ several GPUs, one process
// The reference host is ONE JVM whose parallelism is threads (base:vector/VectorizationProvider.java:79-177,
// base:graph/GraphIndexBuilder.java:440-444), so the sharding of SURVEY §8e has to be reachable from one process: the base
// range-sharded by contiguous node id over the bound devices, every shard scoring all queries on its own stream, the per-shard
// top-k keys (global ids) copied to the first device over NVLink (peer copies) and merged there.
int jv_multi_free(jv_multi m)
{
    if (!m) return JV_OK;
    for (jv_dataset ds : m->shards) jv_dataset_free(ds);
    for (size_t i = 0; i < m->ctx.size(); i++) {
        t_active = m->devices[i];
        cudaSetDevice(m->devices[i]);
        delete m->ctx[i];
    }
    if (!m->devices.empty()) cudaSetDevice(m->devices[0]);
    delete m;
    return JV_OK;
}

int jv_multi_register_bq(const uint64_t *words, int64_t n, int dim, jv_multi *out)
{
    if (!words || !out || n <= 0 || dim <= 0 || n > 0x7fffffffLL) return fail(JV_ERR_INVALID, "multi_register_bq: bad arguments");
    jv_multi m = new jv_multi_s();
    m->kind = KIND_BQ; m->dim = dim; m->n = n;
    const int W = (dim + 63) / 64;
    int rc = multi_register(m, [&](int, int64_t lo, int64_t cnt, jv_dataset *ds) { return jv_dataset_register_bq(words + (size_t)lo * W, cnt, dim, ds); });
    if (rc) { jv_multi_free(m); return rc; }
    *out = m;
    return JV_OK;
}

int jv_multi_register_f32(const float *rows, int64_t n, int dim, jv_multi *out)
{
    if (!rows || !out || n <= 0 || dim <= 0 || n > 0x7fffffffLL) return fail(JV_ERR_INVALID, "multi_register_f32: bad arguments");
    jv_multi m = new jv_multi_s();
    m->kind = KIND_F32; m->dim = dim; m->n = n;
    int rc = multi_register(m, [&](int, int64_t lo, int64_t cnt, jv_dataset *ds) { return jv_dataset_register_f32(rows + (size_t)lo * dim, cnt, dim, ds); });
    if (rc) { jv_multi_free(m); return rc; }
    *out = m;
    return JV_OK;
}

int jv_multi_shard_count(jv_multi m) { return m ? (int)m->shards.size() : 0; }

int jv_multi_shard_info(jv_multi m, int shard, int *device, int64_t *first_row, int64_t *rows)
{
    if (!m || shard < 0 || shard >= (int)m->shards.size()) return fail(JV_ERR_INVALID, "multi_shard_info: bad shard");
    if (device) *device = m->devices[shard];
    if (first_row) *first_row = m->lo[shard];
    if (rows) *rows = m->lo[shard + 1] - m->lo[shard];
    return JV_OK;
}

int jv_multi_topk_bruteforce(jv_multi m, int metric, const float *queries, int nq, int k, int64_t *keys_out)
{
    if (!m || !queries || !keys_out || nq <= 0 || k <= 0 || k > 2048) return fail(JV_ERR_INVALID, "multi_topk_bruteforce: bad arguments");
    const int parts = (int)m->shards.size();
    if ((long long)parts * k > 16384) return fail(JV_ERR_INVALID, "multi_topk_bruteforce: shards * k <= 16384");
    const size_t qb = (size_t)nq * m->dim * 4, kb = (size_t)nq * k * 8;
    std::vector<int> rcs(parts, JV_OK);
    std::vector<std::string> errs(parts);
    // the gathered keys live on the first shard's device: [parts][nq][k]
    ThreadCtx *c0 = m->ctx[0];
    {
        t_active = m->devices[0];
        t_ctx_override = c0;
        cudaSetDevice(m->devices[0]);
        int rc = c0->init();
        if (!rc) rc = grow(m->gathered, kb * parts + kb);
        t_ctx_override = nullptr;
        if (rc) return rc;
    }
    long long *gathered = m->gathered.get<long long>();
    auto work = [&](int i) {
        t_active = m->devices[i];
        t_ctx_override = m->ctx[i];
        ThreadCtx &c = *m->ctx[i];
        int rc = JV_OK;
        do {
            if (cudaSetDevice(m->devices[i]) != cudaSuccess) { rc = fail(JV_ERR_CUDA, "cudaSetDevice"); break; }
            if ((rc = c.init()) || (rc = grow(c.input, qb)) || (rc = grow(c.output, kb))) break;
            if (cudaMemcpyAsync(c.input.get(), queries, qb, cudaMemcpyHostToDevice, c.stream) != cudaSuccess) { rc = fail(JV_ERR_CUDA, "H2D queries"); break; }
            if ((rc = topk_device(m->shards[i], metric, c.input.get<float>(), nq, k, m->lo[i], c.output.get<long long>()))) break;
            // shard keys -> the first device (NVLink peer copy; a plain device copy for shard 0)
            cudaError_t e = cudaMemcpyPeerAsync(gathered + (size_t)i * nq * k, m->devices[0], c.output.get(), m->devices[i], kb, c.stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
            if (e != cudaSuccess) rc = cuda_fail(e, "peer copy of shard keys");
        } while (0);
        rcs[i] = rc;
        if (rc) errs[i] = t_err;
        t_ctx_override = nullptr;
    };
    std::vector<std::thread> th;
    for (int i = 1; i < parts; i++) th.emplace_back(work, i);
    work(0);
    for (auto &t : th) t.join();
    for (int i = 0; i < parts; i++)
        if (rcs[i]) return fail(rcs[i], "shard " + std::to_string(i) + ": " + errs[i]);
    // merge on the first device: [parts][nq][k] -> per query the k best of parts * k
    t_active = m->devices[0];
    t_ctx_override = c0;
    int rc = JV_OK;
    do {
        if (cudaSetDevice(m->devices[0]) != cudaSuccess) { rc = fail(JV_ERR_CUDA, "cudaSetDevice"); break; }
        long long *merged = gathered + (size_t)parts * nq * k;
        cudaError_t e = parts == 1 ? cudaMemcpyAsync(merged, gathered, kb, cudaMemcpyDeviceToDevice, c0->stream)
                                   : launch_topk_merge_strided(gathered, nq, parts, k, merged, c0->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(keys_out, merged, kb, cudaMemcpyDeviceToHost, c0->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c0->stream);
        if (e != cudaSuccess) rc = cuda_fail(e, "merge");
    } while (0);
    t_ctx_override = nullptr;
    return rc;
}

// replicas: graph + data sets registered once per device (jv_gpu_set_device + the ordinary register calls); the query batch is
// split into contiguous slices, one per replica, searched concurrently (no data-path exchange: SURVEY §8e "shard queries")
int jv_multi_graph_search_batch(int replicas, const jv_graph *graphs, const jv_dataset *approx, const jv_dataset *rerankers, int metric,
                                const float *queries, int nq, int topK, int rerankK, const jv_search_options *opts, int32_t *nodes_out,
                                float *scores_out, jv_search_stats *stats)
{
    if (replicas <= 0 || !graphs || !approx || !queries || !nodes_out || !scores_out || nq <= 0) return fail(JV_ERR_INVALID, "multi_graph_search: bad arguments");
    if (opts && opts->accept_bits && opts->accept_stride_words == 0 && replicas > 1) { /* a shared bitset is simply reused by every slice */ }
    const int parts = std::min(replicas, nq);
    const int dim = approx[0]->d.dim;
    // worker threads come and go; their contexts (streams, visited-table scratch) must not: one persistent context per device,
    // calls of this entry point are serialised
    static ThreadCtx *worker_ctx[MAX_DEVICES] = {nullptr};
    static std::mutex worker_mu;
    std::lock_guard<std::mutex> lk(worker_mu);
    for (int i = 0; i < parts; i++) {
        if (!graphs[i] || !approx[i]) return fail(JV_ERR_INVALID, "multi_graph_search: null replica handle");
        if (!worker_ctx[graphs[i]->device]) worker_ctx[graphs[i]->device] = new ThreadCtx();
        for (int j = 0; j < i; j++)
            if (graphs[j]->device == graphs[i]->device) return fail(JV_ERR_INVALID, "multi_graph_search: two replicas on one device");
    }
    std::vector<int> rcs(parts, JV_OK);
    std::vector<std::string> errs(parts);
    std::vector<jv_search_stats> st(parts);
    std::vector<int64_t> lo;
    shard_ranges(nq, parts, lo);
    auto work = [&](int i) {
        const int q0 = (int)lo[i], cq = (int)(lo[i + 1] - lo[i]);
        jv_search_options o2;
        const jv_search_options *op = opts;
        if (opts && opts->accept_bits && opts->accept_stride_words) {
            o2 = *opts;
            o2.accept_bits = opts->accept_bits + (size_t)q0 * opts->accept_stride_words;
            op = &o2;
        }
        t_ctx_override = worker_ctx[graphs[i]->device];
        rcs[i] = jv_graph_search_batch_ex(graphs[i], approx[i], rerankers ? rerankers[i] : nullptr, metric, queries + (size_t)q0 * dim, cq, topK, rerankK, op,
                                          nodes_out + (size_t)q0 * topK, scores_out + (size_t)q0 * topK, &st[i]);
        if (rcs[i]) errs[i] = t_err;
        t_ctx_override = nullptr;
    };
    std::vector<std::thread> th;
    for (int i = 1; i < parts; i++) th.emplace_back(work, i);
    work(0);
    for (auto &t : th) t.join();
    for (int i = 0; i < parts; i++)
        if (rcs[i]) return fail(rcs[i], "replica " + std::to_string(i) + ": " + errs[i]);
    if (stats) {
        memset(stats, 0, sizeof(*stats));
        for (int i = 0; i < parts; i++) {
            stats->visited += st[i].visited; stats->expanded += st[i].expanded; stats->expanded_base += st[i].expanded_base;
            stats->reranked += st[i].reranked; stats->retried += st[i].retried;
            stats->device_ms = std::max(stats->device_ms, st[i].device_ms);  // the replicas run concurrently: the step takes the slowest one
        }
    }
    return JV_OK;
}

// ------------------------------------------------------------------------------------------------ memory helpers
int jv_device_malloc(void **out, size_t bytes)
{
    NEED_INIT();
    if (!out) return fail(JV_ERR_INVALID, "device_malloc: null");
    CK(cudaMalloc(out, bytes ? bytes : 16), "cudaMalloc");
    return JV_OK;
}
int jv_device_free(void *p)
{
    NEED_INIT();
    CK(cudaFree(p), "cudaFree");
    return JV_OK;
}
int jv_memcpy_h2d(void *dst, const void *src, size_t bytes)
{
    NEED_INIT();
    CK(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice), "cudaMemcpy H2D");
    return JV_OK;
}
int jv_memcpy_d2h(void *dst, const void *src, size_t bytes)
{
    NEED_INIT();
    CK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost), "cudaMemcpy D2H");
    return JV_OK;
}
int jv_host_register(void *p, size_t bytes)
{
    NEED_INIT();
    CK(cudaHostRegister(p, bytes, cudaHostRegisterDefault), "cudaHostRegister");
    return JV_OK;
}
int jv_host_unregister(void *p)
{
    NEED_INIT();
    CK(cudaHostUnregister(p), "cudaHostUnregister");
    return JV_OK;
}
int jv_device_synchronize(void)
{
    NEED_INIT();
    CK(cudaDeviceSynchronize(), "cudaDeviceSynchronize");
    return JV_OK;
}

}  // extern "C"
