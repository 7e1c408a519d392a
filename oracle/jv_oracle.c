/*
 * jv_oracle.c — TEST INFRASTRUCTURE ONLY (see jv_oracle.h). Scalar CPU restatement of the JVector scoring
 * hot path. Build: make -C oracle  (gcc -O2 -mfma -ffp-contract=off: only the explicit fmaf() calls fuse).
 * Not linked, loaded or called by the product library.
 */
#define _GNU_SOURCE
#include "jv_oracle.h"
#include <dlfcn.h>
#include <math.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ============================================================================================
 * float32 similarities — base:vector/DefaultVectorUtilSupport.java:41-140 (scalar provider), sequential
 * fp32 accumulation. The reference's SIMD providers differ only in summation order (SURVEY A.2).
 * ========================================================================================== */
float jvo_dot_f32(const float *a, const float *b, int n)
{
    float s = 0.f;
    for (int i = 0; i < n; i++) s += a[i] * b[i];
    return s;
}

float jvo_l2_f32(const float *a, const float *b, int n)
{
    float s = 0.f;
    for (int i = 0; i < n; i++) {
        float d = a[i] - b[i];
        s += d * d;
    }
    return s;
}

/* base:vector/DefaultVectorUtilSupport.java:123-139: (float)(sum / Math.sqrt(aMag * bMag)) */
float jvo_cosine_f32(const float *a, const float *b, int n)
{
    float sum = 0.f, am = 0.f, bm = 0.f;
    for (int i = 0; i < n; i++) {
        sum += a[i] * b[i];
        am += a[i] * a[i];
        bm += b[i] * b[i];
    }
    return (float)((double)sum / sqrt((double)(am * bm)));
}

/* native-c:src/jvector_simd_kernels.cpp:265-287 — sqrtf and an fp32 divide */
float jvo_cosine_native_f32(const float *a, const float *b, int n)
{
    float sum = 0.f, am = 0.f, bm = 0.f;
    for (int i = 0; i < n; i++) {
        sum += a[i] * b[i];
        am += a[i] * a[i];
        bm += b[i] * b[i];
    }
    return sum / sqrtf(am * bm);
}

/* base:vector/VectorSimilarityFunction.java:37-69 */
float jvo_score_from_raw(int metric, float raw)
{
    switch (metric) {
    case JVO_EUCLIDEAN: return 1.f / (1.f + raw);
    case JVO_DOT_PRODUCT: return (1.f + raw) / 2.f;
    default: return (1.f + raw) / 2.f;
    }
}

float jvo_compare_f32(int metric, const float *a, const float *b, int n)
{
    float raw = metric == JVO_EUCLIDEAN ? jvo_l2_f32(a, b, n)
              : metric == JVO_DOT_PRODUCT ? jvo_dot_f32(a, b, n) : jvo_cosine_f32(a, b, n);
    return jvo_score_from_raw(metric, raw);
}

/* ============================================================================================
 * top-k key — base:util/NumericUtils.java:49-65, base:graph/NodeQueue.java:125-137
 * ========================================================================================== */
int32_t jvo_float_to_sortable_int(float f)
{
    int32_t bits;
    memcpy(&bits, &f, 4);
    return bits ^ ((bits >> 31) & 0x7fffffff);
}

int64_t jvo_topk_key(float score, int32_t node)
{
    return (int64_t)(((uint64_t)(uint32_t)jvo_float_to_sortable_int(score)) << 32 | (uint64_t)(uint32_t)(~node));
}

float jvo_key_score(int64_t key)
{
    int32_t s = (int32_t)(key >> 32);
    int32_t bits = s ^ ((s >> 31) & 0x7fffffff);
    float f;
    memcpy(&f, &bits, 4);
    return f;
}

int32_t jvo_key_node(int64_t key) { return (int32_t)~(uint32_t)(key & 0xffffffffu); }

static int cmp_key_desc(const void *x, const void *y)
{
    int64_t a = *(const int64_t *)x, b = *(const int64_t *)y;
    return a > b ? -1 : a < b ? 1 : 0;
}

void jvo_bruteforce_topk_f32(int metric, const float *base, int64_t n, int dim, const float *q, int k, int64_t *keys_out)
{
    int64_t *keys = (int64_t *)malloc(sizeof(int64_t) * (size_t)n);
    for (int64_t i = 0; i < n; i++)
        keys[i] = jvo_topk_key(jvo_compare_f32(metric, q, base + i * dim, dim), (int32_t)i);
    qsort(keys, (size_t)n, sizeof(int64_t), cmp_key_desc);
    for (int i = 0; i < k; i++) keys_out[i] = i < n ? keys[i] : INT64_MIN;
    free(keys);
}

/* ============================================================================================
 * PQ — layout base:quantization/ProductQuantization.java:535-550; encode :507-520,422-443;
 * LUT base:quantization/PQDecoder.java:41-58 + base:vector/DefaultVectorUtilSupport.java:351-365;
 * ADC DefaultVectorUtilSupport.java:303-309; cosine PQDecoder.java:83-135 + VectorUtilSupport.java:152-165;
 * pair table ProductQuantization.java:609-628 + DefaultVectorUtilSupport.java:312-339.
 * codebooks are passed concatenated: codebook m = k*size_m floats starting at k*offsets[m].
 * ========================================================================================== */
void jvo_pq_layout(int dim, int M, int *sizes, int *offsets)
{
    int base = dim / M, rem = dim % M, off = 0;
    for (int m = 0; m < M; m++) {
        sizes[m] = base + (m < rem ? 1 : 0);
        offsets[m] = off;
        off += sizes[m];
    }
}

static const float *cb_of(const float *codebooks, const int *offsets, int k, int m) { return codebooks + (size_t)k * offsets[m]; }

void jvo_pq_encode(const float *codebooks, const int *sizes, const int *offsets, int M, int k,
                   const float *centroid, const float *v, int dim, uint8_t *codes)
{
    float *c = (float *)malloc(sizeof(float) * dim);
    for (int i = 0; i < dim; i++) c[i] = centroid ? v[i] - centroid[i] : v[i];
    for (int m = 0; m < M; m++) {
        const float *cb = cb_of(codebooks, offsets, k, m);
        float best = INFINITY;
        int bi = 0;
        for (int j = 0; j < k; j++) {
            float d = jvo_l2_f32(cb + (size_t)j * sizes[m], c + offsets[m], sizes[m]);
            if (d < best) { best = d; bi = j; }
        }
        codes[m] = (uint8_t)bi;
    }
    free(c);
}

void jvo_pq_lut(const float *codebooks, const int *sizes, const int *offsets, int M, int k,
                const float *centroid, const float *q, int dim, int metric, float *lut)
{
    float *c = (float *)malloc(sizeof(float) * dim);
    for (int i = 0; i < dim; i++) c[i] = centroid ? q[i] - centroid[i] : q[i];
    for (int m = 0; m < M; m++) {
        const float *cb = cb_of(codebooks, offsets, k, m);
        for (int j = 0; j < k; j++) {
            const float *cen = cb + (size_t)j * sizes[m];
            lut[m * k + j] = metric == JVO_EUCLIDEAN ? jvo_l2_f32(cen, c + offsets[m], sizes[m])
                                                      : jvo_dot_f32(cen, c + offsets[m], sizes[m]);
        }
    }
    free(c);
}

void jvo_pq_self_magnitudes(const float *codebooks, const int *sizes, const int *offsets, int M, int k, float *mag)
{
    for (int m = 0; m < M; m++) {
        const float *cb = cb_of(codebooks, offsets, k, m);
        for (int j = 0; j < k; j++) mag[m * k + j] = jvo_dot_f32(cb + (size_t)j * sizes[m], cb + (size_t)j * sizes[m], sizes[m]);
    }
}

float jvo_pq_adc(const float *lut, int k, const uint8_t *codes, int M)
{
    float s = 0.f;
    for (int m = 0; m < M; m++) s += lut[k * m + codes[m]];
    return s;
}

/* native-c:src/jvector_simd_kernels.cpp:821-879: sum / sqrtf(aMag * bMag) */
float jvo_pq_decoded_cosine(const uint8_t *codes, int M, int k, const float *lut, const float *mag, float bMag)
{
    float s = 0.f, a = 0.f;
    for (int m = 0; m < M; m++) {
        s += lut[k * m + codes[m]];
        a += mag[k * m + codes[m]];
    }
    return s / sqrtf(a * bMag);
}

float jvo_pq_score_lut(int metric, const float *lut, const float *mag, float bMag, int k, const uint8_t *codes, int M)
{
    if (metric == JVO_COSINE) return (1.f + jvo_pq_decoded_cosine(codes, M, k, lut, mag, bMag)) / 2.f;
    return jvo_score_from_raw(metric, jvo_pq_adc(lut, k, codes, M));
}

/* base:quantization/PQVectors.java:223-281 */
float jvo_pq_score_direct(const float *codebooks, const int *sizes, const int *offsets, int M, int k,
                          const float *centroid, const float *q, int dim, int metric, const uint8_t *codes)
{
    float *c = (float *)malloc(sizeof(float) * dim);
    for (int i = 0; i < dim; i++) c[i] = centroid ? q[i] - centroid[i] : q[i];
    float sum = 0.f, norm2 = 0.f, res;
    for (int m = 0; m < M; m++) {
        const float *cen = cb_of(codebooks, offsets, k, m) + (size_t)codes[m] * sizes[m];
        if (metric == JVO_EUCLIDEAN) sum += jvo_l2_f32(cen, c + offsets[m], sizes[m]);
        else sum += jvo_dot_f32(cen, c + offsets[m], sizes[m]);
        if (metric == JVO_COSINE) norm2 += jvo_dot_f32(cen, cen, sizes[m]);
    }
    if (metric == JVO_COSINE) {
        float norm1 = jvo_dot_f32(c, c, dim);
        float cosine = sum / (float)sqrt((double)(norm1 * norm2));
        res = (1.f + cosine) / 2.f;
    } else res = jvo_score_from_raw(metric, sum);
    free(c);
    return res;
}

/* base:quantization/PQVectors.java:284-350 */
float jvo_pq_diversity_direct(const float *codebooks, const int *sizes, const int *offsets, int M, int k,
                              int metric, const uint8_t *c1, const uint8_t *c2)
{
    float sum = 0.f, n1 = 0.f, n2 = 0.f;
    for (int m = 0; m < M; m++) {
        const float *a = cb_of(codebooks, offsets, k, m) + (size_t)c1[m] * sizes[m];
        const float *b = cb_of(codebooks, offsets, k, m) + (size_t)c2[m] * sizes[m];
        if (metric == JVO_EUCLIDEAN) sum += jvo_l2_f32(a, b, sizes[m]);
        else sum += jvo_dot_f32(b, a, sizes[m]);
        if (metric == JVO_COSINE) { n1 += jvo_dot_f32(a, a, sizes[m]); n2 += jvo_dot_f32(b, b, sizes[m]); }
    }
    if (metric == JVO_COSINE) return (1.f + sum / (float)sqrt((double)(n1 * n2))) / 2.f;
    return jvo_score_from_raw(metric, sum);
}

void jvo_pq_pair_table(const float *codebooks, const int *sizes, const int *offsets, int M, int k, int metric, float *table)
{
    size_t block = (size_t)k * (k + 1) / 2;
    for (int m = 0; m < M; m++) {
        const float *cb = cb_of(codebooks, offsets, k, m);
        size_t idx = (size_t)m * block;
        for (int i = 0; i < k; i++)
            for (int j = i; j < k; j++) {
                const float *a = cb + (size_t)i * sizes[m], *b = cb + (size_t)j * sizes[m];
                table[idx++] = metric == JVO_EUCLIDEAN ? jvo_l2_f32(a, b, sizes[m]) : jvo_dot_f32(a, b, sizes[m]);
            }
    }
}

float jvo_pq_pair_sum(const float *table, int M, int k, const uint8_t *c1, const uint8_t *c2)
{
    int block = k * (k + 1) / 2;
    float res = 0.f;
    for (int i = 0; i < M; i++) {
        int a = c1[i], b = c2[i];
        int r = a < b ? a : b, c = a < b ? b : a;
        int offsetRow = r * k - (r * (r - 1) / 2);
        res += table[(size_t)i * block + offsetRow + (c - r)];
    }
    return res;
}

/* ImmutablePQVectors.diversityFunctionFor (base:quantization/ImmutablePQVectors.java:63-105): code-vs-code score from the
 * triangular table (assembleAndSumPQ); `table` is the squared-L2 table for EUCLIDEAN, the dot-product table otherwise */
float jvo_pq_diversity_table(int metric, const float *table, int M, int k, const uint8_t *c1, const uint8_t *c2)
{
    float sum = jvo_pq_pair_sum(table, M, k, c1, c2);
    if (metric == JVO_EUCLIDEAN) return 1.f / (1.f + sum);
    if (metric == JVO_DOT_PRODUCT) return (1.f + sum) / 2.f;
    float n1 = jvo_pq_pair_sum(table, M, k, c1, c1), n2 = jvo_pq_pair_sum(table, M, k, c2, c2);
    float cosine = sum / (float)sqrt((double)(n1 * n2));
    return (1.f + cosine) / 2.f;
}

/* KMeansPlusPlusClusterer.getNearestCluster (base:quantization/KMeansPlusPlusClusterer.java:329-342) for a batch of points */
void jvo_kmeans_assign(const float *points, int64_t n, int dim, const float *centroids, int k, int32_t *assign)
{
    for (int64_t p = 0; p < n; p++) {
        float minDistance = 3.402823466e+38f;
        int nearest = 0;
        for (int i = 0; i < k; i++) {
            float d = jvo_l2_f32(points + (size_t)p * dim, centroids + (size_t)i * dim, dim);
            if (d < minDistance) { minDistance = d; nearest = i; }
        }
        assign[p] = nearest;
    }
}

/* ============================================================================================
 * BQ — base:quantization/BinaryQuantization.java:88-110, base:vector/DefaultVectorUtilSupport.java:342-348,
 * base:quantization/BQVectors.java:116-118
 * ========================================================================================== */
void jvo_bq_encode(const float *v, int dim, uint64_t *words)
{
    int W = (dim + 63) / 64;
    for (int i = 0; i < W; i++) {
        uint64_t bits = 0;
        for (int j = 0; j < 64; j++) {
            int idx = i * 64 + j;
            if (idx >= dim) break;
            if (v[idx] > 0) bits |= 1ull << j;
        }
        words[i] = bits;
    }
}

int jvo_hamming(const uint64_t *a, const uint64_t *b, int words)
{
    int hd = 0;
    for (int i = 0; i < words; i++) hd += __builtin_popcountll(a[i] ^ b[i]);
    return hd;
}

float jvo_bq_score(const uint64_t *a, const uint64_t *b, int words, int dim)
{
    return 1.f - (float)jvo_hamming(a, b, words) / (float)dim;
}

/* ============================================================================================
 * NVQ 8-bit — SIMD/native form: jvector-twenty/.../PanamaVectorUtilSupport.java:1164-1237 and
 * native-c:src/jvector_simd_kernels.cpp:1047-1111 (logistic / logit), :1149-1197 (quantize), :1199-1303
 * (loss), :1359-1502,1558-1641 (distances). Element order is natural (the reference's query shuffle is a
 * private lane layout, base:vector/DefaultVectorUtilSupport.java:454 is a no-op).
 * ========================================================================================== */
static inline int32_t f2i(float f) { int32_t i; memcpy(&i, &f, 4); return i; }
static inline float i2f(int32_t i) { float f; memcpy(&f, &i, 4); return f; }

float jvo_nvq_logistic(float v, float alpha, float x0)
{
    float t = fmaf(v, alpha, -alpha * x0);
    int32_t p = signbit(t) ? (int32_t)t : (int32_t)(t + 1.0f); /* truncation toward zero */
    float e = (float)p;
    int32_t m = f2i(fmaf(t - e, 0.5f, 1.0f));
    float r = i2f((int32_t)((uint32_t)m + ((uint32_t)p << 23)));
    return r / (r + 1.0f);
}

float jvo_nvq_logit(float v, float inverseAlpha, float x0)
{
    float z = v / (1.0f - v);
    int32_t t = f2i(z);
    int32_t p = ((t & 0x7f800000) >> 23) - 128;
    float m = i2f((t & 0x007fffff) + 0x3f800000);
    return fmaf(m + (float)p, inverseAlpha, x0);
}

typedef struct { float sa, isa, sx0, bias, scale; } nvq_consts;

static nvq_consts nvq_setup(float alpha, float x0, float minv, float maxv, float levels)
{
    nvq_consts c;
    float delta = maxv - minv;
    c.sa = alpha / delta;
    c.isa = delta / alpha; /* native-c:...:1380 */
    c.sx0 = x0 * delta;
    c.bias = jvo_nvq_logistic(minv, c.sa, c.sx0);
    c.scale = (jvo_nvq_logistic(maxv, c.sa, c.sx0) - c.bias) / levels;
    return c;
}

static inline float nvq_dq(const nvq_consts *c, float byteval)
{
    return jvo_nvq_logit(fmaf(byteval, c->scale, c->bias), c->isa, c->sx0);
}

float jvo_nvq_dequant(uint8_t b, float alpha, float x0, float minv, float maxv)
{
    nvq_consts c = nvq_setup(alpha, x0, minv, maxv, 255.0f);
    return nvq_dq(&c, (float)b);
}

void jvo_nvq_quantize_8bit(const float *v, int n, float alpha, float x0, float minv, float maxv, uint8_t *dst)
{
    float delta = maxv - minv, sa = alpha / delta, sx0 = x0 * delta;
    float bias = jvo_nvq_logistic(minv, sa, sx0);
    float inv = 255.0f / (jvo_nvq_logistic(maxv, sa, sx0) - bias);
    for (int i = 0; i < n; i++) {
        /* the reference is compiled with GCC's default -ffp-contract=fast, which fuses Mul+Add here
         * (pinned against oracle/_ref in tests/test_oracle_ref.py) */
        float a = fmaf(jvo_nvq_logistic(v[i], sa, sx0) - bias, inv, 0.5f);
        int q = (int)a;
        dst[i] = (uint8_t)(q < 0 ? 0 : q > 255 ? 255 : q);
    }
}

float jvo_nvq_loss(const float *v, int n, float alpha, float x0, float minv, float maxv, int nbits)
{
    float levels = (float)((1 << nbits) - 1);
    nvq_consts c = nvq_setup(alpha, x0, minv, maxv, levels);
    float inv = 1.0f / c.scale, s = 0.f;
    for (int i = 0; i < n; i++) {
        float r = (jvo_nvq_logistic(v[i], c.sa, c.sx0) - c.bias) * inv;
        float rq = (float)(int)(r + 0.5f);
        float d = v[i] - nvq_dq(&c, rq);
        s = fmaf(d, d, s);
    }
    return s;
}

float jvo_nvq_uniform_loss(const float *v, int n, float minv, float maxv, int nbits)
{
    float constant = (float)((1 << nbits) - 1), delta = maxv - minv, s = 0.f;
    for (int i = 0; i < n; i++) {
        float r = (v[i] - minv) * (constant / delta);
        float rq = (float)(int)(r + 0.5f);
        float rec = fmaf(rq, delta / constant, minv);
        float d = v[i] - rec;
        s = fmaf(d, d, s);
    }
    return s;
}

float jvo_nvq_dot_8bit(const float *q, const uint8_t *b, int n, float alpha, float x0, float minv, float maxv)
{
    nvq_consts c = nvq_setup(alpha, x0, minv, maxv, 255.0f);
    float s = 0.f;
    for (int i = 0; i < n; i++) s = fmaf(q[i], nvq_dq(&c, (float)b[i]), s);
    return s;
}

float jvo_nvq_l2_8bit(const float *q, const uint8_t *b, int n, float alpha, float x0, float minv, float maxv)
{
    nvq_consts c = nvq_setup(alpha, x0, minv, maxv, 255.0f);
    float s = 0.f;
    for (int i = 0; i < n; i++) {
        float d = q[i] - nvq_dq(&c, (float)b[i]);
        s = fmaf(d, d, s);
    }
    return s;
}

void jvo_nvq_cosine_8bit(const float *q, const uint8_t *b, int n, float alpha, float x0, float minv, float maxv,
                         const float *centroid, float *out2)
{
    nvq_consts c = nvq_setup(alpha, x0, minv, maxv, 255.0f);
    float s = 0.f, nm = 0.f;
    for (int i = 0; i < n; i++) {
        float e = nvq_dq(&c, (float)b[i]) + centroid[i];
        s = fmaf(q[i], e, s);
        nm = fmaf(e, e, nm);
    }
    out2[0] = s;
    out2[1] = nm;
}

/* ---- the loss sums under an explicit summation order ------------------------------------------------------------------
 * The reference defines nvqLoss / nvqUniformLoss only up to the order of the float additions: the scalar provider sums
 * sequentially (base:vector/DefaultVectorUtilSupport.java:493-520), the Panama provider keeps SPECIES_PREFERRED lane
 * accumulators (element i goes to lane i mod lanes) and then reduceLanes (jvector-twenty/.../PanamaVectorUtilSupport.java:
 * 1270-1330), the native provider does the same with Highway lanes (native-c:src/jvector_simd_kernels.cpp:1199-1303).
 * `lanes` selects a member of that family: 1 = sequential (the functions above); 32 = thirty-two strided accumulators folded
 * by a xor butterfly (16, 8, 4, 2, 1), which is the order a 32-lane GPU warp produces. The growth-rate grid search compares
 * these sums, so bit-exact parameters need the same order on both sides; all orders agree to ~1e-6 relative (tests). */
static float lanes_fold(float *acc, int lanes)
{
    float tmp[64];
    for (int o = lanes >> 1; o > 0; o >>= 1) {
        for (int l = 0; l < lanes; l++) tmp[l] = acc[l] + acc[l ^ o];
        memcpy(acc, tmp, sizeof(float) * (size_t)lanes);
    }
    return acc[0];
}

float jvo_nvq_loss_lanes(const float *v, int n, float alpha, float x0, float minv, float maxv, int nbits, int lanes)
{
    if (lanes <= 1) return jvo_nvq_loss(v, n, alpha, x0, minv, maxv, nbits);
    float levels = (float)((1 << nbits) - 1);
    nvq_consts c = nvq_setup(alpha, x0, minv, maxv, levels);
    float inv = 1.0f / c.scale, acc[64] = {0};
    for (int i = 0; i < n; i++) {
        float r = (jvo_nvq_logistic(v[i], c.sa, c.sx0) - c.bias) * inv;
        float rq = (float)(int)(r + 0.5f);
        float d = v[i] - nvq_dq(&c, rq);
        acc[i % lanes] = fmaf(d, d, acc[i % lanes]);
    }
    return lanes_fold(acc, lanes);
}

float jvo_nvq_uniform_loss_lanes(const float *v, int n, float minv, float maxv, int nbits, int lanes)
{
    if (lanes <= 1) return jvo_nvq_uniform_loss(v, n, minv, maxv, nbits);
    float constant = (float)((1 << nbits) - 1), delta = maxv - minv, acc[64] = {0};
    for (int i = 0; i < n; i++) {
        float r = (v[i] - minv) * (constant / delta);
        float rq = (float)(int)(r + 0.5f);
        float rec = fmaf(rq, delta / constant, minv);
        float d = v[i] - rec;
        acc[i % lanes] = fmaf(d, d, acc[i % lanes]);
    }
    return lanes_fold(acc, lanes);
}

/* base:quantization/NVQuantization.java:524-578 (parameter search) */
void jvo_nvq_encode_subvector_lanes(const float *v, int n, int learn, int lanes, float *params_out, uint8_t *bytes_out)
{
    float minv = 3.402823466e+38f, maxv = -3.402823466e+38f;
    for (int i = 0; i < n; i++) {
        if (v[i] < minv) minv = v[i];
        if (v[i] > maxv) maxv = v[i];
    }
    float growth = 1e-2f, mid = 0.f;
    if (learn) {
        float baseline = jvo_nvq_uniform_loss_lanes(v, n, minv, maxv, 8, lanes);
        float coarse = 1e-2f, best = 1.40129846e-45f; /* Float.MIN_VALUE */
        for (float gr = 1e-6f; gr < 20.f; gr += 1.f) {
            float lv = baseline / jvo_nvq_loss_lanes(v, n, gr, 0.f, minv, maxv, 8, lanes);
            if (lv > best) { best = lv; coarse = gr; }
        }
        float fine = coarse;
        for (float gr = coarse - 1; gr < coarse + 1; gr += 0.1f) {
            float lv = baseline / jvo_nvq_loss_lanes(v, n, gr, 0.f, minv, maxv, 8, lanes);
            if (lv > best) { best = lv; fine = gr; }
        }
        growth = fine;
    }
    jvo_nvq_quantize_8bit(v, n, growth, mid, minv, maxv, bytes_out);
    params_out[0] = minv; params_out[1] = maxv; params_out[2] = growth; params_out[3] = mid;
}

void jvo_nvq_encode_subvector(const float *v, int n, int learn, float *params_out, uint8_t *bytes_out)
{
    jvo_nvq_encode_subvector_lanes(v, n, learn, 1, params_out, bytes_out);
}

/* base:quantization/NVQuantization.java:201-251 */
void jvo_nvq_encode_lanes(const float *v, const float *mean, int dim, int nsub, int learn, int lanes, float *params_out, uint8_t *bytes_out)
{
    int *sizes = (int *)malloc(sizeof(int) * nsub * 2), *offsets = sizes + nsub;
    float *c = (float *)malloc(sizeof(float) * dim);
    jvo_pq_layout(dim, nsub, sizes, offsets);
    for (int i = 0; i < dim; i++) c[i] = v[i] - mean[i];
    for (int s = 0; s < nsub; s++) jvo_nvq_encode_subvector_lanes(c + offsets[s], sizes[s], learn, lanes, params_out + 4 * s, bytes_out + offsets[s]);
    free(c);
    free(sizes);
}

void jvo_nvq_encode(const float *v, const float *mean, int dim, int nsub, int learn, float *params_out, uint8_t *bytes_out)
{
    jvo_nvq_encode_lanes(v, mean, dim, nsub, learn, 1, params_out, bytes_out);
}

/* base:quantization/NVQScorer.java:46-137 */
float jvo_nvq_score(int metric, const float *q, const float *mean, int dim, int nsub,
                    const float *params, const uint8_t *bytes)
{
    int *sizes = (int *)malloc(sizeof(int) * nsub * 2), *offsets = sizes + nsub;
    jvo_pq_layout(dim, nsub, sizes, offsets);
    float res;
    if (metric == JVO_DOT_PRODUCT) {
        float bias = jvo_dot_f32(q, mean, dim), acc = 0.f;
        for (int s = 0; s < nsub; s++) {
            const float *p = params + 4 * s;
            acc += jvo_nvq_dot_8bit(q + offsets[s], bytes + offsets[s], sizes[s], p[2], p[3], p[0], p[1]);
        }
        res = (1.f + acc + bias) / 2.f;
    } else if (metric == JVO_EUCLIDEAN) {
        float *sh = (float *)malloc(sizeof(float) * dim), acc = 0.f;
        for (int i = 0; i < dim; i++) sh[i] = q[i] - mean[i];
        for (int s = 0; s < nsub; s++) {
            const float *p = params + 4 * s;
            acc += jvo_nvq_l2_8bit(sh + offsets[s], bytes + offsets[s], sizes[s], p[2], p[3], p[0], p[1]);
        }
        free(sh);
        res = 1.f / (1.f + acc);
    } else {
        float qn = (float)sqrt((double)jvo_dot_f32(q, q, dim)), c0 = 0.f, c1 = 0.f, o[2];
        for (int s = 0; s < nsub; s++) {
            const float *p = params + 4 * s;
            jvo_nvq_cosine_8bit(q + offsets[s], bytes + offsets[s], sizes[s], p[2], p[3], p[0], p[1], mean + offsets[s], o);
            c0 += o[0];
            c1 += o[1];
        }
        float cosine = (c0 / qn) / (float)sqrt((double)c1);
        res = (1.f + cosine) / 2.f;
    }
    free(sizes);
    return res;
}

/* ============================================================================================
 * Optional routing through the reference's own compiled kernels (oracle/_ref/libjvector.so):
 * exactly the downcalls jvector-native/.../NativeVectorUtilSupport.java:95-298 makes.
 * ========================================================================================== */
typedef float (*fn_sim)(const float *, size_t, const float *, size_t, size_t);
typedef float (*fn_adc)(const float *, int, const unsigned char *, int, size_t);
typedef void (*fn_ps)(const float *, int, size_t, int, const float *, int, float *);
typedef void (*fn_psm)(const float *, int, size_t, int, float *);
typedef float (*fn_pqcos)(const unsigned char *, int, size_t, int, const float *, const float *, float);
typedef float (*fn_nvq)(const float *, const unsigned char *, size_t, float, float, float, float);
typedef int64_t (*fn_nvqcos)(const float *, const unsigned char *, size_t, float, float, float, float, const float *);
typedef void (*fn_shuf)(float *, size_t);
typedef void (*fn_nvqq)(const float *, size_t, float, float, float, float, unsigned char *);
typedef float (*fn_nvql)(const float *, size_t, float, float, float, float, int);
typedef float (*fn_nvqu)(const float *, size_t, float, float, int);
typedef const char *(*fn_str)(void);

static struct {
    void *h;
    fn_sim dot, l2, cos;
    fn_adc adc;
    fn_ps ps_dot, ps_l2;
    fn_psm ps_mag;
    fn_pqcos pqcos;
    fn_nvq nvq_dot, nvq_l2;
    fn_nvqcos nvq_cos;
    fn_shuf shuffle;
    fn_nvqq nvq_quant;
    fn_nvql nvq_lossf;
    fn_nvqu nvq_uloss;
    fn_str isa;
} REF;

int jvo_use_ref(const char *path)
{
    if (!path) { memset(&REF, 0, sizeof(REF)); return 0; }
    void *h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
    if (!h) return -1;
    REF.h = h;
    REF.dot = (fn_sim)dlsym(h, "dot_product_f32");
    REF.l2 = (fn_sim)dlsym(h, "euclidean_f32");
    REF.cos = (fn_sim)dlsym(h, "cosine_f32");
    REF.adc = (fn_adc)dlsym(h, "assemble_and_sum_f32");
    REF.ps_dot = (fn_ps)dlsym(h, "calculate_partial_sums_dot_f32");
    REF.ps_l2 = (fn_ps)dlsym(h, "calculate_partial_sums_euclidean_f32");
    REF.ps_mag = (fn_psm)dlsym(h, "calculate_partial_sums_self_magnitude_f32");
    REF.pqcos = (fn_pqcos)dlsym(h, "pq_decoded_cosine_similarity_f32");
    REF.nvq_dot = (fn_nvq)dlsym(h, "nvq_dot_product_8bit");
    REF.nvq_l2 = (fn_nvq)dlsym(h, "nvq_square_l2_distance_8bit");
    REF.nvq_cos = (fn_nvqcos)dlsym(h, "nvq_cosine_8bit_packed");
    REF.shuffle = (fn_shuf)dlsym(h, "nvq_shuffle_query_in_place_8bit");
    REF.nvq_quant = (fn_nvqq)dlsym(h, "nvq_quantize_8bit");
    REF.nvq_lossf = (fn_nvql)dlsym(h, "nvq_loss");
    REF.nvq_uloss = (fn_nvqu)dlsym(h, "nvq_uniform_loss");
    REF.isa = (fn_str)dlsym(h, "jvector_simd_get_active_isa");
    if (!REF.dot || !REF.l2 || !REF.cos || !REF.adc || !REF.ps_dot || !REF.ps_l2 || !REF.ps_mag || !REF.pqcos ||
        !REF.nvq_dot || !REF.nvq_l2 || !REF.nvq_cos || !REF.shuffle || !REF.isa) {
        memset(&REF, 0, sizeof(REF));
        return -2;
    }
    return 0;
}

const char *jvo_ref_isa(void) { return REF.isa ? REF.isa() : "port"; }

/* ============================================================================================
 * score contexts: ScoreFunction.similarityTo(node) for one query
 * (base:graph/similarity/DefaultSearchScoreProvider.java:71-80, base:quantization/PQDecoder.java,
 *  BQVectors.java:108-118, NVQScorer.java)
 * ========================================================================================== */
/* ============================================================================================
 * WARP-ORDER restatements. The float sums of the path are defined up to the order of the additions (SURVEY A.2: the scalar
 * provider sums sequentially, Panama keeps 2 vector accumulators, the native library 4 Highway accumulators; the reference's
 * tests accept 1e-4). A traversal, however, is only reproducible id for id when both sides produce the SAME bits, so the
 * oracle can also evaluate every score in the one order the sm_90a kernels use (jvector_b200/csrc/scorers.cuh): elements
 * dealt to 32 (fp32 rows, NVQ bytes) or 8 (PQ code rows) lane accumulators, fused multiply-adds, lanes folded by a xor
 * butterfly; block-wide sums (query norms) over 256 strided accumulators folded warp by warp. Same arithmetic, same formulas
 * (cited at each function), one fixed member of the family of orders the reference itself ships.
 * jvo_scorer_set_order(s, 1) switches a scorer to it; order 0 (default) is the sequential / reference-kernel arithmetic.
 * ========================================================================================== */
static float block256_sum(const float *acc /* 256 */)
{
    float red[32];
    for (int w = 0; w < 32; w++) red[w] = 0.f;
    for (int w = 0; w < 8; w++) {
        float lanes[32];
        memcpy(lanes, acc + 32 * w, sizeof(lanes));
        red[w] = lanes_fold(lanes, 32);
    }
    return lanes_fold(red, 32);
}

/* prepare_blob's ||q||^2-style sums: element i goes to accumulator i mod 256 */
static float block256_dot(const float *a, const float *b, int n)
{
    float acc[256] = {0};
    for (int i = 0; i < n; i++) acc[i & 255] = fmaf(a[i], b[i], acc[i & 255]);
    return block256_sum(acc);
}

/* score_f32_vec / score_f32_pair: float4 j of the row goes to lane j mod 32; four accumulators per lane (x, y, z, w) */
static float warp_raw_f32(int metric, const float *q, const float *row, int dim, float qnorm2)
{
    float s[32][4] = {{0}}, b0[32] = {0}, b1[32] = {0}, lanes[32];
    for (int i = 0; i < dim; i++) {
        const int l = (i >> 2) & 31, c = i & 3;
        if (metric == JVO_EUCLIDEAN) {
            float d = q[i] - row[i];
            s[l][c] = fmaf(d, d, s[l][c]);
        } else {
            s[l][c] = fmaf(q[i], row[i], s[l][c]);
            if (metric == JVO_COSINE) {
                if (c & 1) b1[l] = fmaf(row[i], row[i], b1[l]);
                else b0[l] = fmaf(row[i], row[i], b0[l]);
            }
        }
    }
    for (int l = 0; l < 32; l++) lanes[l] = (s[l][0] + s[l][1]) + (s[l][2] + s[l][3]);
    float r = lanes_fold(lanes, 32);
    if (metric == JVO_COSINE) {
        for (int l = 0; l < 32; l++) lanes[l] = b0[l] + b1[l];
        r = r / sqrtf(qnorm2 * lanes_fold(lanes, 32));
    }
    return r;
}

float jvo_compare_f32_warp(int metric, const float *q, const float *row, int dim)
{
    return jvo_score_from_raw(metric, warp_raw_f32(metric, q, row, dim, metric == JVO_COSINE ? block256_dot(q, q, dim) : 0.f));
}

/* prepare_blob (PQ branch) and pq_self_mag_kernel: every table entry is one sequential fused chain over the sub-vector */
static void warp_pq_tables(const float *codebooks, const int *sizes, const int *offsets, int M, int k, const float *centroid,
                           const float *q, int dim, int metric, float *lut, float *mag, float *bMag)
{
    float *c = (float *)malloc(sizeof(float) * dim);
    for (int i = 0; i < dim; i++) c[i] = centroid ? q[i] - centroid[i] : q[i];
    for (int m = 0; m < M; m++) {
        const float *cb = cb_of(codebooks, offsets, k, m);
        for (int j = 0; j < k; j++) {
            const float *cen = cb + (size_t)j * sizes[m];
            float t = 0.f, g = 0.f;
            for (int e = 0; e < sizes[m]; e++) {
                if (metric == JVO_EUCLIDEAN) {
                    float d = cen[e] - c[offsets[m] + e];
                    t = fmaf(d, d, t);
                } else t = fmaf(cen[e], c[offsets[m] + e], t);
                g = fmaf(cen[e], cen[e], g);
            }
            lut[m * k + j] = t;
            if (mag) mag[m * k + j] = g;
        }
    }
    *bMag = block256_dot(c, c, dim);
    free(c);
}

/* score_pq: 32-bit word j of the code row (4 codes) goes to lane j mod 8, its 4 entries added in code order; a tail of
 * M mod 4 codes goes one code per lane */
static float warp_pq_score(int metric, const float *lut, const float *mag, float bMag, int k, const uint8_t *codes, int M)
{
    float s[8] = {0}, a[8] = {0};
    const int M4 = M >> 2;
    for (int j = 0; j < M4; j++)
        for (int e = 0; e < 4; e++) {
            const int m = 4 * j + e, idx = m * k + codes[m];
            s[j & 7] = s[j & 7] + lut[idx];
            if (metric == JVO_COSINE) a[j & 7] = a[j & 7] + mag[idx];
        }
    for (int m = 4 * M4; m < M; m++) {
        const int g = (m - 4 * M4) & 7, idx = m * k + codes[m];
        s[g] = s[g] + lut[idx];
        if (metric == JVO_COSINE) a[g] = a[g] + mag[idx];
    }
    float r = lanes_fold(s, 8);
    if (metric == JVO_COSINE) r = r / sqrtf(lanes_fold(a, 8) * bMag);
    return jvo_score_from_raw(metric, r);
}

/* score_nvq: one accumulator per lane across all sub-vectors; a sub-vector whose offset and size are multiples of 4 is dealt
 * four bytes at a time (word j to lane j mod 32), otherwise byte i to lane i mod 32 */
static float warp_nvq_score(int metric, const float *qs /* shifted for L2 */, const float *mean, int nsub, const int *sizes,
                            const int *offsets, const float *params, const uint8_t *bytes, float qbias, float qnorm)
{
    float s[32] = {0}, nm[32] = {0};
    for (int sv = 0; sv < nsub; sv++) {
        const float *pp = params + 4 * sv;
        nvq_consts c = nvq_setup(pp[2], pp[3], pp[0], pp[1], 255.0f);
        const int off = offsets[sv], sz = sizes[sv], vec = ((off | sz) & 3) == 0;
        for (int i = 0; i < sz; i++) {
            const int l = vec ? ((i >> 2) & 31) : (i & 31);
            const float dq = nvq_dq(&c, (float)bytes[off + i]), q = qs[off + i];
            if (metric == JVO_DOT_PRODUCT) s[l] = fmaf(q, dq, s[l]);
            else if (metric == JVO_EUCLIDEAN) {
                float d = q - dq;
                s[l] = fmaf(d, d, s[l]);
            } else {
                float e = dq + mean[off + i];
                s[l] = fmaf(q, e, s[l]);
                nm[l] = fmaf(e, e, nm[l]);
            }
        }
    }
    float r = lanes_fold(s, 32);
    if (metric == JVO_DOT_PRODUCT) return ((1.0f + r) + qbias) / 2.0f;
    if (metric == JVO_EUCLIDEAN) return 1.0f / (1.0f + r);
    float cosine = (r / qnorm) / sqrtf(lanes_fold(nm, 32));
    return (1.0f + cosine) / 2.0f;
}

struct jvo_scorer {
    int kind; /* 0 f32, 1 pq, 2 bq, 3 nvq */
    int metric, dim;
    int64_t n;
    const float *base;
    float *q; /* owned copy (shifted / shuffled as the kind requires) */
    /* pq */
    int M, k;
    const uint8_t *codes;
    float *lut, *mag;
    float bMag;
    /* bq */
    const uint64_t *words;
    uint64_t *qbits;
    int W;
    /* nvq */
    int nsub;
    int *sizes, *offsets;
    const float *params;
    const uint8_t *bytes;
    const float *mean;
    float *mean_sh; /* shuffled copy of mean sub-vectors (cosine, ref path) */
    float qbias, qnorm;
    /* FusedPQ: packed[node] = the codes of node's level-0 neighbours, in neighbour order (jvo_fused_pq_pack) */
    const uint8_t *packed;
    int packed_degree;
    /* warp order (jvo_scorer_set_order) */
    int order;
    const float *codebooks, *centroid;
    float *q_raw;               /* the query as given */
    float *wlut, *wmag, wbMag;  /* PQ tables in warp order */
    float *wq, wqbias, wqnorm;  /* NVQ prepared query in warp order */
};

void jvo_scorer_set_order(jvo_scorer *s, int order)
{
    s->order = order;
    if (!order) return;
    if (s->kind == 1 && !s->wlut) {
        s->wlut = (float *)malloc(sizeof(float) * s->M * s->k);
        s->wmag = (float *)malloc(sizeof(float) * s->M * s->k);
        warp_pq_tables(s->codebooks, s->sizes, s->offsets, s->M, s->k, s->centroid, s->q_raw, s->dim,
                       s->metric == JVO_EUCLIDEAN ? JVO_EUCLIDEAN : JVO_DOT_PRODUCT, s->wlut, s->wmag, &s->wbMag);
    }
    if (s->kind == 3 && !s->wq) {
        /* prepare_blob (NVQ branch): DOT keeps q and adds <q, mean>; L2 shifts q by the mean; COSINE keeps q and needs ||q|| */
        s->wq = (float *)malloc(sizeof(float) * s->dim);
        for (int i = 0; i < s->dim; i++) s->wq[i] = s->metric == JVO_EUCLIDEAN ? s->q_raw[i] - s->mean[i] : s->q_raw[i];
        s->wqbias = block256_dot(s->q_raw, s->mean, s->dim);
        s->wqnorm = sqrtf(block256_dot(s->q_raw, s->q_raw, s->dim));
    }
}

jvo_scorer *jvo_scorer_f32(int metric, const float *base, int64_t n, int dim, const float *q)
{
    jvo_scorer *s = (jvo_scorer *)calloc(1, sizeof(*s));
    s->kind = 0; s->metric = metric; s->dim = dim; s->n = n; s->base = base;
    s->q = (float *)malloc(sizeof(float) * dim);
    memcpy(s->q, q, sizeof(float) * dim);
    s->wqnorm = block256_dot(q, q, dim);
    return s;
}

jvo_scorer *jvo_scorer_pq(int metric, const float *codebooks, int M, int k, int dim, const float *centroid,
                          const uint8_t *codes, int64_t n, const float *q)
{
    jvo_scorer *s = (jvo_scorer *)calloc(1, sizeof(*s));
    s->kind = 1; s->metric = metric; s->dim = dim; s->n = n; s->M = M; s->k = k; s->codes = codes;
    s->codebooks = codebooks; s->centroid = centroid;
    s->q_raw = (float *)malloc(sizeof(float) * dim);
    memcpy(s->q_raw, q, sizeof(float) * dim);
    s->sizes = (int *)malloc(sizeof(int) * 2 * M);
    s->offsets = s->sizes + M;
    jvo_pq_layout(dim, M, s->sizes, s->offsets);
    s->lut = (float *)malloc(sizeof(float) * M * k);
    int lm = metric == JVO_EUCLIDEAN ? JVO_EUCLIDEAN : JVO_DOT_PRODUCT;
    if (REF.h) {
        float *c = (float *)malloc(sizeof(float) * dim);
        for (int i = 0; i < dim; i++) c[i] = centroid ? q[i] - centroid[i] : q[i];
        for (int m = 0; m < M; m++) {
            const float *cb = cb_of(codebooks, s->offsets, k, m);
            (lm == JVO_EUCLIDEAN ? REF.ps_l2 : REF.ps_dot)(cb, m, (size_t)s->sizes[m], k, c, s->offsets[m], s->lut);
        }
        if (metric == JVO_COSINE) {
            s->mag = (float *)malloc(sizeof(float) * M * k);
            for (int m = 0; m < M; m++) REF.ps_mag(cb_of(codebooks, s->offsets, k, m), m, (size_t)s->sizes[m], k, s->mag);
            s->bMag = REF.dot(c, 0, c, 0, (size_t)dim);
        }
        free(c);
    } else {
        jvo_pq_lut(codebooks, s->sizes, s->offsets, M, k, centroid, q, dim, lm, s->lut);
        if (metric == JVO_COSINE) {
            s->mag = (float *)malloc(sizeof(float) * M * k);
            jvo_pq_self_magnitudes(codebooks, s->sizes, s->offsets, M, k, s->mag);
            float *c = (float *)malloc(sizeof(float) * dim);
            for (int i = 0; i < dim; i++) c[i] = centroid ? q[i] - centroid[i] : q[i];
            s->bMag = jvo_dot_f32(c, c, dim);
            free(c);
        }
    }
    return s;
}

jvo_scorer *jvo_scorer_bq(const uint64_t *words, int64_t n, int dim, const float *q)
{
    jvo_scorer *s = (jvo_scorer *)calloc(1, sizeof(*s));
    s->kind = 2; s->dim = dim; s->n = n; s->words = words; s->W = (dim + 63) / 64;
    s->qbits = (uint64_t *)malloc(sizeof(uint64_t) * s->W);
    jvo_bq_encode(q, dim, s->qbits);
    return s;
}

jvo_scorer *jvo_scorer_nvq(int metric, const float *mean, int dim, int nsub, const float *params,
                           const uint8_t *bytes, int64_t n, const float *q)
{
    jvo_scorer *s = (jvo_scorer *)calloc(1, sizeof(*s));
    s->kind = 3; s->metric = metric; s->dim = dim; s->n = n; s->nsub = nsub; s->params = params; s->bytes = bytes; s->mean = mean;
    s->sizes = (int *)malloc(sizeof(int) * 2 * nsub);
    s->offsets = s->sizes + nsub;
    jvo_pq_layout(dim, nsub, s->sizes, s->offsets);
    s->q_raw = (float *)malloc(sizeof(float) * dim);
    memcpy(s->q_raw, q, sizeof(float) * dim);
    s->q = (float *)malloc(sizeof(float) * dim);
    for (int i = 0; i < dim; i++) s->q[i] = metric == JVO_EUCLIDEAN ? q[i] - mean[i] : q[i];
    s->qbias = jvo_dot_f32(q, mean, dim);
    s->qnorm = (float)sqrt((double)jvo_dot_f32(q, q, dim));
    if (REF.h) { /* the reference kernels need their private lane order: NVQScorer.java:57-59,88-90,114-117 */
        s->mean_sh = (float *)malloc(sizeof(float) * dim);
        memcpy(s->mean_sh, mean, sizeof(float) * dim);
        for (int i = 0; i < nsub; i++) {
            REF.shuffle(s->q + s->offsets[i], (size_t)s->sizes[i]);
            REF.shuffle(s->mean_sh + s->offsets[i], (size_t)s->sizes[i]);
        }
    }
    return s;
}

/* FusedPQ.writeInline (base:graph/disk/feature/FusedPQ.java:122-141): for every node, the PQ codes of its level-0 neighbours in
 * neighbour order, zero codes up to maxDegree. packed_out [n][degree][M]. */
void jvo_fused_pq_pack(const int32_t *adj0, int32_t n, int degree, const uint8_t *codes, int M, uint8_t *packed_out)
{
    for (int32_t v = 0; v < n; v++)
        for (int i = 0; i < degree; i++) {
            int32_t f = adj0[(size_t)v * degree + i];
            uint8_t *dst = packed_out + ((size_t)v * degree + i) * M;
            if (f >= 0) memcpy(dst, codes + (size_t)f * M, (size_t)M);
            else memset(dst, 0, (size_t)M);
        }
}

/* FusedPQ.approximateScoreFunctionFor (FusedPQ.java:119-123): a PQ scorer that also knows the packed neighbour codes */
void jvo_scorer_set_packed_neighbors(jvo_scorer *s, const uint8_t *packed, int degree)
{
    s->packed = packed;
    s->packed_degree = degree;
}

/* FusedPQDecoder.similarityToNeighbor (base:quantization/FusedPQDecoder.java:107-114, cosine :187-195): the neighbourIndex-th
 * code row of origin's packed block through the same assembleAndSum / pqDecodedCosineSimilarity as similarityTo */
float jvo_scorer_score_neighbor(jvo_scorer *s, int32_t origin, int neighborIndex)
{
    const uint8_t *c = s->packed + ((size_t)origin * s->packed_degree + neighborIndex) * s->M;
    if (s->order) return warp_pq_score(s->metric, s->wlut, s->wmag, s->wbMag, s->k, c, s->M);
    if (REF.h) {
        if (s->metric == JVO_COSINE) return (1.f + REF.pqcos(c, 0, (size_t)s->M, s->k, s->lut, s->mag, s->bMag)) / 2.f;
        return jvo_score_from_raw(s->metric, REF.adc(s->lut, s->k, c, 0, (size_t)s->M));
    }
    return jvo_pq_score_lut(s->metric, s->lut, s->mag, s->bMag, s->k, c, s->M);
}

float jvo_scorer_score(jvo_scorer *s, int32_t node)
{
    if (s->order) {
        switch (s->kind) {
        case 0: return jvo_score_from_raw(s->metric, warp_raw_f32(s->metric, s->q, s->base + (size_t)node * s->dim, s->dim, s->wqnorm));
        case 1: return warp_pq_score(s->metric, s->wlut, s->wmag, s->wbMag, s->k, s->codes + (size_t)node * s->M, s->M);
        case 2: break; /* integers: one order */
        default: return warp_nvq_score(s->metric, s->wq, s->mean, s->nsub, s->sizes, s->offsets, s->params + (size_t)node * 4 * s->nsub,
                                       s->bytes + (size_t)node * s->dim, s->wqbias, s->wqnorm);
        }
    }
    switch (s->kind) {
    case 0: {
        const float *row = s->base + (size_t)node * s->dim;
        if (REF.h) {
            float raw = s->metric == JVO_EUCLIDEAN ? REF.l2(s->q, 0, row, 0, (size_t)s->dim)
                      : s->metric == JVO_DOT_PRODUCT ? REF.dot(s->q, 0, row, 0, (size_t)s->dim)
                                                     : REF.cos(s->q, 0, row, 0, (size_t)s->dim);
            return jvo_score_from_raw(s->metric, raw);
        }
        return jvo_compare_f32(s->metric, s->q, row, s->dim);
    }
    case 1: {
        const uint8_t *c = s->codes + (size_t)node * s->M;
        if (REF.h) {
            if (s->metric == JVO_COSINE) return (1.f + REF.pqcos(c, 0, (size_t)s->M, s->k, s->lut, s->mag, s->bMag)) / 2.f;
            return jvo_score_from_raw(s->metric, REF.adc(s->lut, s->k, c, 0, (size_t)s->M));
        }
        return jvo_pq_score_lut(s->metric, s->lut, s->mag, s->bMag, s->k, c, s->M);
    }
    case 2: return jvo_bq_score(s->qbits, s->words + (size_t)node * s->W, s->W, s->dim);
    default: {
        const float *p = s->params + (size_t)node * 4 * s->nsub;
        const uint8_t *b = s->bytes + (size_t)node * s->dim;
        if (!REF.h) {
            /* s->q already holds the (shifted) query; undo nothing: jvo_nvq_score shifts itself, so inline here */
            float acc = 0.f, c0 = 0.f, c1 = 0.f, o[2];
            for (int i = 0; i < s->nsub; i++) {
                const float *pp = p + 4 * i;
                const float *qs = s->q + s->offsets[i];
                const uint8_t *bs = b + s->offsets[i];
                if (s->metric == JVO_DOT_PRODUCT) acc += jvo_nvq_dot_8bit(qs, bs, s->sizes[i], pp[2], pp[3], pp[0], pp[1]);
                else if (s->metric == JVO_EUCLIDEAN) acc += jvo_nvq_l2_8bit(qs, bs, s->sizes[i], pp[2], pp[3], pp[0], pp[1]);
                else {
                    jvo_nvq_cosine_8bit(qs, bs, s->sizes[i], pp[2], pp[3], pp[0], pp[1], s->mean + s->offsets[i], o);
                    c0 += o[0]; c1 += o[1];
                }
            }
            if (s->metric == JVO_DOT_PRODUCT) return (1.f + acc + s->qbias) / 2.f;
            if (s->metric == JVO_EUCLIDEAN) return 1.f / (1.f + acc);
            return (1.f + (c0 / s->qnorm) / (float)sqrt((double)c1)) / 2.f;
        } else {
            float acc = 0.f, c0 = 0.f, c1 = 0.f;
            for (int i = 0; i < s->nsub; i++) {
                const float *pp = p + 4 * i;
                const float *qs = s->q + s->offsets[i];
                const uint8_t *bs = b + s->offsets[i];
                if (s->metric == JVO_DOT_PRODUCT) acc += REF.nvq_dot(qs, bs, (size_t)s->sizes[i], pp[2], pp[3], pp[0], pp[1]);
                else if (s->metric == JVO_EUCLIDEAN) acc += REF.nvq_l2(qs, bs, (size_t)s->sizes[i], pp[2], pp[3], pp[0], pp[1]);
                else {
                    int64_t pk = REF.nvq_cos(qs, bs, (size_t)s->sizes[i], pp[2], pp[3], pp[0], pp[1], s->mean_sh + s->offsets[i]);
                    c0 += i2f((int32_t)(pk & 0xffffffff));
                    c1 += i2f((int32_t)(pk >> 32));
                }
            }
            if (s->metric == JVO_DOT_PRODUCT) return (1.f + acc + s->qbias) / 2.f;
            if (s->metric == JVO_EUCLIDEAN) return 1.f / (1.f + acc);
            return (1.f + (c0 / s->qnorm) / (float)sqrt((double)c1)) / 2.f;
        }
    }
    }
}

void jvo_scorer_free(jvo_scorer *s)
{
    if (!s) return;
    free(s->q); free(s->lut); free(s->mag); free(s->qbits); free(s->sizes); free(s->mean_sh);
    free(s->q_raw); free(s->wlut); free(s->wmag); free(s->wq);
    free(s);
}

/* ============================================================================================
 * heaps of int64 keys — base:util/AbstractLongHeap.java / BoundedLongHeap.java / GrowableLongHeap.java via
 * base:graph/NodeQueue.java (MAX_HEAP stores -1 - key in a min-heap; here: explicit max/min flag)
 * ========================================================================================== */
typedef struct { int64_t *a; int size, cap, bound, is_max; } kheap;

static void kh_init(kheap *h, int cap, int bound, int is_max)
{
    h->a = (int64_t *)malloc(sizeof(int64_t) * (size_t)(cap + 1));
    h->size = 0; h->cap = cap; h->bound = bound; h->is_max = is_max;
}
static inline int kh_before(const kheap *h, int64_t x, int64_t y) { return h->is_max ? x > y : x < y; }
static void kh_up(kheap *h, int i)
{
    int64_t v = h->a[i];
    while (i > 1 && kh_before(h, v, h->a[i >> 1])) { h->a[i] = h->a[i >> 1]; i >>= 1; }
    h->a[i] = v;
}
static void kh_down(kheap *h, int i)
{
    int64_t v = h->a[i];
    for (;;) {
        int c = i << 1;
        if (c > h->size) break;
        if (c + 1 <= h->size && kh_before(h, h->a[c + 1], h->a[c])) c++;
        if (!kh_before(h, h->a[c], v)) break;
        h->a[i] = h->a[c];
        i = c;
    }
    h->a[i] = v;
}
static int kh_push(kheap *h, int64_t v)
{
    if (h->bound > 0 && h->size >= h->bound) { /* BoundedLongHeap.java:59-69 (min-heap of the best) */
        if (v < h->a[1]) return 0;
        h->a[1] = v;
        kh_down(h, 1);
        return 1;
    }
    if (h->size == h->cap) {
        h->cap = h->cap * 2 + 16;
        h->a = (int64_t *)realloc(h->a, sizeof(int64_t) * (size_t)(h->cap + 1));
    }
    h->a[++h->size] = v;
    kh_up(h, h->size);
    return 1;
}
static int64_t kh_pop(kheap *h)
{
    int64_t top = h->a[1];
    h->a[1] = h->a[h->size--];
    if (h->size > 0) kh_down(h, 1);
    return top;
}

/* visited set: open addressing */
typedef struct { int32_t *t; uint32_t mask; int count; } iset;
static void is_init(iset *s, int cap_pow2) { s->t = (int32_t *)malloc(sizeof(int32_t) * (size_t)cap_pow2); memset(s->t, 0xff, sizeof(int32_t) * (size_t)cap_pow2); s->mask = (uint32_t)cap_pow2 - 1; s->count = 0; }
static void is_grow(iset *s);
static int is_add(iset *s, int32_t v)
{
    uint32_t h = ((uint32_t)v * 2654435761u) & s->mask;
    while (s->t[h] != -1) {
        if (s->t[h] == v) return 0;
        h = (h + 1) & s->mask;
    }
    s->t[h] = v;
    if (++s->count * 2 > (int)s->mask) is_grow(s);
    return 1;
}
static void is_grow(iset *s)
{
    int32_t *old = s->t;
    uint32_t oldcap = s->mask + 1;
    s->t = (int32_t *)malloc(sizeof(int32_t) * (size_t)oldcap * 2);
    memset(s->t, 0xff, sizeof(int32_t) * (size_t)oldcap * 2);
    s->mask = oldcap * 2 - 1;
    s->count = 0;
    for (uint32_t i = 0; i < oldcap; i++)
        if (old[i] != -1) {
            uint32_t h = ((uint32_t)old[i] * 2654435761u) & s->mask;
            while (s->t[h] != -1) h = (h + 1) & s->mask;
            s->t[h] = old[i];
            s->count++;
        }
    free(old);
}

static const int32_t *graph_neighbors(const jvo_graph *g, int level, int32_t node)
{
    if (level == 0) return g->adj0 + (size_t)node * g->degree;
    int32_t row = g->upper_row[(size_t)(level - 1) * g->n + node];
    if (row < 0) return NULL;
    return g->upper_adj + ((size_t)g->upper_off[level - 1] + row) * g->degree;
}

/* ============================================================================================
 * GraphSearcher — base:graph/GraphSearcher.java:263-282 (internalSearch), :334-353 (initializeInternal),
 * :355-370 (stopSearch), :406-457 (searchOneLayer), :471-507 (reranking), :520-530 (addTopCandidate),
 * :316-332 (setEntryPointsFromPreviousLayer); neighbour loop base:graph/OnHeapGraphIndex.java:475-483;
 * rerank base:graph/NodeQueue.java:168-230. threshold = 0, acceptOrds = ALL, rerankFloor = 0.
 * ========================================================================================== */
typedef struct {
    kheap candidates, results;
    int64_t *evicted; int nev, capev;
    iset visited;
    jvo_search_stats st;
} searcher;

static void ev_add(searcher *S, int64_t key)
{
    if (S->nev == S->capev) { S->capev = S->capev * 2 + 64; S->evicted = (int64_t *)realloc(S->evicted, sizeof(int64_t) * (size_t)S->capev); }
    S->evicted[S->nev++] = key;
}

static int accept_get(const uint32_t *bits, int32_t node) { return !bits || ((bits[node >> 5] >> (node & 31)) & 1u); }

/* searchOneLayer with acceptOrdsThisLayer + threshold (GraphSearcher.java:406-457). The TwoPhaseTracker that a threshold > 0
 * installs (ScoreTracker.java:70-125) is NOT restated: its sliding window survives reset() between queries, so its decisions
 * depend on the searcher's previous queries; threshold here is the admission rule of :427-431 only. */
static void search_one_layer(const jvo_graph *g, searcher *S, jvo_scorer *sf, int rerankK, int level, float threshold, const uint32_t *accept)
{
    S->results.bound = rerankK;
    while (S->candidates.size > 0) {
        int64_t top = S->candidates.a[1];
        float topScore = jvo_key_score(top);
        if (S->results.size >= rerankK && topScore < jvo_key_score(S->results.a[1])) break;
        kh_pop(&S->candidates);
        int32_t node = jvo_key_node(top);
        if (accept_get(accept, node) && topScore >= threshold) {
            /* addTopCandidate (GraphSearcher.java:520-530) */
            if (S->results.size < rerankK) kh_push(&S->results, top);
            else if (topScore > jvo_key_score(S->results.a[1])) { ev_add(S, S->results.a[1]); kh_push(&S->results, top); }
        }
        if (level == 0) S->st.expanded_base++;
        S->st.expanded++;
        const int32_t *nb = graph_neighbors(g, level, node);
        if (!nb) continue;
        for (int i = 0; i < g->degree; i++) {
            int32_t f = nb[i];
            if (f < 0) break;
            if (!is_add(&S->visited, f)) continue;
            /* OnDiskGraphIndex.processNeighbors (base:graph/disk/OnDiskGraphIndex.java:639-661): a scorer that supports
             * similarityToNeighbor scores level-0 neighbours from the expanded node's packed block */
            float sc = (level == 0 && sf->kind == 1 && sf->packed) ? jvo_scorer_score_neighbor(sf, node, i) : jvo_scorer_score(sf, f);
            kh_push(&S->candidates, jvo_topk_key(sc, f));
            S->st.visited++;
        }
    }
}

/* GraphSearcher.search(scoreProvider, topK, rerankK, threshold, rerankFloor, acceptOrds) (GraphSearcher.java:166-181,263-282);
 * accept_bits: bit (node & 31) of word (node >> 5), NULL = Bits.ALL. Upper layers use Bits.ALL and threshold 0 (:273-278). */
int jvo_graph_search_ex(const jvo_graph *g, jvo_scorer *approx, jvo_scorer *reranker, int topK, int rerankK, float threshold,
                        float rerankFloor, const uint32_t *accept_bits, int32_t *nodes_out, float *scores_out, jvo_search_stats *stats)
{
    searcher S;
    memset(&S, 0, sizeof(S));
    kh_init(&S.candidates, 256, 0, 1);
    kh_init(&S.results, rerankK > 0 ? rerankK : 1, rerankK, 0);
    is_init(&S.visited, 1024);
    /* initializeInternal */
    float es = jvo_scorer_score(approx, g->entry_node);
    is_add(&S.visited, g->entry_node);
    kh_push(&S.candidates, jvo_topk_key(es, g->entry_node));
    for (int lvl = g->entry_level; lvl > 0; lvl--) {
        search_one_layer(g, &S, approx, 1, lvl, 0.0f, NULL);
        /* setEntryPointsFromPreviousLayer */
        for (int i = 1; i <= S.results.size; i++) kh_push(&S.candidates, S.results.a[i]);
        for (int i = 0; i < S.nev; i++) kh_push(&S.candidates, S.evicted[i]);
        S.nev = 0;
        S.results.size = 0;
    }
    search_one_layer(g, &S, approx, rerankK, 0, threshold, accept_bits);
    int count;
    if (!reranker) {
        while (S.results.size > topK) kh_pop(&S.results);
        count = S.results.size;
        for (int i = count - 1; i >= 0; i--) {
            int64_t key = kh_pop(&S.results);
            nodes_out[i] = jvo_key_node(key);
            scores_out[i] = jvo_key_score(key);
        }
    } else {
        /* NodeQueue.rerank (NodeQueue.java:168-230): heap-array order; only approximate scores >= rerankFloor are rescored,
         * or the single best one when none is; strict > keeps the first of two equal exact scores */
        kheap rr;
        kh_init(&rr, topK, topK, 0);
        int n = S.results.size, above = 0, bestIndex = -1;
        float bestScore = -INFINITY;
        char *take = (char *)calloc((size_t)n + 1, 1);
        for (int i = 1; i <= n; i++) {
            float sc = jvo_key_score(S.results.a[i]);
            if (sc > bestScore) { bestScore = sc; bestIndex = i; }
            if (sc >= rerankFloor) { take[i] = 1; above++; }
        }
        if (above == 0 && bestIndex >= 1) take[bestIndex] = 1;
        for (int i = 1; i <= n; i++) {
            if (!take[i]) continue;
            int32_t node = jvo_key_node(S.results.a[i]);
            float ex = jvo_scorer_score(reranker, node);
            S.st.reranked++;
            if (rr.size < topK) kh_push(&rr, jvo_topk_key(ex, node));
            else if (ex > jvo_key_score(rr.a[1])) kh_push(&rr, jvo_topk_key(ex, node));
        }
        free(take);
        count = rr.size;
        for (int i = count - 1; i >= 0; i--) {
            int64_t key = kh_pop(&rr);
            nodes_out[i] = jvo_key_node(key);
            scores_out[i] = jvo_key_score(key);
        }
        free(rr.a);
    }
    if (stats) *stats = S.st;
    free(S.candidates.a); free(S.results.a); free(S.evicted); free(S.visited.t);
    return count;
}

int jvo_graph_search(const jvo_graph *g, jvo_scorer *approx, jvo_scorer *reranker, int topK, int rerankK,
                     int32_t *nodes_out, float *scores_out, jvo_search_stats *stats)
{
    return jvo_graph_search_ex(g, approx, reranker, topK, rerankK, 0.0f, 0.0f, NULL, nodes_out, scores_out, stats);
}

/* ---- host memory for the CPU baseline: pages interleaved over the NUMA nodes (what `numactl --interleave=all` does), so that
 *      128 threads gathering random rows do not all hit the one node a single-threaded first touch would have filled ---- */
#include <dirent.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

int jvo_numa_nodes(void)
{
    int n = 0;
    DIR *d = opendir("/sys/devices/system/node");
    if (!d) return 1;
    struct dirent *e;
    while ((e = readdir(d)) != NULL)
        if (strncmp(e->d_name, "node", 4) == 0 && e->d_name[4] >= '0' && e->d_name[4] <= '9') n++;
    closedir(d);
    return n > 0 ? n : 1;
}

void *jvo_alloc_interleaved(size_t bytes)
{
    void *p = mmap(NULL, bytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (p == MAP_FAILED) return NULL;
#ifdef SYS_mbind
    {
        unsigned long mask[16];
        int nodes = jvo_numa_nodes();
        memset(mask, 0, sizeof(mask));
        for (int i = 0; i < nodes && i < 1024; i++) mask[i / (8 * sizeof(unsigned long))] |= 1ul << (i % (8 * sizeof(unsigned long)));
        if (nodes > 1) syscall(SYS_mbind, p, bytes, 3 /* MPOL_INTERLEAVE */, mask, (unsigned long)(nodes + 1), 0u); /* best effort */
    }
#endif
    return p;
}

void jvo_free_interleaved(void *p, size_t bytes) { if (p) munmap(p, bytes); }

/* ---- multi-threaded batch driver (one searcher per thread, queries handed out in small chunks from a shared counter — the
 *      work-stealing ForkJoin pool the reference's parallel query stream runs on balances the same way:
 *      jvector-examples/.../benchmarks/ThroughputBenchmark.java:213, datasets/SiftSmall.java:367-377) ---- */
typedef struct {
    const jvo_graph *g; const jvo_dataset *ds; const float *queries; int nq, topK, rerankK;
    int32_t *nodes; float *scores; int64_t scored; int *next;
} batch_job;
#define JVO_BATCH_CHUNK 4

static void *batch_worker(void *arg)
{
    batch_job *j = (batch_job *)arg;
    const jvo_dataset *ds = j->ds;
    for (;;) {
      const int c0 = __atomic_fetch_add(j->next, JVO_BATCH_CHUNK, __ATOMIC_RELAXED);
      if (c0 >= j->nq) break;
      const int c1 = c0 + JVO_BATCH_CHUNK < j->nq ? c0 + JVO_BATCH_CHUNK : j->nq;
      for (int qi = c0; qi < c1; qi++) {
        const float *q = j->queries + (size_t)qi * ds->dim;
        jvo_scorer *ex = jvo_scorer_f32(ds->metric, ds->base, ds->n, ds->dim, q);
        jvo_scorer *ap = ds->kind == 1 ? jvo_scorer_pq(ds->metric, ds->codebooks, ds->M, ds->k, ds->dim, ds->centroid, ds->codes, ds->n, q) : NULL;
        if (ds->order) { jvo_scorer_set_order(ex, ds->order); if (ap) jvo_scorer_set_order(ap, ds->order); }
        jvo_search_stats st;
        int32_t *no = j->nodes + (size_t)qi * j->topK;
        float *so = j->scores + (size_t)qi * j->topK;
        int c = jvo_graph_search(j->g, ap ? ap : ex, ap ? ex : NULL, j->topK, j->rerankK, no, so, &st);
        for (int i = c; i < j->topK; i++) { no[i] = -1; so[i] = 0.f; }
        j->scored += st.visited + 1 + st.reranked;
        jvo_scorer_free(ex);
        jvo_scorer_free(ap);
      }
    }
    return NULL;
}

double jvo_graph_search_batch(const jvo_graph *g, const jvo_dataset *ds, const float *queries, int nq,
                              int topK, int rerankK, int threads, int32_t *nodes_out, float *scores_out,
                              int64_t *scored_total)
{
    if (threads < 1) threads = 1;
    if (threads > nq) threads = nq > 0 ? nq : 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)threads);
    batch_job *jobs = (batch_job *)calloc((size_t)threads, sizeof(batch_job));
    struct timespec t0, t1;
    int next = 0;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int t = 0; t < threads; t++) {
        jobs[t] = (batch_job){g, ds, queries, nq, topK, rerankK, nodes_out, scores_out, 0, &next};
        pthread_create(&th[t], NULL, batch_worker, &jobs[t]);
    }
    int64_t total = 0;
    for (int t = 0; t < threads; t++) { pthread_join(th[t], NULL); total += jobs[t].scored; }
    clock_gettime(CLOCK_MONOTONIC, &t1);
    if (scored_total) *scored_total = total;
    free(th); free(jobs);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}


/* ---- multi-threaded BQ brute force (CPU baseline of config 4): per query, scan every row with the scalar popcount loop of
 *      base:vector/DefaultVectorUtilSupport.java:342-348, keep the best k by the reference key in a bounded min-heap ---- */
typedef struct { const uint64_t *words; int64_t n; int W, dim; const uint64_t *q; int q0, q1, k; int64_t *keys; } bq_job;

static void *bq_worker(void *arg)
{
    bq_job *j = (bq_job *)arg;
    for (int qi = j->q0; qi < j->q1; qi++) {
        kheap h;
        kh_init(&h, j->k, j->k, 0);
        const uint64_t *qw = j->q + (size_t)qi * j->W;
        for (int64_t r = 0; r < j->n; r++) {
            float sc = jvo_bq_score(qw, j->words + (size_t)r * j->W, j->W, j->dim);
            int64_t key = jvo_topk_key(sc, (int32_t)r);
            if (h.size < j->k || key > h.a[1]) kh_push(&h, key);
        }
        int64_t *out = j->keys + (size_t)qi * j->k;
        int c = h.size;
        for (int i = c; i < j->k; i++) out[i] = INT64_MIN;
        for (int i = c - 1; i >= 0; i--) out[i] = kh_pop(&h);
        free(h.a);
    }
    return NULL;
}

double jvo_bq_bruteforce_batch(const uint64_t *words, int64_t n, int dim, const uint64_t *qwords, int nq, int k, int threads, int64_t *keys_out)
{
    int W = (dim + 63) / 64;
    if (threads < 1) threads = 1;
    if (threads > nq) threads = nq > 0 ? nq : 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)threads);
    bq_job *jobs = (bq_job *)calloc((size_t)threads, sizeof(bq_job));
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int t = 0; t < threads; t++) {
        jobs[t] = (bq_job){words, n, W, dim, qwords, (int)((int64_t)nq * t / threads), (int)((int64_t)nq * (t + 1) / threads), k, keys_out};
        pthread_create(&th[t], NULL, bq_worker, &jobs[t]);
    }
    for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    free(th); free(jobs);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}


/* ---- multi-threaded NVQ encode (CPU baseline of config 5's encode step): NVQuantization.encodeAll parallel stream
 *      (base:quantization/NVQuantization.java:185-193) -> quantizeTo (:524-578), through the reference kernels when loaded ---- */
typedef struct { const float *rows; int64_t r0, r1; int dim, nsub, learn; const float *mean; float *params; uint8_t *bytes; } nvq_job;

static void nvq_encode_sub_ref(const float *v, int n, int learn, float *params_out, uint8_t *bytes_out)
{
    float minv = 3.402823466e+38f, maxv = -3.402823466e+38f;
    for (int i = 0; i < n; i++) { if (v[i] < minv) minv = v[i]; if (v[i] > maxv) maxv = v[i]; }
    float growth = 1e-2f;
    if (learn) {
        float baseline = REF.nvq_uloss(v, (size_t)n, minv, maxv, 8);
        float coarse = 1e-2f, best = 1.40129846e-45f;
        for (float gr = 1e-6f; gr < 20.f; gr += 1.f) {
            float lv = baseline / REF.nvq_lossf(v, (size_t)n, gr, 0.f, minv, maxv, 8);
            if (lv > best) { best = lv; coarse = gr; }
        }
        float fine = coarse;
        for (float gr = coarse - 1; gr < coarse + 1; gr += 0.1f) {
            float lv = baseline / REF.nvq_lossf(v, (size_t)n, gr, 0.f, minv, maxv, 8);
            if (lv > best) { best = lv; fine = gr; }
        }
        growth = fine;
    }
    REF.nvq_quant(v, (size_t)n, growth, 0.f, minv, maxv, bytes_out);
    params_out[0] = minv; params_out[1] = maxv; params_out[2] = growth; params_out[3] = 0.f;
}

static void *nvq_worker(void *arg)
{
    nvq_job *j = (nvq_job *)arg;
    int *sizes = (int *)malloc(sizeof(int) * j->nsub * 2), *offsets = sizes + j->nsub;
    float *c = (float *)malloc(sizeof(float) * j->dim);
    jvo_pq_layout(j->dim, j->nsub, sizes, offsets);
    for (int64_t r = j->r0; r < j->r1; r++) {
        const float *v = j->rows + (size_t)r * j->dim;
        if (REF.h) {
            for (int i = 0; i < j->dim; i++) c[i] = v[i] - j->mean[i];
            for (int s = 0; s < j->nsub; s++)
                nvq_encode_sub_ref(c + offsets[s], sizes[s], j->learn, j->params + ((size_t)r * j->nsub + s) * 4, j->bytes + (size_t)r * j->dim + offsets[s]);
        } else {
            jvo_nvq_encode(v, j->mean, j->dim, j->nsub, j->learn, j->params + (size_t)r * j->nsub * 4, j->bytes + (size_t)r * j->dim);
        }
    }
    free(c); free(sizes);
    return NULL;
}

double jvo_nvq_encode_batch(const float *rows, int64_t n, int dim, int nsub, const float *mean, int learn, int threads, float *params_out, uint8_t *bytes_out)
{
    if (threads < 1) threads = 1;
    if (threads > n) threads = n > 0 ? (int)n : 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)threads);
    nvq_job *jobs = (nvq_job *)calloc((size_t)threads, sizeof(nvq_job));
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int t = 0; t < threads; t++) {
        jobs[t] = (nvq_job){rows, n * t / threads, n * (t + 1) / threads, dim, nsub, learn, mean, params_out, bytes_out};
        pthread_create(&th[t], NULL, nvq_worker, &jobs[t]);
    }
    for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    free(th); free(jobs);
    return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}

/* ============================================================================================
 * Vamana diversity — base:graph/diversity/VamanaDiversityProvider.java:45-95 (diverseBefore = 0)
 * ========================================================================================== */
int jvo_retain_diverse(const float *cand_scores, const int32_t *cand_nodes, int nc, const float *pair_scores,
                       int maxDegree, float alpha, uint8_t *selected)
{
    memset(selected, 0, (size_t)nc);
    int nSelected = 0;
    float currentAlpha = 1.0f;
    while (currentAlpha <= alpha + 1E-6 && nSelected < maxDegree) {
        for (int i = 0; i < nc && nSelected < maxDegree; i++) {
            if (selected[i]) continue;
            int diverse = 1;
            for (int j = 0; j < nc; j++) {
                if (!selected[j]) continue;
                if (cand_nodes[j] == cand_nodes[i]) break;
                if (pair_scores[(size_t)i * nc + j] > cand_scores[i] * currentAlpha) { diverse = 0; break; }
            }
            if (diverse) { selected[i] = 1; nSelected++; }
        }
        currentAlpha += 0.2f;
    }
    return nSelected;
}

/* ============================================================================================
 * Single-threaded Vamana build, no hierarchy — base:graph/GraphIndexBuilder.java:605-671,801-813;
 * base:graph/OnHeapGraphIndex.java:279-282; base:graph/ConcurrentNeighborMap.java:104-110,158-165,
 * 247-262,286-321 (insertDiverse / backlink / insert with overflow); cleanup enforceDegree :214-222.
 * Neighbor lists are kept sorted by score descending (NodeArray).
 * ========================================================================================== */
typedef struct { int32_t *nodes; float *scores; int size; int diverseBefore; } nlist;

static float pair_score(int metric, const float *base, int dim, int a, int b)
{
    const float *x = base + (size_t)a * dim, *y = base + (size_t)b * dim;
    if (REF.h) { /* after jvo_use_ref: the reference's compiled kernels (build-quality comparisons at 100k+ nodes) */
        float raw = metric == JVO_EUCLIDEAN ? REF.l2(x, 0, y, 0, (size_t)dim) : metric == JVO_DOT_PRODUCT ? REF.dot(x, 0, y, 0, (size_t)dim) : REF.cos(x, 0, y, 0, (size_t)dim);
        return jvo_score_from_raw(metric, raw);
    }
    return jvo_compare_f32(metric, x, y, dim);
}

/* retainDiverse over a sorted candidate list, evaluating diversity scores lazily */
static int retain_diverse_lazy(int metric, const float *base, int dim, int32_t *nodes, float *scores, int n,
                               int maxDegree, int diverseBefore, float alpha)
{
    uint8_t *sel = (uint8_t *)calloc((size_t)(n > 0 ? n : 1), 1);
    int lim = diverseBefore < maxDegree ? diverseBefore : maxDegree;
    for (int i = 0; i < lim; i++) sel[i] = 1;
    int nSelected = diverseBefore;
    float currentAlpha = 1.0f;
    while (currentAlpha <= alpha + 1E-6 && nSelected < maxDegree) {
        for (int i = diverseBefore; i < n && nSelected < maxDegree; i++) {
            if (sel[i]) continue;
            int diverse = 1;
            for (int j = 0; j < n; j++) {
                if (!sel[j]) continue;
                if (nodes[j] == nodes[i]) break;
                if (pair_score(metric, base, dim, nodes[i], nodes[j]) > scores[i] * currentAlpha) { diverse = 0; break; }
            }
            if (diverse) { sel[i] = 1; nSelected++; }
        }
        currentAlpha += 0.2f;
    }
    int w = 0;
    for (int i = 0; i < n; i++)
        if (sel[i]) { nodes[w] = nodes[i]; scores[w] = scores[i]; w++; }
    free(sel);
    return w;
}

int32_t jvo_graph_build_f32(int metric, const float *base, int32_t n, int dim, int degree, int beam,
                            float overflow, float alpha, int32_t *adj_out)
{
    int maxOverflow = (int)(degree * overflow);
    int cap = maxOverflow + 1;
    nlist *L = (nlist *)calloc((size_t)n, sizeof(nlist));
    for (int i = 0; i < n; i++) {
        L[i].nodes = (int32_t *)malloc(sizeof(int32_t) * (size_t)cap);
        L[i].scores = (float *)malloc(sizeof(float) * (size_t)cap);
    }
    int32_t *adj_tmp = (int32_t *)malloc(sizeof(int32_t) * (size_t)n * (size_t)cap);
    memset(adj_tmp, 0xff, sizeof(int32_t) * (size_t)n * (size_t)cap);
#define SYNC_ROW(u) do { int32_t *row_ = adj_tmp + (size_t)(u) * cap; \
        for (int i_ = 0; i_ < cap; i_++) row_[i_] = i_ < L[u].size ? L[u].nodes[i_] : -1; } while (0)
    int32_t *res_nodes = (int32_t *)malloc(sizeof(int32_t) * (size_t)(beam + cap + 4));
    float *res_scores = (float *)malloc(sizeof(float) * (size_t)(beam + cap + 4));
    int32_t entry = -1;
    for (int32_t node = 0; node < n; node++) {
        if (entry < 0) { entry = node; continue; }
        /* snapshot view: adjacency padded to cap */
        jvo_graph g;
        memset(&g, 0, sizeof(g));
        g.n = n; g.levels = 1; g.degree = cap; g.entry_node = entry; g.entry_level = 0;
        g.adj0 = adj_tmp; /* rows are kept in sync incrementally (SYNC_ROW) */
        jvo_scorer *sf = jvo_scorer_f32(metric, base, n, dim, base + (size_t)node * dim);
        int cnt = jvo_graph_search(&g, sf, NULL, beam, beam, res_nodes, res_scores, NULL);
        jvo_scorer_free(sf);
        /* insertDiverse(node, candidates) on an empty list */
        int kept = retain_diverse_lazy(metric, base, dim, res_nodes, res_scores, cnt, degree, 0, alpha);
        L[node].size = kept;
        L[node].diverseBefore = kept;
        memcpy(L[node].nodes, res_nodes, sizeof(int32_t) * (size_t)kept);
        memcpy(L[node].scores, res_scores, sizeof(float) * (size_t)kept);
        SYNC_ROW(node);
        /* backlink: insert(node) into every selected neighbour, allowing overflow */
        int hardMax = (int)(overflow * degree);
        for (int i = 0; i < kept; i++) {
            nlist *nb = &L[res_nodes[i]];
            float sc = res_scores[i];
            /* descSortFindRightMostInsertionPoint + duplicate check */
            int ip = 0;
            while (ip < nb->size && !(nb->scores[ip] < sc)) ip++;
            int dup = 0;
            for (int t = ip - 1; t >= 0 && nb->scores[t] == sc; t--) if (nb->nodes[t] == node) dup = 1;
            if (dup) continue;
            memmove(nb->nodes + ip + 1, nb->nodes + ip, sizeof(int32_t) * (size_t)(nb->size - ip));
            memmove(nb->scores + ip + 1, nb->scores + ip, sizeof(float) * (size_t)(nb->size - ip));
            nb->nodes[ip] = node;
            nb->scores[ip] = sc;
            nb->size++;
            if (ip < nb->diverseBefore) nb->diverseBefore = ip;
            if (nb->size > hardMax) {
                nb->size = retain_diverse_lazy(metric, base, dim, nb->nodes, nb->scores, nb->size, degree, nb->diverseBefore, alpha);
                nb->diverseBefore = nb->size;
            }
            SYNC_ROW(res_nodes[i]);
        }
    }
    /* cleanup(): enforceDegree */
    for (int32_t u = 0; u < n; u++) {
        if (L[u].size > degree) {
            L[u].size = retain_diverse_lazy(metric, base, dim, L[u].nodes, L[u].scores, L[u].size, degree, L[u].diverseBefore, alpha);
        }
        for (int i = 0; i < degree; i++) adj_out[(size_t)u * degree + i] = i < L[u].size ? L[u].nodes[i] : -1;
        free(L[u].nodes);
        free(L[u].scores);
    }
    free(L); free(adj_tmp); free(res_nodes); free(res_scores);
    return entry < 0 ? 0 : entry;
}
