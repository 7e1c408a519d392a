// legacy_host.cpp — the 24 symbols of the reference's libjvector.so ABI
// (/root/reference/jvector-native/src/main/native/src/jvector_simd_kernel_list.h:35-61, src/jvector_simd.h:47,53).
//
// The reference binds these with Linker.Option.critical(true) on ON-HEAP segments
// (jvector-native/.../cnative/NativeSimdOps.java:1164,1226,...): the callee gets raw pointers into the Java heap, must
// not block and must return quickly. A CUDA launch cannot live behind that contract, so these entry points stay
// synchronous host functions BY DESIGN (they are the n = 1 case of the SPI, not a fallback for the batched GPU path,
// which has none). They exist so this library can be installed as `libjvector.so` under jvector-native unchanged.
// Arithmetic follows the native reference kernels (native-c:src/jvector_simd_kernels.cpp); NVQ bytes are read in
// natural order, so nvq_shuffle_query_in_place_8bit is the identity (as DefaultVectorUtilSupport.java:454).
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/jvector_b200.h"
#include "legacy_avx512.h"

namespace {

inline int32_t f2i(float f) { int32_t i; memcpy(&i, &f, 4); return i; }
inline float i2f(int32_t i) { float f; memcpy(&f, &i, 4); return f; }

// native-c:...:1047-1077
inline float logistic_nqt(float v, float alpha, float x0)
{
    const float t = fmaf(v, alpha, -alpha * x0);
    const int32_t p = f2i(t) < 0 ? (int32_t)t : (int32_t)(t + 1.0f);
    const int32_t m = f2i(fmaf(t - (float)p, 0.5f, 1.0f));
    const float r = i2f((int32_t)((uint32_t)m + ((uint32_t)p << 23)));
    return r / (r + 1.0f);
}

// native-c:...:1084-1111
inline float logit_nqt(float v, float inv_alpha, float x0)
{
    const float z = v / (1.0f - v);
    const int32_t t = f2i(z);
    const int32_t p = ((t & 0x7f800000) >> 23) - 128;
    const float m = i2f((t & 0x007fffff) + 0x3f800000);
    return fmaf(m + (float)p, inv_alpha, x0);
}

struct Nvq {
    float sa, isa, sx0, bias, scale;
    Nvq(float alpha, float x0, float minv, float maxv, float levels)
    {
        const float delta = maxv - minv;
        sa = alpha / delta;
        isa = delta / alpha;
        sx0 = x0 * delta;
        bias = logistic_nqt(minv, sa, sx0);
        scale = (logistic_nqt(maxv, sa, sx0) - bias) / levels;
    }
    inline float dq(float b) const { return logit_nqt(fmaf(b, scale, bias), isa, sx0); }
    inline jvl::NvqScalars scalars() const { return jvl::NvqScalars{sa, isa, sx0, bias, scale}; }
};

}  // namespace

extern "C" {

// dot_product_f32 / euclidean_f32 / cosine_f32 live in legacy_simd.cpp (vectorised, multi-versioned)

void add_in_place_f32(float *v1, const float *v2, size_t length) { for (size_t i = 0; i < length; i++) v1[i] += v2[i]; }
void add_scalar_in_place_f32(float *v1, float value, size_t length) { for (size_t i = 0; i < length; i++) v1[i] += value; }
void sub_in_place_f32(float *v1, const float *v2, size_t length) { for (size_t i = 0; i < length; i++) v1[i] -= v2[i]; }
void sub_scalar_in_place_f32(float *v1, float value, size_t length) { for (size_t i = 0; i < length; i++) v1[i] -= value; }

float max_f32(const float *v, size_t length)
{
    float m = -3.402823466e+38f;
    for (size_t i = 0; i < length; i++) m = v[i] > m ? v[i] : m;
    return m;
}

void min_in_place_f32(float *v1, const float *v2, size_t length)
{
    for (size_t i = 0; i < length; i++) v1[i] = v2[i] < v1[i] ? v2[i] : v1[i];
}

float assemble_and_sum_f32(const float *data, int dataBase, const unsigned char *baseOffsets, int baseOffsetsOffset, size_t baseOffsetsLength)
{
    const unsigned char *c = baseOffsets + baseOffsetsOffset;
    if (jvl::cpu_has_avx512()) return jvl::assemble_and_sum_avx512(data, dataBase, c, baseOffsetsLength);
    float s = 0.f;
    for (size_t i = 0; i < baseOffsetsLength; i++) s += data[(size_t)dataBase * i + c[i]];
    return s;
}

float assemble_and_sum_pq_f32(const float *data, size_t subspaceCount, const unsigned char *baseOffsets1, int baseOffsetsOffset1,
                              const unsigned char *baseOffsets2, int baseOffsetsOffset2, int clusterCount)
{
    const int k = clusterCount;
    const size_t block = (size_t)k * (k + 1) / 2;
    const unsigned char *c1 = baseOffsets1 + baseOffsetsOffset1, *c2 = baseOffsets2 + baseOffsetsOffset2;
    if (jvl::cpu_has_avx512()) return jvl::assemble_and_sum_pq_avx512(data, subspaceCount, c1, c2, clusterCount);
    float res = 0.f;
    for (size_t i = 0; i < subspaceCount; i++) {
        const int a = c1[i], b = c2[i];
        const int r = a < b ? a : b, c = a < b ? b : a;
        res += data[i * block + (size_t)(r * k - (r * (r - 1) / 2)) + (size_t)(c - r)];
    }
    return res;
}

float pq_decoded_cosine_similarity_f32(const unsigned char *baseOffsets, int baseOffsetsOffset, size_t baseOffsetsLength, int clusterCount,
                                       const float *partialSums, const float *aMagnitude, float bMagnitude)
{
    const unsigned char *c = baseOffsets + baseOffsetsOffset;
    if (jvl::cpu_has_avx512()) return jvl::pq_decoded_cosine_avx512(c, baseOffsetsLength, clusterCount, partialSums, aMagnitude, bMagnitude);
    float s = 0.f, a = 0.f;
    for (size_t i = 0; i < baseOffsetsLength; i++) {
        const size_t idx = (size_t)clusterCount * i + c[i];
        s += partialSums[idx];
        a += aMagnitude[idx];
    }
    return s / sqrtf(a * bMagnitude);
}

void calculate_partial_sums_dot_f32(const float *codebook, int codebookIndex, size_t size, int clusterCount, const float *query, int queryOffset, float *partialSums)
{
    const float *q = query + queryOffset;
    float *out = partialSums + (size_t)codebookIndex * clusterCount;
    if (jvl::cpu_has_avx512()) { jvl::partial_sums_avx512(codebook, size, clusterCount, q, out, 0); return; }
    for (int c = 0; c < clusterCount; c++) {
        const float *cen = codebook + (size_t)c * size;
        float s = 0.f;
        for (size_t j = 0; j < size; j++) s = fmaf(cen[j], q[j], s);
        out[c] = s;
    }
}

void calculate_partial_sums_euclidean_f32(const float *codebook, int codebookIndex, size_t size, int clusterCount, const float *query, int queryOffset, float *partialSums)
{
    const float *q = query + queryOffset;
    float *out = partialSums + (size_t)codebookIndex * clusterCount;
    if (jvl::cpu_has_avx512()) { jvl::partial_sums_avx512(codebook, size, clusterCount, q, out, 1); return; }
    for (int c = 0; c < clusterCount; c++) {
        const float *cen = codebook + (size_t)c * size;
        float s = 0.f;
        for (size_t j = 0; j < size; j++) { const float d = cen[j] - q[j]; s = fmaf(d, d, s); }
        out[c] = s;
    }
}

void calculate_partial_sums_self_magnitude_f32(const float *codebook, int codebookIndex, size_t size, int clusterCount, float *partialSums)
{
    float *out = partialSums + (size_t)codebookIndex * clusterCount;
    if (jvl::cpu_has_avx512()) { jvl::partial_sums_avx512(codebook, size, clusterCount, nullptr, out, 2); return; }
    for (int c = 0; c < clusterCount; c++) {
        const float *cen = codebook + (size_t)c * size;
        float s = 0.f;
        for (size_t j = 0; j < size; j++) s = fmaf(cen[j], cen[j], s);
        out[c] = s;
    }
}

void nvq_quantize_8bit(const float *vector, size_t length, float alpha, float x0, float minValue, float maxValue, unsigned char *destination)
{
    const float delta = maxValue - minValue, sa = alpha / delta, sx0 = x0 * delta;
    const float bias = logistic_nqt(minValue, sa, sx0);
    const float inv = 255.0f / (logistic_nqt(maxValue, sa, sx0) - bias);
    if (jvl::cpu_has_avx512()) { jvl::nvq_quantize_avx512(vector, length, sa, -sa * sx0, bias, inv, destination); return; }
    for (size_t i = 0; i < length; i++) {
        const float a = fmaf(logistic_nqt(vector[i], sa, sx0) - bias, inv, 0.5f);
        const int q = (int)a;
        destination[i] = (unsigned char)(q < 0 ? 0 : q > 255 ? 255 : q);
    }
}

float nvq_loss(const float *vector, size_t length, float alpha, float x0, float minValue, float maxValue, int nBits)
{
    const Nvq c(alpha, x0, minValue, maxValue, (float)((1 << nBits) - 1));
    if (jvl::cpu_has_avx512()) return jvl::nvq_loss_avx512(vector, length, c.scalars(), -c.sa * c.sx0);
    const float inv = 1.0f / c.scale;
    float s = 0.f;
    for (size_t i = 0; i < length; i++) {
        const float r = (logistic_nqt(vector[i], c.sa, c.sx0) - c.bias) * inv;
        const float d = vector[i] - c.dq((float)(int)(r + 0.5f));
        s = fmaf(d, d, s);
    }
    return s;
}

float nvq_uniform_loss(const float *vector, size_t length, float minValue, float maxValue, int nBits)
{
    const float constant = (float)((1 << nBits) - 1), delta = maxValue - minValue;
    if (jvl::cpu_has_avx512()) return jvl::nvq_uniform_loss_avx512(vector, length, minValue, maxValue, constant);
    float s = 0.f;
    for (size_t i = 0; i < length; i++) {
        const float r = (vector[i] - minValue) * (constant / delta);
        const float rec = fmaf((float)(int)(r + 0.5f), delta / constant, minValue);
        const float d = vector[i] - rec;
        s = fmaf(d, d, s);
    }
    return s;
}

float nvq_square_l2_distance_8bit(const float *vector, const unsigned char *quantized, size_t length, float alpha, float x0, float minValue, float maxValue)
{
    const Nvq c(alpha, x0, minValue, maxValue, 255.0f);
    if (jvl::cpu_has_avx512()) return jvl::nvq_l2_avx512(vector, quantized, length, c.scalars());
    float s = 0.f;
    for (size_t i = 0; i < length; i++) { const float d = vector[i] - c.dq((float)quantized[i]); s = fmaf(d, d, s); }
    return s;
}

float nvq_dot_product_8bit(const float *vector, const unsigned char *quantized, size_t length, float alpha, float x0, float minValue, float maxValue)
{
    const Nvq c(alpha, x0, minValue, maxValue, 255.0f);
    if (jvl::cpu_has_avx512()) return jvl::nvq_dot_avx512(vector, quantized, length, c.scalars());
    float s = 0.f;
    for (size_t i = 0; i < length; i++) s = fmaf(vector[i], c.dq((float)quantized[i]), s);
    return s;
}

int64_t nvq_cosine_8bit_packed(const float *vector, const unsigned char *quantized, size_t length, float alpha, float x0, float minValue, float maxValue,
                               const float *centroid)
{
    const Nvq c(alpha, x0, minValue, maxValue, 255.0f);
    float s = 0.f, bm = 0.f;
    if (jvl::cpu_has_avx512()) {
        jvl::nvq_cosine_avx512(vector, quantized, length, c.scalars(), centroid, &s, &bm);
        return ((int64_t)f2i(bm) << 32) | (int64_t)(uint32_t)f2i(s);
    }
    for (size_t i = 0; i < length; i++) {
        const float e = c.dq((float)quantized[i]) + centroid[i];
        s = fmaf(vector[i], e, s);
        bm = fmaf(e, e, bm);
    }
    return ((int64_t)f2i(bm) << 32) | (int64_t)(uint32_t)f2i(s);
}

void nvq_shuffle_query_in_place_8bit(float *vector, size_t length)
{
    (void)vector;
    (void)length;
}

const char *jvector_simd_get_active_isa(void) { return "sm_90a"; }

const char *jvector_simd_get_max_isa_env(void)
{
    static const char *cached = getenv("JVECTOR_MAX_ISA");
    return cached;
}

}  // extern "C"
