/*
 * oracle.c — CPU restatement of Qdrant's vector-scoring hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load it.
 * The product path (qdrant_b200/) never links, imports or calls this file.
 *
 * Every function restates one reference routine with the SAME x86 intrinsics and the SAME
 * reduction order, so that results are bit-identical to what the reference's runtime dispatch
 * selects on an AVX2+FMA host.  Citations are file:line under /root/reference.
 *
 * Build: gcc -O3 -march=haswell -mpopcnt -ffp-contract=off -fPIC -shared (see oracle/Makefile).
 * -ffp-contract=off matters: rustc never contracts `a*b + c`; the explicit _mm256_fmadd_ps
 * calls below ARE fused, exactly like the reference's.
 *
 * Parity pinning: the reference's known-answer tests for this path (SIMD == scalar on fixed
 * vectors; lib/segment/src/spaces/simple_avx.rs:218-256, metric_uint/avx2/dot.rs:77-106, ...)
 * are re-typed in tests/test_oracle_kat.py, and the SQ8 / BQ-scalar inner loops are checked
 * against the reference's own C kernels compiled verbatim into oracle/_ref/libsimd_utils.so.
 */
#include <immintrin.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>

#define API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------
 * f32 metrics — lib/segment/src/spaces/simple_avx.rs, simple_sse.rs, simple.rs
 * ---------------------------------------------------------------------------------------- */

/* simple_avx.rs:10-16 */
static inline float hsum256_ps_avx(__m256 x) {
    __m128 lr_sum = _mm_add_ps(_mm256_extractf128_ps(x, 1), _mm256_castps256_ps128(x));
    __m128 hsum = _mm_hadd_ps(lr_sum, lr_sum);
    float p1 = _mm_cvtss_f32(hsum);
    float p2 = _mm_cvtss_f32(_mm_shuffle_ps(hsum, hsum, 0x55));
    return p1 + p2;
}

/* simple_avx.rs:21-28 */
static inline float four_way_hsum(__m256 a, __m256 b, __m256 c, __m256 d) {
    __m256 sum1 = _mm256_add_ps(a, b);
    __m256 sum2 = _mm256_add_ps(c, d);
    __m256 total = _mm256_add_ps(sum1, sum2);
    return hsum256_ps_avx(total);
}

/* simple_sse.rs:13-17 */
static inline float hsum128_ps_sse(__m128 x) {
    __m128 x64 = _mm_add_ps(x, _mm_movehl_ps(x, x));
    __m128 x32 = _mm_add_ss(x64, _mm_shuffle_ps(x64, x64, 0x55));
    return _mm_cvtss_f32(x32);
}

/* simple_avx.rs:169-213 */
API float qo_dot_avx(const float* v1, const float* v2, size_t n) {
    size_t m = n - (n % 32);
    __m256 s1 = _mm256_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    const float *p1 = v1, *p2 = v2;
    for (size_t i = 0; i < m; i += 32) {
        s1 = _mm256_fmadd_ps(_mm256_loadu_ps(p1), _mm256_loadu_ps(p2), s1);
        s2 = _mm256_fmadd_ps(_mm256_loadu_ps(p1 + 8), _mm256_loadu_ps(p2 + 8), s2);
        s3 = _mm256_fmadd_ps(_mm256_loadu_ps(p1 + 16), _mm256_loadu_ps(p2 + 16), s3);
        s4 = _mm256_fmadd_ps(_mm256_loadu_ps(p1 + 24), _mm256_loadu_ps(p2 + 24), s4);
        p1 += 32; p2 += 32;
    }
    float result = four_way_hsum(s1, s2, s3, s4);
    for (size_t i = 0; i < n - m; i++) result += p1[i] * p2[i];
    return result;
}

/* simple_avx.rs:32-75 */
API float qo_euclid_avx(const float* v1, const float* v2, size_t n) {
    size_t m = n - (n % 32);
    __m256 s1 = _mm256_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    const float *p1 = v1, *p2 = v2;
    for (size_t i = 0; i < m; i += 32) {
        __m256 d1 = _mm256_sub_ps(_mm256_loadu_ps(p1), _mm256_loadu_ps(p2));
        s1 = _mm256_fmadd_ps(d1, d1, s1);
        __m256 d2 = _mm256_sub_ps(_mm256_loadu_ps(p1 + 8), _mm256_loadu_ps(p2 + 8));
        s2 = _mm256_fmadd_ps(d2, d2, s2);
        __m256 d3 = _mm256_sub_ps(_mm256_loadu_ps(p1 + 16), _mm256_loadu_ps(p2 + 16));
        s3 = _mm256_fmadd_ps(d3, d3, s3);
        __m256 d4 = _mm256_sub_ps(_mm256_loadu_ps(p1 + 24), _mm256_loadu_ps(p2 + 24));
        s4 = _mm256_fmadd_ps(d4, d4, s4);
        p1 += 32; p2 += 32;
    }
    float result = four_way_hsum(s1, s2, s3, s4);
    for (size_t i = 0; i < n - m; i++) { float d = p1[i] - p2[i]; result += d * d; }
    return -result;
}

/* simple_avx.rs:79-123 */
API float qo_manhattan_avx(const float* v1, const float* v2, size_t n) {
    const __m256 mask = _mm256_set1_ps(-0.0f);
    size_t m = n - (n % 32);
    __m256 s1 = _mm256_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    const float *p1 = v1, *p2 = v2;
    for (size_t i = 0; i < m; i += 32) {
        __m256 d1 = _mm256_sub_ps(_mm256_loadu_ps(p1), _mm256_loadu_ps(p2));
        s1 = _mm256_add_ps(_mm256_andnot_ps(mask, d1), s1);
        __m256 d2 = _mm256_sub_ps(_mm256_loadu_ps(p1 + 8), _mm256_loadu_ps(p2 + 8));
        s2 = _mm256_add_ps(_mm256_andnot_ps(mask, d2), s2);
        __m256 d3 = _mm256_sub_ps(_mm256_loadu_ps(p1 + 16), _mm256_loadu_ps(p2 + 16));
        s3 = _mm256_add_ps(_mm256_andnot_ps(mask, d3), s3);
        __m256 d4 = _mm256_sub_ps(_mm256_loadu_ps(p1 + 24), _mm256_loadu_ps(p2 + 24));
        s4 = _mm256_add_ps(_mm256_andnot_ps(mask, d4), s4);
        p1 += 32; p2 += 32;
    }
    float result = four_way_hsum(s1, s2, s3, s4);
    for (size_t i = 0; i < n - m; i++) result += fabsf(p1[i] - p2[i]);
    return -result;
}

/* tools.rs:14-16 */
static inline int is_length_zero_or_normalized(float length) {
    return length < FLT_EPSILON || fabsf(length - 1.0f) <= 1.0e-6f;
}

/* simple_avx.rs:127-165 ; writes the (possibly unchanged) vector to out */
API void qo_cosine_preprocess_avx(const float* v, float* out, size_t n) {
    size_t m = n - (n % 32);
    __m256 s1 = _mm256_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    const float* p = v;
    for (size_t i = 0; i < m; i += 32) {
        __m256 a = _mm256_loadu_ps(p);      s1 = _mm256_fmadd_ps(a, a, s1);
        __m256 b = _mm256_loadu_ps(p + 8);  s2 = _mm256_fmadd_ps(b, b, s2);
        __m256 c = _mm256_loadu_ps(p + 16); s3 = _mm256_fmadd_ps(c, c, s3);
        __m256 d = _mm256_loadu_ps(p + 24); s4 = _mm256_fmadd_ps(d, d, s4);
        p += 32;
    }
    float length = four_way_hsum(s1, s2, s3, s4);
    for (size_t i = 0; i < n - m; i++) length += p[i] * p[i];
    if (is_length_zero_or_normalized(length)) { memmove(out, v, n * sizeof(float)); return; }
    length = sqrtf(length);
    for (size_t i = 0; i < n; i++) out[i] = v[i] / length;
}

/* simple_sse.rs:154-204 */
API float qo_dot_sse(const float* v1, const float* v2, size_t n) {
    size_t m = n - (n % 16);
    __m128 s1 = _mm_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    const float *p1 = v1, *p2 = v2;
    for (size_t i = 0; i < m; i += 16) {
        s1 = _mm_add_ps(_mm_mul_ps(_mm_loadu_ps(p1), _mm_loadu_ps(p2)), s1);
        s2 = _mm_add_ps(_mm_mul_ps(_mm_loadu_ps(p1 + 4), _mm_loadu_ps(p2 + 4)), s2);
        s3 = _mm_add_ps(_mm_mul_ps(_mm_loadu_ps(p1 + 8), _mm_loadu_ps(p2 + 8)), s3);
        s4 = _mm_add_ps(_mm_mul_ps(_mm_loadu_ps(p1 + 12), _mm_loadu_ps(p2 + 12)), s4);
        p1 += 16; p2 += 16;
    }
    float result = hsum128_ps_sse(s1) + hsum128_ps_sse(s2) + hsum128_ps_sse(s3) + hsum128_ps_sse(s4);
    for (size_t i = 0; i < n - m; i++) result += p1[i] * p2[i];
    return result;
}

/* simple_sse.rs:20-60 */
API float qo_euclid_sse(const float* v1, const float* v2, size_t n) {
    size_t m = n - (n % 16);
    __m128 s1 = _mm_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    const float *p1 = v1, *p2 = v2;
    for (size_t i = 0; i < m; i += 16) {
        __m128 d1 = _mm_sub_ps(_mm_loadu_ps(p1), _mm_loadu_ps(p2));
        s1 = _mm_add_ps(_mm_mul_ps(d1, d1), s1);
        __m128 d2 = _mm_sub_ps(_mm_loadu_ps(p1 + 4), _mm_loadu_ps(p2 + 4));
        s2 = _mm_add_ps(_mm_mul_ps(d2, d2), s2);
        __m128 d3 = _mm_sub_ps(_mm_loadu_ps(p1 + 8), _mm_loadu_ps(p2 + 8));
        s3 = _mm_add_ps(_mm_mul_ps(d3, d3), s3);
        __m128 d4 = _mm_sub_ps(_mm_loadu_ps(p1 + 12), _mm_loadu_ps(p2 + 12));
        s4 = _mm_add_ps(_mm_mul_ps(d4, d4), s4);
        p1 += 16; p2 += 16;
    }
    float result = hsum128_ps_sse(s1) + hsum128_ps_sse(s2) + hsum128_ps_sse(s3) + hsum128_ps_sse(s4);
    for (size_t i = 0; i < n - m; i++) { float d = p1[i] - p2[i]; result += d * d; }
    return -result;
}

/* simple_sse.rs:64-106 */
API float qo_manhattan_sse(const float* v1, const float* v2, size_t n) {
    const __m128 mask = _mm_set1_ps(-0.0f);
    size_t m = n - (n % 16);
    __m128 s1 = _mm_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    const float *p1 = v1, *p2 = v2;
    for (size_t i = 0; i < m; i += 16) {
        __m128 d1 = _mm_sub_ps(_mm_loadu_ps(p1), _mm_loadu_ps(p2));
        s1 = _mm_add_ps(_mm_andnot_ps(mask, d1), s1);
        __m128 d2 = _mm_sub_ps(_mm_loadu_ps(p1 + 4), _mm_loadu_ps(p2 + 4));
        s2 = _mm_add_ps(_mm_andnot_ps(mask, d2), s2);
        __m128 d3 = _mm_sub_ps(_mm_loadu_ps(p1 + 8), _mm_loadu_ps(p2 + 8));
        s3 = _mm_add_ps(_mm_andnot_ps(mask, d3), s3);
        __m128 d4 = _mm_sub_ps(_mm_loadu_ps(p1 + 12), _mm_loadu_ps(p2 + 12));
        s4 = _mm_add_ps(_mm_andnot_ps(mask, d4), s4);
        p1 += 16; p2 += 16;
    }
    float result = hsum128_ps_sse(s1) + hsum128_ps_sse(s2) + hsum128_ps_sse(s3) + hsum128_ps_sse(s4);
    for (size_t i = 0; i < n - m; i++) result += fabsf(p1[i] - p2[i]);
    return -result;
}

/* simple_sse.rs:110-150 */
API void qo_cosine_preprocess_sse(const float* v, float* out, size_t n) {
    size_t m = n - (n % 16);
    __m128 s1 = _mm_setzero_ps(), s2 = s1, s3 = s1, s4 = s1;
    const float* p = v;
    for (size_t i = 0; i < m; i += 16) {
        __m128 a = _mm_loadu_ps(p);      s1 = _mm_add_ps(_mm_mul_ps(a, a), s1);
        __m128 b = _mm_loadu_ps(p + 4);  s2 = _mm_add_ps(_mm_mul_ps(b, b), s2);
        __m128 c = _mm_loadu_ps(p + 8);  s3 = _mm_add_ps(_mm_mul_ps(c, c), s3);
        __m128 d = _mm_loadu_ps(p + 12); s4 = _mm_add_ps(_mm_mul_ps(d, d), s4);
        p += 16;
    }
    float length = hsum128_ps_sse(s1) + hsum128_ps_sse(s2) + hsum128_ps_sse(s3) + hsum128_ps_sse(s4);
    for (size_t i = 0; i < n - m; i++) length += p[i] * p[i];
    if (is_length_zero_or_normalized(length)) { memmove(out, v, n * sizeof(float)); return; }
    length = sqrtf(length);
    for (size_t i = 0; i < n; i++) out[i] = v[i] / length;
}

/* Rust's `impl Sum for f32` folds from -0.0 (core::iter::traits::accum, float_sum_into_float);
 * identical to folding from the first element except for the sign of an all-(-0.0) sum. */
#define RUST_SUM_INIT (-0.0f)

/* simple.rs:237-239 */
API float qo_dot_scalar(const float* v1, const float* v2, size_t n) {
    float s = RUST_SUM_INIT;
    for (size_t i = 0; i < n; i++) s += v1[i] * v2[i];
    return s;
}
/* simple.rs:214-219 */
API float qo_euclid_scalar(const float* v1, const float* v2, size_t n) {
    float s = RUST_SUM_INIT;
    for (size_t i = 0; i < n; i++) { float d = v1[i] - v2[i]; s += d * d; }
    return -s;
}
/* simple.rs:221-226 */
API float qo_manhattan_scalar(const float* v1, const float* v2, size_t n) {
    float s = RUST_SUM_INIT;
    for (size_t i = 0; i < n; i++) s += fabsf(v1[i] - v2[i]);
    return -s;
}
/* simple.rs:228-235 */
API void qo_cosine_preprocess_scalar(const float* v, float* out, size_t n) {
    float length = RUST_SUM_INIT;
    for (size_t i = 0; i < n; i++) length += v[i] * v[i];
    if (is_length_zero_or_normalized(length)) { memmove(out, v, n * sizeof(float)); return; }
    length = sqrtf(length);
    for (size_t i = 0; i < n; i++) out[i] = v[i] / length;
}

/* Distance enum order follows lib/segment/src/types.rs:313-322: Cosine, Euclid, Dot, Manhattan */
enum { QO_COSINE = 0, QO_EUCLID = 1, QO_DOT = 2, QO_MANHATTAN = 3 };
#define MIN_DIM_SIZE_AVX 32   /* simple.rs:15 */
#define MIN_DIM_SIZE_SIMD 16  /* simple.rs:22 */

/* Metric<f32>::similarity with the runtime dispatch of simple.rs:36-206 on an avx+fma host */
API float qo_similarity_f32(int distance, const float* q, const float* v, size_t n) {
    switch (distance) {
    case QO_COSINE: case QO_DOT:
        if (n >= MIN_DIM_SIZE_AVX) return qo_dot_avx(q, v, n);
        if (n >= MIN_DIM_SIZE_SIMD) return qo_dot_sse(q, v, n);
        return qo_dot_scalar(q, v, n);
    case QO_EUCLID:
        if (n >= MIN_DIM_SIZE_AVX) return qo_euclid_avx(q, v, n);
        if (n >= MIN_DIM_SIZE_SIMD) return qo_euclid_sse(q, v, n);
        return qo_euclid_scalar(q, v, n);
    default:
        if (n >= MIN_DIM_SIZE_AVX) return qo_manhattan_avx(q, v, n);
        if (n >= MIN_DIM_SIZE_SIMD) return qo_manhattan_sse(q, v, n);
        return qo_manhattan_scalar(q, v, n);
    }
}

/* Metric<f32>::preprocess: only Cosine normalises (simple.rs:178-200) */
API void qo_preprocess_f32(int distance, const float* v, float* out, size_t n) {
    if (distance != QO_COSINE) { memmove(out, v, n * sizeof(float)); return; }
    if (n >= MIN_DIM_SIZE_AVX) qo_cosine_preprocess_avx(v, out, n);
    else if (n >= MIN_DIM_SIZE_SIMD) qo_cosine_preprocess_sse(v, out, n);
    else qo_cosine_preprocess_scalar(v, out, n);
}

/* MetricPostProcessing::postprocess (simple.rs:74-78,118-122,163-167,208-212) */
API float qo_postprocess_f32(int distance, float score) {
    if (distance == QO_EUCLID) return sqrtf(fabsf(score));
    if (distance == QO_MANHATTAN) return fabsf(score);
    return score;
}

/* ------------------------------------------------------------------------------------------
 * u8-datatype metrics — lib/segment/src/spaces/metric_uint/{avx2,sse2}/ *.rs, simple_*.rs
 * ---------------------------------------------------------------------------------------- */

/* avx2/dot.rs:9-69 */
API float qo_u8_dot_avx(const uint8_t* v1, const uint8_t* v2, size_t len) {
    __m256i dot_acc = _mm256_setzero_si256();
    const __m256i mask = _mm256_set1_epi16(0xFF);
    const uint8_t *p1 = v1, *p2 = v2;
    for (size_t b = 0; b < len / 32; b++) {
        __m256i a = _mm256_loadu_si256((const __m256i*)p1);
        __m256i c = _mm256_loadu_si256((const __m256i*)p2);
        p1 += 32; p2 += 32;
        __m256i a_lo = _mm256_and_si256(a, mask);
        __m256i a_hi = _mm256_and_si256(_mm256_bsrli_epi128(a, 1), mask);
        __m256i c_lo = _mm256_and_si256(c, mask);
        __m256i c_hi = _mm256_and_si256(_mm256_bsrli_epi128(c, 1), mask);
        dot_acc = _mm256_add_epi32(dot_acc, _mm256_madd_epi16(a_lo, c_lo));
        dot_acc = _mm256_add_epi32(dot_acc, _mm256_madd_epi16(a_hi, c_hi));
    }
    float score = hsum256_ps_avx(_mm256_cvtepi32_ps(dot_acc));
    size_t rem = len % 32;
    if (rem != 0) {
        int32_t r = 0;
        for (size_t i = 0; i < rem; i++) r += (int32_t)p1[i] * (int32_t)p2[i];
        score += (float)r;
    }
    return score;
}

/* avx2/cosine.rs:9-105 */
API float qo_u8_cosine_avx(const uint8_t* v1, const uint8_t* v2, size_t len) {
    __m256i dot_acc = _mm256_setzero_si256(), n1_acc = dot_acc, n2_acc = dot_acc;
    const __m256i mask = _mm256_set1_epi16(0xFF);
    const uint8_t *p1 = v1, *p2 = v2;
    for (size_t b = 0; b < len / 32; b++) {
        __m256i a = _mm256_loadu_si256((const __m256i*)p1);
        __m256i c = _mm256_loadu_si256((const __m256i*)p2);
        p1 += 32; p2 += 32;
        __m256i a_lo = _mm256_and_si256(a, mask);
        __m256i a_hi = _mm256_and_si256(_mm256_bsrli_epi128(a, 1), mask);
        __m256i c_lo = _mm256_and_si256(c, mask);
        __m256i c_hi = _mm256_and_si256(_mm256_bsrli_epi128(c, 1), mask);
        n1_acc = _mm256_add_epi32(n1_acc, _mm256_madd_epi16(a_lo, a_lo));
        n2_acc = _mm256_add_epi32(n2_acc, _mm256_madd_epi16(c_lo, c_lo));
        dot_acc = _mm256_add_epi32(dot_acc, _mm256_madd_epi16(a_lo, c_lo));
        n1_acc = _mm256_add_epi32(n1_acc, _mm256_madd_epi16(a_hi, a_hi));
        n2_acc = _mm256_add_epi32(n2_acc, _mm256_madd_epi16(c_hi, c_hi));
        dot_acc = _mm256_add_epi32(dot_acc, _mm256_madd_epi16(a_hi, c_hi));
    }
    float dot = hsum256_ps_avx(_mm256_cvtepi32_ps(dot_acc));
    float n1 = hsum256_ps_avx(_mm256_cvtepi32_ps(n1_acc));
    float n2 = hsum256_ps_avx(_mm256_cvtepi32_ps(n2_acc));
    size_t rem = len % 32;
    if (rem != 0) {
        int32_t rd = 0, r1 = 0, r2 = 0;
        for (size_t i = 0; i < rem; i++) {
            int32_t x = p1[i], y = p2[i];
            rd += x * y; r1 += x * x; r2 += y * y;
        }
        dot += (float)rd; n1 += (float)r1; n2 += (float)r2;
    }
    float denom = n1 * n2;
    if (denom == 0.0f) return 0.0f;
    return dot / sqrtf(denom);
}

/* avx2/euclid.rs:9-67 */
API float qo_u8_euclid_avx(const uint8_t* v1, const uint8_t* v2, size_t len) {
    __m256i acc = _mm256_setzero_si256();
    const __m256i mask = _mm256_set1_epi16(0xFF);
    const uint8_t *p1 = v1, *p2 = v2;
    for (size_t b = 0; b < len / 32; b++) {
        __m256i a = _mm256_loadu_si256((const __m256i*)p1);
        __m256i c = _mm256_loadu_si256((const __m256i*)p2);
        p1 += 32; p2 += 32;
        __m256i ad = _mm256_max_epu8(_mm256_subs_epu8(a, c), _mm256_subs_epu8(c, a));
        __m256i lo = _mm256_and_si256(ad, mask);
        __m256i hi = _mm256_and_si256(_mm256_bsrli_epi128(ad, 1), mask);
        acc = _mm256_add_epi32(acc, _mm256_madd_epi16(lo, lo));
        acc = _mm256_add_epi32(acc, _mm256_madd_epi16(hi, hi));
    }
    float score = hsum256_ps_avx(_mm256_cvtepi32_ps(acc));
    size_t rem = len % 32;
    if (rem != 0) {
        int32_t r = 0;
        for (size_t i = 0; i < rem; i++) { int32_t d = (int32_t)p1[i] - (int32_t)p2[i]; r += d * d; }
        score += (float)r;
    }
    return -score;
}

/* avx2/manhattan.rs:9-56 */
API float qo_u8_manhattan_avx(const uint8_t* v1, const uint8_t* v2, size_t len) {
    __m256i acc = _mm256_setzero_si256();
    const uint8_t *p1 = v1, *p2 = v2;
    for (size_t b = 0; b < len / 32; b++) {
        __m256i a = _mm256_loadu_si256((const __m256i*)p1);
        __m256i c = _mm256_loadu_si256((const __m256i*)p2);
        p1 += 32; p2 += 32;
        acc = _mm256_add_epi32(acc, _mm256_sad_epu8(a, c));
    }
    float score = hsum256_ps_avx(_mm256_cvtepi32_ps(acc));
    size_t rem = len % 32;
    if (rem != 0) {
        int32_t r = 0;
        for (size_t i = 0; i < rem; i++) r += abs((int32_t)p1[i] - (int32_t)p2[i]);
        score += (float)r;
    }
    return -score;
}

/* scalar references: metric_uint/simple_dot.rs:58-69 etc. (i32 accumulate, one cast) */
API float qo_u8_dot_scalar(const uint8_t* a, const uint8_t* b, size_t n) {
    int32_t s = 0; for (size_t i = 0; i < n; i++) s += (int32_t)a[i] * (int32_t)b[i]; return (float)s;
}
API float qo_u8_euclid_scalar(const uint8_t* a, const uint8_t* b, size_t n) {
    int32_t s = 0; for (size_t i = 0; i < n; i++) { int32_t d = (int32_t)a[i] - (int32_t)b[i]; s += d * d; } return -(float)s;
}
API float qo_u8_manhattan_scalar(const uint8_t* a, const uint8_t* b, size_t n) {
    int32_t s = 0; for (size_t i = 0; i < n; i++) s += abs((int32_t)a[i] - (int32_t)b[i]); return -(float)s;
}
/* metric_uint/simple_cosine.rs:58-78 */
API float qo_u8_cosine_scalar(const uint8_t* a, const uint8_t* b, size_t n) {
    int32_t d = 0, n1 = 0, n2 = 0;
    for (size_t i = 0; i < n; i++) { int32_t x = a[i], y = b[i]; d += x * y; n1 += x * x; n2 += y * y; }
    if (n1 == 0 || n2 == 0) return 0.0f;
    return (float)d / sqrtf((float)n1 * (float)n2);
}

/* ------------------------------------------------------------------------------------------
 * SQ8 — lib/quantization/src/encoded_vectors_u8.rs, lib/quantization/cpp/avx2.c
 * ---------------------------------------------------------------------------------------- */

enum { QO_QD_COSINE = 0, QO_QD_DOT = 1, QO_QD_L1 = 2, QO_QD_L2 = 3 }; /* encoded_vectors.rs:13 */

/* cpp/avx2.c:7-14 */
static inline float hsum256_ps_c(__m256 X) {
    __m128 x128 = _mm_add_ps(_mm256_extractf128_ps(X, 1), _mm256_castps256_ps128(X));
    __m128 x64 = _mm_add_ps(x128, _mm_movehl_ps(x128, x128));
    __m128 x32 = _mm_add_ss(x64, _mm_shuffle_ps(x64, x64, 0x55));
    return _mm_cvtss_f32(x32);
}

/* cpp/avx2.c:25-63 (restated; the verbatim build lives in oracle/_ref/libsimd_utils.so) */
API float qo_sq8_dot_avx(const uint8_t* query_ptr, const uint8_t* vector_ptr, uint32_t dim) {
    const __m256i* v_ptr = (const __m256i*)vector_ptr;
    const __m256i* q_ptr = (const __m256i*)query_ptr;
    __m256i mul1 = _mm256_setzero_si256();
    const __m256i mask_epu32 = _mm256_set1_epi32(0xFFFF);
    for (uint32_t i = 0; i < dim / 32; i++) {
        __m256i v = _mm256_loadu_si256(v_ptr++);
        __m256i q = _mm256_loadu_si256(q_ptr++);
        __m256i s = _mm256_maddubs_epi16(v, q);
        __m256i s_low = _mm256_cvtepi16_epi32(_mm256_castsi256_si128(s));
        __m256i s_high = _mm256_cvtepi16_epi32(_mm256_extractf128_si256(s, 1));
        mul1 = _mm256_add_epi32(mul1, s_low);
        mul1 = _mm256_add_epi32(mul1, s_high);
    }
    if (dim % 32 != 0) {
        __m128i v_short = _mm_loadu_si128((const __m128i*)v_ptr);
        __m128i q_short = _mm_loadu_si128((const __m128i*)q_ptr);
        __m256i v1 = _mm256_cvtepu8_epi16(v_short);
        __m256i q1 = _mm256_cvtepu8_epi16(q_short);
        __m256i s = _mm256_mullo_epi16(v1, q1);
        mul1 = _mm256_add_epi32(mul1, _mm256_and_si256(s, mask_epu32));
        mul1 = _mm256_add_epi32(mul1, _mm256_srli_epi32(s, 16));
    }
    return hsum256_ps_c(_mm256_cvtepi32_ps(mul1));
}

/* cpp/avx2.c:65-122: result is an exact integer converted once to float */
API float qo_sq8_l1_avx(const uint8_t* query_ptr, const uint8_t* vector_ptr, uint32_t dim) {
    /* the u16-lane accumulation + final HSUM256_EPI32 is integer-exact while it does not
     * overflow u16 lanes (dim <= 16 * 65535/127); restated as the equivalent integer sum */
    int32_t sum = 0;
    for (uint32_t i = 0; i < dim; i++) sum += abs((int32_t)query_ptr[i] - (int32_t)vector_ptr[i]);
    return (float)sum;
}

typedef struct {
    uint32_t dim;         /* vector_parameters.dim */
    uint32_t actual_dim;  /* encoded_vectors_u8.rs:622-624 */
    float alpha, offset, multiplier;
    int32_t distance_type; /* QO_QD_* */
    int32_t invert;
} qo_sq8_meta;

/* encoded_vectors_u8.rs:95-98 ; f32::round = half away from zero; NaN as u8 = 0 */
static inline uint8_t sq8_encode_value(const qo_sq8_meta* m, float value) {
    float i = (value - m->offset) / m->alpha;
    /* f32::clamp: NaN stays NaN */
    if (i < 0.0f) i = 0.0f;
    if (i > 127.0f) i = 127.0f;
    float r = roundf(i);
    if (r != r) return 0;
    return (uint8_t)r;
}

/* encoded_vectors_u8.rs:116-134 */
static inline float sq8_get_shift(const qo_sq8_meta* m) {
    float shift;
    if (m->distance_type == QO_QD_DOT || m->distance_type == QO_QD_COSINE)
        shift = (float)m->actual_dim * m->offset * m->offset;
    else
        shift = 0.0f;
    return m->invert ? -shift : shift;
}
API float qo_sq8_get_shift(const qo_sq8_meta* m) { return sq8_get_shift(m); }

/* encoded_vectors_u8.rs:194-225,523-527 with quantile=None: alpha/offset from global min/max
 * (quantile.rs find_min_max_from_iter: plain f32 min/max over all values) */
API void qo_sq8_make_meta(const float* data, uint64_t count, uint32_t dim, int distance_type, int invert,
                          qo_sq8_meta* m) {
    float mn = FLT_MAX, mx = -FLT_MAX;
    for (uint64_t i = 0; i < count * (uint64_t)dim; i++) {
        float v = data[i];
        if (v < mn) mn = v;
        if (v > mx) mx = v;
    }
    m->dim = dim;
    m->actual_dim = dim + (16 - dim % 16) % 16;
    m->alpha = (mx - mn) / 127.0f;
    m->offset = mn;
    m->distance_type = distance_type;
    m->invert = invert;
    float mult;
    if (distance_type == QO_QD_DOT || distance_type == QO_QD_COSINE) mult = m->alpha * m->alpha;
    else if (distance_type == QO_QD_L1) mult = m->alpha;
    else mult = -2.0f * m->alpha * m->alpha;
    m->multiplier = invert ? -mult : mult;
}

/* code + offset for one vector; shared by encode (encoded_vectors_u8.rs:240-283) and
 * encode_int8_query (:583-619).  out_code has actual_dim bytes. Returns the un-shifted offset. */
static float sq8_encode_common(const qo_sq8_meta* m, const float* v, uint8_t* out_code) {
    for (uint32_t i = 0; i < m->dim; i++) out_code[i] = sq8_encode_value(m, v[i]);
    if (m->dim % 16 != 0) {
        float placeholder = (m->distance_type == QO_QD_DOT || m->distance_type == QO_QD_COSINE) ? 0.0f : m->offset;
        uint8_t e = sq8_encode_value(m, placeholder);
        for (uint32_t i = m->dim; i < m->actual_dim; i++) out_code[i] = e;
    }
    float off;
    if (m->distance_type == QO_QD_DOT || m->distance_type == QO_QD_COSINE) {
        float s = RUST_SUM_INIT;
        for (uint32_t i = 0; i < m->actual_dim; i++) s += (float)out_code[i];
        off = s * m->alpha * m->offset;
    } else if (m->distance_type == QO_QD_L1) {
        off = 0.0f;
    } else {
        float s = RUST_SUM_INIT;
        for (uint32_t i = 0; i < m->actual_dim; i++) s += (float)out_code[i] * (float)out_code[i];
        off = s * m->alpha * m->alpha;
    }
    return m->invert ? -off : off;
}

/* rows: count x (4 + actual_dim) bytes, layout [f32 v_off][codes] (encoded_vectors_u8.rs:240-283) */
API void qo_sq8_encode(const qo_sq8_meta* m, const float* data, uint64_t count, uint8_t* rows) {
    size_t stride = 4 + (size_t)m->actual_dim;
    for (uint64_t r = 0; r < count; r++) {
        uint8_t* row = rows + r * stride;
        float off = sq8_encode_common(m, data + r * (uint64_t)m->dim, row + 4);
        float v_off = sq8_get_shift(m) + off;
        memcpy(row, &v_off, 4);
    }
}

/* encoded_vectors_u8.rs:583-619 */
API float qo_sq8_encode_query(const qo_sq8_meta* m, const float* query, uint8_t* out_code) {
    return sq8_encode_common(m, query, out_code);
}

/* encoded_vectors_u8.rs:101-103 */
static inline float sq8_postprocess(const qo_sq8_meta* m, float score, float q_off, float v_off) {
    return m->multiplier * score + q_off + v_off;
}

/* score_point_avx, encoded_vectors_u8.rs:471-490 */
API float qo_sq8_score(const qo_sq8_meta* m, const uint8_t* q_code, float q_off, const uint8_t* row) {
    float v_off; memcpy(&v_off, row, 4);
    float s = (m->distance_type == QO_QD_L1) ? qo_sq8_l1_avx(q_code, row + 4, m->actual_dim)
                                             : qo_sq8_dot_avx(q_code, row + 4, m->actual_dim);
    return sq8_postprocess(m, s, q_off, v_off);
}

/* score_point_avx_internal, encoded_vectors_u8.rs:492-514 + postprocess_internal_score :106-114 */
API float qo_sq8_score_internal(const qo_sq8_meta* m, const uint8_t* row_i, const uint8_t* row_j) {
    float qo, vo; memcpy(&qo, row_i, 4); memcpy(&vo, row_j, 4);
    float s = (m->distance_type == QO_QD_L1) ? qo_sq8_l1_avx(row_i + 4, row_j + 4, m->actual_dim)
                                             : qo_sq8_dot_avx(row_i + 4, row_j + 4, m->actual_dim);
    float q_off = qo - sq8_get_shift(m);
    return sq8_postprocess(m, s, q_off, vo);
}

/* ------------------------------------------------------------------------------------------
 * PQ — lib/quantization/src/encoded_vectors_pq.rs
 * ---------------------------------------------------------------------------------------- */

/* DistanceType::distance, encoded_vectors.rs:119-127 */
static inline float qd_distance(int dt, const float* a, const float* b, uint32_t n) {
    float s = RUST_SUM_INIT;
    if (dt == QO_QD_DOT || dt == QO_QD_COSINE) { for (uint32_t i = 0; i < n; i++) s += a[i] * b[i]; }
    else if (dt == QO_QD_L1) { for (uint32_t i = 0; i < n; i++) s += fabsf(a[i] - b[i]); }
    else { for (uint32_t i = 0; i < n; i++) { float d = a[i] - b[i]; s += d * d; } }
    return s;
}

/* encode_vector, encoded_vectors_pq.rs:301-329.  centroids: n_centroids x dim (row-major full-dim vectors);
 * division: m chunks [start,end) given as starts of step chunk_size (get_vector_division :164-169). */
API void qo_pq_encode(const float* data, uint64_t count, uint32_t dim, uint32_t chunk, const float* centroids,
                      uint32_t n_centroids, uint8_t* codes) {
    uint32_t m = (dim + chunk - 1) / chunk;
    for (uint64_t r = 0; r < count; r++) {
        const float* v = data + r * (uint64_t)dim;
        for (uint32_t j = 0; j < m; j++) {
            uint32_t s = j * chunk, e = s + chunk < dim ? s + chunk : dim;
            float min_d = FLT_MAX; uint32_t min_c = 0;
            for (uint32_t c = 0; c < n_centroids; c++) {
                const float* cd = centroids + (uint64_t)c * dim + s;
                float d = RUST_SUM_INIT;
                for (uint32_t k = 0; k < e - s; k++) { float t = v[s + k] - cd[k]; d += t * t; }
                if (d < min_d) { min_d = d; min_c = c; }
            }
            codes[r * (uint64_t)m + j] = (uint8_t)min_c;
        }
    }
}

/* encode_query (LUT build), encoded_vectors_pq.rs:519-541.  lut: m x n_centroids */
API void qo_pq_encode_query(const float* query, uint32_t dim, uint32_t chunk, const float* centroids,
                            uint32_t n_centroids, int distance_type, int invert, float* lut) {
    uint32_t m = (dim + chunk - 1) / chunk;
    for (uint32_t j = 0; j < m; j++) {
        uint32_t s = j * chunk, e = s + chunk < dim ? s + chunk : dim;
        for (uint32_t c = 0; c < n_centroids; c++) {
            float d = qd_distance(distance_type, query + s, centroids + (uint64_t)c * dim + s, e - s);
            lut[(uint64_t)j * n_centroids + c] = invert ? -d : d;
        }
    }
}

/* score_point_sse, encoded_vectors_pq.rs:411-443 */
API float qo_pq_score(const float* lut, uint32_t n_centroids, const uint8_t* code, uint32_t len) {
    const uint8_t* c = code;
    const float* l = lut;
    __m128 sum128 = _mm_setzero_ps();
    for (uint32_t i = 0; i < len / 4; i++) {
        float buf[4] = { l[c[0]], l[n_centroids + c[1]], l[2 * n_centroids + c[2]], l[3 * n_centroids + c[3]] };
        sum128 = _mm_add_ps(sum128, _mm_loadu_ps(buf));
        c += 4; l += 4 * (size_t)n_centroids;
    }
    __m128 sum64 = _mm_add_ps(sum128, _mm_movehl_ps(sum128, sum128));
    __m128 sum32 = _mm_add_ss(sum64, _mm_shuffle_ps(sum64, sum64, 0x55));
    float sum = _mm_cvtss_f32(sum32);
    for (uint32_t i = 0; i < len % 4; i++) { sum += l[*c]; c++; l += n_centroids; }
    return sum;
}

/* score_internal, encoded_vectors_pq.rs:574-618 */
API float qo_pq_score_internal(const uint8_t* ci, const uint8_t* cj, uint32_t dim, uint32_t chunk,
                               const float* centroids, int distance_type, int invert) {
    uint32_t m = (dim + chunk - 1) / chunk;
    float s = RUST_SUM_INIT;
    for (uint32_t j = 0; j < m; j++) {
        uint32_t st = j * chunk, e = st + chunk < dim ? st + chunk : dim;
        s += qd_distance(distance_type, centroids + (uint64_t)ci[j] * dim + st, centroids + (uint64_t)cj[j] * dim + st, e - st);
    }
    return invert ? -s : s;
}

/* ------------------------------------------------------------------------------------------
 * BQ — lib/quantization/src/encoded_vectors_binary.rs (TBitsStoreType = u128)
 * ---------------------------------------------------------------------------------------- */

enum { QO_BQ_ONE = 0, QO_BQ_TWO = 1, QO_BQ_ONE_AND_HALF = 2 };         /* Encoding :34-39 */
enum { QO_BQQ_SAME = 0, QO_BQQ_SCALAR4 = 1, QO_BQQ_SCALAR8 = 2 };      /* QueryEncoding :48-54 */

/* get_quantized_vector_size_from_params :829-839, bytes per row for u128 words */
API uint32_t qo_bq_row_bytes(uint32_t dim, int encoding) {
    uint64_t ext = dim;
    if (encoding == QO_BQ_TWO) ext = (uint64_t)dim * 2;
    else if (encoding == QO_BQ_ONE_AND_HALF) ext = ((uint64_t)dim * 3 + 1) / 2;
    if (ext < 1) ext = 1;
    uint64_t words = ext / 128 + (ext % 128 != 0);
    return (uint32_t)(words * 16);
}

static inline void set_bit(uint8_t* row, uint64_t i) { row[i >> 3] |= (uint8_t)(1u << (i & 7)); }

/* encode_two_bits_value :636-671 ; stats = (mean, stddev) per coordinate or NULL */
static inline void bq_two_bits_value(float value, const float* mean_std, int* b1, int* b2) {
    if (!mean_std) { *b1 = *b2 = value > 0.0f; return; }
    float mean = mean_std[0], sd = mean_std[1];
    if (sd < FLT_EPSILON) { *b1 = value > 0.0f; *b2 = 0; return; }
    float vz = (value - mean) / sd;
    const float SIGMAS = 2.0f / 3.0f;
    if (vz <= -SIGMAS) { *b1 = 0; *b2 = 0; }
    else if (vz < SIGMAS) { *b1 = 1; *b2 = 0; }
    else { *b1 = 1; *b2 = 1; }
}

/* encode_vector :531-556 + encode_{one_bit,two_bits,one_and_half_bits}_vector :558-634.
 * A u128 word with bit (i % 128) set is, in little-endian memory, byte (i%128)/8 bit i%8: i.e. plain
 * little-endian bit numbering over the row. mean_std: dim x 2 floats or NULL. */
API void qo_bq_encode(const float* v, uint32_t dim, int encoding, const float* mean_std, uint8_t* row) {
    memset(row, 0, qo_bq_row_bytes(dim, encoding));
    for (uint32_t i = 0; i < dim; i++) {
        if (encoding == QO_BQ_ONE) { if (v[i] > 0.0f) set_bit(row, i); continue; }
        int b1, b2;
        bq_two_bits_value(v[i], mean_std ? mean_std + 2 * (size_t)i : NULL, &b1, &b2);
        if (b1) set_bit(row, i);
        if (b2) set_bit(row, encoding == QO_BQ_TWO ? (uint64_t)dim + i : (uint64_t)dim + i / 2);
    }
}

/* _encode_scalar_query_vector :722-757 on the (possibly extended, :692-720) query.
 * out: words(ext) * bits_count u128 words, transposed layout. Returns number of bytes written. */
API uint32_t qo_bq_encode_scalar_query(const float* query, uint32_t dim, int encoding, uint32_t bits_count, uint8_t* out) {
    uint32_t ext = dim;
    if (encoding == QO_BQ_TWO) ext = dim * 2;
    else if (encoding == QO_BQ_ONE_AND_HALF) ext = dim + (dim + 1) / 2;
    float* q = (float*)malloc(sizeof(float) * (ext ? ext : 1));
    memcpy(q, query, sizeof(float) * dim);
    if (encoding == QO_BQ_TWO) memcpy(q + dim, query, sizeof(float) * dim);
    else if (encoding == QO_BQ_ONE_AND_HALF) {
        for (uint32_t i = 0; i < dim; i += 2) {
            /* f32::max: if one is NaN returns the other */
            float a = query[i];
            if (i + 1 < dim) { float b = query[i + 1]; a = fmaxf(a, b); }
            q[dim + i / 2] = a;
        }
    }
    uint32_t n = ext;
    uint32_t words = (n > 0 ? n : 1) / 128 + (((n > 0 ? n : 1) % 128) != 0);
    uint32_t bytes = words * bits_count * 16;
    memset(out, 0, bytes);
    float max_abs = 0.0f;
    for (uint32_t i = 0; i < n; i++) max_abs = fmaxf(max_abs, fabsf(q[i]));
    float mn = -max_abs, mx = max_abs;
    uint64_t ranges = (1ull << bits_count) - 1;
    float delta = (mx - mn) / (float)ranges;
    for (uint32_t i = 0; i < n; i++) {
        uint32_t chunk_index = i / 128, shift = i % 128;
        float shifted = q[i] - mn;
        float delted = delta > FLT_EPSILON ? shifted / delta : 0.0f;
        float rv = roundf(delted);
        /* `as usize` saturates; NaN -> 0 */
        uint64_t rounded = (rv != rv || rv <= 0.0f) ? 0 : (rv >= 1.8446744e19f ? UINT64_MAX : (uint64_t)rv);
        uint64_t quantized = rounded % (ranges + 1);
        for (uint32_t b = 0; b < bits_count; b++) {
            if ((quantized >> b) & 1) {
                uint8_t* word = out + ((size_t)bits_count * chunk_index + b) * 16;
                word[shift >> 3] |= (uint8_t)(1u << (shift & 7));
            }
        }
    }
    free(q);
    return bytes;
}

/* xor_popcnt for u128 words :288-335 (integer-exact on every dispatch tier) */
static inline uint64_t bq_xor_popcnt(const uint8_t* v, const uint8_t* q, uint32_t words) {
    uint64_t r = 0;
    const uint64_t* a = (const uint64_t*)v; const uint64_t* b = (const uint64_t*)q;
    for (uint32_t i = 0; i < words * 2; i++) r += (uint64_t)__builtin_popcountll(a[i] ^ b[i]);
    return r;
}

/* xor_popcnt_scalar :337-410 generic fallback (== what the C kernels compute while < 2^24) */
static inline uint64_t bq_xor_popcnt_scalar(const uint8_t* v, const uint8_t* q, uint32_t words, uint32_t bits) {
    uint64_t r = 0;
    const uint64_t* a = (const uint64_t*)v; const uint64_t* b = (const uint64_t*)q;
    for (uint32_t w = 0; w < words; w++)
        for (uint32_t i = 0; i < bits; i++) {
            uint64_t c = (uint64_t)__builtin_popcountll(a[2 * w] ^ b[2 * ((size_t)w * bits + i)])
                       + (uint64_t)__builtin_popcountll(a[2 * w + 1] ^ b[2 * ((size_t)w * bits + i) + 1]);
            r += c << i;
        }
    return r;
}

/* calculate_metric :766-810 ; query_bits_count = 1 (SameAsStorage), 4 or 8 */
API float qo_bq_score(const uint8_t* vector, const uint8_t* query, uint32_t dim, int encoding, uint32_t query_bits_count,
                      int distance_type, int invert) {
    uint32_t words = qo_bq_row_bytes(dim, encoding) / 16;
    float xor_product;
    if (query_bits_count == 1) xor_product = (float)bq_xor_popcnt(vector, query, words);
    else {
        uint64_t x = bq_xor_popcnt_scalar(vector, query, words, query_bits_count);
        xor_product = (float)x / (float)((1 << query_bits_count) - 1);
    }
    float dimf = (float)dim;
    float zeros = dimf - xor_product;
    int is_dot = distance_type == QO_QD_DOT || distance_type == QO_QD_COSINE;
    if (is_dot) return invert ? xor_product - zeros : zeros - xor_product;
    return invert ? zeros - xor_product : xor_product - zeros;
}

/* ------------------------------------------------------------------------------------------
 * Top-k: FixedLengthPriorityQueue (lib/common/common/src/fixed_length_priority_queue.rs:20-65) over
 * ScoredPointOffset ordered by score only (lib/common/common/src/types.rs:21-25).  The heap is Rust's
 * std BinaryHeap<Reverse<T>> restated (sift_up on push, sift_down after peek_mut swap, heap-sort for
 * into_sorted_vec), so that the surviving set under ties matches the reference.
 * ---------------------------------------------------------------------------------------- */

typedef struct { uint32_t idx; float score; } qo_scored;

/* OrderedFloat total order: NaN is greatest and equal to itself */
static inline int of_cmp(float a, float b) {
    int an = a != a, bn = b != b;
    if (an || bn) return an - bn;
    return (a > b) - (a < b);
}
/* BinaryHeap<Reverse<T>> is a max-heap on Reverse => element "greater" means smaller score */
static inline int rev_le(const qo_scored* a, const qo_scored* b) { return of_cmp(b->score, a->score) <= 0; } /* Reverse(a) <= Reverse(b) */
static inline int rev_ge(const qo_scored* a, const qo_scored* b) { return of_cmp(b->score, a->score) >= 0; }

static void heap_sift_up(qo_scored* d, size_t start, size_t pos) {
    qo_scored elt = d[pos];
    while (pos > start) {
        size_t parent = (pos - 1) / 2;
        if (rev_le(&elt, &d[parent])) break;          /* hole.element() <= hole.get(parent) */
        d[pos] = d[parent]; pos = parent;
    }
    d[pos] = elt;
}
static void heap_sift_down_range(qo_scored* d, size_t pos, size_t end) {
    qo_scored elt = d[pos];
    size_t child = 2 * pos + 1;
    while (end >= 2 && child <= end - 2) {
        child += rev_le(&d[child], &d[child + 1]);    /* pick the greater child; ties -> right */
        if (rev_ge(&elt, &d[child])) { d[pos] = elt; return; }
        d[pos] = d[child]; pos = child; child = 2 * pos + 1;
    }
    if (child == end - 1 && !rev_ge(&elt, &d[child])) { d[pos] = d[child]; pos = child; }
    d[pos] = elt;
}

typedef struct { qo_scored* heap; size_t len, cap; } qo_pq;

static void pq_push(qo_pq* q, qo_scored v) {
    if (q->len < q->cap) { q->heap[q->len] = v; heap_sift_up(q->heap, 0, q->len); q->len++; return; }
    /* peek_mut: x = current min score; if x.0 < value.0 swap, then sift_down(0) on drop */
    if (of_cmp(q->heap[0].score, v.score) < 0) { q->heap[0] = v; heap_sift_down_range(q->heap, 0, q->len); }
}
/* into_sorted_vec of BinaryHeap<Reverse<T>> = ascending in Reverse = descending by score */
static void pq_into_sorted(qo_pq* q) {
    size_t end = q->len;
    while (end > 1) {
        end--;
        qo_scored t = q->heap[0]; q->heap[0] = q->heap[end]; q->heap[end] = t;
        heap_sift_down_range(q->heap, 0, end);
    }
}

API uint32_t qo_topk(const uint32_t* ids, const float* scores, uint64_t n, uint32_t top, qo_scored* out) {
    if (top == 0) return 0;
    qo_pq q = { out, 0, top };
    for (uint64_t i = 0; i < n; i++) { qo_scored v = { ids ? ids[i] : (uint32_t)i, scores[i] }; pq_push(&q, v); }
    pq_into_sorted(&q);
    return (uint32_t)q.len;
}

/* ------------------------------------------------------------------------------------------
 * Brute-force scan: BatchFilteredSearcher::peek_top_iter, lib/segment/src/index/hnsw_index/point_scorer.rs:423-472
 * 64-id chunks (VECTOR_READ_BATCH_SIZE, vector_storage/common.rs:20) x per-query scorers x per-query heaps.
 * deleted: optional bitmap (bit=1 => deleted).  Returns per-query result counts in out_counts.
 * ---------------------------------------------------------------------------------------- */
#define VECTOR_READ_BATCH_SIZE 64

static inline int is_deleted(const uint64_t* bm, uint64_t i) { return bm && ((bm[i >> 6] >> (i & 63)) & 1); }

API void qo_scan_f32(int distance, const float* base, uint64_t row_begin, uint64_t row_end, uint32_t dim,
                     const float* queries_preprocessed, uint32_t n_queries, uint32_t top,
                     const uint64_t* deleted, qo_scored* out, uint32_t* out_counts) {
    qo_pq* pqs = (qo_pq*)malloc(sizeof(qo_pq) * n_queries);
    for (uint32_t q = 0; q < n_queries; q++) { pqs[q].heap = out + (size_t)q * top; pqs[q].len = 0; pqs[q].cap = top; }
    uint32_t chunk[VECTOR_READ_BATCH_SIZE]; float scores[VECTOR_READ_BATCH_SIZE];
    uint64_t next = row_begin;
    for (;;) {
        uint32_t cs = 0;
        while (next < row_end && cs < VECTOR_READ_BATCH_SIZE) { if (!is_deleted(deleted, next)) chunk[cs++] = (uint32_t)next; next++; }
        if (cs == 0) break;
        for (uint32_t q = 0; q < n_queries; q++) {
            const float* qv = queries_preprocessed + (size_t)q * dim;
            for (uint32_t i = 0; i < cs; i++) scores[i] = qo_similarity_f32(distance, qv, base + (uint64_t)chunk[i] * dim, dim);
            if (top) for (uint32_t i = 0; i < cs; i++) { qo_scored v = { chunk[i], scores[i] }; pq_push(&pqs[q], v); }
        }
    }
    for (uint32_t q = 0; q < n_queries; q++) { pq_into_sorted(&pqs[q]); out_counts[q] = (uint32_t)pqs[q].len; }
    free(pqs);
}

API void qo_scan_sq8(const qo_sq8_meta* m, const uint8_t* rows, uint64_t row_begin, uint64_t row_end,
                     const uint8_t* q_codes, const float* q_offs, uint32_t n_queries, uint32_t top,
                     const uint64_t* deleted, qo_scored* out, uint32_t* out_counts) {
    size_t stride = 4 + (size_t)m->actual_dim;
    qo_pq* pqs = (qo_pq*)malloc(sizeof(qo_pq) * n_queries);
    for (uint32_t q = 0; q < n_queries; q++) { pqs[q].heap = out + (size_t)q * top; pqs[q].len = 0; pqs[q].cap = top; }
    uint32_t chunk[VECTOR_READ_BATCH_SIZE]; float scores[VECTOR_READ_BATCH_SIZE];
    uint64_t next = row_begin;
    for (;;) {
        uint32_t cs = 0;
        while (next < row_end && cs < VECTOR_READ_BATCH_SIZE) { if (!is_deleted(deleted, next)) chunk[cs++] = (uint32_t)next; next++; }
        if (cs == 0) break;
        for (uint32_t q = 0; q < n_queries; q++) {
            for (uint32_t i = 0; i < cs; i++)
                scores[i] = qo_sq8_score(m, q_codes + (size_t)q * m->actual_dim, q_offs[q], rows + (uint64_t)chunk[i] * stride);
            if (top) for (uint32_t i = 0; i < cs; i++) { qo_scored v = { chunk[i], scores[i] }; pq_push(&pqs[q], v); }
        }
    }
    for (uint32_t q = 0; q < n_queries; q++) { pq_into_sorted(&pqs[q]); out_counts[q] = (uint32_t)pqs[q].len; }
    free(pqs);
}

API void qo_scan_pq(const uint8_t* codes, uint64_t row_begin, uint64_t row_end, uint32_t m_chunks, uint32_t n_centroids,
                    const float* luts, uint32_t n_queries, uint32_t top,
                    const uint64_t* deleted, qo_scored* out, uint32_t* out_counts) {
    qo_pq* pqs = (qo_pq*)malloc(sizeof(qo_pq) * n_queries);
    for (uint32_t q = 0; q < n_queries; q++) { pqs[q].heap = out + (size_t)q * top; pqs[q].len = 0; pqs[q].cap = top; }
    uint32_t chunk[VECTOR_READ_BATCH_SIZE]; float scores[VECTOR_READ_BATCH_SIZE];
    uint64_t next = row_begin;
    size_t lut_sz = (size_t)m_chunks * n_centroids;
    for (;;) {
        uint32_t cs = 0;
        while (next < row_end && cs < VECTOR_READ_BATCH_SIZE) { if (!is_deleted(deleted, next)) chunk[cs++] = (uint32_t)next; next++; }
        if (cs == 0) break;
        for (uint32_t q = 0; q < n_queries; q++) {
            for (uint32_t i = 0; i < cs; i++)
                scores[i] = qo_pq_score(luts + q * lut_sz, n_centroids, codes + (uint64_t)chunk[i] * m_chunks, m_chunks);
            if (top) for (uint32_t i = 0; i < cs; i++) { qo_scored v = { chunk[i], scores[i] }; pq_push(&pqs[q], v); }
        }
    }
    for (uint32_t q = 0; q < n_queries; q++) { pq_into_sorted(&pqs[q]); out_counts[q] = (uint32_t)pqs[q].len; }
    free(pqs);
}

API void qo_scan_bq(const uint8_t* rows, uint64_t row_begin, uint64_t row_end, uint32_t dim, int encoding,
                    uint32_t query_bits_count, int distance_type, int invert,
                    const uint8_t* q_enc, uint32_t q_stride, uint32_t n_queries, uint32_t top,
                    const uint64_t* deleted, qo_scored* out, uint32_t* out_counts) {
    uint32_t rb = qo_bq_row_bytes(dim, encoding);
    qo_pq* pqs = (qo_pq*)malloc(sizeof(qo_pq) * n_queries);
    for (uint32_t q = 0; q < n_queries; q++) { pqs[q].heap = out + (size_t)q * top; pqs[q].len = 0; pqs[q].cap = top; }
    uint32_t chunk[VECTOR_READ_BATCH_SIZE]; float scores[VECTOR_READ_BATCH_SIZE];
    uint64_t next = row_begin;
    for (;;) {
        uint32_t cs = 0;
        while (next < row_end && cs < VECTOR_READ_BATCH_SIZE) { if (!is_deleted(deleted, next)) chunk[cs++] = (uint32_t)next; next++; }
        if (cs == 0) break;
        for (uint32_t q = 0; q < n_queries; q++) {
            for (uint32_t i = 0; i < cs; i++)
                scores[i] = qo_bq_score(rows + (uint64_t)chunk[i] * rb, q_enc + (size_t)q * q_stride, dim, encoding,
                                        query_bits_count, distance_type, invert);
            if (top) for (uint32_t i = 0; i < cs; i++) { qo_scored v = { chunk[i], scores[i] }; pq_push(&pqs[q], v); }
        }
    }
    for (uint32_t q = 0; q < n_queries; q++) { pq_into_sorted(&pqs[q]); out_counts[q] = (uint32_t)pqs[q].len; }
    free(pqs);
}

/* Whole-storage quantized scoring: out[i] = the per-row score (qo_sq8_score / qo_pq_score / qo_bq_score) of row ids ? ids[i] : i,
 * i < n, for one encoded query */
API void qo_score_rows_sq8(const qo_sq8_meta* m, const uint8_t* rows, uint64_t n, const uint8_t* q_code, float q_off, const uint32_t* ids, float* out) {
    const size_t stride = 4 + (size_t)m->actual_dim;
    for (uint64_t i = 0; i < n; i++) out[i] = qo_sq8_score(m, q_code, q_off, rows + (uint64_t)(ids ? ids[i] : i) * stride);
}
API void qo_score_rows_pq(const uint8_t* codes, uint64_t n, uint32_t m_chunks, uint32_t n_centroids, const float* lut, const uint32_t* ids, float* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = qo_pq_score(lut, n_centroids, codes + (uint64_t)(ids ? ids[i] : i) * m_chunks, m_chunks);
}
API void qo_score_rows_bq(const uint8_t* rows, uint64_t n, uint32_t dim, int encoding, uint32_t query_bits_count, int distance_type, int invert,
                          const uint8_t* q_enc, const uint32_t* ids, float* out) {
    const uint32_t rb = qo_bq_row_bytes(dim, encoding);
    for (uint64_t i = 0; i < n; i++)
        out[i] = qo_bq_score(rows + (uint64_t)(ids ? ids[i] : i) * rb, q_enc, dim, encoding, query_bits_count, distance_type, invert);
}

/* bulk helpers used by tests/bench (score every listed id) */
API void qo_score_points_f32(int distance, const float* base, uint32_t dim, const float* q_pre,
                             const uint32_t* ids, uint64_t n, float* scores) {
    for (uint64_t i = 0; i < n; i++) scores[i] = qo_similarity_f32(distance, q_pre, base + (uint64_t)ids[i] * dim, dim);
}
API void qo_score_rows_f32(int distance, const float* rows, uint64_t n, uint32_t dim, const float* q_pre, float* scores) {
    for (uint64_t i = 0; i < n; i++) scores[i] = qo_similarity_f32(distance, q_pre, rows + i * dim, dim);
}
API void qo_preprocess_rows_f32(int distance, const float* in, float* out, uint64_t n, uint32_t dim) {
    for (uint64_t i = 0; i < n; i++) qo_preprocess_f32(distance, in + i * dim, out + i * dim, dim);
}

/* ------------------------------------------------------------------------------------------
 * f16-datatype metrics — lib/segment/src/spaces/metric_f16/{avx,sse}/ *.rs, simple_*.rs
 * (`half` 2.7.1 f16::to_f32 / from_f32 are IEEE-exact conversions; F16C gives the same values)
 * ---------------------------------------------------------------------------------------- */
static inline float h2f(uint16_t h) { return _cvtsh_ss(h); }

/* metric_f16/avx/{dot.rs:13-69, euclid.rs:13-70, manhattan.rs:13-75}; kind 0 dot, 1 euclid, 2 manhattan */
static float f16_avx(int kind, const uint16_t* v1, const uint16_t* v2, size_t n) {
    const __m256 mask = _mm256_set1_ps(-0.0f);
    size_t m = n - (n % 32);
    __m256 s[4] = { _mm256_setzero_ps(), _mm256_setzero_ps(), _mm256_setzero_ps(), _mm256_setzero_ps() };
    const __m128i* p1 = (const __m128i*)v1; const __m128i* p2 = (const __m128i*)v2;
    for (size_t i = 0; i < m; i += 32) {
        for (int a = 0; a < 4; a++) {
            __m256 x = _mm256_cvtph_ps(_mm_loadu_si128(p1 + a));
            __m256 y = _mm256_cvtph_ps(_mm_loadu_si128(p2 + a));
            if (kind == 0) s[a] = _mm256_fmadd_ps(x, y, s[a]);
            else {
                __m256 d = _mm256_sub_ps(x, y);
                if (kind == 1) s[a] = _mm256_fmadd_ps(d, d, s[a]);
                else s[a] = _mm256_add_ps(_mm256_andnot_ps(mask, d), s[a]);
            }
        }
        p1 += 4; p2 += 4;
    }
    const uint16_t* t1 = (const uint16_t*)p1; const uint16_t* t2 = (const uint16_t*)p2;
    float result = hsum256_ps_avx(s[0]) + hsum256_ps_avx(s[1]) + hsum256_ps_avx(s[2]) + hsum256_ps_avx(s[3]);
    for (size_t i = 0; i < n - m; i++) {
        float a = h2f(t1[i]), b = h2f(t2[i]);
        if (kind == 0) result += a * b;
        else if (kind == 1) { float d = a - b; result += d * d; }
        else result += fabsf(a - b);
    }
    return kind == 0 ? result : -result;
}
API float qo_f16_dot_avx(const uint16_t* a, const uint16_t* b, size_t n) { return f16_avx(0, a, b, n); }
API float qo_f16_euclid_avx(const uint16_t* a, const uint16_t* b, size_t n) { return f16_avx(1, a, b, n); }
API float qo_f16_manhattan_avx(const uint16_t* a, const uint16_t* b, size_t n) { return f16_avx(2, a, b, n); }

/* Metric<f16>::similarity dispatch (metric_f16/simple_dot.rs:17-56 etc.): avx+fma+f16c for n >= 32; the SSE tier
 * converts to f32 and calls the f32 SSE kernels (metric_f16/sse/dot.rs:10-17); scalar tier sums f32 products. */
API float qo_similarity_f16(int distance, const uint16_t* q, const uint16_t* v, size_t n) {
    int kind = (distance == QO_EUCLID) ? 1 : (distance == QO_MANHATTAN ? 2 : 0);
    if (n >= MIN_DIM_SIZE_AVX) return f16_avx(kind, q, v, n);
    float a[32], b[32];
    for (size_t i = 0; i < n; i++) { a[i] = h2f(q[i]); b[i] = h2f(v[i]); }
    if (n >= MIN_DIM_SIZE_SIMD)
        return kind == 0 ? qo_dot_sse(a, b, n) : (kind == 1 ? qo_euclid_sse(a, b, n) : qo_manhattan_sse(a, b, n));
    return kind == 0 ? qo_dot_scalar(a, b, n) : (kind == 1 ? qo_euclid_scalar(a, b, n) : qo_manhattan_scalar(a, b, n));
}
/* scalar f16 reference (metric_f16/simple_dot.rs:65-73) for the SIMD-vs-scalar tolerance KAT */
API float qo_f16_dot_scalar(const uint16_t* a, const uint16_t* b, size_t n) {
    float s = RUST_SUM_INIT;
    for (size_t i = 0; i < n; i++) s += h2f(a[i]) * h2f(b[i]);
    return s;
}

/* ------------------------------------------------------------------------------------------
 * Whole-storage scoring for the f16 / u8 datatypes and the query conversions in front of it
 * ---------------------------------------------------------------------------------------- */

/* Metric<u8>::similarity dispatch: the avx2 kernels for n >= 32, the integer-exact scalar tier below */
static float u8_similarity(int distance, const uint8_t* q, const uint8_t* v, size_t n) {
    const int avx = n >= MIN_DIM_SIZE_AVX;
    switch (distance) {
        case QO_COSINE: return avx ? qo_u8_cosine_avx(q, v, n) : qo_u8_cosine_scalar(q, v, n);
        case QO_EUCLID: return avx ? qo_u8_euclid_avx(q, v, n) : qo_u8_euclid_scalar(q, v, n);
        case QO_MANHATTAN: return avx ? qo_u8_manhattan_avx(q, v, n) : qo_u8_manhattan_scalar(q, v, n);
        default: return avx ? qo_u8_dot_avx(q, v, n) : qo_u8_dot_scalar(q, v, n);
    }
}

/* out[i] = similarity(q, rows[ids ? ids[i] : i]) for i < n; q is already in the storage datatype */
API void qo_score_rows_f16(int distance, const uint16_t* rows, uint64_t n, uint32_t dim, const uint16_t* q, const uint32_t* ids, float* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = qo_similarity_f16(distance, q, rows + (uint64_t)(ids ? ids[i] : i) * dim, dim);
}
API void qo_score_rows_u8(int distance, const uint8_t* rows, uint64_t n, uint32_t dim, const uint8_t* q, const uint32_t* ids, float* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = u8_similarity(distance, q, rows + (uint64_t)(ids ? ids[i] : i) * dim, dim);
}

/* f16::from_f32 (half 2.x): round to nearest, ties to even; overflow to +-inf; subnormal results kept; NaN stays NaN (quiet, top
 * payload bits kept) */
static uint16_t f32_to_f16_bits(float f) {
    uint32_t x;
    memcpy(&x, &f, 4);
    const uint16_t sign = (uint16_t)((x >> 16) & 0x8000u);
    const uint32_t ax = x & 0x7FFFFFFFu;
    if (ax > 0x7F800000u) return (uint16_t)(sign | 0x7E00u | ((ax & 0x7FFFFFu) >> 13));
    if (ax >= 0x47800000u) return (uint16_t)(sign | 0x7C00u);                 /* >= 65536 and inf */
    if (ax >= 0x38800000u)                                                      /* the normal range (>= 2^-14): RNE on the 13 dropped bits */
        return (uint16_t)(sign | (((ax + 0xFFFu + ((ax >> 13) & 1u)) >> 13) - (112u << 10)));   /* a carry out of 0x7BFF is the inf encoding */
    if (ax <= 0x33000000u) return sign;                                         /* <= 2^-25: the tie at 2^-25 goes to the even 0 */
    const uint32_t m = (ax & 0x7FFFFFu) | 0x800000u, shift = 126u - (ax >> 23);  /* units of 2^-24: m * 2^(e - 126) */
    uint32_t r = m >> shift;
    const uint32_t rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1u);
    if (rem > half || (rem == half && (r & 1u))) r++;                           /* may reach 0x400, the smallest normal */
    return (uint16_t)(sign | r);
}
API void qo_f32_to_f16(const float* in, uint64_t n, uint16_t* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = f32_to_f16_bits(in[i]);
}

/* `x as u8` (Rust's saturating float -> int cast): NaN -> 0, truncate toward zero, clamp to 0..255 */
API void qo_f32_to_u8(const float* in, uint64_t n, uint8_t* out) {
    for (uint64_t i = 0; i < n; i++) {
        const float x = in[i];
        out[i] = (x != x || x <= 0.0f) ? 0 : (x >= 255.0f ? 255 : (uint8_t)x);
    }
}

/* ------------------------------------------------------------------------------------------------
 * Custom queries: Query::score_by over the similarities of one stored vector to the example vectors
 *   lib/common/common/src/math.rs:7-18                      fast_sigmoid, scaled_fast_sigmoid
 *   vector_storage/query/reco_query.rs:64-90                RecoBestScoreQuery
 *   vector_storage/query/reco_query.rs:116-133              RecoSumScoresQuery
 *   vector_storage/query/discover_query.rs:16-25,44-50,66-76 DiscoverQuery (rank_by + sigmoid of the target)
 *   vector_storage/query/context_query.rs:52-62,111-119     ContextQuery (loss_by, MARGIN = f32::EPSILON)
 * kinds: 1 reco best score, 2 reco sum scores, 3 discover, 4 context.  sims layout as in include/qb200.h.
 * ------------------------------------------------------------------------------------------------ */
static inline int f32_total_cmp(float a, float b) { /* f32::total_cmp */
    int32_t x, y;
    memcpy(&x, &a, 4);
    memcpy(&y, &b, 4);
    x ^= (int32_t)(((uint32_t)(x >> 31)) >> 1);
    y ^= (int32_t)(((uint32_t)(y >> 31)) >> 1);
    return (x > y) - (x < y);
}
API float qo_fast_sigmoid(float x) { return x / (1.0f + fabsf(x)); }
API float qo_scaled_fast_sigmoid(float x) { return 0.5f * (qo_fast_sigmoid(x) + 1.0f); }

API float qo_custom_score(int kind, uint32_t n_a, uint32_t n_b, const float* sims, uint64_t stride) {
    if (kind == 1) {
        float max_p = -INFINITY, max_n = -INFINITY;
        for (uint32_t e = 0; e < n_a; e++) { float s = sims[e * stride]; if (f32_total_cmp(s, max_p) > 0) max_p = s; }
        for (uint32_t e = 0; e < n_b; e++) { float s = sims[(n_a + e) * stride]; if (f32_total_cmp(s, max_n) > 0) max_n = s; }
        return (max_p > max_n) ? qo_scaled_fast_sigmoid(max_p) : -qo_scaled_fast_sigmoid(max_n);
    } else if (kind == 2) {
        float p = 0.0f, n = 0.0f;
        for (uint32_t e = 0; e < n_a; e++) p += sims[e * stride];
        for (uint32_t e = 0; e < n_b; e++) n += sims[(n_a + e) * stride];
        return p - n;
    } else if (kind == 3) {
        int32_t rank = 0;
        for (uint32_t e = 0; e < n_a; e++) rank += f32_total_cmp(sims[(1 + 2 * e) * stride], sims[(2 + 2 * e) * stride]);
        return (float)rank + qo_scaled_fast_sigmoid(sims[0]);
    } else {
        float sum = 0.0f;
        for (uint32_t e = 0; e < n_a; e++) {
            float difference = sims[(2 * e) * stride] - sims[(2 * e + 1) * stride] - FLT_EPSILON;
            sum += qo_fast_sigmoid(fminf(difference, 0.0f));
        }
        return sum;
    }
}
/* FeedbackQuery::score_by, vector_storage/query/feedback_query.rs:204-226: sims = [target, pos0, neg0, pos1, neg1, ...] */
API float qo_feedback_score(uint32_t n_pairs, float a, const float* partial, const float* sims, uint64_t stride) {
    float score = a * sims[0];
    for (uint32_t e = 0; e < n_pairs; e++) {
        float delta = sims[(1 + 2 * e) * stride] - sims[(2 + 2 * e) * stride];
        score += partial[e] * delta;      /* -ffp-contract=off: product rounded, then added, like rustc */
    }
    return score;
}
/* NaiveFeedbackCoefficients::extract_context_pairs (feedback_query.rs:114-146) with margin 0: every ordered pair (i, j), i != j, in
 * itertools' permutations(2) order, whose score difference exceeds the margin; partial = confidence^b * c.  Returns the pair count. */
API uint32_t qo_feedback_pairs(const float* scores, uint32_t n, float b, float c, uint32_t* pos, uint32_t* neg, float* partial) {
    uint32_t k = 0;
    if (n < 2) return 0;
    for (uint32_t i = 0; i < n; i++)
        for (uint32_t j = 0; j < n; j++) {
            if (i == j) continue;
            float confidence = scores[i] - scores[j];
            if (confidence <= 0.0f) continue;
            pos[k] = i; neg[k] = j; partial[k] = powf(confidence, b) * c; k++;
        }
    return k;
}
/* sims: [examples][stride], one column per candidate */
API void qo_custom_combine(int kind, uint32_t n_a, uint32_t n_b, const float* sims, uint64_t stride, uint64_t n, float* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = qo_custom_score(kind, n_a, n_b, sims + i, stride);
}

/* ------------------------------------------------------------------------------------------------
 * Multivector MaxSim: score_max_similarity, vector_storage/query_scorer/mod.rs:77-98.
 * a = the query's vectors (na x dim), b = the stored point's vectors (nb x dim), both already preprocessed.
 * ------------------------------------------------------------------------------------------------ */
API float qo_maxsim_f32(int distance, const float* a, uint32_t na, const float* b, uint32_t nb, uint32_t dim) {
    float sum = 0.0f;
    for (uint32_t i = 0; i < na; i++) {
        float max_sim = -INFINITY;
        for (uint32_t j = 0; j < nb; j++) {
            float sim = qo_similarity_f32(distance, a + (size_t)i * dim, b + (size_t)j * dim, dim);
            if (sim > max_sim) max_sim = sim;
        }
        sum += max_sim;
    }
    return sum;
}
/* the same fold over precomputed similarities (quantized storages): sims[q * stride + row], point p = rows [off[p], off[p+1]) */
API void qo_maxsim_fold(const float* sims, uint64_t stride, uint32_t n_query, const uint32_t* off, uint64_t n_points, float* out) {
    for (uint64_t p = 0; p < n_points; p++) {
        float sum = 0.0f;
        for (uint32_t q = 0; q < n_query; q++) {
            float max_sim = -INFINITY;
            for (uint32_t r = off[p]; r < off[p + 1]; r++) { float sim = sims[(uint64_t)q * stride + r]; if (sim > max_sim) max_sim = sim; }
            sum += max_sim;
        }
        out[p] = sum;
    }
}
