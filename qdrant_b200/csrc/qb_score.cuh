// qb_score.cuh — device-side per-pair scoring primitives shared by the scan / gather kernels (qb_dense.cu, qb_quant.cu) and the
// device-resident HNSW traversal (qb_hnsw.cu).  Each function restates one reference routine with its accumulation order; see the
// headers of qb_dense.cu / qb_quant.cu for the bit-exactness argument and the reference citations.
#pragma once
#include "qb_common.cuh"

namespace qbs {

// M_COSINE: Uint8 storages only (their cosine is its own chain); f32 cosine rows are normalised and scored with M_DOT
enum { M_DOT = 0, M_EUCLID = 1, M_MANHATTAN = 2, M_COSINE = 3 };

__device__ __forceinline__ float4 shfl_xor4(float4 v, int m) {
    v.x = __shfl_xor_sync(0xFFFFFFFFu, v.x, m);
    v.y = __shfl_xor_sync(0xFFFFFFFFu, v.y, m);
    v.z = __shfl_xor_sync(0xFFFFFFFFu, v.z, m);
    v.w = __shfl_xor_sync(0xFFFFFFFFu, v.w, m);
    return v;
}
__device__ __forceinline__ float4 add4(float4 a, float4 b) {
    return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}

template <int METRIC>
__device__ __forceinline__ float elem_step(float q, float v, float acc) {
    if (METRIC == M_DOT) return __fmaf_rn(q, v, acc);
    float d = __fsub_rn(q, v);
    if (METRIC == M_EUCLID) return __fmaf_rn(d, d, acc);
    return __fadd_rn(fabsf(d), acc);
}
template <int METRIC>
__device__ __forceinline__ float tail_step(float q, float v, float r) {
    if (METRIC == M_DOT) return __fadd_rn(r, __fmul_rn(q, v));
    float d = __fsub_rn(q, v);
    if (METRIC == M_EUCLID) return __fadd_rn(r, __fmul_rn(d, d));
    return __fadd_rn(r, fabsf(d));
}

// AVX tier (dim >= 32).  `row` and `qry` are 16-B aligned; t = lane & 7.  All 8 lanes of the group return r.
template <int METRIC>
__device__ __forceinline__ float score_avx_group8(const float* __restrict__ row, const float* __restrict__ qry, uint32_t dim, int t) {
    const uint32_t nblk = dim >> 5;
    const float4* r4 = reinterpret_cast<const float4*>(row) + t;
    const float4* q4 = reinterpret_cast<const float4*>(qry) + t;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
    for (uint32_t b = 0; b < nblk; ++b) {
        float4 v = r4[b * 8];
        float4 q = q4[b * 8];
        acc.x = elem_step<METRIC>(q.x, v.x, acc.x);
        acc.y = elem_step<METRIC>(q.y, v.y, acc.y);
        acc.z = elem_step<METRIC>(q.z, v.z, acc.z);
        acc.w = elem_step<METRIC>(q.w, v.w, acc.w);
    }
    acc = add4(acc, shfl_xor4(acc, 2));  // (P0+P1), (P2+P3)        four_way_hsum, simple_avx.rs:21-28
    acc = add4(acc, shfl_xor4(acc, 4));  // (P0+P1)+(P2+P3) = T[l]
    acc = add4(acc, shfl_xor4(acc, 1));  // T[i+4]+T[i] = L[i]       hsum256_ps_avx, simple_avx.rs:10-16
    float r = __fadd_rn(__fadd_rn(acc.x, acc.y), __fadd_rn(acc.z, acc.w));
    for (uint32_t i = nblk << 5; i < dim; ++i) r = tail_step<METRIC>(qry[i], row[i], r);
    return (METRIC == M_DOT) ? r : -r;
}

// NQ queries against ONE row: the row's float4 of every 32-block is loaded once and FMA-ed into NQ independent accumulator sets, so a
// batch (or the examples of a custom query) costs one pass over the rows and one row read from shared memory instead of NQ.  Each
// (query, lane) chain is the very chain score_avx_group8 runs, so every result is bit-identical to the single-query function.
// qry + q * q_stride_f = query q (16-B aligned).
template <int METRIC, int NQ>
__device__ __forceinline__ void score_avx_group8_multi(const float* __restrict__ row, const float* __restrict__ qry, uint32_t q_stride_f, uint32_t dim, int t,
                                                       float (&out)[NQ]) {
    const uint32_t nblk = dim >> 5;
    const float4* r4 = reinterpret_cast<const float4*>(row) + t;
    float4 acc[NQ];
#pragma unroll
    for (int q = 0; q < NQ; ++q) acc[q] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 2
    for (uint32_t b = 0; b < nblk; ++b) {
        const float4 v = r4[b * 8];
#pragma unroll
        for (int q = 0; q < NQ; ++q) {
            const float4 w = (reinterpret_cast<const float4*>(qry + (size_t)q * q_stride_f) + t)[b * 8];
            acc[q].x = elem_step<METRIC>(w.x, v.x, acc[q].x);
            acc[q].y = elem_step<METRIC>(w.y, v.y, acc[q].y);
            acc[q].z = elem_step<METRIC>(w.z, v.z, acc[q].z);
            acc[q].w = elem_step<METRIC>(w.w, v.w, acc[q].w);
        }
    }
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
        float4 a = acc[q];
        a = add4(a, shfl_xor4(a, 2));
        a = add4(a, shfl_xor4(a, 4));
        a = add4(a, shfl_xor4(a, 1));
        float r = __fadd_rn(__fadd_rn(a.x, a.y), __fadd_rn(a.z, a.w));
        const float* qq = qry + (size_t)q * q_stride_f;
        for (uint32_t i = nblk << 5; i < dim; ++i) r = tail_step<METRIC>(qq[i], row[i], r);
        out[q] = (METRIC == M_DOT) ? r : -r;
    }
}

// SSE tier (16 <= dim < 32, one 16-block, unfused mul+add) and scalar tier (dim < 16); one thread per pair.
template <int METRIC>
__device__ __forceinline__ float score_small(const float* __restrict__ row, const float* __restrict__ qry, uint32_t dim) {
    float r;
    uint32_t start;
    if (dim >= 16) {
        float p[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            float q = qry[i], v = row[i];
            if (METRIC == M_DOT) p[i] = __fadd_rn(__fmul_rn(q, v), 0.0f);
            else {
                float d = __fsub_rn(q, v);
                p[i] = (METRIC == M_EUCLID) ? __fadd_rn(__fmul_rn(d, d), 0.0f) : __fadd_rn(fabsf(d), 0.0f);
            }
        }
        float h[4];
#pragma unroll
        for (int a = 0; a < 4; ++a)  // hsum128_ps_sse: (x0+x2)+(x1+x3), simple_sse.rs:13-17
            h[a] = __fadd_rn(__fadd_rn(p[4 * a], p[4 * a + 2]), __fadd_rn(p[4 * a + 1], p[4 * a + 3]));
        r = __fadd_rn(__fadd_rn(__fadd_rn(h[0], h[1]), h[2]), h[3]);
        start = 16;
    } else {
        r = -0.0f;  // Rust's f32 Sum folds from -0.0
        start = 0;
    }
    for (uint32_t i = start; i < dim; ++i) r = tail_step<METRIC>(qry[i], row[i], r);
    return (METRIC == M_DOT) ? r : -r;
}

// Uint8 storages (Metric<u8>::similarity, metric_uint/avx2/*.rs, simple_*.rs), shared by the scan (qb_dtype.cu) and the HNSW
// traversal.  dim >= 32: eight i32 lanes, lane i sums bytes 4i..4i+3 of every 32-B block; manhattan uses sad_epu8 (even lanes =
// 8-byte sums, odd = 0); the lanes are converted to f32 and added with hsum256_ps_avx; the n % 32 tail is an integer sum converted
// once.  GPU lane t of an 8-lane group IS AVX lane t.  dim < 32: integer-exact totals.  Rows and query are 4-B aligned.
__device__ __forceinline__ float hsum8(float f) {  // hsum256_ps_avx over the 8 lanes of a group
    f = __fadd_rn(f, __shfl_xor_sync(0xFFFFFFFFu, f, 4));  // lr[i] = f[i+4] + f[i]
    f = __fadd_rn(f, __shfl_xor_sync(0xFFFFFFFFu, f, 1));  // lr0+lr1 | lr2+lr3
    f = __fadd_rn(f, __shfl_xor_sync(0xFFFFFFFFu, f, 2));
    return f;
}

__device__ __forceinline__ float u8_score_avx_group8(int metric, const uint8_t* __restrict__ row, const uint8_t* __restrict__ qry, uint32_t dim, int t) {
    const uint32_t nblk = dim >> 5;
    unsigned int acc = 0, n1 = 0, n2 = 0;
    for (uint32_t b = 0; b < nblk; ++b) {
        const unsigned int v = *reinterpret_cast<const unsigned int*>(row + b * 32 + 4 * t);
        const unsigned int q = *reinterpret_cast<const unsigned int*>(qry + b * 32 + 4 * t);
        if (metric == M_DOT) acc = __dp4a(q, v, acc);
        else if (metric == M_COSINE) { acc = __dp4a(q, v, acc); n1 = __dp4a(q, q, n1); n2 = __dp4a(v, v, n2); }
        else if (metric == M_EUCLID) { const unsigned int d = __vabsdiffu4(q, v); acc = __dp4a(d, d, acc); }
        else acc += __vsadu4(q, v);
    }
    if (metric == M_MANHATTAN) {  // sad_epu8: even lanes hold 8-byte sums, odd lanes 0 (avx2/manhattan.rs:33-35)
        const unsigned int pair = acc + __shfl_xor_sync(0xFFFFFFFFu, acc, 1);
        acc = (t & 1) ? 0u : pair;
    }
    float score = hsum8((float)(int)acc);
    float f1 = 0.f, f2 = 0.f;
    if (metric == M_COSINE) { f1 = hsum8((float)(int)n1); f2 = hsum8((float)(int)n2); }
    const uint32_t rem0 = nblk << 5;
    if (rem0 < dim) {
        int rd = 0, r1 = 0, r2 = 0;
        for (uint32_t i = rem0; i < dim; ++i) {
            const int x = qry[i], y = row[i];
            if (metric == M_DOT) rd += x * y;
            else if (metric == M_COSINE) { rd += x * y; r1 += x * x; r2 += y * y; }
            else if (metric == M_EUCLID) rd += (x - y) * (x - y);
            else rd += abs(x - y);
        }
        score = __fadd_rn(score, (float)rd);
        if (metric == M_COSINE) { f1 = __fadd_rn(f1, (float)r1); f2 = __fadd_rn(f2, (float)r2); }
    }
    if (metric == M_DOT) return score;
    if (metric == M_COSINE) {  // avx2/cosine.rs:97-104
        const float denom = __fmul_rn(f1, f2);
        if (denom == 0.0f) return 0.0f;
        return __fdiv_rn(score, __fsqrt_rn(denom));
    }
    return -score;
}

__device__ __forceinline__ float u8_score_small(int metric, const uint8_t* __restrict__ row, const uint8_t* __restrict__ qry, uint32_t dim) {
    int rd = 0, r1 = 0, r2 = 0;
    for (uint32_t i = 0; i < dim; ++i) {
        const int x = qry[i], y = row[i];
        if (metric == M_DOT) rd += x * y;
        else if (metric == M_COSINE) { rd += x * y; r1 += x * x; r2 += y * y; }
        else if (metric == M_EUCLID) rd += (x - y) * (x - y);
        else rd += abs(x - y);
    }
    if (metric == M_DOT) return (float)rd;
    if (metric == M_COSINE) {
        const float denom = __fmul_rn((float)r1, (float)r2);
        if (denom == 0.0f) return 0.0f;
        return __fdiv_rn((float)rd, __fsqrt_rn(denom));
    }
    return -(float)rd;
}

// SQ8 (EncodedVectorsU8): raw integer score of one stored code row against one query code, 8 lanes per row, 16 B per lane per
// step; every lane of the group returns the value.  l1 = Manhattan on codes (impl_score_l1_avx, cpp/avx2.c:65-122); LANEX =
// the 8-lane partition + HSUM256_PS tree of impl_score_dot_avx (cpp/avx2.c:7-63) for totals that can leave the f32-exact window.
// ld(c) returns the row's 16-B chunk c: sq8_raw_group8 reads an aligned stored row, the HNSW inline-vector search (qb_hnsw_inline.cu)
// a link vector at any byte address; the arithmetic on the chunks is the same.
template <bool LANEX, class LD>
__device__ __forceinline__ float sq8_raw_group8_ld(LD ld, const uint4* __restrict__ qp, uint32_t n_chunks, int t, int l1) {
    float score;
    if (l1) {
        unsigned int acc = 0;
        for (uint32_t c = t; c < n_chunks; c += 8) {
            uint4 v = ld(c), w = qp[c];
            acc += __vsadu4(v.x, w.x) + __vsadu4(v.y, w.y) + __vsadu4(v.z, w.z) + __vsadu4(v.w, w.w);
        }
        acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 1);
        acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 2);
        acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 4);
        score = (float)acc;  // impl_score_l1_avx returns (float)sum, cpp/avx2.c:117-121
    } else if (!LANEX) {
        int acc = 0;
        for (uint32_t c = t; c < n_chunks; c += 8) {
            uint4 v = ld(c), w = qp[c];
            acc = __dp4a((int)v.x, (int)w.x, acc);
            acc = __dp4a((int)v.y, (int)w.y, acc);
            acc = __dp4a((int)v.z, (int)w.z, acc);
            acc = __dp4a((int)v.w, (int)w.w, acc);
        }
        acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 1);
        acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 2);
        acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 4);
        score = (float)acc;  // exact: total < 2^24
    } else {
        // lane partition of impl_score_dot_avx: byte pair j of every 16-B chunk accumulates into i32 lane j
        int ln[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (uint32_t c = t; c < n_chunks; c += 8) {
            uint4 v = ld(c), w = qp[c];
            ln[0] = __dp4a((int)v.x, (int)(w.x & 0x0000FFFFu), ln[0]); ln[1] = __dp4a((int)v.x, (int)(w.x & 0xFFFF0000u), ln[1]);
            ln[2] = __dp4a((int)v.y, (int)(w.y & 0x0000FFFFu), ln[2]); ln[3] = __dp4a((int)v.y, (int)(w.y & 0xFFFF0000u), ln[3]);
            ln[4] = __dp4a((int)v.z, (int)(w.z & 0x0000FFFFu), ln[4]); ln[5] = __dp4a((int)v.z, (int)(w.z & 0xFFFF0000u), ln[5]);
            ln[6] = __dp4a((int)v.w, (int)(w.w & 0x0000FFFFu), ln[6]); ln[7] = __dp4a((int)v.w, (int)(w.w & 0xFFFF0000u), ln[7]);
        }
#pragma unroll
        for (int l = 0; l < 8; ++l) {
            ln[l] += __shfl_xor_sync(0xFFFFFFFFu, ln[l], 1);
            ln[l] += __shfl_xor_sync(0xFFFFFFFFu, ln[l], 2);
            ln[l] += __shfl_xor_sync(0xFFFFFFFFu, ln[l], 4);
        }
        // HSUM256_PS (cpp/avx2.c:7-14): ((l0+l4)+(l2+l6)) + ((l1+l5)+(l3+l7))
        float x0 = __fadd_rn((float)ln[4], (float)ln[0]), x1 = __fadd_rn((float)ln[5], (float)ln[1]);
        float x2 = __fadd_rn((float)ln[6], (float)ln[2]), x3 = __fadd_rn((float)ln[7], (float)ln[3]);
        score = __fadd_rn(__fadd_rn(x0, x2), __fadd_rn(x1, x3));
    }
    return score;
}
template <bool LANEX>
__device__ __forceinline__ float sq8_raw_group8(const uint4* __restrict__ rp, const uint4* __restrict__ qp, uint32_t n_chunks, int t, int l1) {
    return sq8_raw_group8_ld<LANEX>([rp](uint32_t c) { return __ldg(rp + c); }, qp, n_chunks, t, l1);
}

}  // namespace qbs
