// qb_dtype.cu — dense metrics for the Float16 and Uint8 storage datatypes.
//
// Replaces Metric<f16>::similarity (lib/segment/src/spaces/metric_f16/: avx/{dot,euclid,manhattan}.rs,
// sse/*.rs, simple_*.rs) and Metric<u8>::similarity (lib/segment/src/spaces/metric_uint/: avx2/*.rs, sse2/*.rs,
// simple_*.rs) as dispatched on an AVX2+FMA+F16C host.
//
// f16, dim >= 32 : same 4x8 partial-sum layout as f32 (cvtph_ps + fmadd), but the final reduction is
//                  hsum(P0)+hsum(P1)+hsum(P2)+hsum(P3), left-associated (metric_f16/avx/dot.rs:59-62).
// f16, dim <  32 : converted to f32, then the f32 SSE / scalar arithmetic (metric_f16/sse/dot.rs:10-17).
// u8             : qbs::u8_score_avx_group8 (dim >= 32, madd_epi16 pairs, metric_uint/avx2/dot.rs:9-69) and
//                  qbs::u8_score_small (dim < 32, integer-exact) in qb_score.cuh, which the HNSW traversal calls too.
#include <cuda_fp16.h>

#include "qb_internal.h"
#include "qb_score.cuh"   // the u8 chains (u8_score_avx_group8, u8_score_small), shared with the HNSW traversal

using namespace qbs;

namespace {

struct XParams {
    const uint8_t* rows;
    uint32_t stride, dim;
    uint64_t begin, end;
    const uint32_t* ids;
    const uint8_t* q;       // [nq][stride] queries in the storage datatype
    uint32_t nq;
    float* scores;
    int emit_mode;
    int metric;
};

// ---------------------------------------------------------------- f16
__device__ __forceinline__ float f16_step(int metric, float q, float v, float acc) {
    if (metric == M_DOT) return __fmaf_rn(q, v, acc);
    const float d = __fsub_rn(q, v);
    if (metric == M_EUCLID) return __fmaf_rn(d, d, acc);
    return __fadd_rn(fabsf(d), acc);
}
__device__ __forceinline__ float f16_tail(int metric, float q, float v, float r) {
    if (metric == M_DOT) return __fadd_rn(r, __fmul_rn(q, v));
    const float d = __fsub_rn(q, v);
    if (metric == M_EUCLID) return __fadd_rn(r, __fmul_rn(d, d));
    return __fadd_rn(r, fabsf(d));
}

__device__ __forceinline__ float f16_score_avx_group8(int metric, const __half* __restrict__ row, const __half* __restrict__ qry, uint32_t dim, int t) {
    const uint32_t nblk = dim >> 5;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (uint32_t b = 0; b < nblk; ++b) {
        const uint2 vr = *reinterpret_cast<const uint2*>(row + b * 32 + 4 * t);
        const uint2 qr = *reinterpret_cast<const uint2*>(qry + b * 32 + 4 * t);
        const __half2 v01 = *reinterpret_cast<const __half2*>(&vr.x), v23 = *reinterpret_cast<const __half2*>(&vr.y);
        const __half2 q01 = *reinterpret_cast<const __half2*>(&qr.x), q23 = *reinterpret_cast<const __half2*>(&qr.y);
        a0 = f16_step(metric, __low2float(q01), __low2float(v01), a0);
        a1 = f16_step(metric, __high2float(q01), __high2float(v01), a1);
        a2 = f16_step(metric, __low2float(q23), __low2float(v23), a2);
        a3 = f16_step(metric, __high2float(q23), __high2float(v23), a3);
    }
    // hsum256_ps_avx of accumulator a = t/2: lr[i] = P[i+4] + P[i] (lanes t and t^1), then (lr0+lr1)+(lr2+lr3)
    a0 = __fadd_rn(a0, __shfl_xor_sync(0xFFFFFFFFu, a0, 1));
    a1 = __fadd_rn(a1, __shfl_xor_sync(0xFFFFFFFFu, a1, 1));
    a2 = __fadd_rn(a2, __shfl_xor_sync(0xFFFFFFFFu, a2, 1));
    a3 = __fadd_rn(a3, __shfl_xor_sync(0xFFFFFFFFu, a3, 1));
    const float h = __fadd_rn(__fadd_rn(a0, a1), __fadd_rn(a2, a3));
    const int base = (threadIdx.x & 31) & ~7;
    const float h0 = __shfl_sync(0xFFFFFFFFu, h, base + 0), h1 = __shfl_sync(0xFFFFFFFFu, h, base + 2);
    const float h2 = __shfl_sync(0xFFFFFFFFu, h, base + 4), h3 = __shfl_sync(0xFFFFFFFFu, h, base + 6);
    float r = __fadd_rn(__fadd_rn(__fadd_rn(h0, h1), h2), h3);
    for (uint32_t i = nblk << 5; i < dim; ++i) r = f16_tail(metric, __half2float(qry[i]), __half2float(row[i]), r);
    return (metric == M_DOT) ? r : -r;
}

__device__ __forceinline__ float f16_score_small(int metric, const __half* __restrict__ row, const __half* __restrict__ qry, uint32_t dim) {
    float r;
    uint32_t start;
    if (dim >= 16) {
        float p[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const float q = __half2float(qry[i]), v = __half2float(row[i]);
            if (metric == M_DOT) p[i] = __fadd_rn(__fmul_rn(q, v), 0.0f);
            else {
                const float d = __fsub_rn(q, v);
                p[i] = (metric == M_EUCLID) ? __fadd_rn(__fmul_rn(d, d), 0.0f) : __fadd_rn(fabsf(d), 0.0f);
            }
        }
        float h[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) h[a] = __fadd_rn(__fadd_rn(p[4 * a], p[4 * a + 2]), __fadd_rn(p[4 * a + 1], p[4 * a + 3]));
        r = __fadd_rn(__fadd_rn(__fadd_rn(h[0], h[1]), h[2]), h[3]);
        start = 16;
    } else {
        r = -0.0f;
        start = 0;
    }
    for (uint32_t i = start; i < dim; ++i) r = f16_tail(metric, __half2float(qry[i]), __half2float(row[i]), r);
    return (metric == M_DOT) ? r : -r;
}

template <bool IS_F16>
__global__ void __launch_bounds__(256) dense_x_group_kernel(const XParams p, const QbEmit emit) {
    const int t = threadIdx.x & 7;
    const uint64_t groups_per_grid = (uint64_t)gridDim.x * (blockDim.x >> 3);
    const uint64_t g0 = (uint64_t)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3);
    const uint64_t n = p.end - p.begin;
    const uint64_t n_iter = (n + groups_per_grid - 1) / groups_per_grid;
    for (uint64_t it = 0; it < n_iter; ++it) {
        const uint64_t ci = g0 + it * groups_per_grid;
        const bool valid = ci < n;
        const uint64_t cand = p.begin + (valid ? ci : 0);
        const uint32_t row = p.ids ? p.ids[cand] : (uint32_t)cand;
        const uint8_t* rp = p.rows + (size_t)row * p.stride;
        for (uint32_t q = 0; q < p.nq; ++q) {
            const uint8_t* qp = p.q + (size_t)q * p.stride;
            float sc;
            if (IS_F16) {
                const int m = (p.metric == M_COSINE) ? M_DOT : p.metric;
                sc = (p.dim >= 32) ? f16_score_avx_group8(m, reinterpret_cast<const __half*>(rp), reinterpret_cast<const __half*>(qp), p.dim, t)
                                   : f16_score_small(m, reinterpret_cast<const __half*>(rp), reinterpret_cast<const __half*>(qp), p.dim);
            } else {
                sc = (p.dim >= 32) ? u8_score_avx_group8(p.metric, rp, qp, p.dim, t) : u8_score_small(p.metric, rp, qp, p.dim);
            }
            if (valid && t == 0) {
                if (p.emit_mode) qb_emit(emit, q, cand, row, sc);
                else p.scores[(size_t)q * n + ci] = sc;
            }
        }
    }
}

// f32 (preprocessed) -> storage datatype: f16::from_f32 (RNE) / `x as u8` (saturating, truncating, NaN -> 0)
__global__ void convert_queries_kernel(const float* __restrict__ q_pre, uint32_t q_stride_f, uint32_t dim, uint32_t nq, int is_f16, uint8_t* __restrict__ out,
                                       uint32_t out_stride) {
    const uint32_t q = blockIdx.x;
    const float* src = q_pre + (size_t)q * q_stride_f;
    uint8_t* dst = out + (size_t)q * out_stride;
    const uint32_t n_el = is_f16 ? out_stride / 2 : out_stride;
    for (uint32_t i = threadIdx.x; i < n_el; i += blockDim.x) {
        const float x = (i < dim) ? src[i] : 0.0f;
        if (is_f16) reinterpret_cast<__half*>(dst)[i] = __float2half_rn(x);
        else {
            unsigned int u = (x != x) ? 0u : __float2uint_rz(x);
            dst[i] = (uint8_t)(u > 255u ? 255u : u);
        }
    }
}

int metric_code(const qb_storage* s) {
    switch (s->distance) {
        case QB_DIST_EUCLID: return M_EUCLID;
        case QB_DIST_MANHATTAN: return M_MANHATTAN;
        case QB_DIST_COSINE: return M_COSINE;
        default: return M_DOT;
    }
}

qb_status launch_x(const qb_storage* s, XParams& p, const QbEmit& e, cudaStream_t stream) {
    const uint64_t n = p.end - p.begin;
    if (n == 0 || p.nq == 0) return QB_OK;
    p.rows = reinterpret_cast<const uint8_t*>(s->d_rows); p.stride = s->row_stride; p.dim = s->dim; p.metric = metric_code(s);
    uint64_t blocks = ceil_div_u64(n, 256 / 8);
    const uint64_t maxb = (uint64_t)s->sm_count * 8;
    if (blocks > maxb) blocks = maxb;
    if (s->dtype == QB_DT_F16) dense_x_group_kernel<true><<<(unsigned)blocks, 256, 0, stream>>>(p, e);
    else dense_x_group_kernel<false><<<(unsigned)blocks, 256, 0, stream>>>(p, e);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

}  // namespace

qb_status qb_dense_x_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream) {
    XParams p{};
    p.begin = a.row_begin; p.end = a.row_end; p.ids = a.d_ids;
    p.q = reinterpret_cast<const uint8_t*>(a.d_q_enc); p.nq = a.nq; p.scores = nullptr; p.emit_mode = 1;
    return launch_x(s, p, a.emit, stream);
}

qb_status qb_dense_x_score_points(const qb_storage* s, const void* d_q_enc, const uint32_t* d_ids, uint64_t n, float* d_scores, cudaStream_t stream) {
    XParams p{};
    p.begin = 0; p.end = n; p.ids = d_ids;
    p.q = reinterpret_cast<const uint8_t*>(d_q_enc); p.nq = 1; p.scores = d_scores; p.emit_mode = 0;
    QbEmit e{};
    return launch_x(s, p, e, stream);
}

qb_status qb_dense_x_convert_queries(const qb_storage* s, const float* d_q_pre, uint32_t q_stride_f, uint32_t nq, void* d_out, cudaStream_t stream) {
    if (nq == 0) return QB_OK;
    convert_queries_kernel<<<nq, 256, 0, stream>>>(d_q_pre, q_stride_f, s->dim, nq, s->dtype == QB_DT_F16 ? 1 : 0, reinterpret_cast<uint8_t*>(d_out),
                                                   s->row_stride);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}
