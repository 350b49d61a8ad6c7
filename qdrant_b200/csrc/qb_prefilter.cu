// qb_prefilter.cu — single-query dense f32 (dot / cosine) scans at a fraction of the HBM bytes, results unchanged.
// (The default plane is the 6-bit one further down; the bf16 plane described first is the simplest case of the same scheme.)
//
// The single-query scan of qb_dense.cu runs at the HBM copy rate: every query reads dim * 4 bytes per row.  The only way to more
// queries per second is fewer bytes per row — and the scan only has to FIND the rows whose exact score can reach the top-k; it does
// not have to produce their scores.  With a bf16 shadow plane of the rows (RN-even, the same plane the batched tensor-core path of
// qb_sq8_mma.cu keeps) and the query kept in f32:
//     | sum_i q_i bf16(x_i) - sum_i q_i x_i |  <=  2^-9 ||q|| ||x||            (Cauchy-Schwarz on the element-wise rounding errors)
//   + f32 evaluation of either sum, any order:  <=  dim 2^-24 ||q|| ||x|| each
//   =>  |approx - exact|  <=  eps_q := (2^-9 + dim 2^-22) ||q|| max_rows ||x||  (1 + 2^-10)
// Four launches per query, no host synchronisation (the 6-bit plane below takes its sample in its own first stage instead of step 1):
//   1. the EXACT in-kernel-top-k scan (dense_f32_stream_kernel<., LOCALK>) over a prefix of the rows (1/64 of them, 2^14..2^17) -> thr_q = the k-th best exact score
//      of the sample (a lower bound of the final k-th score);
//   2. dense_bf16_filter_kernel: the whole bf16 plane streams through the same TMA-bulk ring (dim * 2 bytes per row); the query sits in
//      REGISTERS (a lane always meets the same dimensions); rows with approx >= thr_q - eps_q are appended to a candidate list — a
//      superset of the rows whose exact score reaches thr_q, hence of the true top-k;
//   3. f32_prefilter_finish_kernel: exact AVX-order scores of the candidates (one CTA per SM, each keeping its own top-k), the top-k of
//      those by the usual keys in the last CTA to finish;
//   4. if the list overflowed (mass ties, a NaN query, a sample without k live rows), step 3 raises a device flag and the exact scan of
//      the whole storage — always enqueued, it exits at once while the flag is down — produces the answer instead.
// (RawScorer results are bit-identical to the exact path: tests/test_gpu_dense.py::test_single_query_prefilter_*.)
#include <algorithm>

#include "qb_internal.h"
#include "qb_localk.cuh"
#include "qb_score.cuh"

qb_status qb_dense_f32_scan_localk(const qb_storage* s, const QbScanArgs& a, uint32_t top, uint64_t* n_slots, cudaStream_t stream, uint64_t min_rows = 65536);   // qb_dense.cu

namespace {

constexpr int PF_CONSUMER_WARPS = 8;
constexpr int PF_MAX_PRODUCERS = 4;
constexpr int PF_PRODUCERS = 2;             // producer warps (one lane each): a bulk copy costs its issuing thread ~500 clocks (wait for the slot, arm the
                                            // barrier, issue), so ONE producer caps a CTA at one 12-KB slot per ~500 clocks — below the HBM rate for these planes
constexpr int PF_THREADS = 32 * (PF_CONSUMER_WARPS + PF_MAX_PRODUCERS);     // launch bound; the launch uses 32 * (consumers + producers)
constexpr uint32_t PF_SLOT_BYTES = 12288;  // target bytes per ring slot (a consumer warp holds one slot while the others are in flight)
constexpr uint32_t PF_CAP = 131072;        // candidate rows per query at most (a few thousand to a few tens of thousands expected on 10M rows)
constexpr uint32_t PF_LIST_CAP = 1u << 21; // first-stage rows of the 6-bit plane per query at most (dense_q5_compact_kernel)

static int pf_producers() { const int o = qb_opt().prefilter_producers; return (o >= 1 && o <= PF_MAX_PRODUCERS) ? o : PF_PRODUCERS; }

struct PfParams {
    const uint8_t* rows;        // bf16 plane
    uint32_t stride;            // bytes per row = row_h * 2 (multiple of 16)
    uint32_t row_h;             // halfs per row
    uint32_t dim;
    uint64_t n_rows;
    const float* q;             // preprocessed f32 query
    uint32_t rows_per_slot, n_slots, slot_bytes;
    const qb_scored_point* samp_out; const uint32_t* samp_cnt; uint32_t top;   // exact top-k of the sample prefix
    const unsigned int* max_norm_bits;                                         // max row norm of the storage (f32 bits)
    uint32_t* cand; unsigned int* cnt; uint32_t cap;
    const uint32_t* deleted; const uint32_t* deleted2;
    int l2_keep;
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}

// One producer lane of a filter kernel's ring: tiles blockIdx.x, blockIdx.x + gridDim.x, ... of `rows_per_slot` rows, every n_prod-th one.
// A tile's copy is rounded up to 16 bytes; planes whose stride is not a multiple of 16 keep that much padding behind their last row.
template <typename P>
__device__ __forceinline__ void pf_produce(const P& p, uint8_t* slots, uint64_t* full, uint64_t* empty, int warp, int n_prod, uint64_t n_local) {
    const uint64_t policy = p.l2_keep ? qb_policy_evict_last() : qb_policy_evict_first();
    // slot / phase / first row advance incrementally: 64-bit divisions in this loop cost more than the copy they issue
    uint32_t s = (uint32_t)warp, ph = 0;                 // n_slots is a multiple of 8, n_prod of 1 / 2 / 4: s wraps exactly
    uint64_t r0 = ((uint64_t)blockIdx.x + (uint64_t)warp * gridDim.x) * p.rows_per_slot;
    const uint64_t r_step = (uint64_t)n_prod * gridDim.x * p.rows_per_slot;
    for (uint64_t i = warp; i < n_local; i += n_prod, r0 += r_step) {
        qb_mbar_wait(&empty[s], ph ^ 1u);
        const uint64_t left = p.n_rows - r0;
        const uint32_t nr = (uint32_t)(left < p.rows_per_slot ? left : p.rows_per_slot);
        const uint32_t bytes = (nr * p.stride + 15u) & ~15u;
        qb_mbar_arrive_expect_tx(&full[s], bytes);
        qb_bulk_g2s(slots + (size_t)s * p.slot_bytes, p.rows + r0 * p.stride, bytes, &full[s], policy);
        s += (uint32_t)n_prod;
        if (s >= p.n_slots) { s -= p.n_slots; ph ^= 1u; }
    }
}

// NCH = 16-byte chunks of a row per lane (row_h <= NCH * 256)
template <int NCH>
__global__ void __launch_bounds__(PF_THREADS, 1) dense_bf16_filter_kernel(const PfParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* slots = smem;
    uint64_t* full = reinterpret_cast<uint64_t*>(slots + (size_t)p.n_slots * p.slot_bytes);
    uint64_t* empty = full + p.n_slots;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t n_tiles = (p.n_rows + p.rows_per_slot - 1) / p.rows_per_slot;
    const uint64_t n_local = (blockIdx.x < n_tiles) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < p.n_slots; ++s) { qb_mbar_init(&full[s], 1); qb_mbar_init(&empty[s], 1); }
        qb_fence_barrier_init();
    }
    __syncthreads();
    const int n_prod = (int)(blockDim.x >> 5) - PF_CONSUMER_WARPS;
    if (warp < n_prod) {
        if (lane == 0) pf_produce(p, slots, full, empty, warp, n_prod, n_local);
        return;
    }
    const int cw = warp - n_prod;
    // this lane's slice of the query: dimensions [ (c * 32 + lane) * 8, + 8 ) for c < NCH, zero past dim
    float qr[NCH][8];
    uint32_t off[NCH];
    float qq = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const uint32_t d0 = (uint32_t)(c * 32 + lane) * 8;
        off[c] = (d0 < p.row_h) ? d0 * 2 : 0;                  // past the row: any valid address, the query slice is zero
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float v = (d0 < p.row_h && d0 + k < p.dim) ? p.q[d0 + k] : 0.f;
            qr[c][k] = v;
            qq = fmaf(v, v, qq);
        }
    }
    qq = warp_sum(qq);
    // thr_q - eps_q, rounded towards "pass"
    float thr_adj;
    {
        const float qn = __fmul_ru(__fsqrt_ru(qq), 1.0001f);
        const float mx = __uint_as_float(*p.max_norm_bits);
        const float c = __fadd_ru(0x1.004p-9f, __fmul_ru((float)p.dim, 0x1p-22f));       // (2^-9)(1 + 2^-10) + dim 2^-22
        const float eps = __fadd_ru(__fmul_ru(__fmul_ru(qn, mx), c), 1.0e-37f);
        const float thr = (*p.samp_cnt >= p.top) ? p.samp_out[p.top - 1].score : __int_as_float(0xff800000);
        thr_adj = __fsub_rd(thr, eps);                           // NaN query -> NaN: `approx < NaN` is false, every row passes (-> fallback)
    }
    uint32_t s = (uint32_t)cw, ph = 0;                            // as in the producers: no 64-bit division per slot
    uint64_t r0 = ((uint64_t)blockIdx.x + (uint64_t)cw * gridDim.x) * p.rows_per_slot;
    const uint64_t r_step = (uint64_t)PF_CONSUMER_WARPS * gridDim.x * p.rows_per_slot;
    for (uint64_t i = cw; i < n_local; i += PF_CONSUMER_WARPS, r0 += r_step) {
        const uint64_t left = p.n_rows - r0;
        const uint32_t nr = (uint32_t)(left < p.rows_per_slot ? left : p.rows_per_slot);
        qb_mbar_wait(&full[s], ph);
        const uint8_t* slot = slots + (size_t)s * p.slot_bytes;
        for (uint32_t r = 0; r < nr; r += 2) {
            const bool two = r + 1 < nr;
            const uint8_t* ra = slot + (size_t)r * p.stride;
            const uint8_t* rb = slot + (size_t)(two ? r + 1 : r) * p.stride;
            float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
                const uint4 va = *reinterpret_cast<const uint4*>(ra + off[c]);
                const uint4 vb = *reinterpret_cast<const uint4*>(rb + off[c]);
                const uint32_t wa[4] = {va.x, va.y, va.z, va.w}, wb[4] = {vb.x, vb.y, vb.z, vb.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    a0 = fmaf(qr[c][2 * k], __uint_as_float(wa[k] << 16), a0);
                    a1 = fmaf(qr[c][2 * k + 1], __uint_as_float(wa[k] & 0xFFFF0000u), a1);
                    b0 = fmaf(qr[c][2 * k], __uint_as_float(wb[k] << 16), b0);
                    b1 = fmaf(qr[c][2 * k + 1], __uint_as_float(wb[k] & 0xFFFF0000u), b1);
                }
            }
            float sa = a0 + a1, sb = b0 + b1;
            // both sums in one butterfly: lanes < 16 end up with row a, lanes >= 16 with row b
            {
                const float send = (lane & 16) ? sa : sb, keep = (lane & 16) ? sb : sa;
                float v = keep + __shfl_xor_sync(0xFFFFFFFFu, send, 16);
#pragma unroll
                for (int o = 8; o; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
                sa = v;
            }
            if ((lane == 0 || (lane == 16 && two)) && !(sa < thr_adj)) {
                const uint32_t id = (uint32_t)(r0 + r + (lane >> 4));
                bool dead = false;
                if (p.deleted) dead = (p.deleted[id >> 5] >> (id & 31)) & 1u;
                if (p.deleted2) dead = dead || ((p.deleted2[id >> 5] >> (id & 31)) & 1u);
                if (!dead) {
                    const unsigned int pos = atomicAdd(p.cnt, 1u);
                    if (pos < p.cap) p.cand[pos] = id;
                }
            }
        }
        __syncwarp();
        if (lane == 0) qb_mbar_arrive(&empty[s]);
        s += PF_CONSUMER_WARPS;
        if (s >= p.n_slots) { s -= p.n_slots; ph ^= 1u; }
    }
}

// ------------------------------------------------------------------------------------------------ int8 shadow plane (a quarter of the bytes)
// x_i ~ s_r c_i, c_i = rint(x_i / s_r) in [-127, 127], s_r = max_i |x_i| / 127 (one f32 scale per row, stored right behind the row's codes);
// the QUERY is split into two int8 levels, q_i ~ s_q (h_i + l_i / 254), so that its own error is negligible and the scan is integer only:
//   H = sum_i h_i c_i, L = sum_i l_i c_i   (dp4a, exact: dim * 127^2 < 2^24 for dim <= 1040),   approx = s_r s_q (H + L / 254)
//   | exact - approx |  <=  s_r (1/2 + 2^-13) ||q||_1          (row rounding:   |x_i - s_r c_i| <= s_r (1/2 + 1e-4))
//                        +  s_r s_q (127 dim / 508)(1 + 0.08)   (query rounding: |q_i - q^_i| <= s_q (1/508 + 2.3e-5), |c_i| <= 127)
//                        +  slack_q = (dim 2^-22 + 2^-17)(1 + sqrt(dim) / 127) ||q|| max||x||     (every f32 evaluation on either side)
// so a row passes iff  s_r * (s_q (H + L / 254) + E_q) >= thr_q - slack_q  with the per-query constant
// E_q = (1/2 + 2^-13) ||q||_1 + 0.27 s_q dim: one FMA, one multiply and one compare per row after two warp-wide integer sums.
__global__ void __launch_bounds__(256) f32_to_q8_rows_kernel(const float* __restrict__ rows, uint64_t stride_f, uint32_t dim, uint64_t n, int8_t* __restrict__ out,
                                                              uint32_t out_stride_b /* codes + 16: the row's f32 scale follows its codes */, unsigned int* __restrict__ max_norm_bits,
                                                              unsigned int* __restrict__ nonfinite) {
    const int t = threadIdx.x & 7;
    const uint64_t groups = (uint64_t)gridDim.x * (blockDim.x >> 3), g0 = (uint64_t)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3);
    const uint64_t n_iter = (n + groups - 1) / groups;
    for (uint64_t it = 0; it < n_iter; ++it) {
        const uint64_t r = g0 + it * groups;
        const bool valid = r < n;
        const float* src = rows + (valid ? r : 0) * stride_f;
        int8_t* dst = out + (valid ? r : 0) * out_stride_b;
        float ss = 0.f, mx = 0.f;
        bool bad = false;
        for (uint32_t i = t; i < dim; i += 8) {
            const float v = src[i];
            bad |= !(fabsf(v) <= 3.0e38f);
            ss = fmaf(v, v, ss);
            mx = fmaxf(mx, fabsf(v));
        }
        ss += __shfl_xor_sync(0xFFFFFFFFu, ss, 1); ss += __shfl_xor_sync(0xFFFFFFFFu, ss, 2); ss += __shfl_xor_sync(0xFFFFFFFFu, ss, 4);
        mx = fmaxf(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, 1)); mx = fmaxf(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, 2)); mx = fmaxf(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, 4));
        bad = __shfl_xor_sync(0xFFFFFFFFu, (int)bad, 1) | __shfl_xor_sync(0xFFFFFFFFu, (int)bad, 2) | __shfl_xor_sync(0xFFFFFFFFu, (int)bad, 4) | (int)bad;
        const bool tiny = !(mx >= 1.0e-30f);                      // zero (or denormal-only) rows: all codes 0, scale = max so that the error bound still holds
        const float sr = tiny ? __fmul_ru(mx, 2.0f) : __fdiv_rn(mx, 127.f);
        const float inv = tiny ? 0.f : __fdiv_rn(127.f, mx);
        for (uint32_t i = t; i < out_stride_b - 16; i += 8) {
            const float v = (i < dim) ? src[i] : 0.f;
            const float c = fminf(fmaxf(rintf(__fmul_rn(v, inv)), -127.f), 127.f);
            if (valid) dst[i] = (int8_t)(int)c;
        }
        if (valid && t == 0) {
            *reinterpret_cast<float4*>(dst + (out_stride_b - 16)) = make_float4(sr, 0.f, 0.f, 0.f);
            if (bad || !(ss <= 3.0e38f)) atomicOr(nonfinite, 1u);
            else atomicMax(max_norm_bits, __float_as_uint(sqrtf(ss) * 1.000001f));
        }
    }
}

struct Pf8Params {
    const uint8_t* rows;        // int8 plane: per row `stride - 16` code bytes, then the row's f32 scale (+ 12 bytes of padding)
    uint32_t stride;            // bytes per row (multiple of 16)
    uint32_t dim;
    uint64_t n_rows;
    const float* q;
    uint32_t rows_per_slot, n_slots, slot_bytes;
    const qb_scored_point* samp_out; const uint32_t* samp_cnt; uint32_t top;
    const unsigned int* max_norm_bits;
    uint32_t* cand; unsigned int* cnt; uint32_t cap;
    const uint32_t* deleted; const uint32_t* deleted2;
    int l2_keep;
};

__device__ __forceinline__ uint32_t pack_s8x4(int a, int b, int c, int d) { return (uint32_t)(a & 255) | ((uint32_t)(b & 255) << 8) | ((uint32_t)(c & 255) << 16) | ((uint32_t)(d & 255) << 24); }

// NCH = 8-byte chunks of a row's codes per lane (stride - 16 <= NCH * 256)
template <int NCH>
__global__ void __launch_bounds__(PF_THREADS, 1) dense_q8_filter_kernel(const Pf8Params p) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* slots = smem;                                       // [n_slots][slot_bytes]
    uint64_t* full = reinterpret_cast<uint64_t*>(slots + (size_t)p.n_slots * p.slot_bytes);
    uint64_t* empty = full + p.n_slots;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t n_tiles = (p.n_rows + p.rows_per_slot - 1) / p.rows_per_slot;
    const uint64_t n_local = (blockIdx.x < n_tiles) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const uint32_t code_b = p.stride - 16;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < p.n_slots; ++s) { qb_mbar_init(&full[s], 1); qb_mbar_init(&empty[s], 1); }
        qb_fence_barrier_init();
    }
    __syncthreads();
    const int n_prod = (int)(blockDim.x >> 5) - PF_CONSUMER_WARPS;
    if (warp < n_prod) {
        if (lane == 0) pf_produce(p, slots, full, empty, warp, n_prod, n_local);
        return;
    }
    const int cw = warp - n_prod;
    // query statistics over the whole vector, then this lane's slice quantised to two int8 levels
    float qv[NCH][8];
    uint32_t off[NCH];
    float qmax = 0.f, q1 = 0.f, q2 = 0.f;
    bool qbad = false;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const uint32_t d0 = (uint32_t)(c * 32 + lane) * 8;
        off[c] = (d0 < code_b) ? d0 : 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float v = (d0 < code_b && d0 + k < p.dim) ? p.q[d0 + k] : 0.f;
            qv[c][k] = v;
            qbad |= !(fabsf(v) <= 3.0e38f);
            qmax = fmaxf(qmax, fabsf(v)); q1 = __fadd_ru(q1, fabsf(v)); q2 = fmaf(v, v, q2);
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        qmax = fmaxf(qmax, __shfl_xor_sync(0xFFFFFFFFu, qmax, o)); q1 = __fadd_ru(q1, __shfl_xor_sync(0xFFFFFFFFu, q1, o)); q2 += __shfl_xor_sync(0xFFFFFFFFu, q2, o);
        qbad |= __shfl_xor_sync(0xFFFFFFFFu, (int)qbad, o) != 0;
    }
    qbad |= (qmax > 0.f && qmax < 1.0e-30f);                     // 127 / qmax would overflow: leave such a query to the exact scan
    const float sq = (qmax > 0.f) ? __fdiv_rn(qmax, 127.f) : 0.f;
    const float inv_sq = (qmax > 0.f && !qbad) ? __fdiv_rn(127.f, qmax) : 0.f;
    uint32_t hq[NCH][2], lq[NCH][2];
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        int h[8], l[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float y = __fmul_rn(qv[c][k], inv_sq);
            const float hf = fminf(fmaxf(rintf(y), -127.f), 127.f);
            h[k] = (int)hf;
            l[k] = (int)fminf(fmaxf(rintf(__fmul_rn(__fsub_rn(y, hf), 254.f)), -127.f), 127.f);
        }
        hq[c][0] = pack_s8x4(h[0], h[1], h[2], h[3]); hq[c][1] = pack_s8x4(h[4], h[5], h[6], h[7]);
        lq[c][0] = pack_s8x4(l[0], l[1], l[2], l[3]); lq[c][1] = pack_s8x4(l[4], l[5], l[6], l[7]);
    }
    // E_q and thr_q - slack_q (rounded towards "pass"); a non-finite query makes every row pass (-> fallback to the exact scan)
    const float qn = __fmul_ru(__fsqrt_ru(q2), 1.0001f);
    const float mxn = __uint_as_float(*p.max_norm_bits);
    const float e_q = __fadd_ru(__fmul_ru(q1, 0x1.001p-1f), __fmul_ru(__fmul_ru(sq, (float)p.dim), 0.27f));      // (1/2 + 2^-13)||q||_1 + s_q dim (127/508)(1 + 0.08)
    const float slack = __fadd_ru(__fmul_ru(__fmul_ru(__fadd_ru(__fmul_ru((float)p.dim, 0x1p-22f), 0x1p-17f), __fadd_ru(1.f, __fdiv_ru(__fsqrt_ru((float)p.dim), 127.f))),
                                            __fmul_ru(qn, mxn)), 1.0e-37f);
    const float thr = (*p.samp_cnt >= p.top) ? p.samp_out[p.top - 1].score : __int_as_float(0xff800000);
    const float thr_adj = qbad ? __int_as_float(0x7fc00000) : __fsub_rd(thr, slack);
    const float k254 = 1.0f / 254.0f;
    uint32_t s = (uint32_t)cw, ph = 0;                            // as in the producers: no 64-bit division per slot
    uint64_t r0 = ((uint64_t)blockIdx.x + (uint64_t)cw * gridDim.x) * p.rows_per_slot;
    const uint64_t r_step = (uint64_t)PF_CONSUMER_WARPS * gridDim.x * p.rows_per_slot;
    for (uint64_t i = cw; i < n_local; i += PF_CONSUMER_WARPS, r0 += r_step) {
        const uint64_t left = p.n_rows - r0;
        const uint32_t nr = (uint32_t)(left < p.rows_per_slot ? left : p.rows_per_slot);
        qb_mbar_wait(&full[s], ph);
        const uint8_t* slot = slots + (size_t)s * p.slot_bytes;
        for (uint32_t r = 0; r < nr; r += 2) {
            const bool two = r + 1 < nr;
            const uint8_t* ra = slot + (size_t)r * p.stride;
            const uint8_t* rb = slot + (size_t)(two ? r + 1 : r) * p.stride;
            int ha = 0, la = 0, hb = 0, lb = 0;
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
                const uint2 va = *reinterpret_cast<const uint2*>(ra + off[c]);
                const uint2 vb = *reinterpret_cast<const uint2*>(rb + off[c]);
                ha = __dp4a((int)va.x, (int)hq[c][0], ha); ha = __dp4a((int)va.y, (int)hq[c][1], ha);
                la = __dp4a((int)va.x, (int)lq[c][0], la); la = __dp4a((int)va.y, (int)lq[c][1], la);
                hb = __dp4a((int)vb.x, (int)hq[c][0], hb); hb = __dp4a((int)vb.y, (int)hq[c][1], hb);
                lb = __dp4a((int)vb.x, (int)lq[c][0], lb); lb = __dp4a((int)vb.y, (int)lq[c][1], lb);
            }
            ha = __reduce_add_sync(0xFFFFFFFFu, ha); la = __reduce_add_sync(0xFFFFFFFFu, la);
            hb = __reduce_add_sync(0xFFFFFFFFu, hb); lb = __reduce_add_sync(0xFFFFFFFFu, lb);
            if (lane < 2 && (lane == 0 || two)) {
                const int H = lane ? hb : ha, L = lane ? lb : la;
                const float v = fmaf(sq, fmaf((float)L, k254, (float)H), e_q);
                const float up = __fmul_ru(*reinterpret_cast<const float*>((lane ? rb : ra) + code_b), v);    // an upper bound of the exact score (up to slack_q)
                if (!(up < thr_adj)) {
                    const uint32_t id = (uint32_t)(r0 + r + lane);
                    bool dead = false;
                    if (p.deleted) dead = (p.deleted[id >> 5] >> (id & 31)) & 1u;
                    if (p.deleted2) dead = dead || ((p.deleted2[id >> 5] >> (id & 31)) & 1u);
                    if (!dead) {
                        const unsigned int pos = atomicAdd(p.cnt, 1u);
                        if (pos < p.cap) p.cand[pos] = id;
                    }
                }
            }
        }
        __syncwarp();
        if (lane == 0) qb_mbar_arrive(&empty[s]);
        s += PF_CONSUMER_WARPS;
        if (s >= p.n_slots) { s -= p.n_slots; ph ^= 1u; }
    }
}

// ------------------------------------------------------------------------------------------------ 6-bit shadow plane, scanned as a 5-bit cascade
// x_i = s_r c_i + r_i, c_i = rint(x_i / s_r) in [-31, 31], s_r = max_i |x_i| / 31.  The code u_i = c_i + 31 = 4 a_i + 2 b_i + e_i is split into
// a 5-bit code w_i = u_i >> 1 = 2 a_i + b_i, streamed for every row, and its low bit e_i, read only for the rows the 5-bit code lets through.
// Main record per row (stride = 5 d_pad / 8 + 12 rounded up to 8 bytes; two records are a multiple of 16), d_pad = dim rounded up to 32:
//   a plane (d_pad / 2 bytes)   byte 8v + 4k + j: a of dim 16v + 8k + j (low nibble) and of dim 16v + 8k + 4 + j (high nibble)
//   b plane (d_pad / 8 bytes)   u16 v: bit 4 P(j) + m = b of dim 16v + 4m + j, P = (0, 2, 1, 3)
//   s_r, rho5 >= ||x - s_r (2w + 1/2 - 31)||_2, rho6 >= ||r||_2   (f32, the norms computed in f64 and rounded up)
// Side plane: the low bits e in the b plane's layout, d_pad / 8 bytes per row (rounded up to 16).
// With t = u16 v, y = (t | t << 12) & 0x0F0F0F0F puts nibble P(j) in byte j, so `(y >> m) & 0x01010101` holds the bits of dims 16v + 4m + j in
// bytes j: OR-ed into the doubled a nibbles it is the dp4a operand 2a + b = w; alone it is the e operand.  The query is split into two int8
// levels as for the int8 plane, q_i ~ s_q (h_i + l_i / 254) =: q^_i.
// Stage 1 (dense_q5_filter_kernel) uses the 5-bit reconstruction x_i ~ s_r c5_i, c5_i = 2 w_i + 1/2 - 31 in [-30.5, 31.5]:
//   H5 = sum_i h_i 2 c5_i = 4 sum h w - 61 sum h, L5 likewise    (integers, |H5| <= 127 * 63 * dim < 2^24: exact in f32)
//   exact - s_r s_q (H5 + L5 / 254) / 2 = sum_i (q_i - q^_i) s_r c5_i + sum_i q_i r5_i, r5_i = r_i + s_r (e_i - 1/2), bounded by the smaller of
//     t1 = s_r E1_5,  E1_5 = (1 + 2^-13) ||q||_1 + 0.066 s_q dim      (|r5_i| <= s_r (1 + 2^-13); |c5_i| <= 31.5, 31.5 (1/508 + 2.3e-5) < 0.066)
//     t2 = ||q||_2 rho5 + e2 (max||x|| + rho5)                        (Cauchy-Schwarz as below; s_r ||c5||_2 <= ||x|| + rho5)
// Stage 1 writes this bound for every row and takes the threshold sample (the exact top-k of the prefix's best rows by approximate score);
// stage 2 (dense_q5_compact_kernel) lists the rows whose bound reaches it.
// Stage 3 (dense_q6_rescreen_kernel) recomputes the 6-bit sums H = sum_i h_i c_i, L likewise, from the main record and the side plane,
//   exact - s_r s_q (H + L / 254) = sum_i (q_i - q^_i) s_r c_i + sum_i q_i r_i, bounded by the smaller of
//     t1 = s_r E1,  E1 = (1/2 + 2^-13) ||q||_1 + s_q dim (31/508)(1 + 0.08)     (|r_i| <= s_r (1/2 + 2^-13), |c_i| <= 31, |q_i - q^_i| <= s_q (1/508 + 2.3e-5))
//     t2 = ||q||_2 rho6 + e2 (max||x|| + rho6),  e2 = s_q sqrt(dim)(1/508 + 2.3e-5)(1 + 0.01) >= ||q - q^||_2   (Cauchy-Schwarz; s_r ||c||_2 <= ||x|| + rho6)
//   and appends the rows that pass to the candidate list.
// Both bounds: + slack_q = 2 (dim 2^-22 + 2^-17) ||q|| max||x||: the exact f32 sum (<= dim 2^-24 ||q|| ||x||) and the kernel's f32 evaluation of
//   the approximation (<= 2^-22 ||q|| (||x|| + rho); rho <= sqrt(dim) (1 + 2^-13) / 31 ||x|| <= 1.04 ||x|| for dim <= 1024, and <= 2 sqrt(dim) ||x||
//   for rows below 1e-30, which the 2^-16 of the slack still covers).
// A row passes a bound iff  approx + min(t1, t2) >= thr_q - slack_q, every bound term rounded towards "pass".  Both bounds hold, so every row
// whose exact score reaches thr_q passes both: the candidate list is a subset of what the 6-bit test alone would pass, and results are unchanged.
// Zero and denormal-only rows (max < 1e-30) keep all-zero codes c (u = 31, c5 = -1/2), s_r = 2 max, rho6 = ||x||: their bounds hold.
// bytes per row of the side plane: d_pad / 8, rounded up to 16
__host__ __device__ constexpr uint32_t q6_lo_stride(uint32_t d_pad) { return (d_pad / 8 + 15) & ~15u; }

__global__ void __launch_bounds__(256) f32_to_q6_rows_kernel(const float* __restrict__ rows, uint64_t stride_f, uint32_t dim, uint32_t d_pad, uint64_t n,
                                                              uint8_t* __restrict__ out, uint32_t out_stride_b, uint8_t* __restrict__ lo_out,
                                                              unsigned int* __restrict__ max_norm_bits, unsigned int* __restrict__ nonfinite) {
    const int t = threadIdx.x & 7;
    const uint64_t groups = (uint64_t)gridDim.x * (blockDim.x >> 3), g0 = (uint64_t)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3);
    const uint64_t n_iter = (n + groups - 1) / groups;
    const uint32_t lo_b = q6_lo_stride(d_pad);
    for (uint64_t it = 0; it < n_iter; ++it) {
        const uint64_t r = g0 + it * groups;
        const bool valid = r < n;
        const float* src = rows + (valid ? r : 0) * stride_f;
        uint8_t* dst = out + (valid ? r : 0) * out_stride_b;
        uint8_t* lo = lo_out + (valid ? r : 0) * lo_b;
        double ss = 0.0;
        float mx = 0.f;
        bool bad = false;
        for (uint32_t i = t; i < dim; i += 8) {
            const float v = src[i];
            bad |= !(fabsf(v) <= 3.0e38f);
            ss += (double)v * (double)v;
            mx = fmaxf(mx, fabsf(v));
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
            ss += __shfl_xor_sync(0xFFFFFFFFu, ss, o); mx = fmaxf(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, o));
            bad |= __shfl_xor_sync(0xFFFFFFFFu, (int)bad, o) != 0;
        }
        const bool tiny = !(mx >= 1.0e-30f);
        const float sr = tiny ? __fmul_ru(mx, 2.0f) : __fdiv_rn(mx, 31.f);
        const float inv = tiny ? 0.f : __fdiv_rn(31.f, mx);
        auto code = [&](uint32_t d) -> int { return (d < dim) ? (int)fminf(fmaxf(rintf(__fmul_rn(src[d], inv)), -31.f), 31.f) : 0; };
        // r_i = x_i - s_r c_i is exact in f64 up to one rounding of the difference (s_r c_i has <= 30 significant bits); likewise for c5_i
        double rr6 = 0.0, rr5 = 0.0;
        for (uint32_t i = t; i < dim; i += 8) {
            const int c = code(i);
            const double e6 = (double)src[i] - (double)sr * (double)c;
            const double e5 = (double)src[i] - (double)sr * ((double)(((c + 31) >> 1) * 2) + 0.5 - 31.0);
            rr6 += e6 * e6; rr5 += e5 * e5;
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) { rr6 += __shfl_xor_sync(0xFFFFFFFFu, rr6, o); rr5 += __shfl_xor_sync(0xFFFFFFFFu, rr5, o); }
        for (uint32_t ab = t; ab < d_pad / 2; ab += 8) {
            const uint32_t d = (ab >> 3) * 16 + ((ab >> 2) & 1) * 8 + (ab & 3);
            if (valid) dst[ab] = (uint8_t)(((code(d) + 31) >> 2) | (((code(d + 4) + 31) >> 2) << 4));
        }
        for (uint32_t v = t; v < d_pad / 16; v += 8) {
            uint32_t hi = 0, lw = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
                for (int m = 0; m < 4; ++m) {
                    const uint32_t u = (uint32_t)(code(v * 16 + 4 * m + j) + 31), bit = 4 * (((j & 1) << 1) | (j >> 1)) + m;
                    hi |= ((u >> 1) & 1u) << bit;
                    lw |= (u & 1u) << bit;
                }
            }
            if (valid) {
                *reinterpret_cast<uint16_t*>(dst + d_pad / 2 + 2 * v) = (uint16_t)hi;
                *reinterpret_cast<uint16_t*>(lo + 2 * v) = (uint16_t)lw;
            }
        }
        if (valid && t == 0) {
            // f64 sums of <= 1024 squares and a square root: relative error < 2^-42, covered by the factor 1 + 2^-40 (then rounded up to f32)
            float* meta = reinterpret_cast<float*>(dst + d_pad / 2 + d_pad / 8);
            meta[0] = sr;
            meta[1] = __double2float_ru(__dmul_ru(sqrt(rr5), 1.0 + 0x1p-40));
            meta[2] = __double2float_ru(__dmul_ru(sqrt(rr6), 1.0 + 0x1p-40));
            for (uint32_t b = d_pad / 2 + d_pad / 8 + 12; b < out_stride_b; ++b) dst[b] = 0;
            for (uint32_t b = d_pad / 8; b < lo_b; ++b) lo[b] = 0;
            if (bad || !(ss <= 3.0e38)) atomicOr(nonfinite, 1u);
            else atomicMax(max_norm_bits, __float_as_uint(__double2float_ru(__dmul_ru(sqrt(ss), 1.0 + 0x1p-40))));
        }
    }
}

struct Pf6Params {
    const uint8_t* rows;        // main records: a plane, b plane, then the row's s_r, rho5, rho6
    const uint8_t* lo;          // side plane: low bits, q6_lo_stride(d_pad) bytes per row
    uint32_t stride;            // bytes per main record (a multiple of 8; two rows are a multiple of 16)
    uint32_t d_pad;             // dim rounded up to 32
    uint32_t dim;
    uint64_t n_rows;
    const float* q;
    uint32_t rows_per_slot, n_slots, slot_bytes;
    qb_scored_point* samp_out; uint32_t* samp_cnt; uint32_t top;              // threshold sample: written by stage 1, read through q6_query
    const unsigned int* max_norm_bits;
    float* up5;                 // stage 1's upper bound of every row
    uint64_t sample_rows;       // the threshold sample: rows of the tiles that start below this
    const uint8_t* f32_rows; uint32_t f32_stride; uint32_t id_base;            // exact rescoring of the sample
    unsigned long long* cta_keys; unsigned int* samp_ticket;                   // per-CTA sample keys, arrival counter of their merge
    uint32_t* list; unsigned int* list_cnt; unsigned int* list_ticket; uint32_t list_cap;   // first-stage list: row ids
    uint32_t* cand; unsigned int* cnt; uint32_t cap;
    const uint32_t* deleted; const uint32_t* deleted2;
    int l2_keep;
};

// The query as both stages see it: lane hl of a half-warp holds the 16-dimension chunks v = c * 16 + hl (zero past dim) as two packed int8
// levels per 4 dimensions; the per-query constants of both bounds, rounded towards "pass".  A non-finite query makes every row pass (-> fallback).
template <int NCH>
struct Q6Query {
    uint32_t hq[NCH][4], lq[NCH][4];
    int sum_h, sum_l;                       // over the whole query
    float sq, e1, e1_5, t2a, t2b, thr_adj;
};

template <int NCH>
__device__ __forceinline__ void q6_query(const Pf6Params& p, int hl, Q6Query<NCH>& Q) {
    const uint32_t n16 = p.d_pad / 16;
    float qmax = 0.f, q1 = 0.f, q2 = 0.f;
    bool qbad = false;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const uint32_t v = (uint32_t)(c * 16 + hl);
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const float x = (v < n16 && v * 16 + k < p.dim) ? p.q[v * 16 + k] : 0.f;
            qbad |= !(fabsf(x) <= 3.0e38f);
            qmax = fmaxf(qmax, fabsf(x)); q1 = __fadd_ru(q1, fabsf(x)); q2 = __fmaf_rn(x, x, q2);
        }
    }
#pragma unroll
    for (int o = 8; o; o >>= 1) {
        qmax = fmaxf(qmax, __shfl_xor_sync(0xFFFFFFFFu, qmax, o)); q1 = __fadd_ru(q1, __shfl_xor_sync(0xFFFFFFFFu, q1, o)); q2 += __shfl_xor_sync(0xFFFFFFFFu, q2, o);
        qbad |= __shfl_xor_sync(0xFFFFFFFFu, (int)qbad, o) != 0;
    }
    qbad |= (qmax > 0.f && qmax < 1.0e-30f);                     // 127 / qmax would overflow: leave such a query to the exact scan
    const float sq = (qmax > 0.f) ? __fdiv_rn(qmax, 127.f) : 0.f;
    const float inv_sq = (qmax > 0.f && !qbad) ? __fdiv_rn(127.f, qmax) : 0.f;
    int sum_h = 0, sum_l = 0;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const uint32_t v = (uint32_t)(c * 16 + hl);
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            int h[4], l[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t d = v * 16 + 4 * m + j;
                const float y = __fmul_rn((v < n16 && d < p.dim) ? p.q[d] : 0.f, inv_sq);
                const float hf = fminf(fmaxf(rintf(y), -127.f), 127.f);
                h[j] = (int)hf;
                l[j] = (int)fminf(fmaxf(rintf(__fmul_rn(__fsub_rn(y, hf), 254.f)), -127.f), 127.f);
                sum_h += h[j]; sum_l += l[j];
            }
            Q.hq[c][m] = pack_s8x4(h[0], h[1], h[2], h[3]);
            Q.lq[c][m] = pack_s8x4(l[0], l[1], l[2], l[3]);
        }
    }
#pragma unroll
    for (int o = 8; o; o >>= 1) { sum_h += __shfl_xor_sync(0xFFFFFFFFu, sum_h, o); sum_l += __shfl_xor_sync(0xFFFFFFFFu, sum_l, o); }
    Q.sum_h = sum_h; Q.sum_l = sum_l; Q.sq = sq;
    const float qn = __fmul_ru(__fsqrt_ru(q2), 1.0001f);
    const float mxn = __uint_as_float(*p.max_norm_bits);
    const float eq = __fmul_ru(__fmul_ru(sq, (float)p.dim), 0.066f);
    Q.e1 = __fadd_ru(__fmul_ru(q1, 0x1.001p-1f), eq);
    Q.e1_5 = __fadd_ru(__fmul_ru(q1, 0x1.0008p+0f), eq);
    const float e2 = __fmul_ru(__fmul_ru(sq, __fsqrt_ru((float)p.dim)), 0.00202f);
    Q.t2a = __fadd_ru(qn, e2); Q.t2b = __fmul_ru(e2, mxn);
    const float slack = __fadd_ru(__fmul_ru(__fmul_ru(__fadd_ru(__fmul_ru((float)p.dim, 0x1p-21f), 0x1p-16f), qn), mxn), 1.0e-37f);
    const float thr = (*p.samp_cnt >= p.top) ? p.samp_out[p.top - 1].score : __int_as_float(0xff800000);
    Q.thr_adj = qbad ? __int_as_float(0x7fc00000) : __fsub_rd(thr, slack);
}

// nibble P(j) of a u16 of the b plane or the side plane to byte j
__device__ __forceinline__ uint32_t q6_spread(uint32_t t) { return (t | (t << 12)) & 0x0F0F0F0Fu; }

// Stage 1: the 5-bit code of every row through the TMA ring.  Half a warp per row.  NCH = 16-dimension chunks of a row per lane (d_pad <= NCH * 256).
// There is no threshold yet: every row's bound goes to p.up5, and stage 2 compares it.  The rows of the tiles that start below p.sample_rows also
// compete, by their approximate score, for each warp's list of the `top` best live rows (qb_localk.cuh).  At the end each CTA re-scores the best
// `top` of its lists exactly, in the finish kernel's order, and the last CTA to finish writes the top `top` of those exact scores to the sample
// slots.  Any `top` live rows give a lower bound of the k-th best exact score, so the threshold holds however well the approximation ranks rows.
constexpr size_t PF_SAMPLE_SMEM = (size_t)QB_LOCALK_WARPS * (QB_LOCALK_SLOTS * 8 + 4 * 8 + 4) + QB_LOCALK_SLOTS * 8;   // lists, queues, counts, exact keys
static_assert(PF_CONSUMER_WARPS == QB_LOCALK_WARPS, "the CTA merge sorts one list per consumer warp");

template <int NCH>
__device__ __forceinline__ void stage1_query(const Pf6Params& p, int hl, Q6Query<NCH>& Q) { q6_query<NCH>(p, hl, Q); }

template <int NCH, bool SAMPLE>
__device__ __forceinline__ void stage1_tile(const Pf6Params& p, const Q6Query<NCH>& Q, const uint8_t* slot, uint32_t nr, uint64_t r0, int lane, LkState& lk,
                                            unsigned long long* lk_queue, unsigned int* lk_count) {
    const int half = lane >> 4, hl = lane & 15;
    // lane hl reads chunk c of a row at a_off + 128 c (a plane) and b_off + 32 c (b plane).  Chunks past d_pad meet a zero query; their reads
    // stay inside the shared memory of the ring: at most 96 bytes past the end of a row, and the ring's barriers (>= 128 bytes) follow its last slot.
    const uint32_t a_off = (uint32_t)hl * 8, b_off = p.d_pad / 2 + (uint32_t)hl * 2;
    const uint32_t meta_off = p.d_pad / 2 + p.d_pad / 8;
    const float sq_half = 0.5f * Q.sq;                             // exact: s_q is 0 or at least 1e-30 / 127
    const float k254 = 1.0f / 254.0f;
    const int corr_h5 = 61 * Q.sum_h, corr_l5 = 61 * Q.sum_l;
    // four rows per step, two per half-warp (rows r + half and r + 2 + half): two independent sum chains per lane, and one reduction and
    // one epilogue for four rows
    for (uint32_t r = 0; r < nr; r += 4) {
        const uint32_t ra = r + (uint32_t)half, rb = ra + 2;
        const bool va = ra < nr, vb = rb < nr;
        const uint8_t* rowa = slot + (size_t)(va ? ra : r) * p.stride;
        const uint8_t* rowb = slot + (size_t)(vb ? rb : r) * p.stride;
        int ha = 0, la = 0, hb = 0, lb = 0;
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
            const uint2 xa = *reinterpret_cast<const uint2*>(rowa + a_off + 128 * c);
            const uint2 xb = *reinterpret_cast<const uint2*>(rowb + a_off + 128 * c);
            const uint32_t ya = q6_spread(*reinterpret_cast<const uint16_t*>(rowa + b_off + 32 * c));
            const uint32_t yb = q6_spread(*reinterpret_cast<const uint16_t*>(rowb + b_off + 32 * c));
            const uint32_t wa[4] = {((xa.x << 1) & 0x1E1E1E1Eu) | (ya & 0x01010101u),        ((xa.x >> 3) & 0x1E1E1E1Eu) | ((ya >> 1) & 0x01010101u),
                                    ((xa.y << 1) & 0x1E1E1E1Eu) | ((ya >> 2) & 0x01010101u), ((xa.y >> 3) & 0x1E1E1E1Eu) | ((ya >> 3) & 0x01010101u)};
            const uint32_t wb[4] = {((xb.x << 1) & 0x1E1E1E1Eu) | (yb & 0x01010101u),        ((xb.x >> 3) & 0x1E1E1E1Eu) | ((yb >> 1) & 0x01010101u),
                                    ((xb.y << 1) & 0x1E1E1E1Eu) | ((yb >> 2) & 0x01010101u), ((xb.y >> 3) & 0x1E1E1E1Eu) | ((yb >> 3) & 0x01010101u)};
#pragma unroll
            for (int m = 0; m < 4; ++m) {
                ha = __dp4a((int)wa[m], (int)Q.hq[c][m], ha); la = __dp4a((int)wa[m], (int)Q.lq[c][m], la);
                hb = __dp4a((int)wb[m], (int)Q.hq[c][m], hb); lb = __dp4a((int)wb[m], (int)Q.lq[c][m], lb);
            }
        }
        // the four half-warp sums in one butterfly: lanes 0-3 of a half end up with sum h w of row a, 4-7 of row b, 8-11 sum l w of row a, 12-15 of row b
        int x0 = ((hl & 8) ? la : ha) + __shfl_xor_sync(0xFFFFFFFFu, (hl & 8) ? ha : la, 8);
        int x1 = ((hl & 8) ? lb : hb) + __shfl_xor_sync(0xFFFFFFFFu, (hl & 8) ? hb : lb, 8);
        int v = ((hl & 4) ? x1 : x0) + __shfl_xor_sync(0xFFFFFFFFu, (hl & 4) ? x0 : x1, 4);
        v += __shfl_xor_sync(0xFFFFFFFFu, v, 2);
        v += __shfl_xor_sync(0xFFFFFFFFu, v, 1);
        const int lsum = __shfl_xor_sync(0xFFFFFFFFu, v, 8);
        const bool mine = (hl == 0 && va) || (hl == 4 && vb);      // lanes 0, 16, 4 and 20 hold rows r, r + 1, r + 2 and r + 3
        float app = 0.f, up = 0.f;
        if (mine) {
            const float* meta = reinterpret_cast<const float*>((hl ? rowb : rowa) + meta_off);
            const float sr = meta[0], rho5 = meta[1];
            const float H5 = (float)(4 * v - corr_h5), L5 = (float)(4 * lsum - corr_l5);     // exact: integers below 2^24
            app = __fmul_rn(sr, __fmul_rn(sq_half, __fmaf_rn(L5, k254, H5)));
            up = __fadd_ru(app, fminf(__fmul_ru(sr, Q.e1_5), __fmaf_ru(rho5, Q.t2a, Q.t2b)));   // an upper bound of the exact score (up to slack_q)
        }
        // lanes 0-3 store the bounds of rows r .. r + 3: one contiguous store per step
        const float u = __shfl_sync(0xFFFFFFFFu, up, ((lane & 1) << 4) | ((lane & 2) << 1));
        if (lane < 4 && r + (uint32_t)lane < nr) p.up5[r0 + r + (uint32_t)lane] = u;
        if (SAMPLE) {
            if (mine && !(app < lk.wthr)) lk_push(p.deleted, p.deleted2, 0u, app, (uint32_t)(r0 + (hl ? rb : ra)), lk_queue, lk_count);
            __syncwarp();
            const unsigned int n_queued = *reinterpret_cast<volatile unsigned int*>(lk_count);
            if (n_queued) lk = lk_drain(lk, lk_queue, lk_count, lane, n_queued);
        }
    }
}

// ------------------------------------------------------------------------------------------------ block-scaled 4-bit plane: the default stage 1
// With one scale per row, a 4-bit step is set by the row's largest coordinate (~3.2 sigma at dim 768) and leaves a residual of ~0.125 ||x||:
// that bound lets about a quarter of the rows through.  Here each 16-dimension chunk b of the lane mapping above has its own scale
//   s_r = max_i |x_i| / 7 (f32),   k_b = ceil(255 max_{i in b} |x_i| / max_i |x_i|) in [1, 255] (0 for an all-zero chunk),   s_b = s_r k_b / 255,
//   x_i = s_b c_i + r_i,  c_i = rint(x_i / s_b) in [-7, 7]
// (k_b is rounded up, so s_b >= max_b / 7 up to a few f32 roundings and |x_i / s_b| < 7.5: the codes need no clamping, |r_i| <= s_b (1/2 + 2^-13)).
// Record per row (stride q4b_stride(d_pad), a multiple of 8; 440 bytes at dim 768 against the 5-bit stage's 496):
//   codes (d_pad / 2 bytes)      byte 8v + 4k + j: c + 8 of dim 16v + 8k + j (low nibble) and of dim 16v + 8k + 4 + j (high nibble), as the 6-bit
//                                plane's a plane: `x & 0x0F0F0F0F` and `(x >> 4) & 0x0F0F0F0F` of the two words of a chunk are dp4a operands of
//                                dims 16v + 4m + j (m = 0..3), the order of the query levels of Q6Query
//   scales (d_pad / 16 bytes)    byte v: k_b of chunk v
//   s_r, rho4 >= ||x - x^||_2    (f32 at a 4-byte boundary; rho4 computed in f64 and rounded up, x^_i = s_b c_i)
// With the query's int8 levels q^_i = s_q (h_i + l_i / 254) and H_b = sum_{i in b} h_i c_i, L_b likewise (dp4a on c + 8, minus 8 sum_b h):
//   approx = sum_b s_b s_q (H_b + L_b / 254) = s_r s_q / 64770 * sum_b k_b (254 H_b + L_b)
//   exact - approx = sum_i (q_i - q^_i) x^_i + sum_i q_i r_i, bounded by the smaller of
//     t1 = sum_b s_b E_b = s_r / 255 sum_b k_b E_b,  E_b = (1/2 + 2^-13) ||q_b||_1 + 0.014 s_q n_b    (|r_i| <= s_b (1/2 + 2^-13); |c_i| <= 7 and
//          |q_i - q^_i| <= s_q (1/508 + 2.3e-5): 7 (1/508 + 2.3e-5) < 0.014; n_b = dims of chunk b below dim)
//     t2 = ||q||_2 rho4 + e2 (max||x|| + rho4)                       (Cauchy-Schwarz as for the 6-bit plane; ||x^||_2 <= ||x|| + rho4)
//   + ev = 2^-19 (||q|| + e2)(max||x|| + rho4): the kernel's f32 evaluation of approx.  254 H_b + L_b is an integer below 2^22 (exact); a lane
//     sums k_b (254 H_b + L_b) over its <= 4 chunks by FMA, the half-warp adds with 4 further roundings, and three products follow: <= 16 roundings
//     of at most 2^-23 each, relative to sum_i |q^_i x^_i| <= ||q^|| ||x^|| <= (||q|| + e2)(max||x|| + rho4).
// A row passes iff  approx + min(t1, t2) + ev >= thr_q - slack_q, every bound term rounded towards "pass", with the 6-bit plane's slack_q
// (which covers the exact f32 sum).  The bound holds for every row, so the first-stage list stays a superset of the rows whose exact score
// reaches thr_q, and stages 2 and 3 run unchanged on it.  Zero and denormal-only rows (max < 1e-30) keep codes 0, k_b = 255, s_r = 2 max, rho4 = ||x||.
__host__ __device__ constexpr uint32_t q4b_meta_off(uint32_t d_pad) { return (d_pad / 2 + d_pad / 16 + 3) & ~3u; }
__host__ __device__ constexpr uint32_t q4b_stride(uint32_t d_pad) { return (q4b_meta_off(d_pad) + 8 + 7) & ~7u; }

__global__ void __launch_bounds__(256) f32_to_q4b_rows_kernel(const float* __restrict__ rows, uint64_t stride_f, uint32_t dim, uint32_t d_pad, uint64_t n,
                                                               uint8_t* __restrict__ out, uint32_t out_stride_b) {
    const int t = threadIdx.x & 7;
    const uint64_t groups = (uint64_t)gridDim.x * (blockDim.x >> 3), g0 = (uint64_t)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3);
    const uint64_t n_iter = (n + groups - 1) / groups;
    const uint32_t meta_off = q4b_meta_off(d_pad);
    for (uint64_t it = 0; it < n_iter; ++it) {
        const uint64_t r = g0 + it * groups;
        const bool valid = r < n;
        const float* src = rows + (valid ? r : 0) * stride_f;
        uint8_t* dst = out + (valid ? r : 0) * out_stride_b;
        float mx = 0.f;
        for (uint32_t i = t; i < dim; i += 8) mx = fmaxf(mx, fabsf(src[i]));
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, o));
        const bool tiny = !(mx >= 1.0e-30f);
        const float sr = tiny ? __fmul_ru(mx, 2.0f) : __fdiv_rn(mx, 7.f);
        const float kr = tiny ? 0.f : __fdiv_rn(255.f, mx);
        double rr = 0.0;
        for (uint32_t v = t; v < d_pad / 16; v += 8) {
            float mb = 0.f;
#pragma unroll
            for (int k = 0; k < 16; ++k) mb = (v * 16 + k < dim) ? fmaxf(mb, fabsf(src[v * 16 + k])) : mb;
            const int kb = tiny ? 255 : (mb > 0.f ? (int)fminf(fmaxf(ceilf(__fmul_rn(mb, kr)), 1.f), 255.f) : 0);
            const float inv = (tiny || kb == 0) ? 0.f : __fdiv_rn(255.f, __fmul_rn(sr, (float)kb));
            uint32_t w0 = 0, w1 = 0;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const float x = (v * 16 + k < dim) ? src[v * 16 + k] : 0.f;
                const int c = (int)fminf(fmaxf(rintf(__fmul_rn(x, inv)), -7.f), 7.f);
                // x - s_b c = (255 x - s_r (k_b c)) / 255: both products exact in f64, then one rounding for the difference and one for the quotient
                const double e = ((double)x * 255.0 - (double)sr * (double)(kb * c)) / 255.0;
                rr += e * e;
                const uint32_t nib = (uint32_t)(c + 8) << (8 * (k & 3) + 4 * ((k >> 2) & 1));    // dim 16v + 4m + j: word m >> 1, byte j, nibble m & 1
                if (k < 8) w0 |= nib; else w1 |= nib;
            }
            if (valid) {
                *reinterpret_cast<uint2*>(dst + 8 * v) = make_uint2(w0, w1);
                dst[d_pad / 2 + v] = (uint8_t)kb;
            }
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) rr += __shfl_xor_sync(0xFFFFFFFFu, rr, o);
        if (valid && t == 0) {
            for (uint32_t b = d_pad / 2 + d_pad / 16; b < meta_off; ++b) dst[b] = 0;
            float* meta = reinterpret_cast<float*>(dst + meta_off);
            meta[0] = sr;
            meta[1] = __double2float_ru(__dmul_ru(sqrt(rr), 1.0 + 0x1p-40));       // as rho5 / rho6 of the 6-bit plane
            for (uint32_t b = meta_off + 8; b < out_stride_b; ++b) dst[b] = 0;
        }
    }
}

// The query for the block-scaled stage: the 6-bit plane's (levels, t2, slack, threshold) and per chunk of this lane the code offset and E_b.
template <int NCH>
struct Q4bQuery {
    Q6Query<NCH> q6;
    int corr[NCH];                // 8 (254 sum h + sum l) over chunk c: the codes are stored as c + 8
    float e1[NCH];                // E_b of chunk c (zero past d_pad)
    float sq_k, k255, ev_a, ev_b; // s_q / 64770; 1/255 rounded up; ev = rho4 ev_a + ev_b
};

template <int NCH>
__device__ __forceinline__ void stage1_query(const Pf6Params& p, int hl, Q4bQuery<NCH>& Q) {
    q6_query<NCH>(p, hl, Q.q6);
    const uint32_t n16 = p.d_pad / 16;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const uint32_t v = (uint32_t)(c * 16 + hl);
        float q1 = 0.f, nb = 0.f;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const bool in = v < n16 && v * 16 + k < p.dim;
            q1 = __fadd_ru(q1, in ? fabsf(p.q[v * 16 + k]) : 0.f);
            nb += in ? 1.f : 0.f;
        }
        int sh = 0, sl = 0;
#pragma unroll
        for (int m = 0; m < 4; ++m) { sh = __dp4a((int)Q.q6.hq[c][m], 0x01010101, sh); sl = __dp4a((int)Q.q6.lq[c][m], 0x01010101, sl); }
        Q.corr[c] = 8 * (254 * sh + sl);
        Q.e1[c] = __fadd_ru(__fmul_ru(q1, 0x1.001p-1f), __fmul_ru(Q.q6.sq, __fmul_ru(nb, 0.014f)));
    }
    Q.sq_k = __fdiv_rn(Q.q6.sq, 64770.f);
    Q.k255 = __fdiv_ru(1.f, 255.f);
    Q.ev_a = __fmul_ru(Q.q6.t2a, 0x1p-19f);
    Q.ev_b = __fmul_ru(Q.ev_a, __uint_as_float(*p.max_norm_bits));
}

// As the 5-bit tile above: four rows per step, two per half-warp; each lane sums k_b (254 H_b + L_b) and k_b E_b over its chunks, and one
// butterfly of these four floats serves the four rows.
template <int NCH, bool SAMPLE>
__device__ __forceinline__ void stage1_tile(const Pf6Params& p, const Q4bQuery<NCH>& Q, const uint8_t* slot, uint32_t nr, uint64_t r0, int lane, LkState& lk,
                                            unsigned long long* lk_queue, unsigned int* lk_count) {
    const int half = lane >> 4, hl = lane & 15;
    // lane hl reads chunk c of a row at c_off + 128 c (codes) and k_off + 16 c (its scale); past d_pad the query is zero and the reads stay
    // inside the ring's shared memory, as in the 5-bit tile
    const uint32_t c_off = (uint32_t)hl * 8, k_off = p.d_pad / 2 + (uint32_t)hl, meta_off = q4b_meta_off(p.d_pad);
    for (uint32_t r = 0; r < nr; r += 4) {
        const uint32_t ra = r + (uint32_t)half, rb = ra + 2;
        const bool va = ra < nr, vb = rb < nr;
        const uint8_t* rowa = slot + (size_t)(va ? ra : r) * p.stride;
        const uint8_t* rowb = slot + (size_t)(vb ? rb : r) * p.stride;
        float aa = 0.f, ta = 0.f, ab = 0.f, tb = 0.f;
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
            const uint2 xa = *reinterpret_cast<const uint2*>(rowa + c_off + 128 * c);
            const uint2 xb = *reinterpret_cast<const uint2*>(rowb + c_off + 128 * c);
            // integer -> float by the exponent trick (exact for |x| < 2^22; I2F is quarter rate and sits on every row's chain)
            const float ka = __fsub_rn(__int_as_float(0x4B000000 | rowa[k_off + 16 * c]), 8388608.f);
            const float kb = __fsub_rn(__int_as_float(0x4B000000 | rowb[k_off + 16 * c]), 8388608.f);
            const uint32_t wa[4] = {xa.x & 0x0F0F0F0Fu, (xa.x >> 4) & 0x0F0F0F0Fu, xa.y & 0x0F0F0F0Fu, (xa.y >> 4) & 0x0F0F0F0Fu};
            const uint32_t wb[4] = {xb.x & 0x0F0F0F0Fu, (xb.x >> 4) & 0x0F0F0F0Fu, xb.y & 0x0F0F0F0Fu, (xb.y >> 4) & 0x0F0F0F0Fu};
            int ha = 0, la = 0, hb = 0, lb = 0;
#pragma unroll
            for (int m = 0; m < 4; ++m) {
                ha = __dp4a((int)wa[m], (int)Q.q6.hq[c][m], ha); la = __dp4a((int)wa[m], (int)Q.q6.lq[c][m], la);
                hb = __dp4a((int)wb[m], (int)Q.q6.hq[c][m], hb); lb = __dp4a((int)wb[m], (int)Q.q6.lq[c][m], lb);
            }
            const float fa = __fsub_rn(__int_as_float(0x4B400000 + 254 * ha + la - Q.corr[c]), 12582912.f);    // |254 H_b + L_b| < 2^22
            const float fb = __fsub_rn(__int_as_float(0x4B400000 + 254 * hb + lb - Q.corr[c]), 12582912.f);
            aa = __fmaf_rn(ka, fa, aa); ta = __fmaf_ru(ka, Q.e1[c], ta);
            ab = __fmaf_rn(kb, fb, ab); tb = __fmaf_ru(kb, Q.e1[c], tb);
        }
        // as in the 5-bit tile: lanes 0-3 of a half end up with the approx sum of row a, 4-7 of row b, 8-11 the t1 sum of row a, 12-15 of row b
        float x0 = __fadd_ru((hl & 8) ? ta : aa, __shfl_xor_sync(0xFFFFFFFFu, (hl & 8) ? aa : ta, 8));
        float x1 = __fadd_ru((hl & 8) ? tb : ab, __shfl_xor_sync(0xFFFFFFFFu, (hl & 8) ? ab : tb, 8));
        float v = __fadd_ru((hl & 4) ? x1 : x0, __shfl_xor_sync(0xFFFFFFFFu, (hl & 4) ? x0 : x1, 4));
        v = __fadd_ru(v, __shfl_xor_sync(0xFFFFFFFFu, v, 2));
        v = __fadd_ru(v, __shfl_xor_sync(0xFFFFFFFFu, v, 1));
        const float tsum = __shfl_xor_sync(0xFFFFFFFFu, v, 8);
        const bool mine = (hl == 0 && va) || (hl == 4 && vb);
        float app = 0.f, up = 0.f;
        if (mine) {
            const float* meta = reinterpret_cast<const float*>((hl ? rowb : rowa) + meta_off);
            const float sr = meta[0], rho4 = meta[1];
            app = __fmul_rn(sr, __fmul_rn(Q.sq_k, v));
            const float t1 = __fmul_ru(sr, __fmul_ru(tsum, Q.k255));
            up = __fadd_ru(__fadd_ru(app, fminf(t1, __fmaf_ru(rho4, Q.q6.t2a, Q.q6.t2b))), __fmaf_ru(rho4, Q.ev_a, Q.ev_b));   // >= exact score - slack_q
        }
        const float u = __shfl_sync(0xFFFFFFFFu, up, ((lane & 1) << 4) | ((lane & 2) << 1));
        if (lane < 4 && r + (uint32_t)lane < nr) p.up5[r0 + r + (uint32_t)lane] = u;
        if (SAMPLE) {
            if (mine && !(app < lk.wthr)) lk_push(p.deleted, p.deleted2, 0u, app, (uint32_t)(r0 + (hl ? rb : ra)), lk_queue, lk_count);
            __syncwarp();
            const unsigned int n_queued = *reinterpret_cast<volatile unsigned int*>(lk_count);
            if (n_queued) lk = lk_drain(lk, lk_queue, lk_count, lane, n_queued);
        }
    }
}

// Stage 1 on either plane (Query = Q6Query: the 5-bit code of the 6-bit plane's main records; Q4bQuery: the block-scaled 4-bit plane)
template <int NCH, class Query>
__device__ __forceinline__ void stage1_run(const Pf6Params& p) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* slots = smem;                                       // [n_slots][slot_bytes]
    uint64_t* full = reinterpret_cast<uint64_t*>(slots + (size_t)p.n_slots * p.slot_bytes);
    uint64_t* empty = full + p.n_slots;
    unsigned long long* lists = reinterpret_cast<unsigned long long*>(empty + p.n_slots);       // [warps][QB_LOCALK_SLOTS]
    unsigned long long* lk_queue = lists + QB_LOCALK_WARPS * QB_LOCALK_SLOTS;                   // [warps][4]
    unsigned int* lk_count = reinterpret_cast<unsigned int*>(lk_queue + QB_LOCALK_WARPS * 4);   // [warps]
    unsigned long long* ex = reinterpret_cast<unsigned long long*>(lk_count + QB_LOCALK_WARPS); // [QB_LOCALK_SLOTS] exact keys of the CTA's sample
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t n_tiles = (p.n_rows + p.rows_per_slot - 1) / p.rows_per_slot;
    const uint64_t n_local = (blockIdx.x < n_tiles) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < p.n_slots; ++s) { qb_mbar_init(&full[s], 1); qb_mbar_init(&empty[s], 1); }
        qb_fence_barrier_init();
    }
    if (threadIdx.x < QB_LOCALK_WARPS) lk_count[threadIdx.x] = 0u;
    __syncthreads();
    const int n_prod = (int)(blockDim.x >> 5) - PF_CONSUMER_WARPS;
    if (warp < n_prod) {
        if (lane == 0) pf_produce(p, slots, full, empty, warp, n_prod, n_local);
        return;
    }
    const int cw = warp - n_prod;
    Query Q;
    stage1_query<NCH>(p, lane & 15, Q);
    // this warp's `top` best sample rows by approximate score (lanes >= top hold the maximum so that they are never the minimum)
    LkState lk{(lane < (int)p.top) ? 0ull : ~0ull, 0ull, __int_as_float(0xff800000)};
    uint32_t s = (uint32_t)cw, ph = 0;                            // as in the producers: no 64-bit division per slot
    uint64_t r0 = ((uint64_t)blockIdx.x + (uint64_t)cw * gridDim.x) * p.rows_per_slot;
    const uint64_t r_step = (uint64_t)PF_CONSUMER_WARPS * gridDim.x * p.rows_per_slot;
    for (uint64_t i = cw; i < n_local; i += PF_CONSUMER_WARPS, r0 += r_step) {
        const uint64_t left = p.n_rows - r0;
        const uint32_t nr = (uint32_t)(left < p.rows_per_slot ? left : p.rows_per_slot);
        qb_mbar_wait(&full[s], ph);
        const uint8_t* slot = slots + (size_t)s * p.slot_bytes;
        // a warp's tiles ascend: the sample tiles come first, and the loop after them does no top-k work
        if (r0 < p.sample_rows) stage1_tile<NCH, true>(p, Q, slot, nr, r0, lane, lk, lk_queue + cw * 4, &lk_count[cw]);
        else stage1_tile<NCH, false>(p, Q, slot, nr, r0, lane, lk, lk_queue + cw * 4, &lk_count[cw]);
        __syncwarp();
        if (lane == 0) qb_mbar_arrive(&empty[s]);
        s += PF_CONSUMER_WARPS;
        if (s >= p.n_slots) { s -= p.n_slots; ph ^= 1u; }
    }
    // CTA merge of the eight lists (consumer warps only, named barrier), exact scores of its best `top` by four warps (one 8-lane group per
    // row), those keys ranked into the CTA's list, and the merge of all lists in the last CTA
    if (lane < QB_LOCALK_SLOTS) lists[cw * QB_LOCALK_SLOTS + lane] = (lk.my_key == ~0ull) ? 0ull : lk.my_key;
    asm volatile("bar.sync 1, %0;" ::"n"(PF_CONSUMER_WARPS * 32) : "memory");
    if (cw == 0) lk_cta_sort(lists, lane);
    asm volatile("bar.sync 1, %0;" ::"n"(PF_CONSUMER_WARPS * 32) : "memory");
    if (cw < QB_LOCALK_SLOTS / 4) {
        const int i = cw * 4 + (lane >> 3);
        const unsigned long long k = (i < (int)p.top) ? lists[i] : 0ull;
        const uint32_t row = k ? qb_key_id(k) : 0u;
        const float sc = qbs::score_avx_group8<qbs::M_DOT>(reinterpret_cast<const float*>(p.f32_rows + (size_t)row * p.f32_stride), p.q, p.dim, lane & 7);
        if ((lane & 7) == 0) ex[i] = k ? qb_pack_key(sc, row + p.id_base) : 0ull;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(PF_CONSUMER_WARPS * 32) : "memory");
    if (cw == 0) {
        if (lane < QB_LOCALK_SLOTS) {
            const unsigned long long k = ex[lane];
            int rank = 0;                                          // descending; equal (empty) keys keep their order
#pragma unroll
            for (int j = 0; j < QB_LOCALK_SLOTS; ++j) rank += (ex[j] > k || (ex[j] == k && j < lane)) ? 1 : 0;
            p.cta_keys[(unsigned long long)blockIdx.x * QB_LOCALK_SLOTS + rank] = k;
        }
        lk_last_cta_merge(p.cta_keys, p.top, p.samp_out, p.samp_cnt, p.samp_ticket, lane);
    }
}

template <int NCH>
__global__ void __launch_bounds__(PF_THREADS, 1) dense_q5_filter_kernel(const Pf6Params p) { stage1_run<NCH, Q6Query<NCH>>(p); }

// p.rows / p.stride: the block-scaled plane (the ring streams it); stages 2 and 3 take the 6-bit plane's
template <int NCH>
__global__ void __launch_bounds__(PF_THREADS, 1) dense_q4b_filter_kernel(const Pf6Params p) { stage1_run<NCH, Q4bQuery<NCH>>(p); }

// Stage 2: rows whose bound reaches the sample threshold, not deleted, to the first-stage list (row ids).  A CTA compacts 16 rows per thread
// per step with ONE atomic: 1-3 % of the rows pass, spread evenly, so an atomic per warp step would meet a pass almost every time, and tens of
// thousands of atomics on one counter serialise.  More rows than list_cap leave the count above it: stage 3 then raises the fallback.
constexpr int PF_COMPACT_THREADS = 256;
template <int NCH>
__global__ void __launch_bounds__(PF_COMPACT_THREADS) dense_q5_compact_kernel(const Pf6Params p) {
    constexpr int UNROLL = 4;                                     // float4 loads in flight per thread
    constexpr int WARPS = PF_COMPACT_THREADS / 32;
    __shared__ float s_thr;
    __shared__ unsigned int s_warp[WARPS], s_base;
    if (threadIdx.x < 32) {
        Q6Query<NCH> Q;
        q6_query<NCH>(p, threadIdx.x & 15, Q);
        if (threadIdx.x == 0) s_thr = Q.thr_adj;
    }
    __syncthreads();
    const float thr_adj = s_thr;                                  // NaN (a non-finite query): every row passes
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t n4 = (p.n_rows + 3) / 4, step = (uint64_t)gridDim.x * PF_COMPACT_THREADS * UNROLL;
    for (uint64_t b = (uint64_t)blockIdx.x * PF_COMPACT_THREADS * UNROLL; b < n4; b += step) {     // uniform per CTA
        float4 u4[UNROLL];
#pragma unroll
        for (int j = 0; j < UNROLL; ++j) {
            const uint64_t i = b + (uint64_t)j * PF_COMPACT_THREADS + threadIdx.x;
            u4[j] = (i < n4) ? __ldcs(reinterpret_cast<const float4*>(p.up5) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        uint32_t mask = 0;                                        // bit 4 j + k: row 4 (b + j * threads + tid) + k
#pragma unroll
        for (int j = 0; j < UNROLL; ++j) {
            const uint64_t i = b + (uint64_t)j * PF_COMPACT_THREADS + threadIdx.x;
            const float u[4] = {u4[j].x, u4[j].y, u4[j].z, u4[j].w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint64_t row = 4 * i + k;
                if (row < p.n_rows && !(u[k] < thr_adj)) {
                    const uint32_t id = (uint32_t)row;
                    bool dead = false;
                    if (p.deleted) dead = (p.deleted[id >> 5] >> (id & 31)) & 1u;
                    if (p.deleted2) dead = dead || ((p.deleted2[id >> 5] >> (id & 31)) & 1u);
                    mask |= dead ? 0u : 1u << (4 * j + k);
                }
            }
        }
        const int c = __popc(mask);
        int incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += t; }
        if (lane == 31) s_warp[warp] = (unsigned int)incl;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned int total = 0;
#pragma unroll
            for (int w = 0; w < WARPS; ++w) { const unsigned int t = s_warp[w]; s_warp[w] = total; total += t; }
            s_base = total ? atomicAdd(p.list_cnt, total) : 0u;
        }
        __syncthreads();
        if (mask) {
            unsigned int pos = s_base + s_warp[warp] + (unsigned int)(incl - c);
            for (uint32_t m = mask; m; m &= m - 1) {
                const int bit = __ffs((int)m) - 1;
                if (pos < p.list_cap) p.list[pos] = (uint32_t)(4 * (b + (uint64_t)(bit >> 2) * PF_COMPACT_THREADS + threadIdx.x) + (bit & 3));
                ++pos;
            }
        }
        __syncthreads();                                          // s_warp / s_base are rewritten by the next step
    }
}

// Stage 3: the 6-bit test of the first-stage list.  Half a warp per entry recomputes the exact 6-bit sums H = sum_i h_i c_i, L likewise, from
// the main record and the side plane: u = c + 31 = 2w + e is a dp4a operand, and H = sum h u - 31 sum h.  The test is the one of the 6-bit
// plane above.  The query's packed int8 levels are staged once per CTA in shared memory.  The last CTA to read the list's count resets it for
// the next query.  An overflowing list leaves the candidate count above cap, so that the finish kernel raises the fallback flag.
constexpr int PF_RESCREEN_THREADS = 256;
template <int NCH>
__global__ void __launch_bounds__(PF_RESCREEN_THREADS) dense_q6_rescreen_kernel(const Pf6Params p) {
    __shared__ uint4 s_hq[NCH * 16], s_lq[NCH * 16];             // chunk v: the query bytes of dims 16v + 4m + j in word m
    __shared__ float s_k[5];
    __shared__ int s_corr[2];
    __shared__ unsigned int s_n;
    if (threadIdx.x == 0) {
        s_n = *reinterpret_cast<volatile unsigned int*>(p.list_cnt);
        __threadfence();
        if (atomicAdd(p.list_ticket, 1u) == gridDim.x - 1) { *p.list_cnt = 0u; *p.list_ticket = 0u; }
    }
    if (threadIdx.x < 32) {
        const int hl = threadIdx.x & 15;
        Q6Query<NCH> Q;
        q6_query<NCH>(p, hl, Q);
        if (threadIdx.x < 16) {
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
                s_hq[c * 16 + hl] = make_uint4(Q.hq[c][0], Q.hq[c][1], Q.hq[c][2], Q.hq[c][3]);
                s_lq[c * 16 + hl] = make_uint4(Q.lq[c][0], Q.lq[c][1], Q.lq[c][2], Q.lq[c][3]);
            }
        }
        if (threadIdx.x == 0) {
            s_k[0] = Q.sq; s_k[1] = Q.e1; s_k[2] = Q.t2a; s_k[3] = Q.t2b; s_k[4] = Q.thr_adj;
            s_corr[0] = 31 * Q.sum_h; s_corr[1] = 31 * Q.sum_l;
        }
    }
    __syncthreads();
    const unsigned int n1 = s_n;
    if (n1 > p.list_cap) {
        if (blockIdx.x == 0 && threadIdx.x == 0) *p.cnt = p.cap + 1u;
        return;
    }
    const float sq = s_k[0], e1 = s_k[1], t2a = s_k[2], t2b = s_k[3], thr_adj = s_k[4];
    const int corr_h = s_corr[0], corr_l = s_corr[1];
    const float k254 = 1.0f / 254.0f;
    const int lane = threadIdx.x & 31, half = lane >> 4, hl = lane & 15;
    uint32_t hq[NCH][4], lq[NCH][4];
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
        const uint4 h = s_hq[c * 16 + hl], l = s_lq[c * 16 + hl];
        hq[c][0] = h.x; hq[c][1] = h.y; hq[c][2] = h.z; hq[c][3] = h.w;
        lq[c][0] = l.x; lq[c][1] = l.y; lq[c][2] = l.z; lq[c][3] = l.w;
    }
    const uint32_t n16 = p.d_pad / 16, lo_b = q6_lo_stride(p.d_pad);
    const uint32_t a_off = (uint32_t)hl * 8, b_off = p.d_pad / 2 + (uint32_t)hl * 2, meta_off = p.d_pad / 2 + p.d_pad / 8;
    const uint32_t warps = gridDim.x * (blockDim.x >> 5), gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    for (uint32_t e0 = 2 * gw; e0 < n1; e0 += 2 * warps) {       // uniform per warp: two entries per step
        const uint32_t e = e0 + (uint32_t)half;
        const bool valid = e < n1;
        const uint32_t row = __ldcg(p.list + (valid ? e : e0));
        const uint8_t* rec = p.rows + (size_t)row * p.stride;
        const uint8_t* lo = p.lo + (size_t)row * lo_b;
        int hs = 0, ls = 0;
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
            if ((uint32_t)(c * 16 + hl) < n16) {
                const uint2 x = __ldg(reinterpret_cast<const uint2*>(rec + a_off + 128 * c));
                const uint32_t y = q6_spread(__ldg(reinterpret_cast<const unsigned short*>(rec + b_off + 32 * c)));
                const uint32_t z = q6_spread(__ldg(reinterpret_cast<const unsigned short*>(lo + 2 * hl + 32 * c)));
                const uint32_t w[4] = {((x.x << 1) & 0x1E1E1E1Eu) | (y & 0x01010101u),        ((x.x >> 3) & 0x1E1E1E1Eu) | ((y >> 1) & 0x01010101u),
                                       ((x.y << 1) & 0x1E1E1E1Eu) | ((y >> 2) & 0x01010101u), ((x.y >> 3) & 0x1E1E1E1Eu) | ((y >> 3) & 0x01010101u)};
#pragma unroll
                for (int m = 0; m < 4; ++m) {
                    const uint32_t u = (w[m] << 1) | ((z >> m) & 0x01010101u);
                    hs = __dp4a((int)u, (int)hq[c][m], hs); ls = __dp4a((int)u, (int)lq[c][m], ls);
                }
            }
        }
        // lanes 0-7 of a half end up with sum h u, 8-15 with sum l u
        int v = ((hl & 8) ? ls : hs) + __shfl_xor_sync(0xFFFFFFFFu, (hl & 8) ? hs : ls, 8);
        v += __shfl_xor_sync(0xFFFFFFFFu, v, 4);
        v += __shfl_xor_sync(0xFFFFFFFFu, v, 2);
        v += __shfl_xor_sync(0xFFFFFFFFu, v, 1);
        const int lsum = __shfl_xor_sync(0xFFFFFFFFu, v, 8);
        if (hl == 0 && valid) {
            const float* meta = reinterpret_cast<const float*>(rec + meta_off);
            const float H = (float)(v - corr_h), L = (float)(lsum - corr_l);                    // exact: integers below 2^24
            const float sr = __ldg(meta), rho6 = __ldg(meta + 2);
            const float app = __fmul_rn(sr, __fmul_rn(sq, __fmaf_rn(L, k254, H)));
            const float up = __fadd_ru(app, fminf(__fmul_ru(sr, e1), __fmaf_ru(rho6, t2a, t2b)));     // an upper bound of the exact score (up to slack_q)
            if (!(up < thr_adj)) {
                const unsigned int pos = atomicAdd(p.cnt, 1u);
                if (pos < p.cap) p.cand[pos] = row;
            }
        }
    }
}

// the ring of any filter kernel above: slots of ~PF_SLOT_BYTES (a multiple of `row_step` rows: the rows a warp takes per step), as many as
// fit, one CTA per SM; `extra_smem` bytes follow the ring's barriers
template <typename P>
qb_status launch_ring(void (*kernel)(P), P& p, int sm_count, cudaStream_t stream, size_t extra_smem = 0, uint32_t row_step = 2) {
    const uint32_t kMaxSmem = 227 * 1024;
    const uint32_t target = qb_opt().prefilter_slot_bytes ? qb_opt().prefilter_slot_bytes : PF_SLOT_BYTES;
    uint32_t rps = target / p.stride / row_step * row_step;
    if (rps < row_step) rps = row_step;
    p.rows_per_slot = rps;
    p.slot_bytes = rps * p.stride;
    uint32_t n_slots = (kMaxSmem - 2048 - (uint32_t)extra_smem) / p.slot_bytes;
    if (n_slots > 64) n_slots = 64;
    n_slots = (n_slots / PF_CONSUMER_WARPS) * PF_CONSUMER_WARPS;
    QB_CHECK(n_slots >= (uint32_t)PF_CONSUMER_WARPS, QB_ERR_INVALID, "prefilter: rows too wide for the ring");
    p.n_slots = n_slots;
    const size_t smem = (size_t)n_slots * p.slot_bytes + (size_t)n_slots * 16 + extra_smem;
    QB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
    const uint64_t n_tiles = ceil_div_u64(p.n_rows, p.rows_per_slot);
    const unsigned grid = (unsigned)std::min<uint64_t>(n_tiles, (uint64_t)sm_count);
    kernel<<<grid, 32 * (PF_CONSUMER_WARPS + pf_producers()), smem, stream>>>(p);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

// the largest key below `prev` among k[0, n) (keys are unique: the id is part of the key), block-wide; 0 when there is none
template <bool GLOBAL>
__device__ unsigned long long block_next_key(const unsigned long long* k, uint32_t n, unsigned long long prev, unsigned long long* s_best) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned long long best = 0ull;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned long long x = GLOBAL ? __ldcg(k + i) : k[i];
        if (x < prev && x > best) best = x;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { const unsigned long long w = __shfl_xor_sync(0xFFFFFFFFu, best, o); best = w > best ? w : best; }
    if (lane == 0) s_best[warp] = best;
    __syncthreads();
    best = s_best[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) best = s_best[w] > best ? s_best[w] : best;
    __syncthreads();
    return best;
}

// exact scores of the candidates in score_avx_group8's order, one contiguous share of the list per CTA (one 8-lane group per candidate); each
// CTA writes its own top-k keys to keys[blockIdx.x * top, + top), and the LAST CTA to finish picks the top-k of those by (score desc, id asc)
// — or raises the fallback flag when the list overflowed / the sample gave no threshold
constexpr int PF_FINISH_THREADS = 256;
__global__ void __launch_bounds__(PF_FINISH_THREADS) f32_prefilter_finish_kernel(const uint8_t* __restrict__ rows, uint32_t stride, uint32_t dim, const float* __restrict__ q,
                                                                   const uint32_t* __restrict__ cand, unsigned int* __restrict__ cnt, uint32_t cap, uint32_t top, uint32_t id_base,
                                                                   unsigned long long* __restrict__ keys, unsigned int* __restrict__ ticket, qb_scored_point* __restrict__ out,
                                                                   uint32_t* __restrict__ out_cnt, unsigned int* __restrict__ fallback, unsigned int* __restrict__ n_fallbacks) {
    extern __shared__ unsigned long long s_keys[];                // ceil(cap / gridDim.x)
    __shared__ unsigned long long s_best[PF_FINISH_THREADS / 32];
    __shared__ unsigned int s_ticket;
    const unsigned int c = *cnt;                                  // nobody resets it before every CTA has drawn its ticket
    const bool bad = c > cap || c < top;                          // overflow, or a sample that could not give a threshold
    const int t = threadIdx.x & 7;
    if (!bad) {
        const uint32_t per = (c + gridDim.x - 1) / gridDim.x, begin = min(c, blockIdx.x * per), m = min(c, begin + per) - begin;
        const uint32_t groups = blockDim.x >> 3, g = threadIdx.x >> 3;
        const uint32_t n_iter = (m + groups - 1) / groups;        // uniform: the 8-lane scorer shuffles with the full warp mask
        for (uint32_t it = 0; it < n_iter; ++it) {
            const uint32_t i = g + it * groups;
            const bool valid = i < m;
            const uint32_t row = valid ? cand[begin + i] : 0u;
            const float sc = qbs::score_avx_group8<qbs::M_DOT>(reinterpret_cast<const float*>(rows + (size_t)row * stride), q, dim, t);
            if (valid && t == 0) s_keys[i] = qb_pack_key(sc, row + id_base);
        }
        __syncthreads();
        unsigned long long prev = ~0ull;
        for (uint32_t r = 0; r < top; ++r) {
            prev = block_next_key<false>(s_keys, m, prev, s_best);
            if (threadIdx.x == 0) keys[(size_t)blockIdx.x * top + r] = prev;
        }
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_ticket = atomicAdd(ticket, 1u);
    __syncthreads();
    if (s_ticket != gridDim.x - 1) return;
    __threadfence();
    if (threadIdx.x == 0) { *cnt = 0u; *ticket = 0u; *fallback = bad ? 1u : 0u; if (bad) atomicAdd(n_fallbacks, 1u); }   // ready for the next query on this context
    if (bad) return;
    unsigned long long prev = ~0ull;
    for (uint32_t r = 0; r < top; ++r) {
        prev = block_next_key<true>(keys, gridDim.x * top, prev, s_best);
        if (threadIdx.x == 0) { qb_scored_point sp; sp.idx = qb_key_id(prev); sp.score = qb_key_score(prev); out[r] = sp; }
    }
    if (threadIdx.x == 0) *out_cnt = top;
}

}  // namespace

// int8 shadow plane (codes + the row's scale) of a dense f32 storage, built on first use and rebuilt after rows were rewritten: +26 % HBM
static qb_status q8_shadow_ensure(qb_storage* s, cudaStream_t stream) {
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->q8_ready) return QB_OK;
    const uint32_t row_b = (uint32_t)round_up_u64(s->dim, 16) + 16;      // codes, then the row's f32 scale in its own 16 bytes: one bulk copy per tile
    if (!s->d_q8) {
        QB_CUDA(cudaMalloc(&s->d_q8, std::max<size_t>((size_t)s->count * row_b, 256)));
        QB_CUDA(cudaMalloc(&s->d_q8_meta, 256));
        s->hbm_bytes += (uint64_t)s->count * row_b;
    }
    s->q8_row_b = row_b;
    QB_CUDA(cudaMemsetAsync(s->d_q8_meta, 0, 256, stream));
    const uint64_t blocks = std::min<uint64_t>(ceil_div_u64(std::max<uint64_t>(s->count, 1), 32), (uint64_t)s->sm_count * 16);
    f32_to_q8_rows_kernel<<<(unsigned)blocks, 256, 0, stream>>>(reinterpret_cast<const float*>(s->d_rows), s->row_stride / 4, s->dim, s->count, s->d_q8, row_b, s->d_q8_meta,
                                                                s->d_q8_meta + 1);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    unsigned int meta[2] = {0, 0};
    QB_CUDA(cudaMemcpyAsync(meta, s->d_q8_meta, 8, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaStreamSynchronize(stream));
    s->q8_ready = true;
    s->q8_usable = meta[1] == 0;
    return QB_OK;
}

// 6-bit shadow plane (main records + the side plane of low bits), built like the int8 plane: +19 % HBM
static qb_status q6_shadow_ensure(qb_storage* s, cudaStream_t stream) {
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->q6_ready) return QB_OK;
    const uint32_t d_pad = (uint32_t)round_up_u64(s->dim, 32);
    const uint32_t row_b = (uint32_t)round_up_u64(d_pad / 2 + d_pad / 8 + 12, 8);
    const size_t bytes = (size_t)s->count * row_b + 16;                  // + 16: a tile's bulk copy is rounded up to 16 bytes (pf_produce)
    const size_t lo_bytes = (size_t)s->count * q6_lo_stride(d_pad);
    if (!s->d_q6) {
        QB_CUDA(cudaMalloc(&s->d_q6_lo, std::max<size_t>(lo_bytes, 256)));
        if (cudaMalloc(&s->d_q6, std::max<size_t>(bytes, 256)) != cudaSuccess) { cudaFree(s->d_q6_lo); s->d_q6_lo = nullptr; s->d_q6 = nullptr; return QB_ERR_CUDA; }
        QB_CUDA(cudaMalloc(&s->d_q6_meta, 256));
        s->hbm_bytes += bytes + lo_bytes;
    }
    s->q6_row_b = row_b;
    QB_CUDA(cudaMemsetAsync(s->d_q6_meta, 0, 256, stream));
    const uint64_t blocks = std::min<uint64_t>(ceil_div_u64(std::max<uint64_t>(s->count, 1), 32), (uint64_t)s->sm_count * 16);
    f32_to_q6_rows_kernel<<<(unsigned)blocks, 256, 0, stream>>>(reinterpret_cast<const float*>(s->d_rows), s->row_stride / 4, s->dim, d_pad, s->count, s->d_q6, row_b,
                                                                s->d_q6_lo, s->d_q6_meta, s->d_q6_meta + 1);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    unsigned int meta[2] = {0, 0};
    QB_CUDA(cudaMemcpyAsync(meta, s->d_q6_meta, 8, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaStreamSynchronize(stream));
    s->q6_ready = true;
    s->q6_usable = meta[1] == 0;
    return QB_OK;
}

// block-scaled 4-bit plane (stage 1 of the 6-bit plane's scan), built like the planes above: +14 % HBM at dim 768, on top of the 6-bit plane
static qb_status q4b_shadow_ensure(qb_storage* s, cudaStream_t stream) {
    std::lock_guard<std::mutex> lk(s->mu);
    if (s->q4b_ready) return QB_OK;
    const uint32_t d_pad = (uint32_t)round_up_u64(s->dim, 32);
    const uint32_t row_b = q4b_stride(d_pad);
    const size_t bytes = (size_t)s->count * row_b + 16;                  // + 16: a tile's bulk copy is rounded up to 16 bytes (pf_produce)
    if (!s->d_q4b) {
        if (cudaMalloc(&s->d_q4b, std::max<size_t>(bytes, 256)) != cudaSuccess) { s->d_q4b = nullptr; return QB_ERR_CUDA; }
        s->hbm_bytes += bytes;
    }
    s->q4b_row_b = row_b;
    const uint64_t blocks = std::min<uint64_t>(ceil_div_u64(std::max<uint64_t>(s->count, 1), 32), (uint64_t)s->sm_count * 16);
    f32_to_q4b_rows_kernel<<<(unsigned)blocks, 256, 0, stream>>>(reinterpret_cast<const float*>(s->d_rows), s->row_stride / 4, s->dim, d_pad, s->count, s->d_q4b, row_b);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    QB_CUDA(cudaStreamSynchronize(stream));
    s->q4b_ready = true;
    return QB_OK;
}

// option prefilter_stage1: 5 = the 5-bit code of the 6-bit plane's main records as stage 1 (no block-scaled plane); anything else = the block-scaled plane
static bool pf_stage1_q4b() { return qb_opt().prefilter_stage1 != 5; }

// option prefilter_plane: 0 = the 6-bit plane, 1 = bf16, 2 = int8 (the integer planes need dim * 127 * 62 < 2^24 and <= 4 chunks per lane: dim <= 1024,
// which every prefiltered storage meets).  Only the selected plane is built; when it cannot be allocated, the bf16 plane is tried.
static int pf_plane() { const int o = qb_opt().prefilter_plane; return (o == 1 || o == 2) ? o : 0; }

// Can this storage answer single-query top-k searches through a shadow-plane prefilter?  Builds the plane on first use.
bool qb_f32_prefilter_usable(qb_storage* s, uint64_t n_rows, uint32_t top, cudaStream_t stream) {
    if (s->kind != QB_KIND_DENSE || s->dtype != QB_DT_F32) return false;
    if (s->distance != QB_DIST_DOT && s->distance != QB_DIST_COSINE) return false;       // the bound is on a dot product
    if (qb_opt().disable_prefilter || n_rows != s->count || n_rows < (1ull << 19) || top > 16 || s->dim < 32 || round_up_u64(s->dim, 8) > 1024) return false;
    if (pf_plane() == 0) {
        if (q6_shadow_ensure(s, stream) == QB_OK) {
            if (s->q6_usable && pf_stage1_q4b() && q4b_shadow_ensure(s, stream) != QB_OK) cudaGetLastError();   // no room: the 5-bit stage 1
            return s->q6_usable;
        }
        cudaGetLastError();                                                               // e.g. no room for the plane: try the bf16 one / stay exact
    } else if (pf_plane() == 2) {
        if (q8_shadow_ensure(s, stream) == QB_OK) return s->q8_usable;
        cudaGetLastError();
    }
    if (qb_f32_shadow_ensure(s, stream) != QB_OK) { cudaGetLastError(); return false; }
    return s->bf16_usable;
}

// d_q = preprocessed query; the exact top-`top` of the storage lands in d_out / d_out_cnt.  `a` = the scan arguments of the exact
// in-kernel-top-k path (emit.cand / final_out / done_counter set up by the caller); scratch = c->d_pf (see qb_f32_prefilter_scratch_bytes),
// d_up5 = s->count floats (rounded up to 4) for the 6-bit plane's per-row bounds.
size_t qb_f32_prefilter_scratch_bytes() { return 256 + (size_t)PF_CAP * 12 + (size_t)PF_LIST_CAP * 4; }

qb_status qb_f32_prefilter_search(qb_storage* s, const QbScanArgs& a, uint32_t top, void* d_scratch, float* d_up5, unsigned int* d_n_fallbacks, qb_scored_point* d_out,
                                  uint32_t* d_out_cnt, cudaEvent_t prof0, cudaEvent_t prof1, cudaStream_t stream) {
    uint8_t* sc = reinterpret_cast<uint8_t*>(d_scratch);
    // scratch: [0,16) cnt | [16,32) fallback flag | [32,48) finish ticket | [48,64) sample count | [64, 64+16*8) sample top-k |
    // [192,208) first-stage count | [208,224) its ticket | [224,240) ticket of the sample merge | from 256: per-CTA top-k keys |
    // candidate rows | first-stage list  (the first 256 bytes are zeroed once, the kernels reset their counters)
    unsigned int* d_cnt = reinterpret_cast<unsigned int*>(sc);
    unsigned int* d_fallback = reinterpret_cast<unsigned int*>(sc + 16);
    uint32_t* d_samp_cnt = reinterpret_cast<uint32_t*>(sc + 48);
    qb_scored_point* d_samp = reinterpret_cast<qb_scored_point*>(sc + 64);
    unsigned int* d_ticket = reinterpret_cast<unsigned int*>(sc + 32);
    unsigned int* d_list_cnt = reinterpret_cast<unsigned int*>(sc + 192);
    unsigned int* d_list_ticket = reinterpret_cast<unsigned int*>(sc + 208);
    unsigned int* d_samp_ticket = reinterpret_cast<unsigned int*>(sc + 224);
    unsigned long long* d_keys = reinterpret_cast<unsigned long long*>(sc + 256);
    uint32_t* d_cand = reinterpret_cast<uint32_t*>(d_keys + PF_CAP);
    uint32_t* d_list = d_cand + PF_CAP;
    const uint64_t n = s->count;
    // the candidate list holds n / 32 rows (at most PF_CAP): re-scoring reads a whole f32 row per candidate, and past 1/32 of the rows the
    // exact scan that a longer list would save is no longer far off
    const uint32_t cap = (uint32_t)std::min<uint64_t>(PF_CAP, n / 32);
    const float* d_q = reinterpret_cast<const float*>(a.d_q_enc);
    const int plane = pf_plane();
    uint64_t n_slots = 0;
    if (plane == 0 && s->q6_ready && s->q6_usable) {
        // 1. stage 1 over the whole 6-bit plane: every row's 5-bit bound, and the exact top-k of the best rows of a prefix by approximate
        //    score as the threshold sample.  The prefix is n / 8 rows: the threshold is then the top-k of 1.25 M rows at 10 M rows, and the
        //    tests that delete all but a few rows of the first third of a storage still find fewer than k live rows in it.
        uint64_t sample = n / 8;
        if (qb_opt().sample_rows) sample = std::min<uint64_t>(n, std::max<uint64_t>(16384, qb_opt().sample_rows & ~(uint64_t)3));   // experiments
        Pf6Params p6{};
        p6.rows = s->d_q6; p6.lo = s->d_q6_lo; p6.stride = s->q6_row_b; p6.d_pad = (uint32_t)round_up_u64(s->dim, 32); p6.dim = s->dim; p6.n_rows = n;
        p6.q = d_q; p6.samp_out = d_samp; p6.samp_cnt = d_samp_cnt; p6.top = top; p6.max_norm_bits = s->d_q6_meta;
        p6.up5 = d_up5; p6.sample_rows = sample;
        p6.f32_rows = reinterpret_cast<const uint8_t*>(s->d_rows); p6.f32_stride = s->row_stride; p6.id_base = a.emit.id_base;
        p6.cta_keys = d_keys; p6.samp_ticket = d_samp_ticket;
        // 2. the rows whose bound reaches the threshold, up to PF_LIST_CAP of them: 1-3 % of the rows on unit-Gaussian data at dim 768, but
        //    far more on wider rows or on a storage whose prefix ranks badly
        p6.list = d_list; p6.list_cnt = d_list_cnt; p6.list_ticket = d_list_ticket; p6.list_cap = (uint32_t)std::min<uint64_t>(PF_LIST_CAP, n);
        p6.cand = d_cand; p6.cnt = d_cnt; p6.cap = cap; p6.deleted = a.emit.deleted; p6.deleted2 = a.emit.deleted2;
        p6.l2_keep = ((uint64_t)n * p6.stride <= (64ull << 20)) ? 1 : 0;
        const unsigned cp_grid = (unsigned)s->sm_count * 8, rs_grid = (unsigned)s->sm_count * 4;
        QB_CHECK((uint64_t)s->sm_count * QB_LOCALK_SLOTS <= PF_CAP, QB_ERR_INVALID, "prefilter: %d CTAs exceed the key buffer", s->sm_count);
        if (prof0) cudaEventRecord(prof0, stream);
        if (pf_stage1_q4b() && s->q4b_ready) {
            // stage 1 on the block-scaled plane: the ring streams its records, every other field stays the 6-bit plane's
            Pf6Params p4 = p6;
            p4.rows = s->d_q4b; p4.stride = s->q4b_row_b;
            switch ((p4.d_pad + 255) / 256) {
                case 1: QB_TRY(launch_ring(dense_q4b_filter_kernel<1>, p4, s->sm_count, stream, PF_SAMPLE_SMEM, 4)); break;
                case 2: QB_TRY(launch_ring(dense_q4b_filter_kernel<2>, p4, s->sm_count, stream, PF_SAMPLE_SMEM, 4)); break;
                case 3: QB_TRY(launch_ring(dense_q4b_filter_kernel<3>, p4, s->sm_count, stream, PF_SAMPLE_SMEM, 4)); break;
                default: QB_TRY(launch_ring(dense_q4b_filter_kernel<4>, p4, s->sm_count, stream, PF_SAMPLE_SMEM, 4)); break;
            }
        } else {
            switch ((p6.d_pad + 255) / 256) {
                case 1: QB_TRY(launch_ring(dense_q5_filter_kernel<1>, p6, s->sm_count, stream, PF_SAMPLE_SMEM, 4)); break;
                case 2: QB_TRY(launch_ring(dense_q5_filter_kernel<2>, p6, s->sm_count, stream, PF_SAMPLE_SMEM, 4)); break;
                case 3: QB_TRY(launch_ring(dense_q5_filter_kernel<3>, p6, s->sm_count, stream, PF_SAMPLE_SMEM, 4)); break;
                default: QB_TRY(launch_ring(dense_q5_filter_kernel<4>, p6, s->sm_count, stream, PF_SAMPLE_SMEM, 4)); break;
            }
        }
        if (prof1) cudaEventRecord(prof1, stream);
        // 2b. the 6-bit test of the listed rows
        switch ((p6.d_pad + 255) / 256) {
            case 1: dense_q5_compact_kernel<1><<<cp_grid, PF_COMPACT_THREADS, 0, stream>>>(p6); dense_q6_rescreen_kernel<1><<<rs_grid, PF_RESCREEN_THREADS, 0, stream>>>(p6); break;
            case 2: dense_q5_compact_kernel<2><<<cp_grid, PF_COMPACT_THREADS, 0, stream>>>(p6); dense_q6_rescreen_kernel<2><<<rs_grid, PF_RESCREEN_THREADS, 0, stream>>>(p6); break;
            case 3: dense_q5_compact_kernel<3><<<cp_grid, PF_COMPACT_THREADS, 0, stream>>>(p6); dense_q6_rescreen_kernel<3><<<rs_grid, PF_RESCREEN_THREADS, 0, stream>>>(p6); break;
            default: dense_q5_compact_kernel<4><<<cp_grid, PF_COMPACT_THREADS, 0, stream>>>(p6); dense_q6_rescreen_kernel<4><<<rs_grid, PF_RESCREEN_THREADS, 0, stream>>>(p6); break;
        }
        QB_LAUNCHED();
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
    } else {
    // 1. exact top-k of a prefix
    // 1/64 of the rows, 2^14..2^17: a shard of a sharded search (1.25M rows at N = 8) should not spend a fifth of its step on the sample
    uint64_t sample = std::min<uint64_t>(131072, std::max<uint64_t>(16384, (n / 64) & ~(uint64_t)3));
    if (qb_opt().sample_rows) sample = std::min<uint64_t>(n, std::max<uint64_t>(16384, qb_opt().sample_rows & ~(uint64_t)3));   // experiments
    QbScanArgs as = a;
    as.row_begin = 0; as.row_end = sample;
    as.emit.final_out = d_samp; as.emit.final_count = d_samp_cnt; as.emit.run_if = nullptr;
    QB_TRY(qb_dense_f32_scan_localk(s, as, top, &n_slots, stream, 4096));
    QB_CHECK(n_slots != 0 && n_slots <= 4096, QB_ERR_CUDA, "prefilter: the sample scan did not launch (%llu slots)", (unsigned long long)n_slots);
    // 2. filter pass over the whole shadow plane
    if (plane == 2 && s->q8_ready && s->q8_usable) {
        Pf8Params p8{};
        p8.rows = reinterpret_cast<const uint8_t*>(s->d_q8); p8.stride = s->q8_row_b; p8.dim = s->dim; p8.n_rows = n;
        p8.q = d_q; p8.samp_out = d_samp; p8.samp_cnt = d_samp_cnt; p8.top = top; p8.max_norm_bits = s->d_q8_meta;
        p8.cand = d_cand; p8.cnt = d_cnt; p8.cap = cap; p8.deleted = a.emit.deleted; p8.deleted2 = a.emit.deleted2;
        p8.l2_keep = ((uint64_t)n * p8.stride <= (64ull << 20)) ? 1 : 0;
        if (prof0) cudaEventRecord(prof0, stream);
        switch ((p8.stride - 16 + 255) / 256) {
            case 1: QB_TRY(launch_ring(dense_q8_filter_kernel<1>, p8, s->sm_count, stream)); break;
            case 2: QB_TRY(launch_ring(dense_q8_filter_kernel<2>, p8, s->sm_count, stream)); break;
            case 3: QB_TRY(launch_ring(dense_q8_filter_kernel<3>, p8, s->sm_count, stream)); break;
            default: QB_TRY(launch_ring(dense_q8_filter_kernel<4>, p8, s->sm_count, stream)); break;
        }
        if (prof1) cudaEventRecord(prof1, stream);
    } else {
    PfParams p{};
    p.rows = reinterpret_cast<const uint8_t*>(s->d_bf16); p.row_h = s->bf16_row_h; p.stride = s->bf16_row_h * 2; p.dim = s->dim; p.n_rows = n;
    p.q = reinterpret_cast<const float*>(a.d_q_enc);
    p.samp_out = d_samp; p.samp_cnt = d_samp_cnt; p.top = top; p.max_norm_bits = s->d_bf16_meta;
    p.cand = d_cand; p.cnt = d_cnt; p.cap = cap; p.deleted = a.emit.deleted; p.deleted2 = a.emit.deleted2;
    p.l2_keep = ((uint64_t)n * p.stride <= (64ull << 20)) ? 1 : 0;
    if (prof0) cudaEventRecord(prof0, stream);
    const uint32_t nch = (p.row_h + 255) / 256;
    switch (nch) {
        case 1: QB_TRY(launch_ring(dense_bf16_filter_kernel<1>, p, s->sm_count, stream)); break;
        case 2: QB_TRY(launch_ring(dense_bf16_filter_kernel<2>, p, s->sm_count, stream)); break;
        case 3: QB_TRY(launch_ring(dense_bf16_filter_kernel<3>, p, s->sm_count, stream)); break;
        default: QB_TRY(launch_ring(dense_bf16_filter_kernel<4>, p, s->sm_count, stream)); break;
    }
    if (prof1) cudaEventRecord(prof1, stream);
    }
    }
    // 3. exact scores + top-k of the survivors (or the fallback flag): one CTA per SM, enough of them that a CTA's share fits in 32 KB
    const unsigned fin_grid = (unsigned)std::max<uint32_t>((uint32_t)s->sm_count, ceil_div_u64(PF_CAP, 4096));
    const size_t fin_smem = (size_t)ceil_div_u64(cap, fin_grid) * sizeof(unsigned long long);
    QB_CHECK((uint64_t)fin_grid * top <= PF_CAP, QB_ERR_INVALID, "prefilter: %u finish CTAs x top %u exceed the key buffer", fin_grid, top);
    f32_prefilter_finish_kernel<<<fin_grid, PF_FINISH_THREADS, fin_smem, stream>>>(reinterpret_cast<const uint8_t*>(s->d_rows), s->row_stride, s->dim, d_q, d_cand, d_cnt, cap,
                                                                                   top, a.emit.id_base, d_keys, d_ticket, d_out, d_out_cnt, d_fallback, d_n_fallbacks);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    // 4. the exact scan of everything: its CTAs return at once unless the flag is up
    QbScanArgs af = a;
    af.row_begin = 0; af.row_end = n;
    af.emit.final_out = d_out; af.emit.final_count = d_out_cnt; af.emit.run_if = d_fallback;
    QB_TRY(qb_dense_f32_scan_localk(s, af, top, &n_slots, stream));
    QB_CHECK(n_slots != 0 && n_slots <= 4096, QB_ERR_CUDA, "prefilter: the fallback scan did not launch (%llu slots)", (unsigned long long)n_slots);
    return QB_OK;
}
