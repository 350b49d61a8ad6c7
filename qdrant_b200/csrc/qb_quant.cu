// qb_quant.cu — quantized scorers on H100: SQ8 (scalar), PQ (product, LUT) and BQ (binary).
//
// Replaces quantization::EncodedVectors::{encode_query, score, score_point, score_internal}
// (lib/quantization/src/encoded_vectors.rs:41-117) for
//   SQ8  EncodedVectorsU8  — lib/quantization/src/encoded_vectors_u8.rs (+ cpp/avx2.c:25-122)
//   PQ   EncodedVectorsPQ  — lib/quantization/src/encoded_vectors_pq.rs:411-443,519-541,574-618
//   BQ   EncodedVectorsBin<u128> — lib/quantization/src/encoded_vectors_binary.rs:558-810
// as called from QuantizedQueryScorer::score_stored_batch (lib/segment/src/vector_storage/quantized/
// quantized_query_scorer.rs:81-93).  All three are integer / table work bounded by HBM or shared-memory
// gathers; none of it is reshaped into a GEMM here (the batched SQ8 tensor-core path lives in qb_sq8_mma.cu).
//
// Exactness notes
//   SQ8  integer dot is exact; the CPU converts 8 i32 lanes to f32 and adds them in the HSUM256_PS tree
//        (cpp/avx2.c:7-14).  Codes are <= 127 and non-negative, so when the total is < 2^24 every partial
//        is exact and any order gives f32(total); beyond that (only possible for actual_dim > 1040) the
//        LANEX variant reproduces the lane partition and the tree.  The epilogue is three separate roundings
//        (encoded_vectors_u8.rs:101-103).
//   PQ   four f32 lanes, lane k sums chunks j = k (mod 4) in ascending j; (s0+s2)+(s1+s3); tail sequential.
//   BQ   popcounts are integers; the float epilogue of calculate_metric is restated literally.
#include <cooperative_groups.h>

#include "qb_internal.h"
#include "qb_score.cuh"

namespace {

// ================================================================== SQ8 ===========================
__device__ __forceinline__ uint8_t sq8_encode_value(float v, float offset, float alpha) {  // encoded_vectors_u8.rs:95-98
    float i = __fdiv_rn(__fsub_rn(v, offset), alpha);
    if (i < 0.0f) i = 0.0f;          // f32::clamp keeps NaN
    if (i > 127.0f) i = 127.0f;
    float r = roundf(i);             // f32::round: half away from zero
    if (r != r) return 0;            // NaN as u8 == 0
    return (uint8_t)r;
}

// one block per query: threads encode elements, thread 0 folds the offset sequentially (f32, Rust order)
__global__ void __launch_bounds__(256) sq8_encode_query_kernel(const float* __restrict__ q_pre, uint32_t q_stride_f, uint32_t dim,
                                                               uint32_t actual_dim, float alpha, float offset, int qdist, int invert,
                                                               uint8_t* __restrict__ codes, float* __restrict__ q_off) {
    const uint32_t q = blockIdx.x;
    const float* src = q_pre + (size_t)q * q_stride_f;
    uint8_t* dst = codes + (size_t)q * actual_dim;
    const bool is_dot = (qdist == QB_QD_DOT || qdist == QB_QD_COSINE);
    const uint8_t pad = sq8_encode_value(is_dot ? 0.0f : offset, offset, alpha);  // :586-596
    for (uint32_t i = threadIdx.x; i < actual_dim; i += blockDim.x) dst[i] = (i < dim) ? sq8_encode_value(src[i], offset, alpha) : pad;
    __syncthreads();
    if (threadIdx.x == 0) {
        float off;
        if (is_dot) {
            float s = -0.0f;
            for (uint32_t i = 0; i < actual_dim; ++i) s = __fadd_rn(s, (float)dst[i]);
            off = __fmul_rn(__fmul_rn(s, alpha), offset);
        } else if (qdist == QB_QD_L1) {
            off = 0.0f;
        } else {
            float s = -0.0f;
            for (uint32_t i = 0; i < actual_dim; ++i) { float c = (float)dst[i]; s = __fadd_rn(s, __fmul_rn(c, c)); }
            off = __fmul_rn(__fmul_rn(s, alpha), alpha);
        }
        q_off[q] = invert ? -off : off;
    }
}

struct Sq8Params {
    const uint8_t* codes;   // [count][ad]
    const float* voff;      // [count]
    uint32_t ad;            // actual_dim (multiple of 16)
    float multiplier;
    int l1;                 // 1: Manhattan on codes
    uint64_t begin, end;
    const uint32_t* ids;
    const uint8_t* q_codes; // [nq][ad]
    const float* q_off;     // [nq]
    uint32_t nq;
    float* scores;
    int emit_mode;
};

// 8 lanes per candidate, 16 B per lane per step.
template <bool LANEX>
__global__ void __launch_bounds__(256) sq8_group_kernel(const Sq8Params p, const QbEmit emit) {
    const int t = threadIdx.x & 7;
    const uint64_t groups_per_grid = (uint64_t)gridDim.x * (blockDim.x >> 3);
    const uint64_t g0 = (uint64_t)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3);
    const uint64_t n = p.end - p.begin;
    const uint64_t n_iter = (n + groups_per_grid - 1) / groups_per_grid;
    const uint32_t n_chunks = p.ad >> 4;
    for (uint64_t it = 0; it < n_iter; ++it) {
        const uint64_t ci = g0 + it * groups_per_grid;
        const bool valid = ci < n;
        const uint64_t cand = p.begin + (valid ? ci : 0);
        const uint32_t row = p.ids ? p.ids[cand] : (uint32_t)cand;
        const uint4* rp = reinterpret_cast<const uint4*>(p.codes + (size_t)row * p.ad);
        const float v_off = p.voff[row];
        for (uint32_t q = 0; q < p.nq; ++q) {
            const uint4* qp = reinterpret_cast<const uint4*>(p.q_codes + (size_t)q * p.ad);
            const float score = qbs::sq8_raw_group8<LANEX>(rp, qp, n_chunks, t, p.l1);
            // postprocess_score: multiplier * score + query_offset + vector_offset (encoded_vectors_u8.rs:101-103)
            const float sc = __fadd_rn(__fadd_rn(__fmul_rn(p.multiplier, score), p.q_off[q]), v_off);
            if (valid && t == 0) {
                if (p.emit_mode) qb_emit(emit, q, cand, row, sc);
                else p.scores[(size_t)q * n + ci] = sc;
            }
        }
    }
}

// encode_internal_vector (encoded_vectors_u8.rs:715-728): query code = stored code, q_off = v_off - shift
__global__ void sq8_internal_query_kernel(const uint8_t* __restrict__ codes, const float* __restrict__ voff, uint32_t ad, uint32_t id,
                                          float shift, uint8_t* __restrict__ q_code, float* __restrict__ q_off) {
    for (uint32_t i = threadIdx.x; i < ad; i += blockDim.x) q_code[i] = codes[(size_t)id * ad + i];
    if (threadIdx.x == 0) q_off[0] = __fsub_rn(voff[id], shift);
}

// repack [f32 v_off][codes] rows -> code plane + offset plane
__global__ void sq8_repack_kernel(const uint8_t* __restrict__ rows, uint32_t row_bytes, uint32_t ad, uint64_t n, uint8_t* __restrict__ codes,
                                  float* __restrict__ voff) {
    const uint64_t total = n * (uint64_t)(ad >> 2);
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t r = i / (ad >> 2);
        const uint32_t w = (uint32_t)(i % (ad >> 2));
        const uint32_t* src = reinterpret_cast<const uint32_t*>(rows + r * row_bytes);  // row_bytes = 4 + ad, 4-B aligned
        reinterpret_cast<uint32_t*>(codes + r * ad)[w] = src[1 + w];
        if (w == 0) voff[r] = __uint_as_float(src[0]);
    }
}

// ================================================================== PQ ============================
// LUT build (encode_query, encoded_vectors_pq.rs:519-541): grid (m, nq), thread c = centroid
__global__ void __launch_bounds__(256) pq_lut_kernel(const float* __restrict__ q_pre, uint32_t q_stride_f, uint32_t dim, uint32_t m,
                                                     const uint32_t* __restrict__ div, const float* __restrict__ centroids,
                                                     uint32_t n_centroids, int qdist, int invert, float* __restrict__ luts) {
    const uint32_t j = blockIdx.x, q = blockIdx.y;
    const uint32_t s = div[2 * j], e = div[2 * j + 1];
    const float* a = q_pre + (size_t)q * q_stride_f + s;
    for (uint32_t c = threadIdx.x; c < n_centroids; c += blockDim.x) {
        const float* b = centroids + (size_t)c * dim + s;
        float acc = -0.0f;  // DistanceType::distance, encoded_vectors.rs:119-127 (sequential f32 sums)
        if (qdist == QB_QD_DOT || qdist == QB_QD_COSINE) {
            for (uint32_t k = 0; k < e - s; ++k) acc = __fadd_rn(acc, __fmul_rn(a[k], b[k]));
        } else if (qdist == QB_QD_L1) {
            for (uint32_t k = 0; k < e - s; ++k) acc = __fadd_rn(acc, fabsf(__fsub_rn(a[k], b[k])));
        } else {
            for (uint32_t k = 0; k < e - s; ++k) { float d = __fsub_rn(a[k], b[k]); acc = __fadd_rn(acc, __fmul_rn(d, d)); }
        }
        luts[((size_t)q * m + j) * n_centroids + c] = invert ? -acc : acc;
    }
}

struct PqParams {
    const uint8_t* codes;   // [count][stride]
    uint32_t stride, m, n_centroids;
    uint64_t begin, end;
    const uint32_t* ids;
    const float* luts;      // [nq][m][n_centroids]
    uint32_t nq;
    float* scores;
    int emit_mode;
    int lut_in_smem;
};

// score_point_sse (encoded_vectors_pq.rs:411-443): one thread per candidate, LUT of the current query in smem
__global__ void __launch_bounds__(512) pq_scan_kernel(const PqParams p, const QbEmit emit) {
    extern __shared__ __align__(16) float lut_s[];
    const uint64_t n = p.end - p.begin;
    const size_t lut_elems = (size_t)p.m * p.n_centroids;
    const uint32_t K = p.n_centroids;
    const uint32_t m4 = p.m & ~3u;
    for (uint32_t q = 0; q < p.nq; ++q) {
        const float* lut = p.luts + (size_t)q * lut_elems;
        if (p.lut_in_smem) {
            __syncthreads();
            const float4* src = reinterpret_cast<const float4*>(lut);
            float4* dst = reinterpret_cast<float4*>(lut_s);
            for (size_t i = threadIdx.x; i < lut_elems / 4; i += blockDim.x) dst[i] = src[i];
            for (size_t i = (lut_elems & ~(size_t)3) + threadIdx.x; i < lut_elems; i += blockDim.x) lut_s[i] = lut[i];
            __syncthreads();
            lut = lut_s;
        }
        for (uint64_t ci = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; ci < n; ci += (uint64_t)gridDim.x * blockDim.x) {
            const uint64_t cand = p.begin + ci;
            const uint32_t row = p.ids ? p.ids[cand] : (uint32_t)cand;
            const uint8_t* code = p.codes + (size_t)row * p.stride;
            float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
            uint32_t j = 0;
            for (; j + 16 <= m4; j += 16) {
                const uint4 cw = *reinterpret_cast<const uint4*>(code + j);
                const uint32_t w[4] = {cw.x, cw.y, cw.z, cw.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float* l = lut + (size_t)(j + 4 * k) * K;
                    s0 = __fadd_rn(s0, l[w[k] & 255u]);
                    s1 = __fadd_rn(s1, l[K + ((w[k] >> 8) & 255u)]);
                    s2 = __fadd_rn(s2, l[2 * K + ((w[k] >> 16) & 255u)]);
                    s3 = __fadd_rn(s3, l[3 * K + (w[k] >> 24)]);
                }
            }
            for (; j < m4; j += 4) {
                const float* l = lut + (size_t)j * K;
                s0 = __fadd_rn(s0, l[code[j]]);
                s1 = __fadd_rn(s1, l[K + code[j + 1]]);
                s2 = __fadd_rn(s2, l[2 * K + code[j + 2]]);
                s3 = __fadd_rn(s3, l[3 * K + code[j + 3]]);
            }
            float sum = __fadd_rn(__fadd_rn(s0, s2), __fadd_rn(s1, s3));
            for (; j < p.m; ++j) sum = __fadd_rn(sum, lut[(size_t)j * K + code[j]]);
            if (p.emit_mode) qb_emit(emit, q, cand, row, sum);
            else p.scores[(size_t)q * n + ci] = sum;
        }
    }
}


// Two queries per pass: their LUTs are interleaved as float2 in shared memory (2 x m x 256 x 4 B = 192 KB at m = 96), so one
// 64-bit shared load serves both queries and every code byte is decoded once per PAIR.  Same four-lane summation order.
__global__ void __launch_bounds__(1024, 1) pq_scan2_kernel(const PqParams p, const QbEmit emit) {
    extern __shared__ __align__(16) float lut_s[];
    float2* lut2 = reinterpret_cast<float2*>(lut_s);
    const uint64_t n = p.end - p.begin;
    const size_t lut_elems = (size_t)p.m * p.n_centroids;
    const uint32_t K = p.n_centroids;
    const uint32_t m4 = p.m & ~3u;
    for (uint32_t q = 0; q < p.nq; q += 2) {
        const bool two = (q + 1 < p.nq);
        const float* la = p.luts + (size_t)q * lut_elems;
        const float* lb = p.luts + (size_t)(two ? q + 1 : q) * lut_elems;
        __syncthreads();
        for (size_t i = threadIdx.x; i < lut_elems; i += blockDim.x) lut2[i] = make_float2(la[i], lb[i]);
        __syncthreads();
        for (uint64_t ci = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; ci < n; ci += (uint64_t)gridDim.x * blockDim.x) {
            const uint64_t cand = p.begin + ci;
            const uint32_t row = p.ids ? p.ids[cand] : (uint32_t)cand;
            const uint8_t* code = p.codes + (size_t)row * p.stride;
            float2 s0 = make_float2(0.f, 0.f), s1 = s0, s2 = s0, s3 = s0;
            uint32_t j = 0;
            for (; j + 16 <= m4; j += 16) {
                const uint4 cw = *reinterpret_cast<const uint4*>(code + j);
                const uint32_t w[4] = {cw.x, cw.y, cw.z, cw.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float2* l = lut2 + (size_t)(j + 4 * k) * K;
                    const float2 a = l[w[k] & 255u], b = l[K + ((w[k] >> 8) & 255u)], c = l[2 * K + ((w[k] >> 16) & 255u)], d = l[3 * K + (w[k] >> 24)];
                    s0.x = __fadd_rn(s0.x, a.x); s0.y = __fadd_rn(s0.y, a.y);
                    s1.x = __fadd_rn(s1.x, b.x); s1.y = __fadd_rn(s1.y, b.y);
                    s2.x = __fadd_rn(s2.x, c.x); s2.y = __fadd_rn(s2.y, c.y);
                    s3.x = __fadd_rn(s3.x, d.x); s3.y = __fadd_rn(s3.y, d.y);
                }
            }
            for (; j < m4; j += 4) {
                const float2* l = lut2 + (size_t)j * K;
                const float2 a = l[code[j]], b = l[K + code[j + 1]], c = l[2 * K + code[j + 2]], d = l[3 * K + code[j + 3]];
                s0.x = __fadd_rn(s0.x, a.x); s0.y = __fadd_rn(s0.y, a.y);
                s1.x = __fadd_rn(s1.x, b.x); s1.y = __fadd_rn(s1.y, b.y);
                s2.x = __fadd_rn(s2.x, c.x); s2.y = __fadd_rn(s2.y, c.y);
                s3.x = __fadd_rn(s3.x, d.x); s3.y = __fadd_rn(s3.y, d.y);
            }
            float sa = __fadd_rn(__fadd_rn(s0.x, s2.x), __fadd_rn(s1.x, s3.x));
            float sb = __fadd_rn(__fadd_rn(s0.y, s2.y), __fadd_rn(s1.y, s3.y));
            for (; j < p.m; ++j) { const float2 t = lut2[(size_t)j * K + code[j]]; sa = __fadd_rn(sa, t.x); sb = __fadd_rn(sb, t.y); }
            qb_emit(emit, q, cand, row, sa);
            if (two) qb_emit(emit, q + 1, cand, row, sb);
        }
    }
}

// Four queries per pass on a CTA PAIR (thread-block cluster of 2): the four LUTs are interleaved as float4, so ONE 16-byte shared
// load serves four queries and — more to the point on random codes — a quarter-warp's 8 gathers spread over 8 sixteen-byte bank
// groups collide less than 32 four-byte gathers over 32 banks.  Four interleaved LUTs are 4 x m x 256 x 4 B = 384 KB at m = 96:
// CTA 0 holds chunks [0, m/2), CTA 1 chunks [m/2, m).  CTA 0 runs the first half of every row's four-lane accumulation and hands the
// 16 partial sums (4 lanes x 4 queries) to CTA 1 through DISTRIBUTED SHARED MEMORY; CTA 1 continues the very same f32 chains — lane
// k keeps adding chunks j = k (mod 4) in ascending j — and finishes with (s0+s2)+(s1+s3): score_point_sse's order exactly
// (encoded_vectors_pq.rs:411-443).  The hand-off is per WARP: thread t of warp w in CTA 0 feeds thread t of warp w in CTA 1 through one
// 64-byte slot: the producer's st.async stores complete transaction bytes on the consumer warp's `full` mbarrier, the consumer's remote
// arrive on the producer warp's `empty` mbarrier frees the slot, so the sixteen warp pairs drift freely — no fence, no CTA-wide
// or cluster-wide barrier inside the row loop — and the consumer frees the slot as soon as it has the partial sums in registers.
// Requires m % 32 == 0 (16-byte code loads per half), m <= 96 (LUT half <= 192 KB).  The launcher walks the code plane in L2-sized
// row blocks and runs ALL query quads over a block before moving on, so HBM sees every code byte once per batch.
constexpr int PQ4_THREADS = 512;
constexpr int PQ4_WARPS = PQ4_THREADS / 32;

__device__ __forceinline__ uint32_t pq4_map_to_cta(const void* smem_ptr, uint32_t cta) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(qb_smem_u32(smem_ptr)), "r"(cta));
    return r;
}
__device__ __forceinline__ void pq4_remote_arrive(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ void pq4_wait_cluster(uint64_t* bar, uint32_t parity) {   // acquire at cluster scope: the data came from the peer CTA
    uint32_t ok = 0;
    long long t0 = 0;
    for (;;) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(qb_smem_u32(bar)), "r"(parity) : "memory");
        if (ok) return;
        if (t0 == 0) t0 = clock64();
        else if (clock64() - t0 > 8000000000ll) __trap();   // a protocol bug must not hang the GPU
    }
}
// asynchronous remote store that credits its 16 bytes to the CONSUMER's mbarrier (st.async ... complete_tx): the producer needs neither
// a fence nor an arrive — the consumer arms the barrier with the 2048 bytes a warp hands over and waits for them
__device__ __forceinline__ void pq4_st_async_f4(uint32_t cluster_addr, float4 v, uint32_t cluster_bar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(cluster_addr), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w), "r"(cluster_bar)
                 : "memory");
}

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(PQ4_THREADS, 1) pq_scan4_kernel(const PqParams p, const QbEmit emit) {
    namespace cg = cooperative_groups;
    extern __shared__ __align__(16) float lut_s[];
    cg::cluster_group cluster = cg::this_cluster();
    const uint32_t rank = cluster.block_rank();
    const uint32_t K = p.n_centroids, mh = p.m >> 1, j0 = rank * mh;
    float4* lut4 = reinterpret_cast<float4*>(lut_s);                 // [mh][K]
    float4* hand = lut4 + (size_t)mh * K;                            // [4][PQ4_THREADS]   (CTA 1's copy is the one in use)
    uint64_t* full = reinterpret_cast<uint64_t*>(hand + 4 * PQ4_THREADS);   // [PQ4_WARPS] in CTA 1: "warp w's partial sums have landed"
    uint64_t* empty = full + PQ4_WARPS;                                     // [PQ4_WARPS] in CTA 0: "warp w's slot may be overwritten"
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid < PQ4_WARPS) { qb_mbar_init(&full[tid], 1); qb_mbar_init(&empty[tid], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    cluster.sync();                                                  // both CTAs' barriers exist before any remote arrive
    const uint32_t hand_remote = pq4_map_to_cta(hand, 1);            // CTA 0 writes into CTA 1's slot
    const uint32_t full_remote = pq4_map_to_cta(&full[warp], 1);
    const uint32_t empty_remote = pq4_map_to_cta(&empty[warp], 0);
    const uint64_t n = p.end - p.begin;
    const uint64_t n_tiles = (n + PQ4_THREADS - 1) / PQ4_THREADS;
    const uint32_t cid = blockIdx.x >> 1, n_clusters = gridDim.x >> 1;
    const size_t lut_elems = (size_t)p.m * K;
    uint32_t it = 0;                                                 // hand-offs done by this warp so far (both CTAs count alike)
    for (uint32_t q0 = 0; q0 < p.nq; q0 += 4) {
        // ---- interleaved LUT half of this CTA: lut4[jl][c] = (lut_q0, lut_q0+1, lut_q0+2, lut_q0+3)[j0 + jl][c]
        const float* l0 = p.luts + (size_t)q0 * lut_elems + (size_t)j0 * K;
        const float* l1 = (q0 + 1 < p.nq) ? l0 + lut_elems : l0;
        const float* l2 = (q0 + 2 < p.nq) ? l0 + 2 * lut_elems : l0;
        const float* l3 = (q0 + 3 < p.nq) ? l0 + 3 * lut_elems : l0;
        __syncthreads();                                             // every warp of this CTA is done with the previous quad's LUT
        for (uint32_t i = tid; i < mh * K; i += PQ4_THREADS) lut4[i] = make_float4(l0[i], l1[i], l2[i], l3[i]);
        __syncthreads();
        for (uint64_t t = cid; t < n_tiles; t += n_clusters, ++it) {
            const uint64_t ci = t * PQ4_THREADS + tid;
            const bool valid = ci < n;
            const uint64_t cand = p.begin + (valid ? ci : 0);
            const uint8_t* code = p.codes + (size_t)cand * p.stride + j0;
            uint4 cw[3];                                             // m <= 96: at most 48 code bytes per half, fetched before any waiting
#pragma unroll
            for (int w = 0; w < 3; ++w) cw[w] = (w * 16u < mh) ? *reinterpret_cast<const uint4*>(code + w * 16) : make_uint4(0, 0, 0, 0);
            float4 s0, s1, s2, s3;
            if (rank == 0) {
                s0 = s1 = s2 = s3 = make_float4(0.f, 0.f, 0.f, 0.f);
            } else {
                if (lane == 0) qb_mbar_arrive_expect_tx(&full[warp], 32u * 64u);   // arm: 32 lanes x 4 float4 arrive through st.async
                pq4_wait_cluster(&full[warp], it & 1u);             // this warp's partial sums of tile `it` have landed
                s0 = hand[0 * PQ4_THREADS + tid]; s1 = hand[1 * PQ4_THREADS + tid]; s2 = hand[2 * PQ4_THREADS + tid]; s3 = hand[3 * PQ4_THREADS + tid];
                __syncwarp();
                if (lane == 0) pq4_remote_arrive(empty_remote);      // slot free again: the producer warp may run ahead into the next tile
            }
#pragma unroll
            for (int w = 0; w < 3; ++w) {
                if (w * 16u >= mh) break;
                const uint32_t wd[4] = {cw[w].x, cw[w].y, cw[w].z, cw[w].w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float4* l = lut4 + (size_t)(w * 16 + 4 * k) * K;
                    const float4 a = l[wd[k] & 255u], b = l[K + ((wd[k] >> 8) & 255u)], c = l[2 * K + ((wd[k] >> 16) & 255u)], d = l[3 * K + (wd[k] >> 24)];
                    s0.x = __fadd_rn(s0.x, a.x); s0.y = __fadd_rn(s0.y, a.y); s0.z = __fadd_rn(s0.z, a.z); s0.w = __fadd_rn(s0.w, a.w);
                    s1.x = __fadd_rn(s1.x, b.x); s1.y = __fadd_rn(s1.y, b.y); s1.z = __fadd_rn(s1.z, b.z); s1.w = __fadd_rn(s1.w, b.w);
                    s2.x = __fadd_rn(s2.x, c.x); s2.y = __fadd_rn(s2.y, c.y); s2.z = __fadd_rn(s2.z, c.z); s2.w = __fadd_rn(s2.w, c.w);
                    s3.x = __fadd_rn(s3.x, d.x); s3.y = __fadd_rn(s3.y, d.y); s3.z = __fadd_rn(s3.z, d.z); s3.w = __fadd_rn(s3.w, d.w);
                }
            }
            if (rank == 0) {
                if (it > 0) pq4_wait_cluster(&empty[warp], (it - 1) & 1u);   // the consumer has taken tile it - 1 out of the slot
                pq4_st_async_f4(hand_remote + (0 * PQ4_THREADS + tid) * 16u, s0, full_remote);
                pq4_st_async_f4(hand_remote + (1 * PQ4_THREADS + tid) * 16u, s1, full_remote);
                pq4_st_async_f4(hand_remote + (2 * PQ4_THREADS + tid) * 16u, s2, full_remote);
                pq4_st_async_f4(hand_remote + (3 * PQ4_THREADS + tid) * 16u, s3, full_remote);
            } else if (valid) {
                const uint32_t row = (uint32_t)cand;
                const float r0 = __fadd_rn(__fadd_rn(s0.x, s2.x), __fadd_rn(s1.x, s3.x));
                const float r1 = __fadd_rn(__fadd_rn(s0.y, s2.y), __fadd_rn(s1.y, s3.y));
                const float r2 = __fadd_rn(__fadd_rn(s0.z, s2.z), __fadd_rn(s1.z, s3.z));
                const float r3 = __fadd_rn(__fadd_rn(s0.w, s2.w), __fadd_rn(s1.w, s3.w));
                qb_emit(emit, q0, cand, row, r0);
                if (q0 + 1 < p.nq) qb_emit(emit, q0 + 1, cand, row, r1);
                if (q0 + 2 < p.nq) qb_emit(emit, q0 + 2, cand, row, r2);
                if (q0 + 3 < p.nq) qb_emit(emit, q0 + 3, cand, row, r3);
            }
        }
    }
    cluster.sync();   // a CTA's shared memory (slot, barriers) must outlive its peer's last remote access
}

// ---------------------------------------------------------------- eight queries per pass: bf16 LUT prefilter + exact rescoring
// The four-query kernel above sits on the shared-memory pipe (random 16-byte gathers, ~10 wavefronts per LDS.128): the only way to more
// lookups per second is more QUERIES per wavefront.  Eight bf16 table entries fit the same 16 bytes, so one gather serves eight queries —
// but a bf16 table cannot give the reference's f32 sums.  It does not have to: the scan only has to find every row whose EXACT score
// reaches the query's threshold.  With  S_q = sum_j max_c |lut_q[j][c]|  the prefilter's score differs from the exact f32 sum by at most
//   2^-9 S_q (round-to-nearest bf16 of every entry) + 2 * m * 2^-24 S_q (both f32 accumulations, any order)  <  (2^-9 + 2^-15) S_q =: margin_q
// so the kernel emits every row with  approx >= thr_q - margin_q  (a superset of the rows the exact filter would pass), a second kernel
// re-scores exactly those survivors with the f32 tables in score_point_sse's order (four lanes, (s0+s2)+(s1+s3)) and rewrites their keys,
// and the selection runs on exact keys: results are bit-identical to the single-query kernel's.  Non-finite table entries make the
// margin inf / NaN: every row passes, the candidate buffer overflows and the host's rerun takes the exact path.
// Layout as above (CTA pair, chunks split, per-warp DSMEM hand-off), except that the approximate sum has no order to keep: one f32 per
// query crosses the pair (32 bytes per thread instead of 256).
constexpr int PQ8_THREADS = 512;
constexpr int PQ8_WARPS = PQ8_THREADS / 32;

__global__ void __launch_bounds__(256) pq8_margin_kernel(const float* __restrict__ luts, uint32_t m, uint32_t K, const float* __restrict__ thr,
                                                         float* __restrict__ thr_adj) {
    __shared__ float s_part[8];
    const uint32_t q = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* lut = luts + (size_t)q * m * K;
    float sum = 0.f;
    for (uint32_t j = warp; j < m; j += 8) {
        float mx = 0.f;
        bool bad = false;
        for (uint32_t c = lane; c < K; c += 32) { const float v = fabsf(lut[(size_t)j * K + c]); bad |= !(v <= 3.0e38f); mx = fmaxf(mx, v); }
        for (int o = 16; o; o >>= 1) { mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); bad |= __shfl_xor_sync(0xffffffffu, (int)bad, o) != 0; }
        sum = __fadd_ru(sum, bad ? __int_as_float(0x7f800000) : mx);      // NaN / inf / beyond bf16's range: no finite margin exists
    }
    if (lane == 0) s_part[warp] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        float S = 0.f;
        for (int w = 0; w < 8; ++w) S = __fadd_ru(S, s_part[w]);
        const float margin = __fadd_ru(__fmul_ru(S, 0x1.04p-9f), 1.0e-37f);   // (2^-9 + 2^-15) S, rounded up, plus the denormal floor
        thr_adj[q] = __fsub_rd(thr[q], margin);
    }
}

__device__ __forceinline__ void pq8_st_async_f4(uint32_t cluster_addr, float4 v, uint32_t cluster_bar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(cluster_addr), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w), "r"(cluster_bar)
                 : "memory");
}
__device__ __forceinline__ uint32_t pq8_pack_bf16(float lo, float hi) {   // round-to-nearest-even bf16 pair, lo in bits [0,16)
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ void pq8_acc(float (&acc)[8], const uint4 v) {
    acc[0] = __fadd_rn(acc[0], __uint_as_float(v.x << 16)); acc[1] = __fadd_rn(acc[1], __uint_as_float(v.x & 0xFFFF0000u));
    acc[2] = __fadd_rn(acc[2], __uint_as_float(v.y << 16)); acc[3] = __fadd_rn(acc[3], __uint_as_float(v.y & 0xFFFF0000u));
    acc[4] = __fadd_rn(acc[4], __uint_as_float(v.z << 16)); acc[5] = __fadd_rn(acc[5], __uint_as_float(v.z & 0xFFFF0000u));
    acc[6] = __fadd_rn(acc[6], __uint_as_float(v.w << 16)); acc[7] = __fadd_rn(acc[7], __uint_as_float(v.w & 0xFFFF0000u));
}

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(PQ8_THREADS, 1) pq_scan8_kernel(const PqParams p, const QbEmit emit /* thr = thr - margin */) {
    namespace cg = cooperative_groups;
    extern __shared__ __align__(16) float lut_s[];
    cg::cluster_group cluster = cg::this_cluster();
    const uint32_t rank = cluster.block_rank();
    const uint32_t K = p.n_centroids, mh = p.m >> 1, j0 = rank * mh;
    uint4* lut8 = reinterpret_cast<uint4*>(lut_s);                   // [mh][K] x 8 bf16 (queries q0 .. q0+7)
    float4* hand = reinterpret_cast<float4*>(lut8 + (size_t)mh * K); // [2][PQ8_THREADS]   (CTA 1's copy is the one in use)
    uint64_t* full = reinterpret_cast<uint64_t*>(hand + 2 * PQ8_THREADS);
    uint64_t* empty = full + PQ8_WARPS;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid < PQ8_WARPS) { qb_mbar_init(&full[tid], 1); qb_mbar_init(&empty[tid], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    cluster.sync();
    const uint32_t hand_remote = pq4_map_to_cta(hand, 1);
    const uint32_t full_remote = pq4_map_to_cta(&full[warp], 1);
    const uint32_t empty_remote = pq4_map_to_cta(&empty[warp], 0);
    const uint64_t n = p.end - p.begin;
    const uint64_t n_tiles = (n + PQ8_THREADS - 1) / PQ8_THREADS;
    const uint32_t cid = blockIdx.x >> 1, n_clusters = gridDim.x >> 1;
    const size_t lut_elems = (size_t)p.m * K;
    uint32_t it = 0;
    for (uint32_t q0 = 0; q0 < p.nq; q0 += 8) {
        const float* l0 = p.luts + (size_t)q0 * lut_elems + (size_t)j0 * K;
        size_t qo[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) qo[i] = (q0 + i < p.nq) ? (size_t)i * lut_elems : 0;   // missing queries of the last group: query q0 again (never emitted)
        __syncthreads();
        for (uint32_t i = tid; i < mh * K; i += PQ8_THREADS) {
            uint4 v;
            v.x = pq8_pack_bf16(l0[qo[0] + i], l0[qo[1] + i]); v.y = pq8_pack_bf16(l0[qo[2] + i], l0[qo[3] + i]);
            v.z = pq8_pack_bf16(l0[qo[4] + i], l0[qo[5] + i]); v.w = pq8_pack_bf16(l0[qo[6] + i], l0[qo[7] + i]);
            lut8[i] = v;
        }
        __syncthreads();
        for (uint64_t t = cid; t < n_tiles; t += n_clusters, ++it) {
            const uint64_t ci = t * PQ8_THREADS + tid;
            const bool valid = ci < n;
            const uint64_t cand = p.begin + (valid ? ci : 0);
            const uint8_t* code = p.codes + (size_t)cand * p.stride + j0;
            uint4 cw[3];
#pragma unroll
            for (int w = 0; w < 3; ++w) cw[w] = (w * 16u < mh) ? *reinterpret_cast<const uint4*>(code + w * 16) : make_uint4(0, 0, 0, 0);
            float a[8], b[8];                                        // two independent chains per query (the order is free here)
#pragma unroll
            for (int i = 0; i < 8; ++i) a[i] = b[i] = 0.f;
#pragma unroll
            for (int w = 0; w < 3; ++w) {
                if (w * 16u >= mh) break;
                const uint32_t wd[4] = {cw[w].x, cw[w].y, cw[w].z, cw[w].w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint4* l = lut8 + (size_t)(w * 16 + 4 * k) * K;
                    const uint4 v0 = l[wd[k] & 255u], v1 = l[K + ((wd[k] >> 8) & 255u)], v2 = l[2 * K + ((wd[k] >> 16) & 255u)], v3 = l[3 * K + (wd[k] >> 24)];
                    pq8_acc(a, v0); pq8_acc(b, v1); pq8_acc(a, v2); pq8_acc(b, v3);
                }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) a[i] = __fadd_rn(a[i], b[i]);
            if (rank == 0) {
                if (it > 0) pq4_wait_cluster(&empty[warp], (it - 1) & 1u);
                pq8_st_async_f4(hand_remote + (0 * PQ8_THREADS + tid) * 16u, make_float4(a[0], a[1], a[2], a[3]), full_remote);
                pq8_st_async_f4(hand_remote + (1 * PQ8_THREADS + tid) * 16u, make_float4(a[4], a[5], a[6], a[7]), full_remote);
            } else {
                if (lane == 0) qb_mbar_arrive_expect_tx(&full[warp], 32u * 32u);
                pq4_wait_cluster(&full[warp], it & 1u);
                const float4 h0 = hand[0 * PQ8_THREADS + tid], h1 = hand[1 * PQ8_THREADS + tid];
                __syncwarp();
                if (lane == 0) pq4_remote_arrive(empty_remote);
                if (valid) {
                    const uint32_t row = (uint32_t)cand;
                    const float r[8] = {__fadd_rn(a[0], h0.x), __fadd_rn(a[1], h0.y), __fadd_rn(a[2], h0.z), __fadd_rn(a[3], h0.w),
                                        __fadd_rn(a[4], h1.x), __fadd_rn(a[5], h1.y), __fadd_rn(a[6], h1.z), __fadd_rn(a[7], h1.w)};
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        if (q0 + i < p.nq) qb_emit(emit, q0 + i, cand, row, r[i]);
                }
            }
        }
    }
    cluster.sync();
}

// ---------------------------------------------------------------- sixteen queries per pass: u8 tables, integer prefilter
// One step further along the same line: SIXTEEN one-byte table entries per 16-byte gather.  Per query the tables are quantised with one
// step for all chunks, u[j][c] = rint((lut[j][c] - min_j) / step), step = max_j(max_c lut[j][c] - min_j) / 255, so that
//   | step * sum_j u[j][code_j] + sum_j min_j  -  sum_j lut[j][code_j] |  <=  m * step * (1/2 + 2^-14)          (real arithmetic)
// and a row whose EXACT f32 score reaches thr_q has  sum_j u >= T_q := floor((thr_q - sum_j min_j - margin_q) / step) - 1  with
// margin_q = m * step * (1/2 + 2^-14) + 4 m 2^-24 sum_j max_c |lut[j][c]|  (quantisation + every f32 rounding on either side, all
// evaluated in double on the device).  The hot loop is integer only: per gather two PRMTs spread the sixteen bytes over eight registers
// of two u16 lanes (sums <= 96 * 255 fit), the accumulators START at 0x8000 - T_q, so "passes" is bit 15 of a lane and the whole
// 16-query test is an OR and an AND.  Survivors are appended without a score and re-scored exactly (pq_rescore_kernel) as above.
// The interleaved u8 tables (nq x m x 256 bytes) and the biases are built once per scan by pq16_prep_kernel; a CTA copies its half
// (192 KB, contiguous) per query group.  Codes of the next row tile are fetched while the current one is gathered.
constexpr int PQ16_THREADS = 512;
constexpr int PQ16_WARPS = PQ16_THREADS / 32;

// one block per (padded) query: tables -> interleaved u8 planes tab16[group][j][c][16], bias[q] = 0x8000 - T_q (u16 in a u32)
__global__ void __launch_bounds__(256) pq16_prep_kernel(const float* __restrict__ luts, uint32_t nq, uint32_t m, uint32_t K, const float* __restrict__ thr,
                                                        uint8_t* __restrict__ tab16, uint32_t* __restrict__ bias) {
    __shared__ float s_min[128], s_rng[8], s_abs[8];
    __shared__ double s_base[8];
    __shared__ int s_bad;
    const uint32_t q = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t* dst = tab16 + ((size_t)(q >> 4) * m * K) * 16 + (q & 15);
    if (q >= nq) {                                                   // padding of the last group: never passes
        for (uint32_t i = threadIdx.x; i < m * K; i += blockDim.x) dst[(size_t)i * 16] = 0;
        if (threadIdx.x == 0) bias[q] = 0u;
        return;
    }
    const float* lut = luts + (size_t)q * m * K;
    if (threadIdx.x == 0) s_bad = 0;
    __syncthreads();
    float rng_w = 0.f, abs_w = 0.f;
    double base_w = 0.0;
    for (uint32_t j = warp; j < m; j += 8) {
        float mn = __int_as_float(0x7f800000), mx = -mn, ab = 0.f;
        bool bad = false;
        for (uint32_t c = lane; c < K; c += 32) { const float v = lut[(size_t)j * K + c]; bad |= !(fabsf(v) <= 3.0e38f); mn = fminf(mn, v); mx = fmaxf(mx, v); ab = fmaxf(ab, fabsf(v)); }
        for (int o = 16; o; o >>= 1) {
            mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); ab = fmaxf(ab, __shfl_xor_sync(0xffffffffu, ab, o));
            bad |= __shfl_xor_sync(0xffffffffu, (int)bad, o) != 0;
        }
        if (bad && lane == 0) s_bad = 1;
        if (lane == 0 && j < 128) s_min[j] = mn;
        rng_w = fmaxf(rng_w, mx - mn); abs_w += ab; base_w += (double)mn;
    }
    if (lane == 0) { s_rng[warp] = rng_w; s_abs[warp] = abs_w; s_base[warp] = base_w; }
    __syncthreads();
    float rng = 0.f;
    double A = 0.0, base = 0.0;
    for (int w = 0; w < 8; ++w) { rng = fmaxf(rng, s_rng[w]); A += (double)s_abs[w] * 1.0001; base += s_base[w]; }
    const bool bad = s_bad != 0 || !(rng <= 3.0e38f) || !(A <= 3.0e38);      // a sum of m entries must stay finite, too
    const float step = bad ? 1.f : fmaxf(rng / 255.f, 1.0e-30f);
    const float inv = 1.f / step;
    for (uint32_t i = threadIdx.x; i < m * K; i += blockDim.x) {
        const float t = __fmul_rn(__fsub_rn(lut[i], s_min[i / K]), inv);
        dst[(size_t)i * 16] = bad ? (uint8_t)0 : (uint8_t)fminf(fmaxf(rintf(t), 0.f), 255.f);
    }
    if (threadIdx.x == 0) {
        uint32_t b;
        const float th = thr[q];
        if (bad || !(fabsf(th) <= 3.0e38f)) {
            b = (th == __int_as_float(0x7f800000) && !bad) ? 0u : 0x8000u;    // +inf threshold: nothing finite reaches it; NaN / -inf / bad tables: everything passes
        } else {
            const double margin = (double)m * (double)step * (0.5 + 1.0 / 16384.0) + 4.0 * (double)m * 5.9604644775390625e-8 * A;
            const double T = floor(((double)th - base - margin) / (double)step) - 1.0;
            b = T <= 0.0 ? 0x8000u : (T >= 32768.0 ? 0u : 0x8000u - (uint32_t)T);
        }
        bias[q] = b;
    }
}

__device__ __forceinline__ void pq16_st_async_u4(uint32_t cluster_addr, uint4 v, uint32_t cluster_bar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(cluster_addr), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w), "r"(cluster_bar)
                 : "memory");
}

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(PQ16_THREADS, 1) pq_scan16_kernel(const PqParams p, const QbEmit emit, const uint8_t* __restrict__ tab16,
                                                                                              const uint32_t* __restrict__ bias) {
    namespace cg = cooperative_groups;
    extern __shared__ __align__(16) float lut_s[];
    cg::cluster_group cluster = cg::this_cluster();
    const uint32_t rank = cluster.block_rank();
    const uint32_t K = p.n_centroids, mh = p.m >> 1, j0 = rank * mh;
    uint4* lut16 = reinterpret_cast<uint4*>(lut_s);                    // [mh][K] x 16 u8 (queries q0 .. q0+15)
    float4* hand = reinterpret_cast<float4*>(lut16 + (size_t)mh * K);  // [2][PQ16_THREADS]   (CTA 1's copy is the one in use)
    uint64_t* full = reinterpret_cast<uint64_t*>(hand + 2 * PQ16_THREADS);
    uint64_t* empty = full + PQ16_WARPS;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid < PQ16_WARPS) { qb_mbar_init(&full[tid], 1); qb_mbar_init(&empty[tid], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    cluster.sync();
    const uint32_t hand_remote = pq4_map_to_cta(hand, 1);
    const uint32_t full_remote = pq4_map_to_cta(&full[warp], 1);
    const uint32_t empty_remote = pq4_map_to_cta(&empty[warp], 0);
    const uint64_t n = p.end - p.begin;
    const uint64_t n_tiles = (n + PQ16_THREADS - 1) / PQ16_THREADS;
    const uint32_t cid = blockIdx.x >> 1, n_clusters = gridDim.x >> 1;
    uint32_t it = 0;
    for (uint32_t q0 = 0; q0 < p.nq; q0 += 16) {
        const uint4* src = reinterpret_cast<const uint4*>(tab16) + ((size_t)(q0 >> 4) * p.m + j0) * K;
        __syncthreads();
        for (uint32_t i = tid; i < mh * K; i += PQ16_THREADS) lut16[i] = src[i];
        uint32_t init[8];                                            // accumulator layout: word 2k = queries (4k, 4k+2), word 2k+1 = (4k+1, 4k+3)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            init[2 * k] = rank ? 0u : (bias[q0 + 4 * k] | (bias[q0 + 4 * k + 2] << 16));
            init[2 * k + 1] = rank ? 0u : (bias[q0 + 4 * k + 1] | (bias[q0 + 4 * k + 3] << 16));
        }
        __syncthreads();
        uint4 cw[3], cn[3];
        {
            const uint64_t ci = (uint64_t)cid * PQ16_THREADS + tid;
            const uint8_t* code = p.codes + (size_t)(p.begin + (ci < n ? ci : 0)) * p.stride + j0;
#pragma unroll
            for (int w = 0; w < 3; ++w) cn[w] = (w * 16u < mh && cid < n_tiles) ? *reinterpret_cast<const uint4*>(code + w * 16) : make_uint4(0, 0, 0, 0);
        }
        for (uint64_t t = cid; t < n_tiles; t += n_clusters, ++it) {
            const uint64_t ci = t * PQ16_THREADS + tid;
            const bool valid = ci < n;
            const uint64_t cand = p.begin + (valid ? ci : 0);
#pragma unroll
            for (int w = 0; w < 3; ++w) cw[w] = cn[w];
            if (t + n_clusters < n_tiles) {                          // next tile's codes: in flight while this tile gathers
                const uint64_t cj = (t + n_clusters) * PQ16_THREADS + tid;
                const uint8_t* code = p.codes + (size_t)(p.begin + (cj < n ? cj : 0)) * p.stride + j0;
#pragma unroll
                for (int w = 0; w < 3; ++w) cn[w] = (w * 16u < mh) ? *reinterpret_cast<const uint4*>(code + w * 16) : make_uint4(0, 0, 0, 0);
            }
            uint32_t a[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) a[i] = init[i];
#pragma unroll
            for (int w = 0; w < 3; ++w) {
                if (w * 16u >= mh) break;
                const uint32_t wd[4] = {cw[w].x, cw[w].y, cw[w].z, cw[w].w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint4* l = lut16 + (size_t)(w * 16 + 4 * k) * K;
                    const uint4 v[4] = {l[wd[k] & 255u], l[K + ((wd[k] >> 8) & 255u)], l[2 * K + ((wd[k] >> 16) & 255u)], l[3 * K + (wd[k] >> 24)]};
#pragma unroll
                    for (int x = 0; x < 4; ++x) {
                        a[0] += __byte_perm(v[x].x, 0, 0x4240); a[1] += __byte_perm(v[x].x, 0, 0x4341);
                        a[2] += __byte_perm(v[x].y, 0, 0x4240); a[3] += __byte_perm(v[x].y, 0, 0x4341);
                        a[4] += __byte_perm(v[x].z, 0, 0x4240); a[5] += __byte_perm(v[x].z, 0, 0x4341);
                        a[6] += __byte_perm(v[x].w, 0, 0x4240); a[7] += __byte_perm(v[x].w, 0, 0x4341);
                    }
                }
            }
            if (rank == 0) {
                if (it > 0) pq4_wait_cluster(&empty[warp], (it - 1) & 1u);
                pq16_st_async_u4(hand_remote + (0 * PQ16_THREADS + tid) * 16u, make_uint4(a[0], a[1], a[2], a[3]), full_remote);
                pq16_st_async_u4(hand_remote + (1 * PQ16_THREADS + tid) * 16u, make_uint4(a[4], a[5], a[6], a[7]), full_remote);
            } else {
                if (lane == 0) qb_mbar_arrive_expect_tx(&full[warp], 32u * 32u);
                pq4_wait_cluster(&full[warp], it & 1u);
                const uint4 h0 = reinterpret_cast<const uint4*>(hand)[0 * PQ16_THREADS + tid], h1 = reinterpret_cast<const uint4*>(hand)[1 * PQ16_THREADS + tid];
                __syncwarp();
                if (lane == 0) pq4_remote_arrive(empty_remote);
                a[0] += h0.x; a[1] += h0.y; a[2] += h0.z; a[3] += h0.w; a[4] += h1.x; a[5] += h1.y; a[6] += h1.z; a[7] += h1.w;
                const uint32_t any = (a[0] | a[1] | a[2] | a[3] | a[4] | a[5] | a[6] | a[7]) & 0x80008000u;
                if (any && valid) {
                    const uint32_t row = (uint32_t)cand;
                    if (!qb_is_deleted(emit, row)) {
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const uint32_t q = q0 + 4 * (i >> 1) + (i & 1) + 2 * h;
                                if ((a[i] >> (15 + 16 * h)) & 1u) {
                                    const unsigned int pos = atomicAdd(&emit.cnt[q], 1u);
                                    if (pos < emit.cap) emit.cand[(unsigned long long)q * emit.cap + pos] = qb_pack_key(0.f, row + emit.id_base);
                                }
                            }
                        }
                    }
                }
            }
        }
    }
    cluster.sync();
}

// exact f32 score of every survivor of the prefilter, in score_point_sse's order; the candidate's key is rewritten in place
__global__ void __launch_bounds__(128) pq_rescore_kernel(const PqParams p, const QbEmit emit) {
    const uint32_t q = blockIdx.y;
    const unsigned long long cnt = min((unsigned long long)emit.cnt[q], emit.cap);
    const uint32_t K = p.n_centroids, m4 = p.m & ~3u;
    const float* lut = p.luts + (size_t)q * p.m * K;
    for (unsigned long long pos = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; pos < cnt; pos += (unsigned long long)gridDim.x * blockDim.x) {
        unsigned long long* slot = emit.cand + (unsigned long long)q * emit.cap + pos;
        const uint32_t id = qb_key_id(*slot);
        const uint8_t* code = p.codes + (size_t)(id - emit.id_base) * p.stride;
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        uint32_t j = 0;
        for (; j < m4; j += 4) {
            const float* l = lut + (size_t)j * K;
            s0 = __fadd_rn(s0, l[code[j]]);
            s1 = __fadd_rn(s1, l[K + code[j + 1]]);
            s2 = __fadd_rn(s2, l[2 * K + code[j + 2]]);
            s3 = __fadd_rn(s3, l[3 * K + code[j + 3]]);
        }
        float sum = __fadd_rn(__fadd_rn(s0, s2), __fadd_rn(s1, s3));
        for (; j < p.m; ++j) sum = __fadd_rn(sum, lut[(size_t)j * K + code[j]]);
        *slot = qb_pack_key(sum, id);
    }
}

// score_internal (encoded_vectors_pq.rs:574-618): decode both codes through the centroids; single pair
__global__ void pq_score_internal_kernel(const uint8_t* __restrict__ codes, uint32_t stride, uint32_t m, const uint32_t* __restrict__ div,
                                         const float* __restrict__ centroids, uint32_t dim, int qdist, int invert, uint32_t a, uint32_t b,
                                         float* __restrict__ out) {
    if (threadIdx.x != 0) return;
    float total = -0.0f;
    for (uint32_t j = 0; j < m; ++j) {
        const uint32_t s = div[2 * j], e = div[2 * j + 1];
        const float* x = centroids + (size_t)codes[(size_t)a * stride + j] * dim + s;
        const float* y = centroids + (size_t)codes[(size_t)b * stride + j] * dim + s;
        float acc = -0.0f;
        if (qdist == QB_QD_DOT || qdist == QB_QD_COSINE) {
            for (uint32_t k = 0; k < e - s; ++k) acc = __fadd_rn(acc, __fmul_rn(x[k], y[k]));
        } else if (qdist == QB_QD_L1) {
            for (uint32_t k = 0; k < e - s; ++k) acc = __fadd_rn(acc, fabsf(__fsub_rn(x[k], y[k])));
        } else {
            for (uint32_t k = 0; k < e - s; ++k) { float d = __fsub_rn(x[k], y[k]); acc = __fadd_rn(acc, __fmul_rn(d, d)); }
        }
        total = __fadd_rn(total, acc);
    }
    out[0] = invert ? -total : total;
}

// ================================================================== BQ ============================
__device__ __forceinline__ void bq_two_bits(float value, const float* ms, bool& b1, bool& b2) {  // :636-671
    if (!ms) { b1 = b2 = value > 0.0f; return; }
    const float mean = ms[0], sd = ms[1];
    if (sd < 1.1920929e-07f) { b1 = value > 0.0f; b2 = false; return; }
    const float vz = __fdiv_rn(__fsub_rn(value, mean), sd);
    const float SIG = 2.0f / 3.0f;
    if (vz <= -SIG) { b1 = false; b2 = false; }
    else if (vz < SIG) { b1 = true; b2 = false; }
    else { b1 = true; b2 = true; }
}

// one block per query.  Binary query (SameAsStorage) or transposed scalar query (4 / 8 bits).
__global__ void __launch_bounds__(256) bq_encode_query_kernel(const float* __restrict__ q_pre, uint32_t q_stride_f, uint32_t dim, int enc,
                                                              int bits, const float* __restrict__ mean_std, uint32_t row_bytes,
                                                              uint32_t* __restrict__ out /* [nq][row_bytes*bits/4] */) {
    __shared__ float s_max[256];
    const uint32_t q = blockIdx.x;
    const float* src = q_pre + (size_t)q * q_stride_f;
    const uint32_t words = row_bytes * (uint32_t)bits / 4;
    uint32_t* dst = out + (size_t)q * words;
    for (uint32_t i = threadIdx.x; i < words; i += blockDim.x) dst[i] = 0u;
    __syncthreads();
    if (bits == 1) {
        for (uint32_t i = threadIdx.x; i < dim; i += blockDim.x) {
            const float v = src[i];
            if (enc == QB_BQ_ONE_BIT) {
                if (v > 0.0f) atomicOr(&dst[i >> 5], 1u << (i & 31));
            } else {
                bool b1, b2;
                bq_two_bits(v, mean_std ? mean_std + 2 * (size_t)i : nullptr, b1, b2);
                if (b1) atomicOr(&dst[i >> 5], 1u << (i & 31));
                if (b2) {
                    const uint32_t jx = (enc == QB_BQ_TWO_BITS) ? dim + i : dim + i / 2;
                    atomicOr(&dst[jx >> 5], 1u << (jx & 31));
                }
            }
        }
        return;
    }
    // extended query (encode_scalar_query_vector :692-720)
    uint32_t ext = dim;
    if (enc == QB_BQ_TWO_BITS) ext = 2 * dim;
    else if (enc == QB_BQ_ONE_AND_HALF_BITS) ext = dim + (dim + 1) / 2;
    auto ext_value = [&](uint32_t i) -> float {
        if (i < dim) return src[i];
        if (enc == QB_BQ_TWO_BITS) return src[i - dim];
        const uint32_t k = 2 * (i - dim);
        return (k + 1 < dim) ? fmaxf(src[k], src[k + 1]) : src[k];
    };
    float mx = 0.0f;
    for (uint32_t i = threadIdx.x; i < ext; i += blockDim.x) mx = fmaxf(mx, fabsf(ext_value(i)));
    s_max[threadIdx.x] = mx;
    __syncthreads();
    for (int st = 128; st > 0; st >>= 1) {
        if ((int)threadIdx.x < st) s_max[threadIdx.x] = fmaxf(s_max[threadIdx.x], s_max[threadIdx.x + st]);
        __syncthreads();
    }
    const float max_abs = s_max[0];
    const float mn = -max_abs;
    const unsigned long long ranges = (1ull << bits) - 1ull;
    const float delta = __fdiv_rn(__fsub_rn(max_abs, mn), (float)ranges);
    for (uint32_t i = threadIdx.x; i < ext; i += blockDim.x) {
        const float shifted = __fsub_rn(ext_value(i), mn);
        const float delted = (delta > 1.1920929e-07f) ? __fdiv_rn(shifted, delta) : 0.0f;
        const float rv = roundf(delted);
        unsigned long long rounded = (rv != rv || rv <= 0.0f) ? 0ull : (rv >= 1.8446744e19f ? 0xFFFFFFFFFFFFFFFFull : (unsigned long long)rv);
        const unsigned long long quantized = rounded % (ranges + 1ull);
        const uint32_t chunk = i >> 7, shift = i & 127;
        for (int b = 0; b < bits; ++b)
            if ((quantized >> b) & 1ull) {
                const uint32_t word32 = ((uint32_t)bits * chunk + (uint32_t)b) * 4 + (shift >> 5);
                atomicOr(&dst[word32], 1u << (shift & 31));
            }
    }
}

struct BqParams {
    const uint8_t* rows;    // [count][row_bytes]
    uint32_t row_bytes, dim;
    int bits;               // 1, 4, 8
    int is_dot, invert;
    uint64_t begin, end;
    const uint32_t* ids;
    const uint8_t* q_enc;   // [nq][row_bytes*bits]
    uint32_t nq;
    float* scores;
    int emit_mode;
};

__device__ __forceinline__ unsigned int popc128(uint4 a, uint4 b) {
    return __popc(a.x ^ b.x) + __popc(a.y ^ b.y) + __popc(a.z ^ b.z) + __popc(a.w ^ b.w);
}

// calculate_metric (encoded_vectors_binary.rs:766-810): 8 lanes per candidate, one u128 word per lane per step
__global__ void __launch_bounds__(256) bq_group_kernel(const BqParams p, const QbEmit emit) {
    const int t = threadIdx.x & 7;
    const uint64_t groups_per_grid = (uint64_t)gridDim.x * (blockDim.x >> 3);
    const uint64_t g0 = (uint64_t)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3);
    const uint64_t n = p.end - p.begin;
    const uint64_t n_iter = (n + groups_per_grid - 1) / groups_per_grid;
    const uint32_t n_words = p.row_bytes >> 4;
    const float dimf = (float)p.dim;
    for (uint64_t it = 0; it < n_iter; ++it) {
        const uint64_t ci = g0 + it * groups_per_grid;
        const bool valid = ci < n;
        const uint64_t cand = p.begin + (valid ? ci : 0);
        const uint32_t row = p.ids ? p.ids[cand] : (uint32_t)cand;
        const uint4* rp = reinterpret_cast<const uint4*>(p.rows + (size_t)row * p.row_bytes);
        for (uint32_t q = 0; q < p.nq; ++q) {
            const uint4* qp = reinterpret_cast<const uint4*>(p.q_enc + (size_t)q * p.row_bytes * p.bits);
            unsigned int acc = 0;
            if (p.bits == 1) {
                for (uint32_t w = t; w < n_words; w += 8) acc += popc128(__ldg(rp + w), __ldg(qp + w));
            } else {
                for (uint32_t w = t; w < n_words; w += 8) {
                    const uint4 v = __ldg(rp + w);
                    for (int b = 0; b < p.bits; ++b) acc += popc128(v, __ldg(qp + (size_t)w * p.bits + b)) << b;
                }
            }
            acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 1);
            acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 2);
            acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 4);
            float xr = (float)acc;
            if (p.bits != 1) xr = __fdiv_rn(xr, (float)((1 << p.bits) - 1));
            const float zeros = __fsub_rn(dimf, xr);
            // (Dot, invert) -> xor - zeros ; (Dot, !invert) -> zeros - xor ; (L1/L2, invert) -> zeros - xor ; else xor - zeros
            const bool zeros_minus_xor = p.is_dot ? !p.invert : (p.invert != 0);
            const float sc = zeros_minus_xor ? __fsub_rn(zeros, xr) : __fsub_rn(xr, zeros);
            if (valid && t == 0) {
                if (p.emit_mode) qb_emit(emit, q, cand, row, sc);
                else p.scores[(size_t)q * n + ci] = sc;
            }
        }
    }
}

unsigned grid_for_groups(uint64_t n, int sm_count) {
    uint64_t blocks = ceil_div_u64(n, 256 / 8);
    uint64_t maxb = (uint64_t)sm_count * 8;
    if (blocks > maxb) blocks = maxb;
    if (blocks == 0) blocks = 1;
    return (unsigned)blocks;
}

}  // namespace

// ---------------------------------------------------------------- SQ8 host launchers
qb_status qb_sq8_repack(const qb_storage* s, const uint8_t* d_rows_in, uint32_t row_bytes, uint64_t first, uint64_t n, cudaStream_t stream) {
    if (n == 0) return QB_OK;
    uint64_t total = n * (uint64_t)(s->actual_dim >> 2);
    uint64_t blocks = ceil_div_u64(total, 256);
    if (blocks > 132 * 32) blocks = 132 * 32;
    sq8_repack_kernel<<<(unsigned)blocks, 256, 0, stream>>>(d_rows_in, row_bytes, s->actual_dim, n, s->d_codes + first * s->actual_dim,
                                                            s->d_voff + first);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

qb_status qb_sq8_encode_queries(const qb_storage* s, const float* d_q_pre, uint32_t q_stride_f, uint32_t nq, uint8_t* d_codes, float* d_q_off,
                                cudaStream_t stream) {
    if (nq == 0) return QB_OK;
    sq8_encode_query_kernel<<<nq, 256, 0, stream>>>(d_q_pre, q_stride_f, s->dim, s->actual_dim, s->alpha, s->offset, (int)s->qdist, s->invert,
                                                    d_codes, d_q_off);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

static float sq8_shift_host(const qb_storage* s) {  // get_shift, encoded_vectors_u8.rs:116-134
    float shift = 0.0f;
    if (s->qdist == QB_QD_DOT || s->qdist == QB_QD_COSINE) {
        volatile float a = (float)s->actual_dim * s->offset;
        shift = a * s->offset;
    }
    return s->invert ? -shift : shift;
}

qb_status qb_sq8_internal_query(const qb_storage* s, uint32_t id, uint8_t* d_code, float* d_q_off, cudaStream_t stream) {
    sq8_internal_query_kernel<<<1, 256, 0, stream>>>(s->d_codes, s->d_voff, s->actual_dim, id, sq8_shift_host(s), d_code, d_q_off);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

static qb_status sq8_launch(const qb_storage* s, Sq8Params& p, const QbEmit& e, cudaStream_t stream) {
    const uint64_t n = p.end - p.begin;
    if (n == 0 || p.nq == 0) return QB_OK;
    p.codes = s->d_codes; p.voff = s->d_voff; p.ad = s->actual_dim; p.multiplier = s->multiplier;
    p.l1 = (s->qdist == QB_QD_L1) ? 1 : 0;
    const bool lanex = (uint64_t)s->actual_dim * 127ull * 127ull >= (1ull << 24);
    if (lanex) sq8_group_kernel<true><<<grid_for_groups(n, s->sm_count), 256, 0, stream>>>(p, e);
    else sq8_group_kernel<false><<<grid_for_groups(n, s->sm_count), 256, 0, stream>>>(p, e);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

qb_status qb_sq8_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream) {
    Sq8Params p{};
    p.begin = a.row_begin; p.end = a.row_end; p.ids = a.d_ids;
    p.q_codes = reinterpret_cast<const uint8_t*>(a.d_q_enc); p.q_off = a.d_q_off; p.nq = a.nq;
    p.scores = nullptr; p.emit_mode = 1;
    return sq8_launch(s, p, a.emit, stream);
}

qb_status qb_sq8_score_points(const qb_storage* s, const void* d_q_enc, const float* d_q_off, const uint32_t* d_ids, uint64_t n, float* d_scores,
                              cudaStream_t stream) {
    Sq8Params p{};
    p.begin = 0; p.end = n; p.ids = d_ids;
    p.q_codes = reinterpret_cast<const uint8_t*>(d_q_enc); p.q_off = d_q_off; p.nq = 1;
    p.scores = d_scores; p.emit_mode = 0;
    QbEmit e{};
    return sq8_launch(s, p, e, stream);
}

// ---------------------------------------------------------------- PQ host launchers
qb_status qb_pq_build_luts(const qb_storage* s, const float* d_q_pre, uint32_t q_stride_f, uint32_t nq, float* d_luts, cudaStream_t stream) {
    if (nq == 0) return QB_OK;
    dim3 grid(s->pq_m, nq);
    pq_lut_kernel<<<grid, 256, 0, stream>>>(d_q_pre, q_stride_f, s->dim, s->pq_m, s->d_pq_div, s->d_centroids, s->n_centroids, (int)s->qdist,
                                            s->invert, d_luts);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

static qb_status pq_launch(const qb_storage* s, PqParams& p, const QbEmit& e, cudaStream_t stream, float* d_thr_adj = nullptr, void* scratch = nullptr,
                           size_t scratch_bytes = 0) {
    const uint64_t n = p.end - p.begin;
    if (n == 0 || p.nq == 0) return QB_OK;
    p.codes = s->d_pq_codes; p.stride = s->pq_stride; p.m = s->pq_m; p.n_centroids = s->n_centroids;
    const size_t lut_bytes = (size_t)s->pq_m * s->n_centroids * sizeof(float);
    const int qpp = qb_opt().pq_queries_per_pass;   // 0 = automatic; 1 / 2 / 4 force a kernel (experiments)
    const size_t smem4 = 2 * lut_bytes + (size_t)4 * PQ4_THREADS * 16 + (size_t)2 * PQ4_WARPS * 8;   // interleaved LUT half (4 queries x m/2 chunks) + hand-off slot + barriers
    const uint32_t nq16 = (p.nq + 15u) & ~15u;
    const size_t tab_bytes = (size_t)nq16 * s->pq_m * s->n_centroids;
    const size_t smem16 = 2 * lut_bytes + (size_t)2 * PQ16_THREADS * 16 + (size_t)2 * PQ16_WARPS * 8;   // 16 u8 tables x m/2 chunks = the same bytes again
    if (p.emit_mode && !e.dense && scratch && scratch_bytes >= tab_bytes + (size_t)nq16 * 4 + 256 && !p.ids && (qpp == 0 || qpp == 16) && p.nq >= 9 && s->pq_m % 32 == 0 &&
        s->pq_m <= 128 && s->n_centroids == 256 && smem16 <= 227 * 1024 && n >= 65536 && s->sm_count >= 2) {
        // batched filter passes: sixteen queries per gather through u8 tables, integer thresholds; survivors re-scored exactly (pq_scan16_kernel)
        QB_CUDA(cudaFuncSetAttribute(pq_scan16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem16));
        uint8_t* tab16 = reinterpret_cast<uint8_t*>(scratch);
        uint32_t* bias = reinterpret_cast<uint32_t*>(tab16 + ((tab_bytes + 255) & ~(size_t)255));
        pq16_prep_kernel<<<nq16, 256, 0, stream>>>(p.luts, p.nq, p.m, p.n_centroids, e.thr, tab16, bias);
        QB_LAUNCHED();
        const uint64_t block_rows = std::max<uint64_t>(65536, (48ull << 20) / s->pq_stride);
        const unsigned grid = (unsigned)(s->sm_count & ~1);
        for (uint64_t b0 = p.begin; b0 < p.end; b0 += block_rows) {
            PqParams pb = p;
            pb.begin = b0; pb.end = std::min<uint64_t>(p.end, b0 + block_rows);
            pq_scan16_kernel<<<grid, PQ16_THREADS, smem16, stream>>>(pb, e, tab16, bias);
            QB_LAUNCHED();
        }
        pq_rescore_kernel<<<dim3(8, p.nq), 128, 0, stream>>>(p, e);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
    const size_t smem8 = 2 * lut_bytes + (size_t)2 * PQ8_THREADS * 16 + (size_t)2 * PQ8_WARPS * 8;   // 8 bf16 tables x m/2 chunks = the same bytes
    if (p.emit_mode && !e.dense && d_thr_adj && !p.ids && (qpp == 0 || qpp == 8) && p.nq >= 5 && s->pq_m % 32 == 0 && smem8 <= 227 * 1024 && n >= 65536 && s->sm_count >= 2) {
        // batched filter passes: eight queries per gather through bf16 tables; survivors re-scored exactly (see pq_scan8_kernel)
        QB_CUDA(cudaFuncSetAttribute(pq_scan8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem8));
        pq8_margin_kernel<<<p.nq, 256, 0, stream>>>(p.luts, p.m, p.n_centroids, e.thr, d_thr_adj);
        QB_LAUNCHED();
        QbEmit e8 = e;
        e8.thr = d_thr_adj;
        const uint64_t block_rows = std::max<uint64_t>(65536, (48ull << 20) / s->pq_stride);
        const unsigned grid = (unsigned)(s->sm_count & ~1);
        for (uint64_t b0 = p.begin; b0 < p.end; b0 += block_rows) {
            PqParams pb = p;
            pb.begin = b0; pb.end = std::min<uint64_t>(p.end, b0 + block_rows);
            pq_scan8_kernel<<<grid, PQ8_THREADS, smem8, stream>>>(pb, e8);
            QB_LAUNCHED();
        }
        pq_rescore_kernel<<<dim3(8, p.nq), 128, 0, stream>>>(p, e);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
    if (p.emit_mode && !p.ids && (qpp == 0 || qpp == 4) && p.nq >= 3 && s->pq_m % 32 == 0 && smem4 <= 227 * 1024 && n >= 65536 && s->sm_count >= 2) {
        // batched scans: four queries per pass on CTA pairs; row blocks sized to stay in L2 while every query quad visits them
        QB_CUDA(cudaFuncSetAttribute(pq_scan4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem4));
        const uint64_t block_rows = std::max<uint64_t>(65536, (48ull << 20) / s->pq_stride);
        const unsigned grid = (unsigned)(s->sm_count & ~1);
        for (uint64_t b0 = p.begin; b0 < p.end; b0 += block_rows) {
            PqParams pb = p;
            pb.begin = b0; pb.end = std::min<uint64_t>(p.end, b0 + block_rows);
            pq_scan4_kernel<<<grid, PQ4_THREADS, smem4, stream>>>(pb, e);
            QB_LAUNCHED();
        }
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
    if (p.emit_mode && (qpp == 0 || qpp == 2 || qpp == 4) && p.nq >= 2 && 2 * lut_bytes <= 224 * 1024 && n >= 65536) {
        // batched scans: two queries per pass (interleaved LUTs)
        QB_CUDA(cudaFuncSetAttribute(pq_scan2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        uint64_t blocks2 = ceil_div_u64(n, 1024);
        if (blocks2 > (uint64_t)s->sm_count) blocks2 = (uint64_t)s->sm_count;
        pq_scan2_kernel<<<(unsigned)blocks2, 1024, 2 * lut_bytes, stream>>>(p, e);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
    p.lut_in_smem = (lut_bytes <= 200 * 1024 && n >= 4096) ? 1 : 0;
    const size_t smem = p.lut_in_smem ? lut_bytes : 0;
    if (smem > 48 * 1024) QB_CUDA(cudaFuncSetAttribute(pq_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    uint64_t blocks = ceil_div_u64(n, 512);
    uint64_t maxb = p.lut_in_smem ? (uint64_t)s->sm_count * (smem > 100 * 1024 ? 1 : 2) : (uint64_t)s->sm_count * 4;
    if (blocks > maxb) blocks = maxb;
    pq_scan_kernel<<<(unsigned)blocks, 512, smem, stream>>>(p, e);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

// bytes of per-call scratch the sixteen-query prefilter wants for a batch of nq queries (interleaved u8 tables + biases)
size_t qb_pq_scratch_bytes(const qb_storage* s, uint32_t nq) {
    if (s->kind != QB_KIND_PQ || nq < 9) return 0;
    const size_t nq16 = ((size_t)nq + 15) & ~(size_t)15;
    return nq16 * s->pq_m * s->n_centroids + nq16 * 4 + 512;
}

qb_status qb_pq_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream) {
    PqParams p{};
    p.begin = a.row_begin; p.end = a.row_end; p.ids = a.d_ids;
    p.luts = reinterpret_cast<const float*>(a.d_q_enc); p.nq = a.nq;
    p.scores = nullptr; p.emit_mode = 1;
    return pq_launch(s, p, a.emit, stream, a.d_thr_scratch, a.d_scratch, a.scratch_bytes);
}

qb_status qb_pq_score_points(const qb_storage* s, const void* d_q_enc, const uint32_t* d_ids, uint64_t n, float* d_scores, cudaStream_t stream) {
    PqParams p{};
    p.begin = 0; p.end = n; p.ids = d_ids;
    p.luts = reinterpret_cast<const float*>(d_q_enc); p.nq = 1;
    p.scores = d_scores; p.emit_mode = 0;
    QbEmit e{};
    return pq_launch(s, p, e, stream);
}

qb_status qb_pq_score_internal(const qb_storage* s, uint32_t a, uint32_t b, float* d_out, cudaStream_t stream) {
    pq_score_internal_kernel<<<1, 32, 0, stream>>>(s->d_pq_codes, s->pq_stride, s->pq_m, s->d_pq_div, s->d_centroids, s->dim, (int)s->qdist,
                                                   s->invert, a, b, d_out);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

// ---------------------------------------------------------------- BQ host launchers
static int bq_bits(const qb_storage* s) { return s->bq_qenc == QB_BQQ_SCALAR4 ? 4 : (s->bq_qenc == QB_BQQ_SCALAR8 ? 8 : 1); }

qb_status qb_bq_encode_queries(const qb_storage* s, const float* d_q_pre, uint32_t q_stride_f, uint32_t nq, int force_binary, void* d_out,
                               cudaStream_t stream) {
    if (nq == 0) return QB_OK;
    const int bits = force_binary ? 1 : bq_bits(s);
    bq_encode_query_kernel<<<nq, 256, 0, stream>>>(d_q_pre, q_stride_f, s->dim, (int)s->bq_enc, bits, s->d_mean_std, s->bq_row_bytes,
                                                   reinterpret_cast<uint32_t*>(d_out));
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

static qb_status bq_launch(const qb_storage* s, BqParams& p, const QbEmit& e, cudaStream_t stream) {
    const uint64_t n = p.end - p.begin;
    if (n == 0 || p.nq == 0) return QB_OK;
    p.rows = s->d_bq_rows; p.row_bytes = s->bq_row_bytes; p.dim = s->dim;
    p.is_dot = (s->qdist == QB_QD_DOT || s->qdist == QB_QD_COSINE) ? 1 : 0;
    p.invert = s->invert;
    bq_group_kernel<<<grid_for_groups(n, s->sm_count), 256, 0, stream>>>(p, e);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

qb_status qb_bq_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream) {
    BqParams p{};
    p.bits = bq_bits(s);
    p.begin = a.row_begin; p.end = a.row_end; p.ids = a.d_ids;
    p.q_enc = reinterpret_cast<const uint8_t*>(a.d_q_enc); p.nq = a.nq;
    p.scores = nullptr; p.emit_mode = 1;
    return bq_launch(s, p, a.emit, stream);
}

qb_status qb_bq_score_points(const qb_storage* s, const void* d_q_enc, int bits, const uint32_t* d_ids, uint64_t n, float* d_scores,
                             cudaStream_t stream) {
    BqParams p{};
    p.bits = bits;
    p.begin = 0; p.end = n; p.ids = d_ids;
    p.q_enc = reinterpret_cast<const uint8_t*>(d_q_enc); p.nq = 1;
    p.scores = d_scores; p.emit_mode = 0;
    QbEmit e{};
    return bq_launch(s, p, e, stream);
}
