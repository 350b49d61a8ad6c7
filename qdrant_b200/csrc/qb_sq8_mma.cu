// qb_sq8_mma.cu — batched SQ8 scoring on the Hopper tensor cores (wgmma.mma_async, register accumulators, TMA, mbarriers).
//
// The one dense contraction on the path (north_star): many queries x one segment.  In the reference every
// (query, vector) pair is a separate impl_score_dot_avx call (lib/quantization/cpp/avx2.c:25-63) made from
// QuantizedQueryScorer::score_stored_batch (quantized_query_scorer.rs:81-93) inside the peek_top_iter loop
// (point_scorer.rs:453-462), i.e. the batch re-reads each 64-vector chunk once per query.  Here it is
//      D[vectors x N queries] (s32, registers)  +=  A[vectors x K] (u8 codes, smem via TMA)  x  B[N x K]^T (u8 query codes)
// with the integer dot exact by construction, followed by the reference's epilogue
//      score = multiplier * f32(dot) + q_off[q] + v_off[v]              (encoded_vectors_u8.rs:101-103)
// and the fused threshold filter that feeds the top-k selection (the N x 10M score matrix is never materialised).
//
// One persistent CTA per SM, 9 warps:
//   warps 0-7  two consumer warpgroups: each owns 64 rows of every 128-row tile and all n_blk <= 128 columns, issues
//              wgmma.m64n32k32 (u8) per 32-column chunk straight from the shared-memory ring, and filters its accumulators
//              in registers: an integer prefilter of min/max instructions per 16 dot products, exact scoring only for the
//              rare survivors.
//   warp 8     TMA producer: the CTA's query block B stays resident in shared memory (128-B-swizzled K-blocks); vector-code
//              tiles A (128 rows x 128 B) stream through a ring of as many stages as shared memory leaves (4..8); tiles are
//              L2-prefetched three tiles ahead.
// A consumer keeps one wgmma group in flight: the stage of K-block k is released once the MMAs of K-block k + 1 are issued
// and those of k have retired.
//
// The per-query part of the threshold is moved INTO the accumulator, so that the filter needs no shared-memory load per
// element: one extra K = 32 MMA per tile multiplies a constant A tile (fifteen 127s and a 1 per 16 bytes) with a per-query
// "bias" row
//      D' = dot + bias_q,   bias_q = 2 * ceil((T - t_q) / 2),   t_q = (thr_q - q_off_q) / multiplier - slack
// after which ONE integer threshold serves every query of the batch and a row only needs
//      max(D'[...]) >= T - row_term
// with both sides in registers.  Survivors of that test are re-scored exactly (dot = D' - bias_q) against their own
// query's threshold.
//
// Exactness: codes are <= 127, so dot <= 127^2 * K.  While dot < 2^24 the CPU's lane-wise f32 tree equals f32(dot)
// exactly (all partial sums are non-negative integers <= dot).  If any dot >= 2^24 (possible only for K > 1040) the
// kernel raises a flag and the host reruns the batch on the lane-exact CUDA-core kernel.
//
// F16 = true: the same pipeline for DENSE f32 storages (dot / cosine) — "batched multi-query x segment scoring on tensor cores" for
// full-precision vectors.  bf16 inputs cannot reproduce the reference's f32 FMA chains, so the tensor cores only PREFILTER:
//      approx = bf16(row) . bf16(query)   (wgmma.m64n32k16 bf16, f32 accumulators; a bf16 shadow plane of the rows lives beside the f32 plane)
//      |approx - exact| <= eps_q = (2^-8 + 2^-18 + K 2^-22) |q| max|row|  (RN-even input rounding of both operands + f32 accumulation) + slack
// a row survives when approx >= thr_q - eps_q, and every survivor is re-scored by the bit-exact AVX-order kernel before the
// selection sees it (f32_rescore_kernel).  thr_q comes from exactly scored samples, so it never exceeds the final k-th score:
// nothing that belongs to the top-k can be filtered out, and the reported scores are the exact ones.
#include <cuda.h>
#include <stdlib.h>

#include "qb_internal.h"
#include "qb_score.cuh"

namespace {

constexpr int MMA_M = 128;                   // rows per tile: 64 per consumer warpgroup
constexpr int WG_M = 64;                     // rows of one wgmma
constexpr int KB = 128;                      // K bytes per smem block (one 128-B swizzle atom wide), for A stages and B blocks
constexpr int A_STAGE_BYTES = MMA_M * KB;    // 16 KB
constexpr int MIN_STAGES = 4;
constexpr int MAX_STAGES = 8;
constexpr int NC = 32;                       // columns (queries) per wgmma
constexpr int N_MAX = 128;                   // columns per CTA: 4 chunks x 16 accumulator registers per thread
#ifndef QB_MMA_PF
#define QB_MMA_PF 3
#endif
constexpr int CONSUMER_WARPS = 8;
constexpr int THREADS = 32 * (CONSUMER_WARPS + 1);
constexpr int WARP_TMA = CONSUMER_WARPS;
constexpr int T_CLAMP = 1 << 29;
constexpr int BIAS_KB = 32;                  // K bytes of the bias MMA (one u8 k32 / bf16 k16 instruction)
constexpr int BIAS_HALF_MAX = 127 * 127 * 15 + 126;  // largest representable bias / 2

struct MmaParams {
    const float* voff;
    uint64_t n_rows;
    uint32_t ad;             // K bytes
    uint32_t n_qblocks;
    uint32_t nq;             // real number of queries
    uint32_t n_workers;      // CTAs per query block
    uint32_t stages;         // A ring depth, MIN_STAGES..MAX_STAGES
    float multiplier;
    const float* q_off;      // [nq]
    const uint8_t* bias_rows;  // [nq_pad][32] per-query B rows of the bias MMA; null = no bias / no prefilter (sample pass)
    const int* bias_i;       // [nq_pad] the integer each row adds to its query's dot products
    const int* t_int;        // [1] the batch-wide threshold T on dot + bias
    unsigned int* flags;     // 2: a dot product reached 2^24; 8: a survivor segment overflowed
    int check_exact;
    uint32_t seg_cap;        // survivors of (query, CTA of its block group) go to a private segment of this many slots (0 = global atomics)
    int debug;               // QB_MMA_DEBUG perf experiments: 1 = epilogue skips its work, 2 = no bias MMA (every element re-scored), 4 = prefilter never passes, 8 = no A loads, 16 = no L2 prefetch
};

// Everything the survivor path needs, in shared memory: the out-of-line slow path takes ONE pointer, and nothing it reads sits
// in per-thread local memory.
struct EpiShared {
    float thr[N_MAX];          // exact per-query thresholds (+inf for padding)
    float qoff[N_MAX];
    int bias[N_MAX];
    unsigned int cnt[N_MAX];   // survivors of this CTA per query
    unsigned long long* cand;
    unsigned long long cap;
    unsigned long long dense_base;
    unsigned int* gcnt;
    unsigned int* flags;
    float multiplier;
    uint32_t seg_cap, seg_index, q_base, nq, id_base;
    int dense, check_exact;
};
constexpr size_t SMALL_SMEM = sizeof(EpiShared) + (2 * MAX_STAGES + 1) * 8 + 16;  // + barriers

// ---------------------------------------------------------------------------------------------- PTX helpers
__device__ __forceinline__ bool elect_one() {  // one lane of a converged warp
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* smem_dst, int32_t c0, int32_t c1, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
            qb_smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(qb_smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* map, int32_t c0, int32_t c1) {  // into L2 only
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1) : "memory");
}
// wgmma shared-memory matrix descriptor (sm_90): K-major, 128-B swizzle, 8 rows x 128 B between swizzle atoms
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);     // start address  [0,14)
    d |= (uint64_t)1 << 16;                          // leading byte offset: unused for swizzled K-major, canonical value 1
    d |= (uint64_t)((8 * KB) >> 4) << 32;            // stride byte offset [32,46)
    d |= (uint64_t)1 << 62;                          // layout [62,64): 1 = SWIZZLE_128B
    return d;
}
// 32-B swizzle, rows of 32 B, 8-row groups 256 B apart (the bias MMA's operands; both 16-B halves of every row are identical,
// so the swizzle's chunk permutation is immaterial)
__device__ __forceinline__ uint64_t make_smem_desc_sw32(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)((8 * BIAS_KB) >> 4) << 32;
    d |= (uint64_t)3 << 62;                          // 3 = SWIZZLE_32B
    return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
__device__ __forceinline__ void acc_fence(uint32_t (&d)[16]) {
#pragma unroll
    for (int i = 0; i < 16; ++i) asm volatile("" : "+r"(d[i])::"memory");
}
// D[64 x 32] (+)= A[64 x 32 B] . B[32 x 32 B]^T; u8 x u8 -> s32, or (F16) bf16 x bf16 -> f32 held as raw bits
template <bool F16>
__device__ __forceinline__ void wgmma_n32(uint32_t (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    if (F16)
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]),
              "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
            : "l"(a_desc), "l"(b_desc), "r"(accumulate));
    else
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.u8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p;\n\t}"
            : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]),
              "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
            : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// ---------------------------------------------------------------------------------------------- epilogue
// Exact epilogue of one (vector, query) pair: int -> f32 (exact), three roundings (encoded_vectors_u8.rs:101-103), emit.
// Survivors go to a segment private to (query, CTA): the slot comes from a SHARED-memory counter, the store is fire-and-forget.
__device__ __forceinline__ void epilogue_exact(EpiShared* es, uint32_t acc, uint32_t n, uint64_t row, bool valid_row, bool dead, float v_off) {
    const uint32_t q = es->q_base + n;
    if (q >= es->nq) return;
    const uint32_t dot = acc - (uint32_t)es->bias[n];
    float f = __uint_as_float(dot | 0x4B000000u) - 8388608.0f;  // exact for dot < 2^23
    if (dot >= 0x800000u) {
        f = (float)dot;
        if (es->check_exact && dot >= 0x1000000u) atomicOr(es->flags, 2u);
    }
    const float sc = __fadd_rn(__fadd_rn(__fmul_rn(es->multiplier, f), es->qoff[n]), v_off);
    if (es->dense) {
        if (valid_row) es->cand[(unsigned long long)q * es->cap + (row - es->dense_base)] = dead ? 0ull : qb_pack_key(sc, (uint32_t)row + es->id_base);
    } else if (sc >= es->thr[n] && !dead) {
        const uint32_t seg_cap = es->seg_cap;
        if (seg_cap) {
            const unsigned int pos = atomicAdd(&es->cnt[n], 1u);
            if (pos < seg_cap) es->cand[(unsigned long long)q * es->cap + (unsigned long long)es->seg_index * seg_cap + pos] = qb_pack_key(sc, (uint32_t)row + es->id_base);
            else atomicOr(es->flags, 8u);  // segment full: the host reruns this batch with global counters
        } else {
            const unsigned int pos = atomicAdd(&es->gcnt[q], 1u);
            if (pos < es->cap) es->cand[(unsigned long long)q * es->cap + pos] = qb_pack_key(sc, (uint32_t)row + es->id_base);
        }
    }
}

// F16 prefilter survivors: (query, row) pairs whose bf16 approximation reached the batch threshold; the key carries the approximate
// score and the LOCAL row — f32_rescore_kernel replaces it with the exact score (or drops it) before any selection.
__device__ __forceinline__ void epilogue_approx(EpiShared* es, float val, uint32_t n, uint64_t row, bool valid_row, bool dead) {
    const uint32_t q = es->q_base + n;
    if (q >= es->nq || !valid_row || dead) return;
    const float approx = __fsub_rn(val, __int_as_float(es->bias[n]));
    const uint32_t seg_cap = es->seg_cap;
    if (seg_cap) {
        const unsigned int pos = atomicAdd(&es->cnt[n], 1u);
        if (pos < seg_cap) es->cand[(unsigned long long)q * es->cap + (unsigned long long)es->seg_index * seg_cap + pos] = qb_pack_key(approx, (uint32_t)row);
        else atomicOr(es->flags, 8u);
    } else {
        const unsigned int pos = atomicAdd(&es->gcnt[q], 1u);
        if (pos < es->cap) es->cand[(unsigned long long)q * es->cap + pos] = qb_pack_key(approx, (uint32_t)row);
    }
}

// Slow path of a 32-column chunk: at least one lane of the warp holds a value at or above its row's threshold.  ONE out-of-line copy
// per variant (the 16 accumulator values travel in registers): the hot loop stays straight-line code.
// wgmma accumulator layout (m64nN): value j of a thread sits in row  row_lo + 8 * ((j >> 1) & 1)  and column
// 8 * (j >> 2) + 2 * (lane & 3) + (j & 1) of the chunk, row_lo = 16 * (warp in warpgroup) + lane / 4.
// row_flags: bit 0 / 1 = valid / deleted for row_lo, bits 2 / 3 the same for row_lo + 8.
template <bool F16>
__device__ __noinline__ void epilogue_hits(EpiShared* es, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3, uint32_t r4, uint32_t r5, uint32_t r6, uint32_t r7,
                                           uint32_t r8, uint32_t r9, uint32_t r10, uint32_t r11, uint32_t r12, uint32_t r13, uint32_t r14, uint32_t r15, uint32_t c,
                                           uint32_t t_lo, uint32_t t_hi, uint64_t row_lo, uint32_t row_flags, float voff_lo, float voff_hi) {
    uint32_t mask = 0;
#define QB_HIT(j)                                                                                                          \
    {                                                                                                                      \
        const uint32_t t = ((j) & 2) ? t_hi : t_lo;                                                                        \
        const bool hit = F16 ? (__uint_as_float(r##j) >= __uint_as_float(t)) : ((int)r##j >= (int)t);                    \
        mask |= hit ? (1u << (j)) : 0u;                                                                                    \
    }
    QB_HIT(0) QB_HIT(1) QB_HIT(2) QB_HIT(3) QB_HIT(4) QB_HIT(5) QB_HIT(6) QB_HIT(7) QB_HIT(8) QB_HIT(9) QB_HIT(10) QB_HIT(11) QB_HIT(12) QB_HIT(13) QB_HIT(14) QB_HIT(15)
#undef QB_HIT
    const uint32_t lane_col = 2u * (threadIdx.x & 3u);
    while (mask) {  // divergent: usually one lane, one column
        const uint32_t j = (uint32_t)__ffs((int)mask) - 1u;
        mask &= mask - 1u;
        // register select tree (no local-memory indexing)
        const bool b0 = j & 1u, b1 = j & 2u, b2 = j & 4u, b3 = j & 8u;
        const uint32_t s0 = b0 ? r1 : r0, s1 = b0 ? r3 : r2, s2 = b0 ? r5 : r4, s3 = b0 ? r7 : r6, s4 = b0 ? r9 : r8, s5 = b0 ? r11 : r10, s6 = b0 ? r13 : r12,
                       s7 = b0 ? r15 : r14;
        const uint32_t u0 = b1 ? s1 : s0, u1 = b1 ? s3 : s2, u2 = b1 ? s5 : s4, u3 = b1 ? s7 : s6;
        const uint32_t w0 = b2 ? u1 : u0, w1 = b2 ? u3 : u2;
        const uint32_t v = b3 ? w1 : w0;
        const uint32_t n = c * NC + 8u * (j >> 2) + lane_col + (j & 1u);
        const uint64_t row = row_lo + (b1 ? 8u : 0u);
        const uint32_t fl = b1 ? (row_flags >> 2) : row_flags;
        if (F16) epilogue_approx(es, __uint_as_float(v), n, row, (fl & 1u) != 0, (fl & 2u) != 0);
        else epilogue_exact(es, v, n, row, (fl & 1u) != 0, (fl & 2u) != 0, b1 ? voff_hi : voff_lo);
    }
}

// Filter one 32-column chunk held by this thread (two rows x 8 columns).  t_lo / t_hi = batch threshold - row term (registers only).
template <bool F16>
__device__ __forceinline__ void epilogue_chunk(EpiShared* es, const uint32_t (&r)[16], uint32_t c, uint32_t t_lo, uint32_t t_hi, uint64_t row_lo, uint32_t row_flags,
                                               float voff_lo, float voff_hi) {
    bool hit;
    if (F16) {
        float m_lo = __uint_as_float(r[0]), m_hi = __uint_as_float(r[2]);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            if (j & 2) m_hi = fmaxf(m_hi, __uint_as_float(r[j]));
            else m_lo = fmaxf(m_lo, __uint_as_float(r[j]));
        }
        hit = m_lo >= __uint_as_float(t_lo) || m_hi >= __uint_as_float(t_hi);
    } else {
        int m_lo = (int)r[0], m_hi = (int)r[2];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            if (j & 2) m_hi = max(m_hi, (int)r[j]);
            else m_lo = max(m_lo, (int)r[j]);
        }
        hit = m_lo >= (int)t_lo || m_hi >= (int)t_hi;
    }
    if (__any_sync(0xFFFFFFFFu, hit))
        epilogue_hits<F16>(es, r[0], r[1], r[2], r[3], r[4], r[5], r[6], r[7], r[8], r[9], r[10], r[11], r[12], r[13], r[14], r[15], c, t_lo, t_hi, row_lo, row_flags,
                           voff_lo, voff_hi);
}

// per-row inputs of the epilogue: validity, delete bit, v_off and the row term of the prefilter
struct RowIn {
    bool valid, dead;
    float v_off;
    int vi;
};
template <bool F16>
__device__ __forceinline__ RowIn row_in(const MmaParams& p, const QbEmit& emit, uint64_t row, bool pre) {
    RowIn r;
    r.valid = row < p.n_rows;
    r.v_off = (r.valid && !F16) ? p.voff[row] : 0.0f;
    r.dead = !r.valid || qb_is_deleted(emit, (uint32_t)(r.valid ? row : 0));
    r.vi = 0;
    if (pre && !F16) {  // score >= thr  <=>  dot >= t_query - v_off/mult; everything is rounded towards "pass"
        const float vm = r.v_off / p.multiplier;
        const float up = ceilf(vm + 1.0e-5f * fabsf(vm)) + 2.0f;
        r.vi = (int)fminf(fmaxf(up, (float)-T_CLAMP), (float)T_CLAMP);
    }
    return r;
}

// ---------------------------------------------------------------------------------------------- the kernel
template <int NCH, bool F16>
__global__ void __launch_bounds__(THREADS, 1)
sq8_mma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const MmaParams p, const QbEmit emit) {
    constexpr uint32_t n_blk = NCH * NC;
    extern __shared__ __align__(1024) uint8_t smem[];
    if ((qb_smem_u32(smem) & 1023u) != 0u) __trap();      // 128-B swizzle atoms need 1024-B alignment (no static smem precedes)
    const uint32_t n_kb = (p.ad + KB - 1) / KB;
    const uint32_t b_block_bytes = n_blk * KB;
    const uint32_t stages = p.stages;
    uint8_t* b_s = smem;
    uint8_t* a_s = b_s + (size_t)n_kb * b_block_bytes;
    uint8_t* a_const = a_s + (size_t)stages * A_STAGE_BYTES;    // [128 rows][32 B] constant A operand of the bias MMA
    uint8_t* b_bias = a_const + MMA_M * BIAS_KB;                // [n_blk rows][32 B] per-query bias rows
    EpiShared* es = reinterpret_cast<EpiShared*>(b_bias + (size_t)n_blk * BIAS_KB);
    uint64_t* full_a = reinterpret_cast<uint64_t*>(es + 1);     // [stages]
    uint64_t* empty_a = full_a + MAX_STAGES;                    // [stages]
    uint64_t* b_full = empty_a + MAX_STAGES;                    // [1]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t qblock = blockIdx.x % p.n_qblocks;
    const uint32_t worker = blockIdx.x / p.n_qblocks;
    const uint64_t n_tiles = (p.n_rows + MMA_M - 1) / MMA_M;
    const uint64_t my_tiles = (worker < n_tiles) ? (n_tiles - worker + p.n_workers - 1) / p.n_workers : 0;
    const uint32_t q_base = qblock * n_blk;
    const bool use_bias = p.bias_rows != nullptr;

    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < stages; ++s) { qb_mbar_init(&full_a[s], 1); qb_mbar_init(&empty_a[s], CONSUMER_WARPS); }
        qb_mbar_init(b_full, 1);
        es->cand = emit.cand; es->cap = emit.cap; es->dense_base = emit.dense_base; es->gcnt = emit.cnt; es->flags = p.flags;
        es->multiplier = p.multiplier; es->seg_cap = p.seg_cap; es->seg_index = worker; es->q_base = q_base; es->nq = p.nq;
        es->id_base = emit.id_base; es->dense = emit.dense; es->check_exact = p.check_exact;
    }
    for (uint32_t i = threadIdx.x; i < N_MAX; i += blockDim.x) {
        const uint32_t q = q_base + i;
        const bool real = i < n_blk && q < p.nq;
        es->thr[i] = real ? (emit.dense ? __int_as_float(0xff800000) : emit.thr[q]) : __int_as_float(0x7f800000);  // +inf: padding never emits
        es->qoff[i] = (real && !F16) ? p.q_off[q] : 0.0f;
        es->bias[i] = (real && use_bias) ? p.bias_i[q] : 0;
        es->cnt[i] = 0u;
    }
    // bias MMA operands, written with ordinary stores (both 16-B halves of a row are identical: swizzle-agnostic)
    for (uint32_t i = threadIdx.x; i < MMA_M * BIAS_KB / 16; i += blockDim.x)
        reinterpret_cast<uint4*>(a_const)[i] = F16 ? make_uint4(0x3F803F80u, 0u, 0u, 0u)                          // bf16 (1, 1, 0, 0, 0, 0, 0, 0)
                                                   : make_uint4(0x7F7F7F7Fu, 0x7F7F7F7Fu, 0x7F7F7F7Fu, 0x017F7F7Fu);  // bytes 0-14 = 127, byte 15 = 1
    if (use_bias)
        for (uint32_t i = threadIdx.x; i < n_blk * BIAS_KB / 16; i += blockDim.x)
            reinterpret_cast<uint4*>(b_bias)[i] = reinterpret_cast<const uint4*>(p.bias_rows + (size_t)q_base * BIAS_KB)[i];
    qb_fence_barrier_init();  // mbarrier inits + the generic-proxy stores above become visible to the async proxy (TMA / wgmma)
    __syncthreads();

    if (warp == WARP_TMA) {
        // ------------------------------------------------------------ TMA producer (warp-uniform loop, one elected lane issues)
        const uint64_t pol_keep = qb_policy_evict_last();
        const uint64_t pol_stream = qb_policy_evict_first();
        if (elect_one()) {  // resident query block
            qb_mbar_arrive_expect_tx(b_full, n_kb * b_block_bytes);
            for (uint32_t kb = 0; kb < n_kb; ++kb) tma_load_2d(&map_b, b_full, b_s + (size_t)kb * b_block_bytes, (int32_t)(kb * KB), (int32_t)q_base, pol_keep);
        }
        __syncwarp();
        uint32_t s = 0, ph = 0;
        constexpr uint64_t PF = QB_MMA_PF;  // L2 prefetch distance in tiles: hides the HBM latency that the smem ring cannot
        for (uint64_t ti = 0; ti < my_tiles; ++ti) {
            const int32_t row0 = (int32_t)((worker + ti * p.n_workers) * MMA_M);
            if (!(p.debug & 16) && elect_one()) {  // the n_qblocks groups of a worker walk the same tiles: each prefetches its share of the K-blocks
                for (uint64_t d = (ti == 0) ? 0 : PF; d <= PF; ++d)
                    if (ti + d < my_tiles)
                        for (uint32_t ka = qblock; ka < n_kb; ka += p.n_qblocks)
                            tma_prefetch_2d(&map_a, (int32_t)(ka * KB), (int32_t)((worker + (ti + d) * p.n_workers) * MMA_M));
            }
            __syncwarp();
            for (uint32_t ka = 0; ka < n_kb; ++ka) {
                qb_mbar_wait(&empty_a[s], ph ^ 1u);
                if (elect_one()) {
                    if (p.debug & 8) qb_mbar_arrive(&full_a[s]);  // timing experiment: stages are "filled" without moving data
                    else {
                        qb_mbar_arrive_expect_tx(&full_a[s], A_STAGE_BYTES);
                        tma_load_2d(&map_a, &full_a[s], a_s + (size_t)s * A_STAGE_BYTES, (int32_t)(ka * KB), row0, p.n_qblocks > 1 ? pol_keep : pol_stream);
                    }
                }
                __syncwarp();
                if (++s == stages) { s = 0; ph ^= 1u; }
            }
        }
    } else {
        // ------------------------------------------------------------ consumer warpgroups: MMAs, then the epilogue on the accumulators
        const uint32_t wg = (uint32_t)warp >> 2;
        const uint32_t row_off = wg * WG_M + (uint32_t)(warp & 3) * 16 + ((uint32_t)lane >> 2);  // row_lo within the tile
        const bool pre = use_bias && (F16 || p.multiplier > 0.0f);
        const int t_int = pre ? ((p.debug & 4) ? 0x7fffffff - T_CLAMP : *p.t_int) : -T_CLAMP;  // one threshold for the whole batch, in a register
        const float t_f16 = (F16 && pre) ? __int_as_float(*p.t_int) : __int_as_float(0xff800000);  // F16: the same word holds the f32 threshold
        // descriptors differ only in their 14-bit start-address field (low word): the high word is hoisted out of the loop
        const uint64_t a_desc0 = make_smem_desc(qb_smem_u32(a_s + wg * WG_M * KB)), b_desc0 = make_smem_desc(qb_smem_u32(b_s));
        const uint32_t a_hi = (uint32_t)(a_desc0 >> 32), a_lo0 = (uint32_t)a_desc0;
        const uint32_t b_hi = (uint32_t)(b_desc0 >> 32), b_lo0 = (uint32_t)b_desc0;
        const uint64_t bias_a_desc = make_smem_desc_sw32(qb_smem_u32(a_const + wg * WG_M * BIAS_KB)), bias_b_desc = make_smem_desc_sw32(qb_smem_u32(b_bias));
        uint32_t acc[NCH][16];
#pragma unroll
        for (int c = 0; c < NCH; ++c)
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[c][i] = 0u;
        qb_mbar_wait(b_full, 0);
        uint32_t s = 0, ph = 0;
        for (uint64_t ti = 0; ti < my_tiles; ++ti) {
            const uint64_t row_lo = (worker + ti * p.n_workers) * MMA_M + row_off;
            const RowIn lo = row_in<F16>(p, emit, row_lo, pre), hi = row_in<F16>(p, emit, row_lo + 8, pre);  // loads in flight under the MMAs
            uint32_t s_prev = 0;
            for (uint32_t ka = 0; ka < n_kb; ++ka) {
                qb_mbar_wait(&full_a[s], ph);
                wg_fence();
#pragma unroll
                for (int c = 0; c < NCH; ++c) acc_fence(acc[c]);
                const uint32_t a_lo = a_lo0 + s * (A_STAGE_BYTES >> 4);
                const uint32_t b_lo = b_lo0 + ka * (b_block_bytes >> 4);  // stage ka pairs with K-block ka
#pragma unroll
                for (uint32_t j = 0; j < KB / 32; ++j)  // +32 B inside the swizzled row per K-step (32 u8 codes, or 16 bf16 values); past ad the TMA boxes hold zeros
#pragma unroll
                    for (int c = 0; c < NCH; ++c)
                        wgmma_n32<F16>(acc[c], ((uint64_t)a_hi << 32) | (a_lo + 2 * j), ((uint64_t)b_hi << 32) | (b_lo + c * (NC * KB >> 4) + 2 * j),
                                       (ka | j) != 0 ? 1u : 0u);
                wg_commit();
                if (ka > 0) {  // the MMAs of K-block ka - 1 have retired: its stage goes back to the producer
                    wg_wait<1>();
                    __syncwarp();
                    if (lane == 0) qb_mbar_arrive(&empty_a[s_prev]);
                }
                s_prev = s;
                if (++s == stages) { s = 0; ph ^= 1u; }
            }
            if (use_bias) {  // D += bias_q in every row
                wg_fence();
#pragma unroll
                for (int c = 0; c < NCH; ++c) wgmma_n32<F16>(acc[c], bias_a_desc, bias_b_desc + (uint64_t)(c * NC * BIAS_KB >> 4), 1u);
                wg_commit();
            }
            wg_wait<0>();
#pragma unroll
            for (int c = 0; c < NCH; ++c) acc_fence(acc[c]);
            __syncwarp();
            if (lane == 0) qb_mbar_arrive(&empty_a[s_prev]);
            if (p.debug & 1) continue;
            const uint32_t row_flags = (lo.valid ? 1u : 0u) | (lo.dead ? 2u : 0u) | (hi.valid ? 4u : 0u) | (hi.dead ? 8u : 0u);
            const uint32_t t_lo = F16 ? __float_as_uint(t_f16) : (uint32_t)(t_int - lo.vi);
            const uint32_t t_hi = F16 ? __float_as_uint(t_f16) : (uint32_t)(t_int - hi.vi);
#pragma unroll
            for (int c = 0; c < NCH; ++c) epilogue_chunk<F16>(es, acc[c], (uint32_t)c, t_lo, t_hi, row_lo, row_flags, lo.v_off, hi.v_off);
        }
    }
}

// ---------------------------------------------------------------------------------------------- batch preparation
// Per-query bias rows for the main pass (one CTA, after the threshold selection of the sample pass):
//   t_q   = (thr_q - q_off_q) / multiplier - slack        the integer dot a row (with v_off = 0) must reach; conservative
//   T     = min(max_q t_q, min_q t_q + 2 * BIAS_HALF_MAX) the batch threshold on dot + bias
//   h_q   = clamp(ceil((T - t_q) / 2), 0, BIAS_HALF_MAX),  bias_q = 2 h_q
// so that dot >= t_q implies dot + bias_q >= floor(T) for every query.  h_q = 127 * (b_0 + ... + b_14) + b_15 with bytes <= 127;
// the row stores the 16 bytes twice (K = 32), the constant A operand holds (127 x 15, 1) twice.
__global__ void __launch_bounds__(1024) qb_mma_bias_kernel(const float* __restrict__ thr, const float* __restrict__ q_off, float mult, uint32_t nq, uint32_t n_pad,
                                                           uint8_t* __restrict__ bias_rows, int* __restrict__ bias_i, int* __restrict__ t_out) {
    __shared__ double s_min[32], s_max[32];
    __shared__ double s_T;
    auto t_of = [&](uint32_t i) -> double {
        const double tq = ((double)thr[i] - (double)q_off[i]) / (double)mult;
        double t = tq - (8.0 + 1.0e-5 * fabs(tq));
        if (!(t > -(double)T_CLAMP)) t = -(double)T_CLAMP;  // also catches NaN and thr = -inf (no threshold: everything passes)
        if (t > (double)T_CLAMP) t = (double)T_CLAMP;
        return t;
    };
    double mn = 1e300, mx = -1e300;
    for (uint32_t i = threadIdx.x; i < nq; i += blockDim.x) { const double t = t_of(i); mn = fmin(mn, t); mx = fmax(mx, t); }
    for (int o = 16; o > 0; o >>= 1) { mn = fmin(mn, __shfl_xor_sync(0xFFFFFFFFu, mn, o)); mx = fmax(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, o)); }
    if ((threadIdx.x & 31) == 0) { s_min[threadIdx.x >> 5] = mn; s_max[threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { mn = fmin(mn, s_min[w]); mx = fmax(mx, s_max[w]); }
        const double T = floor(fmin(mx, mn + 2.0 * (double)BIAS_HALF_MAX));
        s_T = T;
        *t_out = (int)T;
    }
    __syncthreads();
    const double T = s_T;
    for (uint32_t i = threadIdx.x; i < n_pad; i += blockDim.x) {
        int h = 0;
        if (i < nq) {
            const double d = ceil((T - t_of(i)) * 0.5);
            h = d <= 0.0 ? 0 : (d >= (double)BIAS_HALF_MAX ? BIAS_HALF_MAX : (int)d);
        }
        bias_i[i] = 2 * h;
        int coarse = h / 127;  // <= 127 * 15
        const int fine = h % 127;
        uint32_t w[4] = {0, 0, 0, 0};
        for (int k = 0; k < 15; ++k) {
            const int b = coarse > 127 ? 127 : coarse;
            coarse -= b;
            w[k >> 2] |= (uint32_t)b << (8 * (k & 3));
        }
        w[3] |= (uint32_t)fine << 24;
        const uint4 v = make_uint4(w[0], w[1], w[2], w[3]);
        reinterpret_cast<uint4*>(bias_rows + (size_t)i * BIAS_KB)[0] = v;
        reinterpret_cast<uint4*>(bias_rows + (size_t)i * BIAS_KB)[1] = v;
    }
}


// ---------------------------------------------------------------------------------------------- F16 (dense f32 storages): helpers
__device__ __forceinline__ uint16_t bf16_rne(float f) {       // round to nearest even (finite inputs)
    uint32_t u = __float_as_uint(f);
    u += 0x7FFFu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
}
__device__ __forceinline__ float bf16_to_f32(uint16_t h) { return __uint_as_float((uint32_t)h << 16); }

// f32 rows -> bf16 shadow rows (zero padded to the shadow stride); also max |row| (as float bits, rows are finite or the flag is raised)
__global__ void __launch_bounds__(256) f32_to_bf16_rows_kernel(const float* __restrict__ rows, uint64_t stride_f, uint32_t dim, uint64_t n, uint16_t* __restrict__ out,
                                                                uint32_t out_stride_h, unsigned int* __restrict__ max_norm_bits, unsigned int* __restrict__ nonfinite) {
    const int t = threadIdx.x & 7;
    const uint64_t groups = (uint64_t)gridDim.x * (blockDim.x >> 3), g0 = (uint64_t)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3);
    const uint64_t n_iter = (n + groups - 1) / groups;
    for (uint64_t it = 0; it < n_iter; ++it) {
        const uint64_t r = g0 + it * groups;
        const bool valid = r < n;
        const float* src = rows + (valid ? r : 0) * stride_f;
        uint16_t* dst = out + (valid ? r : 0) * out_stride_h;
        float ss = 0.f;
        bool bad = false;
        for (uint32_t i = t; i < out_stride_h; i += 8) {
            const float v = (i < dim) ? src[i] : 0.f;
            bad |= !(fabsf(v) <= 3.0e38f);
            ss = fmaf(v, v, ss);
            if (valid) dst[i] = bf16_rne(v);
        }
        ss += __shfl_xor_sync(0xFFFFFFFFu, ss, 1); ss += __shfl_xor_sync(0xFFFFFFFFu, ss, 2); ss += __shfl_xor_sync(0xFFFFFFFFu, ss, 4);
        if (valid && t == 0) {
            if (bad || !(ss <= 3.0e38f)) atomicOr(nonfinite, 1u);
            else atomicMax(max_norm_bits, __float_as_uint(sqrtf(ss) * 1.000001f));   // non-negative floats order like their bit patterns
        }
    }
}

// queries: bf16 B rows [nq_pad][row_h] + eps_q; thresholds -> bias rows (two bf16 halves, hi + lo, duplicated in both 16-B halves of the
// 32-B row so that the 32-B swizzle is immaterial), the f32 bias each query adds and the batch threshold T.  One CTA.
__global__ void __launch_bounds__(1024) f16_prepare_kernel(const float* __restrict__ q, uint32_t q_stride_f, uint32_t dim, uint32_t row_h, uint32_t nq, uint32_t n_pad,
                                                           const float* __restrict__ thr, const unsigned int* __restrict__ max_norm_bits, uint16_t* __restrict__ qb,
                                                           uint8_t* __restrict__ bias_rows, int* __restrict__ bias_f, int* __restrict__ t_out, unsigned int* __restrict__ flags) {
    __shared__ float s_t[1024];
    __shared__ float s_T;
    const float R = __uint_as_float(*max_norm_bits);
    // eps_q and t_q = thr_q - eps_q (thread per query, strided)
    float tmax = __int_as_float(0xff800000);
    for (uint32_t i = threadIdx.x; i < n_pad; i += blockDim.x) {
        const float* src = q + (size_t)(i < nq ? i : 0) * q_stride_f;
        uint16_t* dst = qb + (size_t)i * row_h;
        double ss = 0.0;
        for (uint32_t k = 0; k < row_h; ++k) {
            const float v = (i < nq && k < dim) ? src[k] : 0.f;
            ss += (double)v * (double)v;
            dst[k] = bf16_rne(v);
        }
        if (i < nq) {
            const float qn = (float)sqrt(ss) * 1.000001f;
            if (!(qn <= 3.0e38f)) atomicOr(flags, 1u);      // NaN / inf in a query: OrderedFloat semantics need the exact path
            // |approx - exact| <= (2^-8 + 2^-18 + K 2^-22) |q| |x|  (+ the rounding of adding the bias in the accumulator, + slack)
            const float eps = (0.00390625f + 3.9e-6f + (float)row_h * 2.4e-7f) * qn * R * 1.01f + 1.0e-6f * (1.0f + fabsf(thr[i]));
            const float t = thr[i] - eps;                  // -inf stays -inf: no threshold yet, everything must pass
            reinterpret_cast<float*>(bias_f)[i] = t;         // parked; turned into the bias below
            if (t > -3.0e38f && t > tmax) tmax = t;
        }
    }
    s_t[threadIdx.x] = tmax;
    __syncthreads();
    if (threadIdx.x == 0) {
        float T = __int_as_float(0xff800000);
        for (uint32_t i = 0; i < blockDim.x; ++i) T = fmaxf(T, s_t[i]);
        if (!(T > -3.0e38f)) T = 0.0f;                       // no query has a threshold: T is arbitrary, every bias is "pass everything"
        s_T = T;
        *reinterpret_cast<float*>(t_out) = T;
    }
    __syncthreads();
    const float T = s_T;
    for (uint32_t i = threadIdx.x; i < n_pad; i += blockDim.x) {
        float b = 0.0f;
        if (i < nq) {
            const float t = reinterpret_cast<float*>(bias_f)[i];
            b = (t > -3.0e38f) ? (T - t) * 1.0000002f + 1.0e-30f : 1.0e30f;     // rounded towards "pass"
            if (!(b >= 0.0f)) b = 0.0f;
        }
        // b / 2 = x + y with x = bf16 truncation, y = the remainder rounded UP to bf16: 2 (x + y) >= b, exactly representable in f32
        const float h = 0.5f * b;
        const uint16_t x = (uint16_t)(__float_as_uint(h) >> 16);
        const float rem = h - bf16_to_f32(x);
        uint32_t yu = __float_as_uint(rem);
        uint16_t y = (uint16_t)(yu >> 16);
        if ((yu & 0xFFFFu) != 0u) y += 1;                    // round the non-negative remainder up
        const float applied = 2.0f * (bf16_to_f32(x) + bf16_to_f32(y));
        bias_f[i] = __float_as_int(i < nq ? applied : 0.0f);
        uint32_t w0 = (uint32_t)x | ((uint32_t)y << 16);
        if (i >= nq) w0 = 0u;
        const uint4 v = make_uint4(w0, 0u, 0u, 0u);
        reinterpret_cast<uint4*>(bias_rows + (size_t)i * BIAS_KB)[0] = v;
        reinterpret_cast<uint4*>(bias_rows + (size_t)i * BIAS_KB)[1] = v;
    }
}

// Replace every surviving (approx score, local row) key by the exact AVX-order f32 score, or by "empty" when the exact score misses the
// query's threshold: 8 lanes per candidate, the same chains as every other f32 path.  Lists are counted (cnt[q], capped at cap).
__global__ void __launch_bounds__(256) f32_rescore_kernel(const uint8_t* __restrict__ rows, uint32_t stride, uint32_t dim, const float* __restrict__ q, uint32_t q_stride_f,
                                                          uint32_t nq, unsigned long long* __restrict__ cand, const unsigned int* __restrict__ cnt, unsigned long long cap,
                                                          const float* __restrict__ thr, uint32_t id_base) {
    const int t = threadIdx.x & 7;
    const uint32_t g = (blockIdx.x * (blockDim.x >> 3)) + (threadIdx.x >> 3), n_groups = gridDim.x * (blockDim.x >> 3);
    for (uint32_t qi = blockIdx.y; qi < nq; qi += gridDim.y) {
        const unsigned int c = min((unsigned long long)cnt[qi], cap);
        const float* qv = q + (size_t)qi * q_stride_f;
        const float th = thr[qi];
        unsigned long long* list = cand + (unsigned long long)qi * cap;
        const uint32_t n_iter = (c + n_groups - 1) / n_groups;
        for (uint32_t it = 0; it < n_iter; ++it) {
            const uint32_t i = g + it * n_groups;
            const bool valid = i < c;
            const unsigned long long key = valid ? list[i] : 0ull;
            const uint32_t row = valid ? qb_key_id(key) : 0u;
            const float sc = qbs::score_avx_group8<qbs::M_DOT>(reinterpret_cast<const float*>(rows + (size_t)row * stride), qv, dim, t);
            if (valid && t == 0) list[i] = (key != 0ull && !(sc < th)) ? qb_pack_key(sc, row + id_base) : 0ull;
        }
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

qb_status make_map_u8(CUtensorMap* m, const void* base, uint64_t inner_bytes, uint64_t rows, uint32_t box_inner, uint32_t box_rows) {
    EncodeTiledFn fn = get_encode_fn();
    QB_CHECK(fn, QB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t gdim[2] = {inner_bytes, rows};
    cuuint64_t gstride[1] = {inner_bytes};
    cuuint32_t box[2] = {box_inner, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    QB_CHECK(r == CUDA_SUCCESS, QB_ERR_CUDA, "cuTensorMapEncodeTiled failed: %d", (int)r);
    return QB_OK;
}

constexpr size_t SMEM_MAX = 227 * 1024;
// shared memory of everything but the A ring: resident query block and its bias rows, the bias MMA's constant A tile, small arrays
size_t fixed_smem(uint32_t k_bytes, uint32_t n_blk) {
    return (size_t)n_blk * ((size_t)((k_bytes + KB - 1) / KB) * KB + BIAS_KB) + MMA_M * BIAS_KB + SMALL_SMEM;
}
// query block width: the fixed part and a ring of MIN_STAGES must fit; equal-width blocks, multiples of one wgmma's N
uint32_t block_for_bytes(uint32_t k_bytes, uint32_t nq) {
    uint32_t n_blk = N_MAX;
    while (n_blk >= NC && fixed_smem(k_bytes, n_blk) + MIN_STAGES * A_STAGE_BYTES > SMEM_MAX) n_blk -= NC;
    if (n_blk < NC) return 0;
    const uint32_t n_qblocks = (nq + n_blk - 1) / n_blk;
    return (((nq + n_qblocks - 1) / n_qblocks) + NC - 1) & ~(NC - 1);
}
uint32_t block_for(const qb_storage* s, uint32_t nq) { return block_for_bytes(s->actual_dim, nq); }

// one CTA per (worker, query block); the ring takes what shared memory the fixed part leaves, up to MAX_STAGES
template <bool F16>
qb_status launch_mma(const CUtensorMap& map_a, const CUtensorMap& map_b, MmaParams p, const QbEmit& emit, uint32_t n_blk, cudaStream_t stream) {
    QB_CHECK(n_blk % NC == 0 && n_blk >= NC && n_blk <= N_MAX, QB_ERR_INVALID, "mma scan: query block width %u", n_blk);
    const size_t fixed = fixed_smem(p.ad, n_blk);
    QB_CHECK(fixed + MIN_STAGES * A_STAGE_BYTES <= SMEM_MAX, QB_ERR_INVALID, "mma scan: shared memory %zu exceeds 227 KB", fixed + MIN_STAGES * A_STAGE_BYTES);
    p.stages = (uint32_t)std::min<size_t>(MAX_STAGES, (SMEM_MAX - fixed) / A_STAGE_BYTES);
    const size_t smem = fixed + (size_t)p.stages * A_STAGE_BYTES;
    void (*k)(const CUtensorMap, const CUtensorMap, const MmaParams, const QbEmit) = nullptr;
    switch (n_blk / NC) {
        case 1: k = sq8_mma_kernel<1, F16>; break;
        case 2: k = sq8_mma_kernel<2, F16>; break;
        case 3: k = sq8_mma_kernel<3, F16>; break;
        default: k = sq8_mma_kernel<4, F16>; break;
    }
    QB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<p.n_workers * p.n_qblocks, THREADS, smem, stream>>>(map_a, map_b, p, emit);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

}  // namespace

// The epilogue's filter (sc >= thr) drops a NaN score, which the CUDA-core scan keeps (OrderedFloat: NaN is the greatest score), so
// the tensor cores only take storages whose scores are finite: score = multiplier * dot + q_off + v_off with dot <= actual_dim * 127^2,
// |q_off| <= actual_dim * 127 * |alpha * offset| (dot / cosine) or actual_dim * 127^2 * alpha^2 (L2).  A bound that is not finite or
// not clear of FLT_MAX (metadata from rows holding +-inf: alpha = inf, every offset 0 * inf = NaN) sends the batch to the CUDA cores.
static bool sq8_scores_finite(const qb_storage* s) {
    const double d = (double)s->actual_dim * 127.0 * 127.0, a = fabs((double)s->alpha), o = fabs((double)s->offset);
    const double q = (s->qdist == QB_QD_L2) ? d * a * a : (double)s->actual_dim * 127.0 * a * o;
    return fabs((double)s->multiplier) * d + q + (double)s->voff_absmax < 1.0e38;   // false for inf and NaN
}

// Can this (storage, batch) use the tensor-core path?  Returns the query block width (0 = no).
uint32_t qb_sq8_mma_block(const qb_storage* s, uint32_t nq) {
    if (s->kind != QB_KIND_SQ8 || s->qdist == QB_QD_L1) return 0;
    if (nq < 32 || s->count < 4 * 128) return 0;
    if (!sq8_scores_finite(s)) return 0;
    return block_for(s, nq);
}
// scratch the filter-mode scan needs (bias rows, bias integers, the batch threshold)
size_t qb_sq8_mma_scratch_bytes(const qb_storage*, uint32_t nq_pad) { return (size_t)nq_pad * (BIAS_KB + 4) + 256; }

// d_q_codes: [>= nq_pad][ad] u8 query codes (rows past nq are never scored).  Dense emit = sample pass (no thresholds yet);
// filter emit = main pass: queries are sorted by threshold first, survivors land in per-(query, CTA) segments and *seg_len
// (if given) returns the fixed length of each query's candidate row (zero = empty slot).
qb_status qb_sq8_mma_scan(const qb_storage* s, const uint8_t* d_q_codes, uint32_t nq_pad, const float* d_q_off, uint32_t nq, uint32_t n_blk,
                          uint64_t row_begin, uint64_t row_end, const QbEmit& emit, unsigned int* d_flags, unsigned long long* seg_len, void* d_scratch,
                          size_t scratch_bytes, cudaStream_t stream) {
    if (seg_len) *seg_len = 0;
    QB_CHECK(row_begin == 0, QB_ERR_INVALID, "sq8_mma_scan: scans start at row 0");
    QB_CHECK(emit.dense || (emit.thr && emit.cnt), QB_ERR_INVALID, "sq8_mma_scan: filter mode needs thresholds and counters");
    const uint32_t ad = s->actual_dim;
    const uint32_t n_qblocks = (nq + n_blk - 1) / n_blk;
    QB_CHECK(nq_pad >= n_qblocks * n_blk && nq_pad % 16 == 0, QB_ERR_INVALID, "sq8_mma_scan: query buffer not padded");
    MmaParams p{};
    p.voff = s->d_voff; p.n_rows = row_end; p.ad = ad; p.n_qblocks = n_qblocks; p.nq = nq;
    p.multiplier = s->multiplier; p.q_off = d_q_off; p.flags = d_flags;
    p.check_exact = ((uint64_t)ad * 127ull * 127ull >= (1ull << 24)) ? 1 : 0;
    p.debug = qb_opt().mma_debug;
    if (!emit.dense && s->multiplier > 0.0f && !(p.debug & 2)) {
        QB_CHECK(d_scratch && scratch_bytes >= qb_sq8_mma_scratch_bytes(s, nq_pad), QB_ERR_INVALID, "sq8_mma_scan: scratch too small");
        uint8_t* sc = reinterpret_cast<uint8_t*>(d_scratch);
        uint8_t* bias_rows = sc;                                                       // [nq_pad][32]
        int* bias_i = reinterpret_cast<int*>(sc + (size_t)nq_pad * BIAS_KB);            // [nq_pad]
        int* t_int = bias_i + nq_pad;
        qb_mma_bias_kernel<<<1, 1024, 0, stream>>>(emit.thr, d_q_off, s->multiplier, nq, nq_pad, bias_rows, bias_i, t_int);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        p.bias_rows = bias_rows; p.bias_i = bias_i; p.t_int = t_int;
    }
    CUtensorMap map_a, map_b;
    QB_TRY(make_map_u8(&map_a, s->d_codes, ad, row_end, KB, MMA_M));
    QB_TRY(make_map_u8(&map_b, d_q_codes, ad, nq_pad, KB, n_blk));
    const uint64_t n_tiles = (row_end + MMA_M - 1) / MMA_M;
    uint32_t workers = (uint32_t)s->sm_count / n_qblocks;
    if (workers < 1) workers = 1;
    if (workers > n_tiles) workers = (uint32_t)n_tiles;
    p.n_workers = workers;
    const uint32_t n_seg = workers;  // CTAs that ever see a given query
    if (!emit.dense && seg_len && !qb_opt().mma_no_segments) {
        uint64_t seg = (emit.cap / n_seg) & ~15ull;
        const uint64_t seg_max = qb_opt().mma_seg_cap ? qb_opt().mma_seg_cap : 256;   // slots per (query, CTA): the selection scans all of them
        if (seg > seg_max) seg = seg_max;
        if (seg >= 64) {
            p.seg_cap = (uint32_t)seg;
            *seg_len = (unsigned long long)n_seg * seg;
            QB_CUDA(cudaMemset2DAsync(emit.cand, emit.cap * 8, 0, (size_t)n_seg * seg * 8, nq, stream));
        }
    }
    return launch_mma<false>(map_a, map_b, p, emit, n_blk, stream);
}

// ---------------------------------------------------------------------------------------------- dense f32 batches (F16 prefilter + exact rescoring)
// bf16 shadow plane of a dense f32 storage, built on first use (and rebuilt after rows were rewritten): +50 % HBM for the storage, the
// price of reading 2 bytes per element instead of 4 on every batched pass and of feeding the tensor cores.
qb_status qb_f32_shadow_ensure(qb_storage* s, cudaStream_t stream) {
    std::lock_guard<std::mutex> lk(s->mu);          // concurrent first batches build it once
    if (s->bf16_ready) return QB_OK;
    const uint32_t row_h = (uint32_t)round_up_u64(s->dim, 8);
    if (!s->d_bf16) {
        QB_CUDA(cudaMalloc(&s->d_bf16, std::max<size_t>((size_t)s->count * row_h * 2, 256)));
        QB_CUDA(cudaMalloc(&s->d_bf16_meta, 256));
        s->hbm_bytes += (uint64_t)s->count * row_h * 2;
    }
    s->bf16_row_h = row_h;
    QB_CUDA(cudaMemsetAsync(s->d_bf16_meta, 0, 256, stream));
    const uint64_t blocks = std::min<uint64_t>(ceil_div_u64(std::max<uint64_t>(s->count, 1), 32), (uint64_t)s->sm_count * 16);
    f32_to_bf16_rows_kernel<<<(unsigned)blocks, 256, 0, stream>>>(reinterpret_cast<const float*>(s->d_rows), s->row_stride / 4, s->dim, s->count, s->d_bf16, row_h,
                                                                  s->d_bf16_meta, s->d_bf16_meta + 1);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    unsigned int meta[2] = {0, 0};
    QB_CUDA(cudaMemcpyAsync(meta, s->d_bf16_meta, 8, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaStreamSynchronize(stream));
    s->bf16_ready = true;
    s->bf16_usable = meta[1] == 0;      // NaN / inf rows: OrderedFloat ranks NaN scores highest, only the exact kernels honour that
    return QB_OK;
}

// Query block width of the tensor-core prefilter for a dense f32 storage (0 = not applicable).
uint32_t qb_f32_mma_block(qb_storage* s, uint32_t nq, cudaStream_t stream) {
    if (s->kind != QB_KIND_DENSE || s->dtype != QB_DT_F32) return 0;
    if (s->distance != QB_DIST_DOT && s->distance != QB_DIST_COSINE) return 0;   // the approximation bounds a dot product
    if (nq < 32 || s->count < 65536 || s->dim < 32 || qb_opt().disable_mma) return 0;
    if (qb_f32_shadow_ensure(s, stream) != QB_OK) { cudaGetLastError(); return 0; }  // e.g. no room for the shadow plane: stay on the exact kernels
    if (!s->bf16_usable) return 0;                                                // NaN / inf rows: only the exact kernels honour OrderedFloat
    const uint32_t k_bytes = (uint32_t)round_up_u64(s->dim, 8) * 2;
    return block_for_bytes(k_bytes, nq);
}
size_t qb_f32_mma_scratch_bytes(const qb_storage* s, uint32_t nq_pad) { return (size_t)nq_pad * ((size_t)round_up_u64(s->dim, 8) * 2 + BIAS_KB + 4) + 512; }

// Filter pass over rows [0, row_end): survivors of the bf16 prefilter are re-scored exactly and land, with their exact scores, in the
// counted candidate lists of `emit` (emit.thr = exact per-query thresholds).  d_q_pre = preprocessed f32 queries [nq][q_stride_f].
// Returns QB_ERR_UNSUPPORTED (nothing launched) when the storage holds non-finite values: the caller takes the exact path.
qb_status qb_f32_mma_scan(qb_storage* s, const float* d_q_pre, uint32_t q_stride_f, uint32_t nq, uint32_t nq_pad, uint32_t n_blk, uint64_t row_end, const QbEmit& emit,
                          unsigned int* d_flags, void* d_scratch, size_t scratch_bytes, cudaStream_t stream) {
    QB_CHECK(!emit.dense && emit.thr && emit.cnt, QB_ERR_INVALID, "f32_mma_scan: filter mode only");
    QB_CHECK(s->bf16_ready && s->bf16_usable, QB_ERR_INVALID, "f32_mma_scan: no usable bf16 shadow (qb_f32_mma_block decides)");
    const uint32_t row_h = s->bf16_row_h, ad = row_h * 2;
    const uint32_t n_qblocks = (nq + n_blk - 1) / n_blk;
    QB_CHECK(nq_pad >= n_qblocks * n_blk && nq_pad % 16 == 0, QB_ERR_INVALID, "f32_mma_scan: query block not padded");
    QB_CHECK(d_scratch && scratch_bytes >= qb_f32_mma_scratch_bytes(s, nq_pad), QB_ERR_INVALID, "f32_mma_scan: scratch too small");
    uint8_t* sc = reinterpret_cast<uint8_t*>(d_scratch);
    uint16_t* qb = reinterpret_cast<uint16_t*>(sc);
    uint8_t* bias_rows = sc + round_up_u64((size_t)nq_pad * ad, 256);
    int* bias_f = reinterpret_cast<int*>(bias_rows + (size_t)nq_pad * BIAS_KB);
    int* t_word = bias_f + nq_pad;
    f16_prepare_kernel<<<1, 1024, 0, stream>>>(d_q_pre, q_stride_f, s->dim, row_h, nq, nq_pad, emit.thr, s->d_bf16_meta, qb, bias_rows, bias_f, t_word, d_flags);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    MmaParams p{};
    p.voff = nullptr; p.n_rows = row_end; p.ad = ad; p.n_qblocks = n_qblocks; p.nq = nq;
    p.multiplier = 1.0f; p.q_off = nullptr; p.flags = d_flags; p.check_exact = 0; p.debug = qb_opt().mma_debug;
    p.bias_rows = bias_rows; p.bias_i = bias_f; p.t_int = t_word; p.seg_cap = 0;
    CUtensorMap map_a, map_b;
    QB_TRY(make_map_u8(&map_a, s->d_bf16, ad, row_end, KB, MMA_M));
    QB_TRY(make_map_u8(&map_b, qb, ad, nq_pad, KB, n_blk));
    const uint64_t n_tiles = (row_end + MMA_M - 1) / MMA_M;
    uint32_t workers = (uint32_t)s->sm_count / n_qblocks;
    if (workers < 1) workers = 1;
    if (workers > n_tiles) workers = (uint32_t)n_tiles;
    p.n_workers = workers;
    QB_TRY(launch_mma<true>(map_a, map_b, p, emit, n_blk, stream));
    // exact scores for the survivors (and only them)
    const dim3 grid(8, std::min<uint32_t>(nq, (uint32_t)s->sm_count * 4));
    f32_rescore_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const uint8_t*>(s->d_rows), s->row_stride, s->dim, d_q_pre, q_stride_f, nq, emit.cand, emit.cnt, emit.cap,
                                                 emit.thr, emit.id_base);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}
