// qb_dense.cu — f32 dense metrics (dot / cosine / euclid / manhattan) on H100.
//
// Replaces: Metric<f32>::similarity / preprocess (lib/segment/src/spaces/simple.rs:36-206) as dispatched on an
// AVX2+FMA host — dot_similarity_avx / euclid_similarity_avx / manhattan_similarity_avx / cosine_preprocess_avx
// (simple_avx.rs:32-213), the SSE tier for 16 <= dim < 32 (simple_sse.rs) and the scalar tier below that
// (simple.rs:214-239) — as called per (query, point) pair by MetricQueryScorer::score_stored_batch
// (vector_storage/query_scorer/metric_query_scorer.rs:81-92) from the brute-force scan loop
// (index/hnsw_index/point_scorer.rs:423-472) and from HNSW hops (FilteredScorer::score_points, :265-295).
//
// Bit-exactness (SURVEY Appendix A): the AVX kernels keep 32 partial sums P[a][l] (4 ymm accumulators x 8 lanes),
// element e of every 32-block is FMA-ed into P[e/8][e%8] in block order, then reduced as
// T[l]=(P0[l]+P1[l])+(P2[l]+P3[l]); L[i]=T[i+4]+T[i]; r=(L0+L1)+(L2+L3); the n%32 tail is added unfused.
// Here 8 consecutive lanes own one row; lane t owns the four positions e=4t..4t+3 (one float4 per block), so the
// FMA chains are identical, and the tree is three shuffles (xor 2, 4, 1) + the in-lane hadd.  All arithmetic uses
// explicit _rn intrinsics so nvcc can neither contract nor re-associate.
//
// Streaming scan (the HBM-bound headline kernel): persistent CTAs, one per SM; a producer lane feeds a ring of
// shared-memory slots with 1-D bulk async copies (cp.async.bulk, the TMA engine; rows are contiguous so no tensor
// map is needed), completion on mbarriers; 8 consumer warps each own every 8th slot, read rows and the query from
// shared memory with conflict-free 128-bit loads and emit candidates that pass the per-query threshold.
#include "qb_internal.h"
#include "qb_fold.cuh"
#include "qb_localk.cuh"
#include "qb_score.cuh"

namespace {

using namespace qbs;

// ------------------------------------------------------------------------------------------------
// streaming scan kernel
// ------------------------------------------------------------------------------------------------
constexpr int STREAM_CONSUMER_WARPS = 8;
constexpr int STREAM_THREADS = 32 * (STREAM_CONSUMER_WARPS + 1);

struct StreamParams {
    const uint8_t* rows;        // storage base
    uint32_t stride;            // bytes per row (multiple of 16)
    uint32_t dim;
    uint64_t row_begin, row_end;
    const float* q;             // [nq][stride/4] preprocessed queries (device)
    uint32_t nq;
    uint32_t rows_per_slot;     // multiple of 4
    uint32_t n_slots;
    uint32_t slot_bytes;        // rows_per_slot * stride
    uint32_t q_smem_bytes;      // nq * stride rounded up to 128
    int l2_keep;                // 1: data set fits L2 -> keep it resident (evict_last); 0: stream (evict_first)
    // custom queries: the nq "queries" are the example vectors of ONE query and a row's nq similarities are folded (Query::score_by,
    // qb_fold.cuh) into the single score that is emitted for query slot 0; fold_kind = 0: plain batch, every query emits its own score
    int fold_kind;
    uint32_t fold_na, fold_nb;
    const float* fold_coef;
};

// one row against the p.nq queries staged in shared memory, row read once (score_avx_group8_multi); emits per query, or the fold
template <int METRIC, int NQ>
__device__ __forceinline__ void stream_score_multi(const StreamParams& p, const QbEmit& emit, const float* rp, const float* q_s, uint32_t stride_f, int t, bool valid,
                                                   uint64_t slot) {
    float sc[NQ];
    // queries past p.nq alias query 0 (computed, never emitted)
    score_avx_group8_multi<METRIC, NQ>(rp, q_s, (NQ == 1) ? 0u : stride_f, p.dim, t, sc);
    if (!(valid && t == 0)) return;
    if (p.fold_kind) {
        const float f = qbf::fold(p.fold_kind, p.fold_na, p.fold_nb, p.fold_coef, [&](uint32_t e) { return sc[e < (uint32_t)NQ ? e : 0]; });
        qb_emit(emit, 0, slot, (uint32_t)slot, f);
    } else {
#pragma unroll
        for (int q = 0; q < NQ; ++q)
            if ((uint32_t)q < p.nq) qb_emit(emit, q, slot, (uint32_t)slot, sc[q]);
    }
}

// LOCALK (single query, top <= 16): instead of a threshold pass + filtered emission, every consumer warp keeps its own k best keys
// in registers (qb_localk.cuh), so ONE scan + one small select replaces sample pass + threshold select + filter pass + select.
static_assert(STREAM_CONSUMER_WARPS == QB_LOCALK_WARPS, "the CTA merge sorts one list per consumer warp");

template <int METRIC, bool LOCALK>
__global__ void __launch_bounds__(STREAM_THREADS, 1) dense_f32_stream_kernel(const StreamParams p, const QbEmit emit) {
    extern __shared__ __align__(128) uint8_t smem[];
    if (LOCALK && emit.run_if && *emit.run_if == 0u) return;      // conditional launch (uniform): the prefilter path answered already
    float* q_s = reinterpret_cast<float*>(smem);
    uint8_t* slots = smem + p.q_smem_bytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(slots + (size_t)p.n_slots * p.slot_bytes);
    uint64_t* empty = full + p.n_slots;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t n_rows = p.row_end - p.row_begin;
    const uint64_t n_tiles = (n_rows + p.rows_per_slot - 1) / p.rows_per_slot;
    const uint64_t n_local = (blockIdx.x < n_tiles) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < p.n_slots; ++s) { qb_mbar_init(&full[s], 1); qb_mbar_init(&empty[s], 1); }
        qb_fence_barrier_init();
    }
    if (LOCALK && threadIdx.x < STREAM_CONSUMER_WARPS)
        reinterpret_cast<unsigned int*>(reinterpret_cast<unsigned long long*>(empty + p.n_slots) + STREAM_CONSUMER_WARPS * (QB_LOCALK_SLOTS + 4))[threadIdx.x] = 0u;
    // stage the queries (small, L2-resident) into shared memory; slots up to the next power of two repeat query 0 (the multi-query
    // scorer is instantiated for 2 / 4 / 8 / 16 queries and never emits the padding)
    {
        uint32_t nq_pad = 1;
        while (nq_pad < p.nq) nq_pad <<= 1;
        const uint32_t per = p.stride >> 4, n4 = nq_pad * per;
        const float4* src = reinterpret_cast<const float4*>(p.q);
        float4* dst = reinterpret_cast<float4*>(q_s);
        for (uint32_t i = threadIdx.x; i < n4; i += blockDim.x) dst[i] = (i / per < p.nq) ? src[i] : src[i % per];
    }
    __syncthreads();

    if (warp == 0) {
        if (lane == 0) {
            const uint64_t policy = p.l2_keep ? qb_policy_evict_last() : qb_policy_evict_first();
            // slot, phase and first row advance incrementally: a 64-bit division per copy costs the issuing thread more than the copy
            uint32_t s = 0, ph = 0;
            uint64_t r0 = p.row_begin + (uint64_t)blockIdx.x * p.rows_per_slot;
            const uint64_t r_step = (uint64_t)gridDim.x * p.rows_per_slot;
            for (uint64_t i = 0; i < n_local; ++i, r0 += r_step) {
                qb_mbar_wait(&empty[s], ph ^ 1u);
                const uint64_t left = p.row_end - r0;
                const uint32_t nr = (uint32_t)(left < p.rows_per_slot ? left : p.rows_per_slot);
                const uint32_t bytes = nr * p.stride;
                qb_mbar_arrive_expect_tx(&full[s], bytes);
                qb_bulk_g2s(slots + (size_t)s * p.slot_bytes, p.rows + r0 * p.stride, bytes, &full[s], policy);
                if (++s == p.n_slots) { s = 0; ph ^= 1u; }
            }
        }
    } else {
        const int cw = warp - 1;
        const int grp = lane >> 3, t = lane & 7;
        const uint32_t stride_f = p.stride >> 2;
        // LOCALK state: this warp's k best keys (lanes >= k hold the maximum so that they are never the minimum) and their minimum
        unsigned long long my_key = (LOCALK && lane < (int)emit.local_k) ? 0ull : ~0ull;
        unsigned long long wmin = 0ull;
        float wthr = __int_as_float(0xff800000);  // score of wmin once the list is full
        unsigned long long* lk_queue = reinterpret_cast<unsigned long long*>(empty + p.n_slots) + STREAM_CONSUMER_WARPS * QB_LOCALK_SLOTS;  // [8][4]
        unsigned int* lk_count = reinterpret_cast<unsigned int*>(lk_queue + STREAM_CONSUMER_WARPS * 4);                                   // [8]
        uint32_t s = (uint32_t)cw, ph = 0;                        // n_slots is a multiple of STREAM_CONSUMER_WARPS: s wraps exactly
        uint64_t r0 = p.row_begin + ((uint64_t)blockIdx.x + (uint64_t)cw * gridDim.x) * p.rows_per_slot;
        const uint64_t r_step = (uint64_t)STREAM_CONSUMER_WARPS * gridDim.x * p.rows_per_slot;
        for (uint64_t i = cw; i < n_local; i += STREAM_CONSUMER_WARPS, r0 += r_step, s += STREAM_CONSUMER_WARPS) {
            if (s >= p.n_slots) { s -= p.n_slots; ph ^= 1u; }
            const uint64_t left = p.row_end - r0;
            const uint32_t nr = (uint32_t)(left < p.rows_per_slot ? left : p.rows_per_slot);
            qb_mbar_wait(&full[s], ph);
            const float* slot = reinterpret_cast<const float*>(slots + (size_t)s * p.slot_bytes);
            for (uint32_t quad = 0; quad * 4 < nr; ++quad) {
                const uint32_t rin = quad * 4 + grp;
                const bool valid = rin < nr;
                const float* rp = slot + (size_t)(valid ? rin : nr - 1) * stride_f;
                if (LOCALK) {
                    // hot path = one float compare on one lane in eight; the few rows that beat the warp's current k-th score are
                    // queued in shared memory and folded into the register list by the whole warp right after the quad
                    const float sc = score_avx_group8<METRIC>(rp, q_s, p.dim, t);
                    if ((quad + 1) * 4 >= nr) {  // last quad: the slot's bytes are all in registers -> give it back to the producer BEFORE
                        __syncwarp();            // the bookkeeping (the kernel lives on bytes in flight: hold time is bandwidth)
                        if (lane == 0) qb_mbar_arrive(&empty[s]);
                    }
                    if (valid && t == 0 && !(sc < wthr)) lk_push(emit.deleted, emit.deleted2, emit.id_base, sc, (uint32_t)(r0 + rin), lk_queue + cw * 4, &lk_count[cw]);
                    __syncwarp();
                    const unsigned int n_queued = *reinterpret_cast<volatile unsigned int*>(&lk_count[cw]);
                    if (n_queued) {
                        const LkState st = lk_drain(LkState{my_key, wmin, wthr}, lk_queue + cw * 4, &lk_count[cw], lane, n_queued);
                        my_key = st.my_key; wmin = st.wmin; wthr = st.wthr;
                    }
                } else if (p.nq == 1 && !p.fold_kind) {
                    const float sc = score_avx_group8<METRIC>(rp, q_s, p.dim, t);
                    if (valid && t == 0) qb_emit(emit, 0, r0 + rin, (uint32_t)(r0 + rin), sc);
                } else if (p.nq <= 2) stream_score_multi<METRIC, 2>(p, emit, rp, q_s, stride_f, t, valid, r0 + rin);
                else if (p.nq <= 4) stream_score_multi<METRIC, 4>(p, emit, rp, q_s, stride_f, t, valid, r0 + rin);
                else if (p.nq <= 8) stream_score_multi<METRIC, 8>(p, emit, rp, q_s, stride_f, t, valid, r0 + rin);
                else stream_score_multi<METRIC, 16>(p, emit, rp, q_s, stride_f, t, valid, r0 + rin);
            }
            if (!LOCALK) {
                __syncwarp();
                if (lane == 0) qb_mbar_arrive(&empty[s]);
            }
        }
        if (LOCALK) {
            // CTA merge of the eight lists.  Only the consumer warps meet at a NAMED barrier: with __syncthreads() the 31 idle lanes of the
            // producer warp would sit in the barrier from the first cycle on and share issue slots with the one lane that feeds the ring.
            unsigned long long* lists = reinterpret_cast<unsigned long long*>(empty + p.n_slots);
            if (lane < QB_LOCALK_SLOTS) lists[cw * QB_LOCALK_SLOTS + lane] = (my_key == ~0ull) ? 0ull : my_key;
            asm volatile("bar.sync 1, %0;" ::"n"(STREAM_CONSUMER_WARPS * 32) : "memory");
            if (cw == 0) {  // four keys per lane, bitonic sort of 128 in shared memory, keep the first 16
                lk_cta_sort(lists, lane);
                if (lane < QB_LOCALK_SLOTS) emit.cand[(unsigned long long)blockIdx.x * QB_LOCALK_SLOTS + lane] = (lane < (int)emit.local_k) ? lists[lane] : 0ull;
                if (emit.done_counter) lk_last_cta_merge(emit.cand, emit.local_k, emit.final_out, emit.final_count, emit.done_counter, lane);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// group kernel: 8 lanes per candidate, rows read straight from global memory (gather lists, huge dims,
// RawScorer::score_points).  Either emits candidates (emit_mode) or writes scores[i].
// ------------------------------------------------------------------------------------------------
struct GroupParams {
    const uint8_t* rows;
    uint32_t stride, dim;
    uint64_t begin, end;        // candidate index range
    const uint32_t* ids;        // optional: candidate i -> row ids[i]; null: row = i
    const float* q;             // [nq][stride/4]
    uint32_t nq;
    float* scores;              // score mode: scores[q * (end-begin) + (i-begin)]
    int emit_mode;
};

template <int METRIC>
__global__ void __launch_bounds__(256) dense_f32_group_kernel(const GroupParams p, const QbEmit emit) {
    const int t = threadIdx.x & 7;
    const uint64_t groups_per_grid = (uint64_t)gridDim.x * (blockDim.x >> 3);
    const uint64_t g0 = (uint64_t)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3);
    const uint32_t stride_f = p.stride >> 2;
    const uint64_t n = p.end - p.begin;
    // all 32 lanes of a warp must stay in the loop together (shuffles): iterate on the warp's first group
    const uint64_t n_iter = (n + groups_per_grid - 1) / groups_per_grid;
    for (uint64_t it = 0; it < n_iter; ++it) {
        const uint64_t ci = g0 + it * groups_per_grid;
        const bool valid = ci < n;
        const uint64_t cand = p.begin + (valid ? ci : 0);
        const uint32_t row = p.ids ? p.ids[cand] : (uint32_t)cand;
        const float* rp = reinterpret_cast<const float*>(p.rows + (size_t)row * p.stride);
        for (uint32_t q = 0; q < p.nq; ++q) {
            float sc = score_avx_group8<METRIC>(rp, p.q + (size_t)q * stride_f, p.dim, t);
            if (valid && t == 0) {
                if (p.emit_mode) qb_emit(emit, q, cand, row, sc);
                else p.scores[(size_t)q * n + ci] = sc;
            }
        }
    }
}

// one thread per candidate for dim < 32
template <int METRIC>
__global__ void __launch_bounds__(256) dense_f32_small_kernel(const GroupParams p, const QbEmit emit) {
    const uint64_t n = p.end - p.begin;
    const uint32_t stride_f = p.stride >> 2;
    for (uint64_t ci = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; ci < n; ci += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t cand = p.begin + ci;
        const uint32_t row = p.ids ? p.ids[cand] : (uint32_t)cand;
        const float* rp = reinterpret_cast<const float*>(p.rows + (size_t)row * p.stride);
        for (uint32_t q = 0; q < p.nq; ++q) {
            float sc = score_small<METRIC>(rp, p.q + (size_t)q * stride_f, p.dim);
            if (p.emit_mode) qb_emit(emit, q, cand, row, sc);
            else p.scores[(size_t)q * n + ci] = sc;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Metric::preprocess (cosine normalisation; identity copy otherwise) — rows in, rows out (strided, zero padded)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool length_zero_or_normalized(float len) {  // spaces/tools.rs:14-16
    return len < 1.1920929e-07f || fabsf(__fsub_rn(len, 1.0f)) <= 1.0e-6f;
}

__global__ void __launch_bounds__(256) preprocess_rows_kernel(int normalize, uint32_t dim, uint64_t n, const float* in,
                                                              uint64_t in_stride_f, float* out, uint64_t out_stride_f) {
    const int t = threadIdx.x & 7;
    const uint64_t groups_per_grid = (uint64_t)gridDim.x * (blockDim.x >> 3);
    const uint64_t g0 = (uint64_t)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3);
    const uint64_t n_iter = (n + groups_per_grid - 1) / groups_per_grid;
    const bool aligned = ((in_stride_f & 3) == 0) && ((reinterpret_cast<uintptr_t>(in) & 15) == 0);
    for (uint64_t it = 0; it < n_iter; ++it) {
        const uint64_t r = g0 + it * groups_per_grid;
        const bool valid = r < n;
        const float* src = in + (valid ? r : 0) * in_stride_f;
        float len = 0.f;
        bool scale = false;
        if (normalize) {
            if (dim >= 32 && aligned) len = score_avx_group8<M_DOT>(src, src, dim, t);
            else if (dim >= 32) {
                // unaligned host layout: same arithmetic with scalar loads (lane t owns positions 4t..4t+3)
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                const uint32_t nblk = dim >> 5;
                for (uint32_t b = 0; b < nblk; ++b) {
                    const float* s4 = src + b * 32 + 4 * t;
                    acc.x = __fmaf_rn(s4[0], s4[0], acc.x); acc.y = __fmaf_rn(s4[1], s4[1], acc.y);
                    acc.z = __fmaf_rn(s4[2], s4[2], acc.z); acc.w = __fmaf_rn(s4[3], s4[3], acc.w);
                }
                acc = add4(acc, shfl_xor4(acc, 2)); acc = add4(acc, shfl_xor4(acc, 4)); acc = add4(acc, shfl_xor4(acc, 1));
                len = __fadd_rn(__fadd_rn(acc.x, acc.y), __fadd_rn(acc.z, acc.w));
                for (uint32_t i = nblk << 5; i < dim; ++i) len = __fadd_rn(len, __fmul_rn(src[i], src[i]));
            } else len = score_small<M_DOT>(src, src, dim);
            scale = !length_zero_or_normalized(len);
            if (scale) len = __fsqrt_rn(len);
        }
        __syncwarp();  // in-place: every lane has finished reading the row before any lane rewrites it
        if (valid) {
            float* dst = out + r * out_stride_f;
            if (in == out && !scale) {
                for (uint64_t i = dim + t; i < out_stride_f; i += 8) dst[i] = 0.f;
            } else {
                for (uint64_t i = t; i < out_stride_f; i += 8) {
                    float x = (i < dim) ? src[i] : 0.f;
                    dst[i] = (scale && i < dim) ? __fdiv_rn(x, len) : x;
                }
            }
        }
    }
}

template <int METRIC>
qb_status launch_group(const GroupParams& gp, const QbEmit& emit, int sm_count, cudaStream_t stream) {
    const uint64_t n = gp.end - gp.begin;
    if (n == 0) return QB_OK;
    if (gp.dim >= 32) {
        uint64_t blocks = ceil_div_u64(n, 256 / 8);
        uint64_t maxb = (uint64_t)sm_count * 8;
        if (blocks > maxb) blocks = maxb;
        dense_f32_group_kernel<METRIC><<<(unsigned)blocks, 256, 0, stream>>>(gp, emit);
    } else {
        uint64_t blocks = ceil_div_u64(n, 256);
        uint64_t maxb = (uint64_t)sm_count * 8;
        if (blocks > maxb) blocks = maxb;
        dense_f32_small_kernel<METRIC><<<(unsigned)blocks, 256, 0, stream>>>(gp, emit);
    }
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

template <int METRIC, bool LOCALK = false>
qb_status launch_stream(const StreamParams& sp_in, const QbEmit& emit, int sm_count, cudaStream_t stream, bool* done, unsigned* grid_out = nullptr) {
    StreamParams sp = sp_in;
    *done = false;
    const uint32_t kMaxSmem = 227 * 1024;
    uint32_t nq_pad = 1;
    while (nq_pad < sp.nq) nq_pad <<= 1;
    sp.q_smem_bytes = (uint32_t)round_up_u64((uint64_t)nq_pad * sp.stride, 128);
    uint32_t rps = (16384 / sp.stride) & ~3u;
    if (rps < 4) rps = 4;
    sp.rows_per_slot = rps;
    sp.slot_bytes = rps * sp.stride;
    if (sp.q_smem_bytes + 2048 >= kMaxSmem) return QB_OK;
    uint32_t budget = kMaxSmem - sp.q_smem_bytes - 2048;
    uint32_t n_slots = budget / sp.slot_bytes;
    if (n_slots > 64) n_slots = 64;
    n_slots = (n_slots / STREAM_CONSUMER_WARPS) * STREAM_CONSUMER_WARPS;
    if (n_slots < STREAM_CONSUMER_WARPS) return QB_OK;  // rows too wide for the ring: caller uses the group kernel
    sp.n_slots = n_slots;
    // ring + barriers (+ the per-warp top-k lists of the LOCALK merge; the 1024-byte reserve above covers them)
    const size_t smem = (size_t)sp.q_smem_bytes + (size_t)n_slots * sp.slot_bytes + (size_t)n_slots * 16 +
                        (LOCALK ? (size_t)STREAM_CONSUMER_WARPS * (QB_LOCALK_SLOTS * 8 + 4 * 8 + 4) : 0);
    QB_CUDA(cudaFuncSetAttribute(dense_f32_stream_kernel<METRIC, LOCALK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
    const uint64_t n_tiles = ceil_div_u64(sp.row_end - sp.row_begin, sp.rows_per_slot);
    unsigned grid = (unsigned)(n_tiles < (uint64_t)sm_count ? n_tiles : (uint64_t)sm_count);
    if (grid_out) *grid_out = grid;
    dense_f32_stream_kernel<METRIC, LOCALK><<<grid, STREAM_THREADS, smem, stream>>>(sp, emit);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    *done = true;
    return QB_OK;
}

int metric_of(qb_distance d) {
    switch (d) {
        case QB_DIST_EUCLID: return M_EUCLID;
        case QB_DIST_MANHATTAN: return M_MANHATTAN;
        default: return M_DOT;  // cosine = dot on normalised vectors (simple.rs:174-176)
    }
}

}  // namespace

// ---------------------------------------------------------------- host entry points for dense f32
qb_status qb_dense_f32_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream) {
    const int metric = metric_of(s->distance);
    const uint64_t n = a.row_end - a.row_begin;
    if (n == 0 || a.nq == 0) return QB_OK;
    // streaming ring for contiguous ranges of wide-enough rows; queries are processed in chunks that fit smem
    if (!a.d_ids && s->dim >= 32 && n >= 1024) {
        const uint32_t q_chunk_max = 16;
        bool all_done = true;
        for (uint32_t q0 = 0; q0 < a.nq && all_done; q0 += q_chunk_max) {
            const uint32_t qn = (a.nq - q0 < q_chunk_max) ? a.nq - q0 : q_chunk_max;
            StreamParams sp{};
            sp.rows = reinterpret_cast<const uint8_t*>(s->d_rows);
            sp.stride = s->row_stride; sp.dim = s->dim;
            sp.row_begin = a.row_begin; sp.row_end = a.row_end;
            sp.q = reinterpret_cast<const float*>(a.d_q_enc) + (size_t)q0 * (s->row_stride / 4);
            sp.nq = qn;
            sp.l2_keep = (s->hbm_bytes <= (64ull << 20)) ? 1 : 0;
            QbEmit e = a.emit;
            if (e.thr) e.thr += q0;
            if (e.cnt) e.cnt += q0;
            e.cand += (unsigned long long)q0 * e.cap;
            bool done = false;
            qb_status st;
            switch (metric) {
                case M_EUCLID: st = launch_stream<M_EUCLID>(sp, e, s->sm_count, stream, &done); break;
                case M_MANHATTAN: st = launch_stream<M_MANHATTAN>(sp, e, s->sm_count, stream, &done); break;
                default: st = launch_stream<M_DOT>(sp, e, s->sm_count, stream, &done); break;
            }
            QB_TRY(st);
            if (!done) { all_done = false; QB_CHECK(q0 == 0, QB_ERR_CUDA, "stream kernel configuration changed mid-batch"); }
        }
        if (all_done) return QB_OK;
    }
    GroupParams gp{};
    gp.rows = reinterpret_cast<const uint8_t*>(s->d_rows);
    gp.stride = s->row_stride; gp.dim = s->dim;
    gp.begin = a.row_begin; gp.end = a.row_end;
    gp.ids = a.d_ids; gp.q = reinterpret_cast<const float*>(a.d_q_enc); gp.nq = a.nq;
    gp.scores = nullptr; gp.emit_mode = 1;
    switch (metric) {
        case M_EUCLID: return launch_group<M_EUCLID>(gp, a.emit, s->sm_count, stream);
        case M_MANHATTAN: return launch_group<M_MANHATTAN>(gp, a.emit, s->sm_count, stream);
        default: return launch_group<M_DOT>(gp, a.emit, s->sm_count, stream);
    }
}

// Custom query over a contiguous row range in ONE pass: the a.nq encoded "queries" are the example vectors, every row's similarities are
// folded in the kernel (no [examples][rows] matrix, rows read once).  *done = false when the shape does not suit the streaming kernel.
qb_status qb_dense_f32_scan_fold(const qb_storage* s, const QbScanArgs& a, int kind, uint32_t n_a, uint32_t n_b, const float* d_coef, bool* done, cudaStream_t stream) {
    *done = false;
    const uint64_t n = a.row_end - a.row_begin;
    if (a.d_ids || s->dim < 32 || n < 1024 || a.nq < 1 || a.nq > 16) return QB_OK;
    StreamParams sp{};
    sp.rows = reinterpret_cast<const uint8_t*>(s->d_rows);
    sp.stride = s->row_stride; sp.dim = s->dim;
    sp.row_begin = a.row_begin; sp.row_end = a.row_end;
    sp.q = reinterpret_cast<const float*>(a.d_q_enc);
    sp.nq = a.nq;
    sp.l2_keep = (s->hbm_bytes <= (64ull << 20)) ? 1 : 0;
    sp.fold_kind = kind; sp.fold_na = n_a; sp.fold_nb = n_b; sp.fold_coef = d_coef;
    switch (metric_of(s->distance)) {
        case M_EUCLID: return launch_stream<M_EUCLID>(sp, a.emit, s->sm_count, stream, done);
        case M_MANHATTAN: return launch_stream<M_MANHATTAN>(sp, a.emit, s->sm_count, stream, done);
        default: return launch_stream<M_DOT>(sp, a.emit, s->sm_count, stream, done);
    }
}

// Single-query scan with per-CTA top-k lists (top <= 16): writes *n_slots candidate keys (zeros = empty) to a.emit.cand.
// *n_slots = 0 when the shape does not suit the streaming kernel (the caller then takes the generic path).
qb_status qb_dense_f32_scan_localk(const qb_storage* s, const QbScanArgs& a, uint32_t top, uint64_t* n_slots, cudaStream_t stream, uint64_t min_rows) {
    *n_slots = 0;
    const uint64_t n = a.row_end - a.row_begin;
    if (a.d_ids || a.nq != 1 || top > (uint32_t)QB_LOCALK_SLOTS || s->dim < 32 || n < min_rows) return QB_OK;
    StreamParams sp{};
    sp.rows = reinterpret_cast<const uint8_t*>(s->d_rows);
    sp.stride = s->row_stride; sp.dim = s->dim;
    sp.row_begin = a.row_begin; sp.row_end = a.row_end;
    sp.q = reinterpret_cast<const float*>(a.d_q_enc);
    sp.nq = 1;
    sp.l2_keep = (s->hbm_bytes <= (64ull << 20)) ? 1 : 0;
    QbEmit e = a.emit;
    e.local_k = top;
    bool done = false;
    unsigned grid = 0;
    qb_status st;
    switch (metric_of(s->distance)) {
        case M_EUCLID: st = launch_stream<M_EUCLID, true>(sp, e, s->sm_count, stream, &done, &grid); break;
        case M_MANHATTAN: st = launch_stream<M_MANHATTAN, true>(sp, e, s->sm_count, stream, &done, &grid); break;
        default: st = launch_stream<M_DOT, true>(sp, e, s->sm_count, stream, &done, &grid); break;
    }
    QB_TRY(st);
    if (done) *n_slots = (uint64_t)grid * QB_LOCALK_SLOTS;
    return QB_OK;
}

qb_status qb_dense_f32_score_points(const qb_storage* s, const void* d_q_enc, const uint32_t* d_ids, uint64_t n, float* d_scores,
                                    cudaStream_t stream) {
    GroupParams gp{};
    gp.rows = reinterpret_cast<const uint8_t*>(s->d_rows);
    gp.stride = s->row_stride; gp.dim = s->dim;
    gp.begin = 0; gp.end = n; gp.ids = d_ids;
    gp.q = reinterpret_cast<const float*>(d_q_enc); gp.nq = 1;
    gp.scores = d_scores; gp.emit_mode = 0;
    QbEmit e{};
    switch (metric_of(s->distance)) {
        case M_EUCLID: return launch_group<M_EUCLID>(gp, e, s->sm_count, stream);
        case M_MANHATTAN: return launch_group<M_MANHATTAN>(gp, e, s->sm_count, stream);
        default: return launch_group<M_DOT>(gp, e, s->sm_count, stream);
    }
}

qb_status qb_launch_preprocess_rows(qb_distance distance, uint32_t dim, uint64_t n, const float* in, uint64_t in_stride_f, float* out,
                                    uint64_t out_stride_f, cudaStream_t stream) {
    if (n == 0) return QB_OK;
    uint64_t blocks = ceil_div_u64(n, 256 / 8);
    if (blocks > 132 * 16) blocks = 132 * 16;
    preprocess_rows_kernel<<<(unsigned)blocks, 256, 0, stream>>>(distance == QB_DIST_COSINE ? 1 : 0, dim, n, in, in_stride_f, out, out_stride_f);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}
