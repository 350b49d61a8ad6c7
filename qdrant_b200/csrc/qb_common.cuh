// qb_common.cuh — shared device/host helpers for libqdrant_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/qb200.h"

// ------------------------------------------------------------------------------------------------
// host-side error plumbing
// ------------------------------------------------------------------------------------------------
void qb_set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_qb_launches;

#define QB_CUDA(call)                                                                          \
    do {                                                                                       \
        cudaError_t _e = (call);                                                               \
        if (_e != cudaSuccess) {                                                               \
            qb_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
            return (_e == cudaErrorMemoryAllocation) ? QB_ERR_OOM : QB_ERR_CUDA;               \
        }                                                                                      \
    } while (0)

#define QB_CHECK(cond, status, ...)      \
    do {                                 \
        if (!(cond)) {                   \
            qb_set_error(__VA_ARGS__);   \
            return (status);             \
        }                                \
    } while (0)

#define QB_TRY(expr)                    \
    do {                                \
        qb_status _s = (expr);          \
        if (_s != QB_OK) return _s;     \
    } while (0)

struct QbOptions {
    bool disable_localk = false, disable_mma = false, mma_no_segments = false, verbose = false;
    int mma_debug = 0;
    int pq_queries_per_pass = 0;   // 0 = automatic
    int hnsw_threads = 0;          // 0 / 128 (default) or 256 threads per traversal CTA
    bool hnsw_no_prefetch = false;
    int prefilter_producers = 0;       // single-query prefilter: producer warps per CTA (0 = default)
    uint32_t prefilter_slot_bytes = 0; // single-query prefilter: target bytes per ring slot (0 = default)
    int prefilter_plane = 0;          // single-query prefilter: 0 = 6-bit shadow plane when the storage allows it, 1 = bf16, 2 = int8 shadow plane
    int prefilter_stage1 = 0;         // first stage of the 6-bit plane's scan: 5 = its own 5-bit codes (no extra plane), otherwise the block-scaled 4-bit plane
    bool disable_prefilter = false;   // single-query dense f32 searches: always the exact f32 scan (no bf16 shadow plane, qb_prefilter.cu)
    uint32_t mma_seg_cap = 0;      // 0 = 256 survivor slots per (query, CTA) segment of the tensor-core scan
    uint64_t sample_rows = 0;
    uint32_t hnsw_heal_stack = 0;  // qb_hnsw_build_incremental: DFS stack entries per CTA on the first run (0 = 16384)
};
QbOptions& qb_opt();

#define QB_LAUNCHED() (g_qb_launches.fetch_add(1, std::memory_order_relaxed))

static inline uint64_t ceil_div_u64(uint64_t a, uint64_t b) { return (a + b - 1) / b; }
static inline uint64_t round_up_u64(uint64_t a, uint64_t b) { return ceil_div_u64(a, b) * b; }

// ------------------------------------------------------------------------------------------------
// candidate keys: (orderable(score) << 32) | ~id  — descending u64 order == (score desc, id asc).
// ScoredPointOffset orders by OrderedFloat(score) only (lib/common/common/src/types.rs:21-25); the id
// tie-break is ours and makes results independent of CTA scheduling.  Scores keep their bit pattern: -0.0 is NOT folded
// into +0.0 (OrderedFloat calls them equal, so ranking -0.0 just below +0.0 is one of the orders the reference allows, and
// a returned -0.0 stays -0.0); every NaN maps to one key above +inf (OrderedFloat: NaN is the greatest value and equal
// to itself) and comes back as the canonical quiet NaN.  Key 0 is reserved as "empty".
// ------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t qb_orderable(float s) {
    uint32_t u;
#ifdef __CUDA_ARCH__
    u = __float_as_uint(s);
#else
    memcpy(&u, &s, 4);
#endif
    if ((u & 0x7FFFFFFFu) > 0x7F800000u) return 0xFFC00000u;  // NaN (either sign): above +inf; decodes to 0x7FC00000
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float qb_unorderable(uint32_t o) {
    uint32_t u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
__host__ __device__ __forceinline__ unsigned long long qb_pack_key(float score, uint32_t id) {
    return ((unsigned long long)qb_orderable(score) << 32) | (unsigned long long)(0xFFFFFFFFu - id);
}
__host__ __device__ __forceinline__ uint32_t qb_key_id(unsigned long long k) { return 0xFFFFFFFFu - (uint32_t)(k & 0xFFFFFFFFull); }
__host__ __device__ __forceinline__ float qb_key_score(unsigned long long k) { return qb_unorderable((uint32_t)(k >> 32)); }

// ------------------------------------------------------------------------------------------------
// Emission of (query, id, score) candidates from scan kernels (see qb_topk.cu for the selection side)
//   dense mode : cand[q*cap + (id - dense_base)] = key        (no atomics; used for sample / small scans)
//   filter mode: if score >= thr[q]: append via atomicAdd(cnt[q])
// ------------------------------------------------------------------------------------------------
struct QbEmit {
    const float* thr;               // per query threshold (filter mode)
    unsigned int* cnt;              // per query candidate counter (filter mode)
    unsigned long long* cand;       // [n_queries][cap]
    const uint32_t* deleted;        // resident soft-delete bits (32-bit words) or null
    const uint32_t* deleted2;       // per-call soft-delete bits or null
    unsigned long long cap;         // per-query capacity
    unsigned long long dense_base;  // dense mode: position = slot - dense_base
    int dense;                      // 1 = dense mode
    uint32_t id_base;               // added to reported ids (row offset of this shard inside the sharded segment set)
    uint32_t local_k;               // per-CTA top-k mode of the dense streaming kernel: entries kept per warp / written per CTA
    // per-CTA top-k mode: the LAST CTA to finish merges the per-CTA lists and writes the query's final top-k here (no select launch)
    qb_scored_point* final_out; uint32_t* final_count; unsigned int* done_counter;
    const unsigned int* run_if;     // per-CTA top-k mode: when set, the scan runs only if *run_if != 0 (device-side fallback of qb_prefilter.cu)
};

#ifdef __CUDACC__
__device__ __forceinline__ bool qb_is_deleted(const QbEmit& e, uint32_t id) {
    bool d = false;
    if (e.deleted) d = (e.deleted[id >> 5] >> (id & 31)) & 1u;
    if (e.deleted2) d = d || ((e.deleted2[id >> 5] >> (id & 31)) & 1u);
    return d;
}
// `slot` is the position of the candidate in scan order (row index for full scans, index into the id list
// for filtered scans); `id` is the point offset reported to the caller.
__device__ __forceinline__ void qb_emit(const QbEmit& e, uint32_t q, unsigned long long slot, uint32_t id, float score) {
    if (e.dense) {
        unsigned long long key = qb_is_deleted(e, id) ? 0ull : qb_pack_key(score, id + e.id_base);
        e.cand[(unsigned long long)q * e.cap + (slot - e.dense_base)] = key;
    } else {
        if (!(score < e.thr[q]) && !qb_is_deleted(e, id)) {   // NaN ranks highest: it passes
            unsigned int pos = atomicAdd(&e.cnt[q], 1u);
            if (pos < e.cap) e.cand[(unsigned long long)q * e.cap + pos] = qb_pack_key(score, id + e.id_base);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// mbarrier + bulk async copy (TMA engine, 1-D) helpers.  SASS: SYNCS.*, UBLKCP.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t qb_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void qb_mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(qb_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void qb_fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void qb_mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(qb_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void qb_mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(qb_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool qb_mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(qb_smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must trap (visible error) instead of hanging the GPU box.
__device__ __forceinline__ void qb_mbar_wait(uint64_t* bar, uint32_t parity) {
    if (qb_mbar_try_wait(bar, parity)) return;
    long long t0 = clock64();
    while (!qb_mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 8000000000ll) __trap();  // ~4 s at 2 GHz
    }
}
// same, for producers that run far ahead of their consumers: back off between polls so the spin does not compete for issue slots
__device__ __forceinline__ void qb_mbar_wait_relaxed(uint64_t* bar, uint32_t parity) {
    if (qb_mbar_try_wait(bar, parity)) return;
    long long t0 = clock64();
    while (!qb_mbar_try_wait(bar, parity)) {
        __nanosleep(100);
        if (clock64() - t0 > 8000000000ll) __trap();
    }
}
// global -> shared bulk copy, completion signalled on an mbarrier (bytes, src, dst 16-B aligned)
__device__ __forceinline__ void qb_bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            qb_smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(qb_smem_u32(bar)), "l"(policy)
        : "memory");
}
__device__ __forceinline__ uint64_t qb_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t qb_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
#endif  // __CUDACC__
