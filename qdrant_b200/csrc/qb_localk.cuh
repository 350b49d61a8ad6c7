// qb_localk.cuh — per-warp top-k lists in registers, the CTA merge of eight of them and the last-CTA merge of the per-CTA lists.
// Used by the single-query exact scan (qb_dense.cu, LOCALK) and by the threshold sample of the 6-bit prefilter (qb_prefilter.cu).
#pragma once
#include "qb_common.cuh"

namespace {

// Every consumer warp keeps its own k best keys in registers (lane i < 16 holds entry i; an insertion is two warp-wide min reductions and
// happens ~k ln(rows/k) times per warp), the CTA merges its eight lists at the end and writes QB_LOCALK_SLOTS keys: the top-k of the union
// of the per-CTA lists is the global top-k.
constexpr int QB_LOCALK_SLOTS = 16;
constexpr int QB_LOCALK_WARPS = 8;

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xFFFFFFFFu, v, o);
        v = w < v ? w : v;
    }
    return v;
}

// Both rare paths are out of line on purpose: inlined, they changed the unrolling of the dot-product loop of the exact scan (60 instead of
// 292 FFMA in the loop body) and the kernel lost 10 % of its bandwidth.
struct LkState { unsigned long long my_key, wmin; float wthr; };
__device__ __noinline__ void lk_push(const uint32_t* deleted, const uint32_t* deleted2, uint32_t id_base, float sc, uint32_t id, unsigned long long* queue,
                                     unsigned int* count) {
    bool dead = false;
    if (deleted) dead = (deleted[id >> 5] >> (id & 31)) & 1u;
    if (deleted2) dead = dead || ((deleted2[id >> 5] >> (id & 31)) & 1u);
    if (!dead) queue[atomicAdd(count, 1u)] = qb_pack_key(sc, id + id_base);
}
__device__ __noinline__ LkState lk_drain(LkState st, const unsigned long long* queue, unsigned int* count, int lane, unsigned int n_queued) {
    for (unsigned int j = 0; j < n_queued; ++j) {
        const unsigned long long k_new = queue[j];
        if (k_new > st.wmin) {  // warp-uniform: replace the smallest entry
            const unsigned int holders = __ballot_sync(0xFFFFFFFFu, st.my_key == st.wmin);
            if (lane == __ffs((int)holders) - 1) st.my_key = k_new;
            st.wmin = warp_min_u64(st.my_key);
        }
    }
    __syncwarp();
    if (lane == 0) *count = 0u;
    __syncwarp();
    st.wthr = (st.wmin != 0ull) ? qb_key_score(st.wmin) : __int_as_float(0xff800000);
    return st;
}

// CTA merge, one warp: bitonic sort of the eight lists (lists[w * QB_LOCALK_SLOTS + i], 0 = empty) in shared memory, descending; the CTA's
// top-16 end up in lists[0, 16).  The consumer warps meet at a NAMED barrier before it: with __syncthreads() the idle lanes of a producer
// warp would sit in the barrier from the first cycle on and share issue slots with the lane that feeds the ring.
__device__ __forceinline__ void lk_cta_sort(unsigned long long* lists, int lane) {
    constexpr int N = QB_LOCALK_WARPS * QB_LOCALK_SLOTS;
    for (int k = 2; k <= N; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < N; i += 32) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = lists[i], b = lists[ixj];
                    const bool desc = ((i & k) == 0);
                    if (desc ? (a < b) : (a > b)) { lists[i] = b; lists[ixj] = a; }
                }
            }
            __syncwarp();
        }
}

// One warp per CTA, after it wrote the CTA's sorted list to all[blockIdx.x * QB_LOCALK_SLOTS, + QB_LOCALK_SLOTS): the last CTA standing merges
// the per-CTA lists.  Each is sorted descending, so the global top-k is a gridDim-way merge of list heads — k rounds of (best head per lane,
// warp arg-max, the winner advances) instead of a separate select launch.  Writes the top-k (fewer when the lists hold fewer keys) and its
// length, and resets the arrival counter for the next launch.
__device__ __forceinline__ void lk_last_cta_merge(const unsigned long long* all, uint32_t local_k, qb_scored_point* final_out, uint32_t* final_count,
                                                  unsigned int* done_counter, int lane) {
    __threadfence();
    __syncwarp();
    unsigned int ticket = 0;
    if (lane == 0) ticket = atomicAdd(done_counter, 1u);
    ticket = __shfl_sync(0xFFFFFFFFu, ticket, 0);
    if (ticket != gridDim.x - 1) return;
    __threadfence();
    constexpr int PER = 8;                           // lists per lane: up to 256 CTAs
    unsigned int pos[PER];
    unsigned long long head[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        const unsigned int l = lane + 32u * i;
        pos[i] = 0;
        head[i] = (l < gridDim.x) ? __ldcg(all + (unsigned long long)l * QB_LOCALK_SLOTS) : 0ull;
    }
    unsigned int n_out = 0;
    for (unsigned int r = 0; r < local_k; ++r) {
        unsigned long long best = 0ull;
        int bi = 0;
#pragma unroll
        for (int i = 0; i < PER; ++i) if (head[i] > best) { best = head[i]; bi = i; }
        unsigned long long wbest = best;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { const unsigned long long w = __shfl_xor_sync(0xFFFFFFFFu, wbest, o); wbest = w > wbest ? w : wbest; }
        if (wbest == 0ull) break;                    // fewer than k keys in all lists
        if (best == wbest) {                         // keys are unique: exactly one lane owns the winner
#pragma unroll
            for (int i = 0; i < PER; ++i)
                if (i == bi) {
                    pos[i] += 1;
                    const unsigned int l = lane + 32u * i;
                    head[i] = (pos[i] < (unsigned int)QB_LOCALK_SLOTS) ? __ldcg(all + (unsigned long long)l * QB_LOCALK_SLOTS + pos[i]) : 0ull;
                }
            qb_scored_point sp;
            sp.idx = qb_key_id(wbest); sp.score = qb_key_score(wbest);
            final_out[r] = sp;
        }
        n_out = r + 1;
    }
    if (lane == 0) { *final_count = n_out; *done_counter = 0u; }
}

}  // namespace
