// qb_mmr.cuh — the selection skeleton of the MMR kernels, shared by qb_mmr.cu (dense vectors) and qb_mmr_maxsim.cu (multivectors).
//
// One thread-block cluster per query; the query's candidates (input indices 0..n) are split into C contiguous slices, one per CTA, and
// every CTA keeps the same replicated position arrays (rem: position -> input index, where: input index -> position, u16).  The pieces
// below are the parts of that selection that do not depend on how a pair is scored: the dedup, the numbering of the kept candidates
// across the cluster, the cluster argmax of a step through DSMEM and the swap_remove.  Each is force-inlined into its kernel.
// qb_mmr.cu's mmr_kernel states the dedup and the numbering (steps 1 and 2) inline: routed through mmr_dedup / mmr_positions it
// compiles to other SASS (two registers fewer, another schedule), and that kernel keeps the code it was checked with.
#pragma once
#include <cooperative_groups.h>

#include "qb_internal.h"
#include "qb_score.cuh"

namespace qb_mmr {

namespace cg = cooperative_groups;
using namespace qbs;

constexpr uint32_t MMR_THREADS = 512;
constexpr uint32_t MMR_WARPS = MMR_THREADS / 32;
constexpr uint16_t MMR_GONE = 0xFFFF;                 // `where` of a candidate that is selected, a duplicate or out of range

// CTAs per cluster for lists of up to n candidates
static inline uint32_t mmr_ctas(uint32_t n) { return n <= 256 ? 1u : n <= 1024 ? 2u : n <= 4096 ? 4u : 8u; }

// OrderedFloat as an unsigned key: NaN above everything and equal to NaN, -0.0 == +0.0
__device__ __forceinline__ uint32_t ord_key(float s) { return qb_orderable(s == 0.0f ? 0.0f : s); }
// (value, position): the larger wins, the later position on equal values (max_by_key keeps the last maximum); never 0
__device__ __forceinline__ unsigned long long pos_key(float s, uint32_t pos) { return ((unsigned long long)ord_key(s) << 32) | pos; }

__device__ __forceinline__ unsigned long long block_max(unsigned long long v, unsigned long long* wbest) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xFFFFFFFFu, v, o);
        v = w > v ? w : v;
    }
    const uint32_t warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) wbest[warp] = v;
    __syncthreads();
    v = 0;
    for (uint32_t w = 0; w < MMR_WARPS; ++w) v = wbest[w] > v ? wbest[w] : v;
    return v;
}

// 1. unique_by(id), first occurrence kept; an id that local_of(id, &local) rejects is dropped.  lrow = local row, or ~0 when not kept
template <class LocalOf>
__device__ __forceinline__ void mmr_dedup(uint32_t tid, const qb_scored_point* cand, uint32_t lo, uint32_t hi, uint32_t* lrow, LocalOf local_of) {
    for (uint32_t i = lo + tid; i < hi; i += MMR_THREADS) {
        const uint32_t id = cand[i].idx;
        uint32_t local;
        bool keep = local_of(id, local);
        for (uint32_t j = 0; keep && j < i; ++j) keep = __ldg(&cand[j].idx) != id;
        lrow[i - lo] = keep ? local : 0xFFFFFFFFu;
    }
    __syncthreads();
}

// 2. positions: the kept candidates in input order, numbered across the cluster (kpos: scratch of the slice's size, each one's rank
// within the slice); cnt[0] = the slice's kept count.  Returns the cluster's kept count; every CTA's rem / where are complete after it.
__device__ __forceinline__ uint32_t mmr_positions(uint32_t tid, cg::cluster_group& cluster, uint32_t C, uint32_t rank, uint32_t lo, uint32_t hi,
                                                  const uint32_t* lrow, uint32_t* kpos, unsigned long long* wbest, uint32_t* cnt, uint16_t* rem,
                                                  uint16_t* where) {
    uint32_t run = 0;
    for (uint32_t base = lo; base < hi; base += MMR_THREADS) {
        const uint32_t i = base + tid;
        const bool f = i < hi && lrow[i - lo] != 0xFFFFFFFFu;
        const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, f), lane = tid & 31, warp = tid >> 5;
        if (lane == 0) reinterpret_cast<uint32_t*>(wbest)[warp] = __popc(ballot);
        __syncthreads();
        uint32_t off = run, total = 0;
        for (uint32_t w = 0; w < MMR_WARPS; ++w) {
            const uint32_t c = reinterpret_cast<uint32_t*>(wbest)[w];
            if (w < warp) off += c;
            total += c;
        }
        if (f) kpos[i - lo] = off + __popc(ballot & ((1u << lane) - 1u));
        __syncthreads();
        run += total;
    }
    if (tid == 0) cnt[0] = run;
    cluster.sync();
    uint32_t offset = 0, n_keep = 0;
    for (uint32_t r = 0; r < C; ++r) {
        const uint32_t c = *cluster.map_shared_rank(cnt, r);
        if (r < rank) offset += c;
        n_keep += c;
    }
    for (uint32_t i = lo + tid; i < hi; i += MMR_THREADS) {
        const bool f = lrow[i - lo] != 0xFFFFFFFFu;
        const uint32_t pos = f ? offset + kpos[i - lo] : MMR_GONE;
        for (uint32_t r = 0; r < C; ++r) {
            cluster.map_shared_rank(where, r)[i] = (uint16_t)pos;
            if (f) cluster.map_shared_rank(rem, r)[pos] = (uint16_t)i;
        }
    }
    cluster.sync();   // every CTA's rem / where complete; the last remote access of the slot counts
    return n_keep;
}

// 4. cluster argmax of a step: every CTA reads every CTA's slot after one barrier, and takes the same pick
__device__ __forceinline__ unsigned long long mmr_cluster_best(uint32_t tid, cg::cluster_group& cluster, uint32_t C, unsigned long long best,
                                                               unsigned long long* wbest, unsigned long long* slot, uint32_t par) {
    best = block_max(best, wbest);
    if (tid == 0) slot[par] = best;
    cluster.sync();
    for (uint32_t r = 0; r < C; ++r) {
        const unsigned long long v = cluster.map_shared_rank(slot, r)[par];
        best = v > best ? v : best;
    }
    return best;
}

// 5. IndexSet::swap_remove of the pick at position pos (input index sel) on this CTA's copy of the positions; one thread
__device__ __forceinline__ void mmr_swap_remove(uint16_t* rem, uint16_t* where, uint32_t pos, uint32_t sel, uint32_t remaining) {
    const uint32_t moved = rem[remaining - 1];
    rem[pos] = (uint16_t)moved;
    where[moved] = (uint16_t)pos;
    where[sel] = MMR_GONE;
}

}  // namespace qb_mmr
