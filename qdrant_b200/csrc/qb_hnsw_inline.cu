// qb_hnsw_inline.cu — HNSW search over a graph with inline vectors (GraphLinksFormat::CompressedWithVectors, loaded by
// qb_hnsw_create_with_vectors in qb_hnsw.cu), batched over queries.
//
// Restates GraphLayers::search_with_vectors (graph_layers.rs:564-596) with
//   search_entry_with_vectors / _on_level_with_vectors   graph_layers.rs:396-452   (greedy descent on the inline link vectors)
//   search_on_level_with_vectors                         graph_layers.rs:336-394   (level 0: two search contexts)
//   FilteredBytesScorer::score_points                    point_scorer.rs:139-153   (filter, truncate to level_m, score the bytes)
// A level-0 record holds the point's original vector (base) and, after its links, each neighbour's quantized vector (link vector).
// The beam ("links context") runs on SQ8 scores of the link vectors inside the record being expanded; every candidate the beam pops
// is scored exactly from its base vector into a second list ("base context"), whose best `top` entries are the result.
//
// One CTA (128 threads) per query in flight, as in hnsw_search_kernel (qb_hnsw_traverse.cuh), whose visited bitmaps and logs, key
// merge and score chains this kernel shares:
//  * link scores: sq8_raw_group8_ld + postprocess_score over the inline bytes, one 8-lane group per link.  A link vector starts at any
//    byte (its layout has alignment 1), so every 16-byte step is assembled from five aligned 4-byte loads and funnel shifts
//    (hv_ld16); the integer dot products see the same bytes in the same lanes, so the score has the bits of the storage's chain.
//    Only the links that survive the visited check and the filter are read (not the whole record).
//  * base scores: the f32 chain of qb_score.cuh for the metric (score_avx_group8 at dim >= 32, score_small below) on a copy of the
//    base vector in shared memory, bit for bit qb_score_points on a dense f32 storage.
//  * the entry point is scored from the storage's own SQ8 row (links_scorer_raw.score_point, graph_layers.rs:403).
//
// Pops.  The reference's links context pushes every point that entered `nearest` into a max-heap `candidates` and pops its best:
// if that candidate is below lower_bound() the loop ends, but the candidate is still base-scored first (graph_layers.rs:358-365).
// Under keyed (score desc, id asc) comparisons every point ever evicted from `nearest` is below every point still in it, so the
// heap top is the best unexpanded entry of `nearest` when there is one, and otherwise the best key ever evicted from `nearest`
// while unexpanded — the only pop that can end the loop with a base score.  The kernel keeps that key as a running maximum:
//  * an old entry of `nearest` pushed out by a hop (merge rank >= ef) while unexpanded is a candidate the heap still holds;
//  * a new key of the hop that does not make the final list (a "loser") was pushed in the reference one by one, in stored link
//    order, and entered the heap iff at its push fewer than ef keys above it were present.  For the largest loser that entered,
//    those keys are exactly the old keys above it (none of them can have been evicted yet, or it would not have entered) plus the
//    hop's winners pushed before it; a larger loser that did not enter has at least ef such keys.  So the largest loser that
//    entered is the largest loser with count_greater(old, k) + (winners pushed before it) < ef, a test each loser runs alone.
// Duplicate ids within one list are outside the contract (reference-built graphs have none): the first copy is scored, later copies
// are dropped from the merge.
#include "qb_hnsw_traverse.cuh"

namespace {

constexpr int HV_THREADS = 128;
static_assert(HNSW_MAX_LIST <= HV_THREADS, "hv_collect reads a list with one thread per link");

struct HvParams {
    // plain arrays (the regular search's) and the resident records
    const uint64_t* level_offsets; const uint32_t* reindex; const uint32_t* neighbors; const uint64_t* offsets;
    const uint8_t* blob;            // the records (total_neighbors_bytes, padded)
    const uint64_t* lvoff;          // per entry: byte offset of its first link vector in blob
    const uint64_t* boff;           // per point: byte offset of its level-0 record = its base vector
    uint32_t n_points, m, m0, link_size;
    // storage (SQ8: the entry point's score) and the two scorers
    const uint8_t* codes; const float* voff; uint32_t ad; float multiplier; int l1; uint32_t dim;
    // queries: preprocessed f32 (stride pre_stride floats) and SQ8 encoded
    const float* q_pre; uint32_t pre_stride; const uint8_t* q_enc; uint32_t q_bytes; const float* q_off;
    uint32_t nq, top, ef, entry, entry_level;
    const uint32_t* deleted; const uint32_t* deleted2;
    uint32_t* visited; uint64_t visited_words; uint32_t* vlog; uint32_t vlog_cap; unsigned int* work;
    qb_scored_point* out; uint32_t* out_counts; uint32_t id_base;
    unsigned long long* stats;      // [0] hops, [1] link-scored points (entry included), [2] base-scored points
};

// four bytes at any address (the record blob is padded, so the word after the last one is readable)
__device__ __forceinline__ uint32_t hv_ld32(const uint8_t* a) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(a) & ~uintptr_t(3));
    return __funnelshift_r(__ldg(w), __ldg(w + 1), (uint32_t)(reinterpret_cast<uintptr_t>(a) & 3u) * 8u);
}
__device__ __forceinline__ uint4 hv_ld16(const uint8_t* a) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(a) & ~uintptr_t(3));
    const uint32_t s = (uint32_t)(reinterpret_cast<uintptr_t>(a) & 3u) * 8u;
    const uint32_t w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2), w3 = __ldg(w + 3), w4 = __ldg(w + 4);
    return make_uint4(__funnelshift_r(w0, w1, s), __funnelshift_r(w1, w2, s), __funnelshift_r(w2, w3, s), __funnelshift_r(w3, w4, s));
}

// EncodedVectorsU8::score_bytes of one inline link vector [f32 v_off][ad codes]; every lane of the 8-lane group returns it
template <bool LANEX>
__device__ __forceinline__ float hv_link_score(const HvParams& p, const uint4* qc, float q_off, const uint8_t* vec, int t) {
    const uint8_t* codes = vec + 4;
    const float raw = sq8_raw_group8_ld<LANEX>([&](uint32_t c) { return hv_ld16(codes + 16u * c); }, qc, p.ad >> 4, t, p.l1);
    return __fadd_rn(__fadd_rn(__fmul_rn(p.multiplier, raw), q_off), __uint_as_float(hv_ld32(vec)));   // postprocess_score
}

struct HvSmem {
    float* qf;                      // preprocessed query
    uint4* qc;                      // encoded query
    float* bv;                      // the popped candidate's base vector
    unsigned long long* keys[2]; uint8_t* flags[2];
    unsigned long long* newk; uint32_t* ids; uint32_t* lidx; float* sc; uint32_t* rank;
    unsigned long long* res;        // base context: the best `top` keys, sorted
};

// scores ids[0 .. n) (their link vectors: record link lidx[i]) into sc
template <bool LANEX>
__device__ __forceinline__ void hv_score_links(const HvParams& p, const HvSmem& sm, float q_off, uint64_t lv, uint32_t n) {
    constexpr int GROUPS = HV_THREADS / 8;
    const int g = threadIdx.x >> 3, t = threadIdx.x & 7;
    for (uint32_t i = g; i < ((n + GROUPS - 1) / GROUPS) * GROUPS; i += GROUPS) {   // whole warps stay converged for the shuffles
        const uint32_t j = i < n ? i : 0;
        const float s = hv_link_score<LANEX>(p, sm.qc, q_off, p.blob + lv + (size_t)sm.lidx[j] * p.link_size, t);
        if (i < n && t == 0) sm.sc[i] = s;
    }
}

// level list of `idx` (plain entry index): links that pass the filter (and, on level 0, were not visited), in stored order, truncated
// to `limit`, into ids / lidx; returns how many (all threads)
__device__ __forceinline__ uint32_t hv_collect(const HvParams& p, const HvSmem& sm, uint64_t idx, uint32_t limit, const uint32_t* visited,
                                               unsigned int* s_warp_cnt) {
    const int tid = threadIdx.x;
    const uint64_t b = p.offsets[idx], e = p.offsets[idx + 1];
    const uint32_t cnt = (uint32_t)min(e - b, (uint64_t)HNSW_MAX_LIST);
    const uint32_t l = (uint32_t)tid < cnt ? p.neighbors[b + tid] : HNSW_EMPTY;
    bool keep = l < p.n_points && !hnsw_filtered_out(p, l);
    if (keep && visited) keep = ((visited[l >> 5] >> (l & 31)) & 1u) == 0u;
    const unsigned int bal = __ballot_sync(0xFFFFFFFFu, keep);
    if ((tid & 31) == 0) s_warp_cnt[tid >> 5] = __popc(bal);
    __syncthreads();
    uint32_t pos = __popc(bal & ((1u << (tid & 31)) - 1u));
    for (int w = 0; w < (tid >> 5); ++w) pos += s_warp_cnt[w];
    const uint32_t total = s_warp_cnt[0] + s_warp_cnt[1] + s_warp_cnt[2] + s_warp_cnt[3];
    if (keep && pos < limit) { sm.ids[pos] = l; sm.lidx[pos] = (uint32_t)tid; }
    __syncthreads();
    return min(total, limit);
}

template <bool LANEX, int BKIND, int METRIC>
__global__ void __launch_bounds__(HV_THREADS) hnsw_inline_kernel(const HvParams p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ unsigned int s_q, s_best, s_len, s_nlog, s_cur, s_changed, s_nvalid, s_rlen, s_warp_cnt[4];
    __shared__ float s_cur_score, s_base;
    __shared__ unsigned long long s_evict, s_hop_ev;
    const int tid = threadIdx.x;
    const uint32_t ef = p.ef;
    HvSmem sm;
    {
        uint8_t* b = smem_raw;
        const uint32_t fb = (p.dim * 4u + 15u) & ~15u;
        sm.qf = reinterpret_cast<float*>(b); b += fb;
        sm.bv = reinterpret_cast<float*>(b); b += fb;
        sm.qc = reinterpret_cast<uint4*>(b); b += (p.q_bytes + 15u) & ~15u;
        sm.keys[0] = reinterpret_cast<unsigned long long*>(b); b += (size_t)ef * 8;
        sm.keys[1] = reinterpret_cast<unsigned long long*>(b); b += (size_t)ef * 8;
        sm.res = reinterpret_cast<unsigned long long*>(b); b += (size_t)p.top * 8;
        sm.newk = reinterpret_cast<unsigned long long*>(b); b += HNSW_MAX_LINKS * 8;
        sm.ids = reinterpret_cast<uint32_t*>(b); b += HNSW_MAX_LINKS * 4;
        sm.lidx = reinterpret_cast<uint32_t*>(b); b += HNSW_MAX_LINKS * 4;
        sm.sc = reinterpret_cast<float*>(b); b += HNSW_MAX_LINKS * 4;
        sm.rank = reinterpret_cast<uint32_t*>(b); b += HNSW_MAX_LINKS * 4;
        sm.flags[0] = b; b += (ef + 15u) & ~15u;
        sm.flags[1] = b;
    }
    uint32_t* visited = p.visited + (size_t)blockIdx.x * p.visited_words;
    uint32_t* vlog = p.vlog + (size_t)blockIdx.x * p.vlog_cap;
    unsigned long long hops = 0, evals = 0, bevals = 0;   // thread 0 only

    for (;;) {
        if (tid == 0) s_q = atomicAdd(p.work, 1u);
        __syncthreads();
        const uint32_t q = s_q;
        if (q >= p.nq) break;
        for (uint32_t i = tid; i < p.dim; i += HV_THREADS) sm.qf[i] = p.q_pre[(size_t)q * p.pre_stride + i];
        {
            const uint4* src = reinterpret_cast<const uint4*>(p.q_enc + (size_t)q * p.q_bytes);
            for (uint32_t i = tid; i < (p.q_bytes + 15u) / 16u; i += HV_THREADS) sm.qc[i] = src[i];
        }
        const float q_off = p.q_off[q];
        if (tid == 0) { s_nlog = 0; s_rlen = 0; s_evict = 0ull; }
        __syncthreads();

        // ---- the entry point, scored from the storage's SQ8 row (warp 0; its four groups compute the same value)
        if (tid < 32) {
            const float raw = sq8_raw_group8<LANEX>(reinterpret_cast<const uint4*>(p.codes + (size_t)p.entry * p.ad), sm.qc, p.ad >> 4, tid & 7, p.l1);
            if (tid == 0) {
                s_cur = p.entry;
                s_cur_score = __fadd_rn(__fadd_rn(__fmul_rn(p.multiplier, raw), q_off), p.voff[p.entry]);
                ++hops; ++evals;
            }
        }
        __syncthreads();
        // ---- search_entry_on_level_with_vectors, entry level .. 1: move only to a strictly better link, the first in stored order
        for (uint32_t lvl = p.entry_level; lvl >= 1; --lvl) {
            for (;;) {
                const uint32_t cur = s_cur;
                const uint64_t idx = p.level_offsets[lvl] + p.reindex[cur];
                const uint32_t n = hv_collect(p, sm, idx, p.m, nullptr, s_warp_cnt);
                hv_score_links<LANEX>(p, sm, q_off, p.lvoff[idx], n);
                __syncthreads();
                if (tid == 0) {
                    bool changed = false;
                    uint32_t c = cur; float cs = s_cur_score;
                    for (uint32_t i = 0; i < n; ++i) if (sm.sc[i] > cs) { changed = true; c = sm.ids[i]; cs = sm.sc[i]; }
                    s_cur = c; s_cur_score = cs; s_changed = changed ? 1u : 0u;
                    if (n) { ++hops; evals += n; }
                }
                __syncthreads();
                if (!s_changed) break;
            }
        }

        // ---- search_on_level_with_vectors (level 0)
        if (tid == 0) {
            const uint32_t e0 = s_cur;
            sm.keys[0][0] = qb_pack_key(s_cur_score, e0);
            sm.flags[0][0] = 0;
            s_len = 1;
            atomicOr(&visited[e0 >> 5], 1u << (e0 & 31));
            vlog[0] = e0; s_nlog = 1;
        }
        __syncthreads();
        int cb = 0;
        for (;;) {
            unsigned long long* keys = sm.keys[cb];
            uint8_t* flags = sm.flags[cb];
            const uint32_t len = s_len;
            // 1. the heap's top: the best unexpanded entry of `nearest`, else the best key evicted while unexpanded (below lower_bound)
            if (tid == 0) s_best = 0xFFFFFFFFu;
            __syncthreads();
            for (uint32_t i = tid; i < len; i += HV_THREADS) if (!flags[i]) atomicMin(&s_best, i);
            __syncthreads();
            const uint32_t best = s_best;
            const bool last = best == 0xFFFFFFFFu;
            if (last && s_evict == 0ull) break;
            const uint32_t cand = qb_key_id(last ? s_evict : keys[best]);
            // 2. base score of the candidate into the base context
            {
                const uint8_t* bsrc = p.blob + p.boff[cand];
                for (uint32_t i = tid; i < p.dim; i += HV_THREADS) sm.bv[i] = __uint_as_float(hv_ld32(bsrc + 4u * i));
                __syncthreads();
                if (BKIND == HK_DENSE_AVX) {
                    if (tid < 32) {
                        const float s = score_avx_group8<METRIC>(sm.bv, sm.qf, p.dim, tid & 7);
                        if (tid == 0) s_base = s;
                    }
                } else if (tid == 0) {
                    s_base = score_small<METRIC>(sm.bv, sm.qf, p.dim);
                }
                __syncthreads();
                const unsigned long long k = qb_pack_key(s_base, cand);
                const uint32_t rlen = s_rlen;
                const uint32_t r = count_greater(sm.res, rlen, k);
                __syncthreads();
                if (r < p.top) {
                    // shift [r, min(rlen, top - 1)) up by one, from the top down, a block of threads at a time
                    for (int hi = (int)min(rlen, p.top - 1); hi > (int)r; hi -= HV_THREADS) {
                        const int i = hi - 1 - tid;
                        const unsigned long long v = i >= (int)r ? sm.res[i] : 0ull;
                        __syncthreads();
                        if (i >= (int)r) sm.res[i + 1] = v;
                        __syncthreads();
                    }
                    if (tid == 0) { sm.res[r] = k; s_rlen = min(rlen + 1, p.top); }
                }
                if (tid == 0) { ++bevals; if (!last) flags[best] = 1; }
                __syncthreads();
            }
            if (last) break;
            // 3. its unvisited links that pass the filter, in stored order, truncated to m0 after the filter
            const uint32_t n = hv_collect(p, sm, cand, p.m0, visited, s_warp_cnt);
            if (n == 0) continue;
            if (tid == 0) { ++hops; evals += n; s_nvalid = 0; s_hop_ev = 0ull; }
            // 4. score from the inline link vectors; mark the scored points visited
            hv_score_links<LANEX>(p, sm, q_off, p.lvoff[cand], n);
            __syncthreads();
            if ((uint32_t)tid < n) {
                const uint32_t l = sm.ids[tid];
                bool dup = false;
                for (uint32_t j = 0; j < (uint32_t)tid; ++j) dup = dup || sm.ids[j] == l;
                unsigned long long k = 0ull;
                const uint32_t lp = s_nlog + (uint32_t)tid;
                if (lp < p.vlog_cap) vlog[lp] = l;
                if (!dup) {
                    k = qb_pack_key(sm.sc[tid], l);
                    atomicOr(&visited[l >> 5], 1u << (l & 31));
                    atomicAdd(&s_nvalid, 1u);
                }
                sm.newk[tid] = k;
            }
            __syncthreads();
            const uint32_t nvalid = s_nvalid;
            if (tid == 0) s_nlog += n;
            // 5. final ranks of the new keys (rank >= ef: a loser)
            if ((uint32_t)tid < n) {
                const unsigned long long k = sm.newk[tid];
                uint32_t r = 0xFFFFFFFFu;
                if (k) {
                    r = count_greater(keys, len, k);
                    for (uint32_t j = 0; j < n; ++j) r += (sm.newk[j] > k) ? 1u : 0u;
                }
                sm.rank[tid] = r;
            }
            __syncthreads();
            // 6. merge into the other buffer, and the best key this hop pushed out of `nearest` while unexpanded
            unsigned long long* nk = sm.keys[cb ^ 1];
            uint8_t* nf = sm.flags[cb ^ 1];
            for (uint32_t i = tid; i < len; i += HV_THREADS) {
                const unsigned long long k = keys[i];
                uint32_t r = i;
                for (uint32_t j = 0; j < n; ++j) r += (sm.newk[j] > k) ? 1u : 0u;
                if (r < ef) { nk[r] = k; nf[r] = flags[i]; }
                else if (!flags[i]) atomicMax(&s_hop_ev, k);
            }
            if ((uint32_t)tid < n && sm.newk[tid]) {
                const unsigned long long k = sm.newk[tid];
                const uint32_t r = sm.rank[tid];
                if (r < ef) {
                    nk[r] = k; nf[r] = 0;
                } else {
                    uint32_t wb = 0;   // winners pushed before this key
                    for (uint32_t j = 0; j < (uint32_t)tid; ++j) wb += (sm.newk[j] && sm.rank[j] < ef) ? 1u : 0u;
                    if (count_greater(keys, len, k) + wb < ef) atomicMax(&s_hop_ev, k);
                }
            }
            __syncthreads();
            if (tid == 0) {
                s_len = min(len + nvalid, ef);
                if (s_hop_ev > s_evict) s_evict = s_hop_ev;
            }
            cb ^= 1;
            __syncthreads();
        }

        // ---- results: the base context's nearest, best first, `top` of them
        {
            const uint32_t cnt = s_rlen;
            for (uint32_t i = tid; i < cnt; i += HV_THREADS) {
                qb_scored_point sp;
                sp.idx = qb_key_id(sm.res[i]) + p.id_base;
                sp.score = qb_key_score(sm.res[i]);
                p.out[(size_t)q * p.top + i] = sp;
            }
            if (tid == 0) p.out_counts[q] = cnt;
        }
        {
            const uint32_t nlog = s_nlog;
            if (nlog <= p.vlog_cap) {
                for (uint32_t i = tid; i < nlog; i += HV_THREADS) visited[vlog[i] >> 5] = 0u;
            } else {
                for (uint64_t i = tid; i < p.visited_words; i += HV_THREADS) visited[i] = 0u;
            }
        }
        __syncthreads();
    }
    if (tid == 0 && p.stats) { atomicAdd(&p.stats[0], hops); atomicAdd(&p.stats[1], evals); atomicAdd(&p.stats[2], bevals); }
}

template <bool LANEX, int BKIND, int METRIC>
qb_status hv_launch(const HvParams& p, unsigned grid_cap, int sm_count, size_t smem, cudaStream_t stream, unsigned* grid_out, bool dry) {
    auto* k = hnsw_inline_kernel<LANEX, BKIND, METRIC>;
    QB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, HV_THREADS, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    const unsigned grid = std::min<unsigned>((unsigned)sm_count * (unsigned)per_sm, grid_cap);
    *grid_out = grid;
    if (dry) return QB_OK;
    k<<<grid, HV_THREADS, smem, stream>>>(p);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

template <bool LANEX, int BKIND>
qb_status hv_launch_metric(int metric, const HvParams& p, unsigned grid_cap, int sm_count, size_t smem, cudaStream_t stream, unsigned* grid, bool dry) {
    if (metric == M_EUCLID) return hv_launch<LANEX, BKIND, M_EUCLID>(p, grid_cap, sm_count, smem, stream, grid, dry);
    if (metric == M_MANHATTAN) return hv_launch<LANEX, BKIND, M_MANHATTAN>(p, grid_cap, sm_count, smem, stream, grid, dry);
    return hv_launch<LANEX, BKIND, M_DOT>(p, grid_cap, sm_count, smem, stream, grid, dry);
}

qb_status hv_dispatch(bool lanex, int bkind, int metric, const HvParams& p, unsigned grid_cap, int sm_count, size_t smem, cudaStream_t stream, unsigned* grid,
                      bool dry) {
    if (lanex) return bkind == HK_DENSE_AVX ? hv_launch_metric<true, HK_DENSE_AVX>(metric, p, grid_cap, sm_count, smem, stream, grid, dry)
                                            : hv_launch_metric<true, HK_DENSE_SMALL>(metric, p, grid_cap, sm_count, smem, stream, grid, dry);
    return bkind == HK_DENSE_AVX ? hv_launch_metric<false, HK_DENSE_AVX>(metric, p, grid_cap, sm_count, smem, stream, grid, dry)
                                 : hv_launch_metric<false, HK_DENSE_SMALL>(metric, p, grid_cap, sm_count, smem, stream, grid, dry);
}

}  // namespace

qb_status qb_hnsw_inline_launch(qb_hnsw* g, const float* d_q_pre, uint32_t pre_stride, const void* d_q_enc, const float* d_q_off, uint32_t nq, uint32_t top,
                                uint32_t ef, uint32_t entry, uint32_t entry_level, const uint32_t* d_deleted2, qb_scored_point* d_out, uint32_t* d_counts,
                                cudaStream_t stream) {
    qb_storage* s = g->st;
    QB_CHECK(g->d_blob, QB_ERR_UNSUPPORTED, "hnsw_search_with_vectors: the graph has no inline vectors (load it with qb_hnsw_create_with_vectors)");
    QB_CHECK(entry < g->n_points, QB_ERR_INVALID, "hnsw_search_with_vectors: entry point %u out of range", entry);
    QB_CHECK(entry_level < std::max<uint32_t>(g->levels, 1), QB_ERR_INVALID, "hnsw_search_with_vectors: entry level %u but the graph has %u levels", entry_level,
             g->levels);
    ef = std::max(ef, top);   // graph_layers.rs:590
    QB_CHECK(ef <= HNSW_MAX_EF, QB_ERR_UNSUPPORTED, "hnsw_search_with_vectors: ef %u > %u", ef, HNSW_MAX_EF);
    HvParams p{};
    p.level_offsets = g->d_level_offsets; p.reindex = g->d_reindex; p.neighbors = g->d_neighbors; p.offsets = g->d_offsets;
    p.blob = g->d_blob; p.lvoff = g->d_lvoff; p.boff = g->d_boff;
    p.n_points = g->n_points; p.m = g->m; p.m0 = g->m0; p.link_size = g->link_size;
    p.codes = s->d_codes; p.voff = s->d_voff; p.ad = s->actual_dim; p.multiplier = s->multiplier; p.l1 = (s->qdist == QB_QD_L1) ? 1 : 0; p.dim = s->dim;
    p.q_pre = d_q_pre; p.pre_stride = pre_stride; p.q_enc = reinterpret_cast<const uint8_t*>(d_q_enc); p.q_bytes = (uint32_t)qb_encoded_query_bytes(s);
    p.q_off = d_q_off;
    p.nq = nq; p.top = top; p.ef = ef; p.entry = entry; p.entry_level = entry_level;
    p.deleted = s->d_deleted; p.deleted2 = d_deleted2;
    p.out = d_out; p.out_counts = d_counts; p.id_base = s->id_base; p.stats = g->d_stats + 4;
    const size_t smem = 2 * (size_t)((s->dim * 4u + 15u) & ~15u) + ((p.q_bytes + 15u) & ~15u) + (size_t)ef * 16 + (size_t)top * 8 + HNSW_MAX_LINKS * 24 +
                        2 * (size_t)((ef + 15u) & ~15u);
    QB_CHECK(smem <= 200 * 1024, QB_ERR_UNSUPPORTED, "hnsw_search_with_vectors: dim %u, ef %u and top %u need %zu B of shared memory", s->dim, ef, top, smem);
    const bool lanex = (uint64_t)s->actual_dim * 127ull * 127ull >= (1ull << 24);   // as the SQ8 traversal picks its chain (qb_hnsw.cu)
    const int bkind = s->dim >= 32 ? HK_DENSE_AVX : HK_DENSE_SMALL;
    const int metric = s->distance == QB_DIST_EUCLID ? M_EUCLID : (s->distance == QB_DIST_MANHATTAN ? M_MANHATTAN : M_DOT);
    unsigned max_grid = 0;
    QB_TRY(hv_dispatch(lanex, bkind, metric, p, ~0u, s->sm_count, smem, stream, &max_grid, true));
    const unsigned grid = std::min<unsigned>(max_grid, nq);
    // per-CTA visited bitmaps + logs, shared with the regular search on this handle (grown on demand; every kernel leaves them clean)
    const uint64_t words = ceil_div_u64(g->n_points, 32);
    if (g->visited_slots < max_grid || g->visited_words != words) {
        cudaFree(g->d_visited); cudaFree(g->d_vlog); g->d_visited = nullptr; g->d_vlog = nullptr; g->visited_slots = 0;
        g->vlog_cap = 32768;
        QB_CUDA(cudaMalloc(&g->d_visited, std::max<size_t>((size_t)max_grid * words * 4, 256)));
        QB_CUDA(cudaMalloc(&g->d_vlog, (size_t)max_grid * g->vlog_cap * 4));
        QB_CUDA(cudaMemsetAsync(g->d_visited, 0, std::max<size_t>((size_t)max_grid * words * 4, 256), stream));
        g->visited_slots = max_grid; g->visited_words = words;
    }
    p.visited = g->d_visited; p.visited_words = words; p.vlog = g->d_vlog; p.vlog_cap = g->vlog_cap; p.work = g->d_work;
    QB_CUDA(cudaMemsetAsync(g->d_work, 0, 4, stream));
    unsigned used = 0;
    return hv_dispatch(lanex, bkind, metric, p, grid, s->sm_count, smem, stream, &used, false);
}
