// qb_hnsw.cu — device-resident HNSW graph search, batched over queries (BASELINE config 5).
//
// Replaces, for a whole batch of queries at once, the reference's per-query traversal
//   GraphLayers::search            lib/segment/src/index/hnsw_index/graph_layers.rs:530-561
//   search_entry / _on_level       graph_layers.rs:247-316   (greedy descent, beam 1, through the upper levels)
//   search_on_level                graph_layers.rs:108-148   (beam search on level 0)
//   SearchContext::process_candidate / lower_bound           search_context.rs:8-41
//   FilteredScorer::score_points   point_scorer.rs:265-295   (filter, truncate to level_m, score)
// which calls the scorer once per hop with <= m0 ids.  Through a per-call GPU boundary that loop is launch/latency bound
// (round 1: 10x slower than the CPU scorer); here the loop itself runs on the device: one persistent CTA per in-flight
// query (128 threads), graph links resident in HBM, the query in shared memory, the hop's neighbours scored by the CTA's 8-lane groups
// with the SAME bit-exact per-pair arithmetic as the scan kernels (qb_score.cuh), so a hop costs three dependent memory
// round trips (links, visited flags, vectors) and no host interaction.  Throughput comes from many queries in flight
// (SMs x resident CTAs), not from one fast query.
//
// State per query (shared memory): `nearest` = the ef best (score desc, id asc) keys seen so far, kept SORTED, with one
// "expanded" flag each.  In the reference `candidates` (a max-heap) only ever holds points that entered `nearest`; a point
// evicted from `nearest` is strictly worse than lower_bound() and popping it ends the search, so
//   "pop the best candidate; stop if it is below lower_bound"  ==  "take the best not-yet-expanded entry of nearest; stop if none".
// A hop's scored points are merged into the sorted list in parallel (rank = own index + number of keys of the other list
// that are greater), which equals pushing them one by one when scores are distinct; equal scores are ordered by id (the
// reference leaves that to heap order), as everywhere in this library.
// Visited set: one bitmap per resident CTA in HBM/L2 (test-and-set with atomicOr), un-set at the end of a query from a log
// of the ids it touched.
//
// Graph layout: the reference's plain `links.bin` (graph_links/header.rs:9-20, view.rs:121-135, serializer.rs:53-200) is
// taken as is for the upper levels (level_offsets, reindex, neighbors, offsets); level 0 — every hop of the beam search —
// is re-laid at upload as a fixed-stride [n][m0] table so a hop needs ONE coalesced 128-B read instead of offsets -> range.
#include <algorithm>

#include "qb_internal.h"
#include "qb_score.cuh"

using namespace qbs;

namespace {

#ifndef QB_HNSW_LINK_PREFETCH
#define QB_HNSW_LINK_PREFETCH 1      // build-time experiment knob
#endif
constexpr uint32_t HNSW_MAX_LINKS = 64;      // links scored per hop (m0 <= 64)
constexpr uint32_t HNSW_EMPTY = 0xFFFFFFFFu;
constexpr uint32_t HNSW_MAX_EF = 4096;

enum { HK_DENSE_AVX = 0, HK_DENSE_SMALL = 1, HK_SQ8 = 2, HK_SQ8_LANEX = 3 };

struct HnswParams {
    // graph
    const uint32_t* links0;        // [n][m0], HNSW_EMPTY padded
    const uint64_t* level_offsets; // [levels]
    const uint32_t* reindex;       // [n]
    const uint32_t* neighbors;     // plain neighbours (all levels; only levels >= 1 are read here)
    const uint64_t* offsets;       // [total_offsets]
    uint32_t n_points, m, m0, levels;
    // storage
    const uint8_t* rows; uint32_t stride; uint32_t dim;             // dense f32
    const uint8_t* codes; const float* voff; uint32_t ad; float multiplier; int l1;   // SQ8
    // queries
    const uint8_t* q_enc; uint32_t q_bytes; const float* q_off;
    uint32_t nq, top, ef;
    uint32_t entry, entry_level;
    const uint32_t* deleted; const uint32_t* deleted2;
    // per-CTA scratch
    uint32_t* visited; uint64_t visited_words;   // [grid][visited_words]
    uint32_t* vlog; uint32_t vlog_cap;           // [grid][vlog_cap]
    unsigned int* work;                          // next query index
    // results
    qb_scored_point* out; uint32_t* out_counts; uint32_t id_base;
    unsigned long long* stats;                   // [0] hops (scorer calls), [1] scored points
    int prefetch;                                // 1: bulk-prefetch the surviving neighbours' vectors into L2 before scoring
};

struct HnswSmem {
    unsigned long long* keys[2];
    uint8_t* flags[2];
    unsigned long long* newk;   // [HNSW_MAX_LINKS]
    uint32_t* ids;              // [HNSW_MAX_LINKS]
    float* sc;                  // [HNSW_MAX_LINKS]
    const uint8_t* q;           // query
};

template <int KIND, int METRIC>
__device__ __forceinline__ float score_one(const HnswParams& p, const uint8_t* q_smem, float q_off, uint32_t id, int t) {
    if (KIND == HK_DENSE_AVX) {
        return score_avx_group8<METRIC>(reinterpret_cast<const float*>(p.rows + (size_t)id * p.stride), reinterpret_cast<const float*>(q_smem), p.dim, t);
    } else if (KIND == HK_DENSE_SMALL) {
        return score_small<METRIC>(reinterpret_cast<const float*>(p.rows + (size_t)id * p.stride), reinterpret_cast<const float*>(q_smem), p.dim);
    } else {
        const float raw = sq8_raw_group8<KIND == HK_SQ8_LANEX>(reinterpret_cast<const uint4*>(p.codes + (size_t)id * p.ad), reinterpret_cast<const uint4*>(q_smem),
                                                               p.ad >> 4, t, p.l1);
        return __fadd_rn(__fadd_rn(__fmul_rn(p.multiplier, raw), q_off), p.voff[id]);   // postprocess_score, encoded_vectors_u8.rs:101-103
    }
}

// scores ids[0..n) into sc[0..n): one 8-lane group per id (dense small dims: one thread per id)
template <int KIND, int METRIC, int NT>
__device__ __forceinline__ void score_list(const HnswParams& p, const HnswSmem& sm, float q_off, uint32_t n) {
    constexpr int HNSW_GROUPS = NT / 8;
    const int tid = threadIdx.x;
    if (KIND == HK_DENSE_SMALL) {
        if ((uint32_t)tid < n) sm.sc[tid] = score_one<KIND, METRIC>(p, sm.q, q_off, sm.ids[tid], 0);
    } else {
        const int g = tid >> 3, t = tid & 7;
        for (uint32_t i = g; i < ((n + HNSW_GROUPS - 1) / HNSW_GROUPS) * HNSW_GROUPS; i += HNSW_GROUPS) {   // whole warps stay converged for the shuffles
            const uint32_t id = sm.ids[i < n ? i : 0];
            const float s = score_one<KIND, METRIC>(p, sm.q, q_off, id, t);
            if (i < n && t == 0) sm.sc[i] = s;
        }
    }
}

// one TMA-engine instruction pulls a whole vector (dim * 4 bytes) from HBM into L2, so that the group's demand loads — which the
// compiler keeps only 3-4 deep — are L2 hits instead of HBM round trips
__device__ __forceinline__ void prefetch_row_l2(const void* p, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
template <int KIND>
__device__ __forceinline__ void prefetch_point(const HnswParams& p, uint32_t id) {
    if (KIND == HK_DENSE_AVX || KIND == HK_DENSE_SMALL) prefetch_row_l2(p.rows + (size_t)id * p.stride, p.stride);
    else prefetch_row_l2(p.codes + (size_t)id * p.ad, p.ad);
}

__device__ __forceinline__ bool hnsw_filtered_out(const HnswParams& p, uint32_t id) {
    bool d = false;
    if (p.deleted) d = (p.deleted[id >> 5] >> (id & 31)) & 1u;
    if (p.deleted2) d = d || ((p.deleted2[id >> 5] >> (id & 31)) & 1u);
    return d;
}

template <int KIND, int METRIC, int NT>
__global__ void __launch_bounds__(NT) hnsw_search_kernel(const HnswParams p) {
    constexpr int HNSW_THREADS = NT;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ unsigned int s_q, s_best, s_n, s_nvalid, s_len, s_nlog, s_cur, s_changed, s_warp_cnt[2];
    __shared__ float s_cur_score;
    const int tid = threadIdx.x;
    const uint32_t ef = p.ef;
    HnswSmem sm;
    {
        uint8_t* b = smem_raw;
        sm.q = b; b += (p.q_bytes + 15u) & ~15u;
        sm.keys[0] = reinterpret_cast<unsigned long long*>(b); b += (size_t)ef * 8;
        sm.keys[1] = reinterpret_cast<unsigned long long*>(b); b += (size_t)ef * 8;
        sm.newk = reinterpret_cast<unsigned long long*>(b); b += HNSW_MAX_LINKS * 8;
        sm.ids = reinterpret_cast<uint32_t*>(b); b += HNSW_MAX_LINKS * 4;
        sm.sc = reinterpret_cast<float*>(b); b += HNSW_MAX_LINKS * 4;
        sm.flags[0] = b; b += (ef + 15u) & ~15u;
        sm.flags[1] = b;
    }
    uint32_t* visited = p.visited + (size_t)blockIdx.x * p.visited_words;
    uint32_t* vlog = p.vlog + (size_t)blockIdx.x * p.vlog_cap;
    unsigned long long hops = 0, evals = 0;   // thread 0 only

    for (;;) {
        if (tid == 0) s_q = atomicAdd(p.work, 1u);
        __syncthreads();
        const uint32_t q = s_q;
        if (q >= p.nq) break;
        // ---- query into shared memory
        {
            const uint4* src = reinterpret_cast<const uint4*>(p.q_enc + (size_t)q * p.q_bytes);
            uint4* dst = reinterpret_cast<uint4*>(const_cast<uint8_t*>(sm.q));
            for (uint32_t i = tid; i < (p.q_bytes + 15u) / 16u; i += HNSW_THREADS) dst[i] = src[i];
        }
        const float q_off = p.q_off ? p.q_off[q] : 0.0f;
        if (tid == 0) { s_nlog = 0; sm.ids[0] = p.entry; }
        __syncthreads();

        // ---- search_entry: greedy descent from the entry point's level to level 1 (graph_layers.rs:247-316)
        score_list<KIND, METRIC, NT>(p, sm, q_off, 1);      // score_point(entry)
        __syncthreads();
        if (tid == 0) { s_cur = p.entry; s_cur_score = sm.sc[0]; ++hops; ++evals; }
        __syncthreads();
        for (uint32_t lvl = p.entry_level; lvl >= 1; --lvl) {
            // search_entry_on_level re-scores its entry point on every level (graph_layers.rs:298-301): same value, but the scorer call
            // and the scored point are metered, so they are counted here too
            if (tid == 0 && lvl != p.entry_level) { ++hops; ++evals; }
            for (;;) {
                const uint32_t cur = s_cur;
                // links of `cur` on this level: neighbors[offsets[idx] .. offsets[idx + 1]), idx = level_offsets[lvl] + reindex[cur] (view.rs:203-215)
                if (tid < 32) {
                    const uint64_t idx = p.level_offsets[lvl] + p.reindex[cur];
                    const uint64_t b = p.offsets[idx], e = p.offsets[idx + 1];
                    uint32_t cnt = 0;
                    // filter (check_batched keeps matches in order), then truncate to level_m (point_scorer.rs:270-277)
                    for (uint64_t base = b; base < e && cnt < p.m; base += 32) {
                        const uint64_t i = base + tid;
                        const uint32_t l = i < e ? p.neighbors[i] : HNSW_EMPTY;
                        const bool keep = l != HNSW_EMPTY && l < p.n_points && !hnsw_filtered_out(p, l);
                        const unsigned int bal = __ballot_sync(0xFFFFFFFFu, keep);
                        const uint32_t pos = cnt + __popc(bal & ((1u << tid) - 1u));
                        if (keep && pos < p.m && pos < HNSW_MAX_LINKS) { sm.ids[pos] = l; if (p.prefetch) prefetch_point<KIND>(p, l); }
                        cnt += __popc(bal);
                    }
                    if (tid == 0) s_n = min(min(cnt, p.m), HNSW_MAX_LINKS);
                }
                __syncthreads();
                const uint32_t n = s_n;
                score_list<KIND, METRIC, NT>(p, sm, q_off, n);
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

        // ---- search_on_level(level 0, ef): nearest = [level entry], entry visited
        if (tid == 0) {
            const uint32_t e0 = s_cur;
            sm.keys[0][0] = qb_pack_key(s_cur_score, e0);
            sm.flags[0][0] = 0;
            s_len = 1;
            atomicOr(&visited[e0 >> 5], 1u << (e0 & 31));
            vlog[0] = e0; s_nlog = 1;
        }
        __syncthreads();
        int cb = 0;   // current buffer
        for (;;) {
            unsigned long long* keys = sm.keys[cb];
            uint8_t* flags = sm.flags[cb];
            const uint32_t len = s_len;
            // 1. best not-yet-expanded entry
            if (tid == 0) s_best = 0xFFFFFFFFu;
            __syncthreads();
            for (uint32_t i = tid; i < len; i += HNSW_THREADS) if (!flags[i]) atomicMin(&s_best, i);
            __syncthreads();
            const uint32_t best = s_best;
            if (best == 0xFFFFFFFFu) break;
            const uint32_t cand = qb_key_id(keys[best]);
            // 2. its level-0 links that pass the filter and were not visited (test-and-set), in link order
            if (tid < 64) {
                const uint32_t l = (uint32_t)tid < p.m0 ? p.links0[(size_t)cand * p.m0 + tid] : HNSW_EMPTY;
                bool keep = l < p.n_points && !hnsw_filtered_out(p, l);
                if (keep) keep = ((atomicOr(&visited[l >> 5], 1u << (l & 31)) >> (l & 31)) & 1u) == 0u;
                const unsigned int bal = __ballot_sync(0xFFFFFFFFu, keep);
                if ((tid & 31) == 0) s_warp_cnt[tid >> 5] = __popc(bal);
                __syncwarp();
                // two warps: positions of warp 1 follow warp 0's
                asm volatile("bar.sync 1, 64;" ::: "memory");
                const uint32_t pos = ((tid >> 5) ? s_warp_cnt[0] : 0u) + __popc(bal & ((1u << (tid & 31)) - 1u));
                if (keep) {
                    if (p.prefetch) prefetch_point<KIND>(p, l);          // HBM -> L2 for the whole vector, in flight while the list is published
                    sm.ids[pos] = l;
                    const uint32_t lp = s_nlog + pos;
                    if (lp < p.vlog_cap) vlog[lp] = l;
                }
                if (tid == 0) { flags[best] = 1; s_n = s_warp_cnt[0] + s_warp_cnt[1]; }
            }
            __syncthreads();
            const uint32_t n = s_n;
            if (tid == 0) { s_nlog += n; if (n) { ++hops; evals += n; } s_nvalid = 0; }
            if (n == 0) { __syncthreads(); continue; }
            // 3. score
            score_list<KIND, METRIC, NT>(p, sm, q_off, n);
            __syncthreads();
            // 4. keys of the new points; the ones that cannot enter a full list are dropped here (key 0 = empty)
            const unsigned long long lower = (len == ef) ? keys[ef - 1] : 0ull;
            if ((uint32_t)tid < n) {
                unsigned long long k = qb_pack_key(sm.sc[tid], sm.ids[tid]);
                if (k <= lower) k = 0ull; else atomicAdd(&s_nvalid, 1u);
                sm.newk[tid] = k;
            }
            __syncthreads();
            const uint32_t nvalid = s_nvalid;
            if (nvalid == 0) continue;
            // 5. merge into the other buffer: rank = own index + number of greater keys in the other list
            unsigned long long* nk = sm.keys[cb ^ 1];
            uint8_t* nf = sm.flags[cb ^ 1];
            for (uint32_t i = tid; i < len; i += HNSW_THREADS) {
                const unsigned long long k = keys[i];
                uint32_t r = i;
                for (uint32_t j = 0; j < n; ++j) r += (sm.newk[j] > k) ? 1u : 0u;
                if (r < ef) { nk[r] = k; nf[r] = flags[i]; }
            }
            if ((uint32_t)tid >= HNSW_THREADS - HNSW_MAX_LINKS) {   // the last two warps place the new keys
                const uint32_t j = (uint32_t)tid - (HNSW_THREADS - HNSW_MAX_LINKS);
                const unsigned long long k = j < n ? sm.newk[j] : 0ull;
                if (k) {
                    uint32_t r = 0;
                    for (uint32_t j2 = 0; j2 < n; ++j2) r += (sm.newk[j2] > k) ? 1u : 0u;
                    uint32_t lo = 0, hi = len;   // first index with keys[idx] < k (keys are distinct and descending)
                    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (keys[mid] > k) lo = mid + 1; else hi = mid; }
                    r += lo;
                    if (r < ef) {
                        nk[r] = k; nf[r] = 0;
                        // every point that enters `nearest` is a future candidate: pull its level-0 link row (one 128-byte line at m0 = 32) into L2 now
                        if (QB_HNSW_LINK_PREFETCH && p.prefetch) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.links0 + (size_t)qb_key_id(k) * p.m0));
                    }
                }
            }
            __syncthreads();
            if (tid == 0) s_len = min(len + nvalid, ef);
            cb ^= 1;
            __syncthreads();
        }

        // ---- results: into_iter_sorted().take(top) (graph_layers.rs:560)
        {
            const unsigned long long* keys = sm.keys[cb];
            const uint32_t len = s_len, cnt = min(len, p.top);
            for (uint32_t i = tid; i < cnt; i += HNSW_THREADS) {
                qb_scored_point sp;
                sp.idx = qb_key_id(keys[i]) + p.id_base;
                sp.score = qb_key_score(keys[i]);
                p.out[(size_t)q * p.top + i] = sp;
            }
            if (tid == 0) p.out_counts[q] = cnt;
        }
        // ---- un-set the visited bits this query set
        {
            const uint32_t nlog = s_nlog;
            if (nlog <= p.vlog_cap) {
                for (uint32_t i = tid; i < nlog; i += HNSW_THREADS) visited[vlog[i] >> 5] = 0u;
            } else {
                for (uint64_t i = tid; i < p.visited_words; i += HNSW_THREADS) visited[i] = 0u;
            }
        }
        __syncthreads();
    }
    if (tid == 0 && p.stats) { atomicAdd(&p.stats[0], hops); atomicAdd(&p.stats[1], evals); }
}

template <int KIND, int NT>
qb_status launch_kind(int metric, const HnswParams& p, unsigned grid, size_t smem, cudaStream_t stream) {
#define QB_HNSW_LAUNCH(M)                                                                                              \
    do {                                                                                                               \
        QB_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<KIND, M, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        hnsw_search_kernel<KIND, M, NT><<<grid, NT, smem, stream>>>(p);                                                \
    } while (0)
    if (KIND == HK_SQ8 || KIND == HK_SQ8_LANEX) QB_HNSW_LAUNCH(M_DOT);
    else if (metric == M_EUCLID) QB_HNSW_LAUNCH(M_EUCLID);
    else if (metric == M_MANHATTAN) QB_HNSW_LAUNCH(M_MANHATTAN);
    else QB_HNSW_LAUNCH(M_DOT);
#undef QB_HNSW_LAUNCH
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

template <int KIND, int METRIC, int NT>
int occupancy_of(size_t smem) {
    int nb = 0;
    cudaFuncSetAttribute(hnsw_search_kernel<KIND, METRIC, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, hnsw_search_kernel<KIND, METRIC, NT>, NT, smem) != cudaSuccess) nb = 1;
    return nb < 1 ? 1 : nb;
}
template <int NT>
int occupancy_dispatch(int kind, int metric, size_t smem) {
    switch (kind) {
        case HK_DENSE_AVX: return metric == M_EUCLID ? occupancy_of<HK_DENSE_AVX, M_EUCLID, NT>(smem) : metric == M_MANHATTAN ? occupancy_of<HK_DENSE_AVX, M_MANHATTAN, NT>(smem) : occupancy_of<HK_DENSE_AVX, M_DOT, NT>(smem);
        case HK_DENSE_SMALL: return metric == M_EUCLID ? occupancy_of<HK_DENSE_SMALL, M_EUCLID, NT>(smem) : metric == M_MANHATTAN ? occupancy_of<HK_DENSE_SMALL, M_MANHATTAN, NT>(smem) : occupancy_of<HK_DENSE_SMALL, M_DOT, NT>(smem);
        case HK_SQ8: return occupancy_of<HK_SQ8, M_DOT, NT>(smem);
        default: return occupancy_of<HK_SQ8_LANEX, M_DOT, NT>(smem);
    }
}
template <int NT>
qb_status launch_dispatch(int kind, int metric, const HnswParams& p, unsigned grid, size_t smem, cudaStream_t stream) {
    switch (kind) {
        case HK_DENSE_AVX: return launch_kind<HK_DENSE_AVX, NT>(metric, p, grid, smem, stream);
        case HK_DENSE_SMALL: return launch_kind<HK_DENSE_SMALL, NT>(metric, p, grid, smem, stream);
        case HK_SQ8: return launch_kind<HK_SQ8, NT>(metric, p, grid, smem, stream);
        default: return launch_kind<HK_SQ8_LANEX, NT>(metric, p, grid, smem, stream);
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------ host side
static size_t hnsw_smem_bytes(uint32_t q_bytes, uint32_t ef) {
    return (size_t)((q_bytes + 15u) & ~15u) + (size_t)ef * 16 + HNSW_MAX_LINKS * 16 + 2 * (size_t)((ef + 15u) & ~15u);
}

__global__ void hnsw_links0_kernel(const uint32_t* __restrict__ neighbors, const uint64_t* __restrict__ offsets, uint32_t n, uint32_t m0, uint32_t* __restrict__ links0) {
    const uint64_t total = (uint64_t)n * m0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t p = (uint32_t)(i / m0), k = (uint32_t)(i % m0);
        const uint64_t b = offsets[p], e = offsets[p + 1];   // level 0: idx = point id (view.rs:205-206)
        links0[i] = (b + k < e) ? neighbors[b + k] : 0xFFFFFFFFu;
    }
}

extern "C" qb_status qb_hnsw_create_plain(qb_storage* s, const uint8_t* links_bin, uint64_t n_bytes, uint32_t m, uint32_t m0, qb_hnsw** out) {
    QB_CHECK(s && links_bin && out, QB_ERR_INVALID, "hnsw_create_plain: null argument");
    *out = nullptr;
    QB_CHECK(m >= 1 && m0 >= 1 && m0 <= HNSW_MAX_LINKS && m <= HNSW_MAX_LINKS, QB_ERR_UNSUPPORTED, "hnsw_create_plain: m %u / m0 %u outside [1,%u]", m, m0, HNSW_MAX_LINKS);
    QB_CHECK(n_bytes >= 64, QB_ERR_INVALID, "hnsw_create_plain: %llu bytes is smaller than HeaderPlain", (unsigned long long)n_bytes);
    uint64_t hdr[5];
    memcpy(hdr, links_bin, sizeof(hdr));   // point_count, levels_count, total_neighbors_count, total_offset_count, offsets_padding_bytes
    const uint64_t n = hdr[0], levels = hdr[1], n_nb = hdr[2], n_off = hdr[3], pad = hdr[4];
    QB_CHECK(n == s->count, QB_ERR_INVALID, "hnsw_create_plain: graph has %llu points, storage %llu", (unsigned long long)n, (unsigned long long)s->count);
    QB_CHECK(pad == 0 || pad == 4, QB_ERR_INVALID, "hnsw_create_plain: offsets padding %llu", (unsigned long long)pad);
    QB_CHECK(levels <= 64 && n_off >= n + 1, QB_ERR_INVALID, "hnsw_create_plain: bad header (levels %llu, offsets %llu)", (unsigned long long)levels, (unsigned long long)n_off);
    const uint64_t need = 64 + 8 * levels + 4 * n + 4 * n_nb + pad + 8 * n_off;
    QB_CHECK(n_bytes >= need, QB_ERR_INVALID, "hnsw_create_plain: %llu bytes, header describes %llu", (unsigned long long)n_bytes, (unsigned long long)need);
    const uint8_t* p_lo = links_bin + 64;
    const uint8_t* p_re = p_lo + 8 * levels;
    const uint8_t* p_nb = p_re + 4 * n;
    const uint8_t* p_of = p_nb + 4 * n_nb + pad;
    {   // level offsets index the offsets table: validate before the device ever follows them
        std::vector<uint64_t> lo(levels);
        memcpy(lo.data(), p_lo, 8 * levels);
        for (uint64_t l = 0; l < levels; ++l) QB_CHECK(lo[l] < n_off, QB_ERR_INVALID, "hnsw_create_plain: level offset %llu out of range", (unsigned long long)l);
    }
    cudaError_t ce = cudaSetDevice(s->device);
    if (ce != cudaSuccess) { qb_set_error("hnsw_create_plain: %s", cudaGetErrorString(ce)); return QB_ERR_CUDA; }
    qb_hnsw* g = new qb_hnsw();
    g->st = s; g->n_points = (uint32_t)n; g->m = m; g->m0 = m0; g->levels = (uint32_t)levels;
    bool ok = cudaMalloc(&g->d_links0, std::max<size_t>((size_t)n * m0 * 4, 256)) == cudaSuccess &&
              cudaMalloc(&g->d_level_offsets, std::max<size_t>(8 * levels, 256)) == cudaSuccess &&
              cudaMalloc(&g->d_reindex, std::max<size_t>(4 * n, 256)) == cudaSuccess &&
              cudaMalloc(&g->d_neighbors, std::max<size_t>(4 * n_nb, 256)) == cudaSuccess &&
              cudaMalloc(&g->d_offsets, 8 * n_off + 256) == cudaSuccess && cudaMalloc(&g->d_work, 256) == cudaSuccess &&
              cudaMalloc(&g->d_stats, 256) == cudaSuccess;
    if (!ok) { qb_set_error("hnsw_create_plain: cudaMalloc failed: %s", cudaGetErrorString(cudaGetLastError())); qb_hnsw_destroy(g); return QB_ERR_OOM; }
    g->hbm_bytes = (uint64_t)n * m0 * 4 + 8 * levels + 4 * n + 4 * n_nb + 8 * n_off;
    ce = cudaMemcpy(g->d_level_offsets, p_lo, 8 * levels, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_reindex, p_re, 4 * n, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_neighbors, p_nb, 4 * n_nb, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_offsets, p_of, 8 * n_off, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemset(g->d_stats, 0, 256);
    if (ce == cudaSuccess && n) {
        hnsw_links0_kernel<<<(unsigned)std::min<uint64_t>(ceil_div_u64(n * m0, 256), 132 * 16), 256>>>(g->d_neighbors, g->d_offsets, (uint32_t)n, m0, g->d_links0);
        QB_LAUNCHED();
        ce = cudaDeviceSynchronize();
    }
    if (ce != cudaSuccess) { qb_set_error("hnsw_create_plain: upload: %s", cudaGetErrorString(ce)); qb_hnsw_destroy(g); return QB_ERR_CUDA; }
    *out = g;
    return QB_OK;
}

extern "C" void qb_hnsw_destroy(qb_hnsw* g) {
    if (!g) return;
    if (g->st) cudaSetDevice(g->st->device);
    cudaDeviceSynchronize();
    cudaFree(g->d_links0); cudaFree(g->d_level_offsets); cudaFree(g->d_reindex); cudaFree(g->d_neighbors); cudaFree(g->d_offsets);
    cudaFree(g->d_visited); cudaFree(g->d_vlog); cudaFree(g->d_work); cudaFree(g->d_stats);
    cudaGetLastError();
    delete g;
}

extern "C" qb_status qb_hnsw_info(const qb_hnsw* g, uint32_t* n_points, uint32_t* levels, uint64_t* hbm_bytes) {
    QB_CHECK(g, QB_ERR_INVALID, "hnsw_info: null graph");
    if (n_points) *n_points = g->n_points;
    if (levels) *levels = g->levels;
    if (hbm_bytes) *hbm_bytes = g->hbm_bytes;
    return QB_OK;
}

// queries already encoded (d_q_enc / d_q_off); results to device buffers; enqueued on `stream`, no synchronisation
qb_status qb_hnsw_launch(qb_hnsw* g, const void* d_q_enc, const float* d_q_off, uint32_t nq, uint32_t top, uint32_t ef, uint32_t entry, uint32_t entry_level,
                         const uint32_t* d_deleted2, qb_scored_point* d_out, uint32_t* d_counts, cudaStream_t stream) {
    qb_storage* s = g->st;
    QB_CHECK(entry < g->n_points, QB_ERR_INVALID, "hnsw_search: entry point %u out of range", entry);
    QB_CHECK(entry_level < std::max<uint32_t>(g->levels, 1), QB_ERR_INVALID, "hnsw_search: entry level %u but the graph has %u levels", entry_level, g->levels);
    ef = std::max(ef, top);   // graph_layers.rs:551
    QB_CHECK(ef <= HNSW_MAX_EF, QB_ERR_UNSUPPORTED, "hnsw_search: ef %u > %u", ef, HNSW_MAX_EF);
    int kind;
    if (s->kind == QB_KIND_DENSE && s->dtype == QB_DT_F32) kind = s->dim >= 32 ? HK_DENSE_AVX : HK_DENSE_SMALL;
    else if (s->kind == QB_KIND_SQ8) kind = ((uint64_t)s->actual_dim * 127ull * 127ull >= (1ull << 24)) ? HK_SQ8_LANEX : HK_SQ8;
    else { qb_set_error("hnsw_search: device traversal supports dense f32 and SQ8 storages (others go through qb_score_points per hop)"); return QB_ERR_UNSUPPORTED; }
    const int metric = s->distance == QB_DIST_EUCLID ? M_EUCLID : (s->distance == QB_DIST_MANHATTAN ? M_MANHATTAN : M_DOT);
    HnswParams p{};
    p.links0 = g->d_links0; p.level_offsets = g->d_level_offsets; p.reindex = g->d_reindex; p.neighbors = g->d_neighbors; p.offsets = g->d_offsets;
    p.n_points = g->n_points; p.m = g->m; p.m0 = g->m0; p.levels = g->levels;
    p.rows = reinterpret_cast<const uint8_t*>(s->d_rows); p.stride = s->row_stride; p.dim = s->dim;
    p.codes = s->d_codes; p.voff = s->d_voff; p.ad = s->actual_dim; p.multiplier = s->multiplier; p.l1 = (s->qdist == QB_QD_L1) ? 1 : 0;
    p.q_enc = reinterpret_cast<const uint8_t*>(d_q_enc); p.q_bytes = (uint32_t)qb_encoded_query_bytes(s); p.q_off = (s->kind == QB_KIND_SQ8) ? d_q_off : nullptr;
    p.nq = nq; p.top = top; p.ef = ef; p.entry = entry; p.entry_level = entry_level;
    p.deleted = s->d_deleted; p.deleted2 = d_deleted2;
    p.out = d_out; p.out_counts = d_counts; p.id_base = s->id_base; p.stats = g->d_stats;
    const size_t smem = hnsw_smem_bytes(p.q_bytes, ef);
    QB_CHECK(smem <= 200 * 1024, QB_ERR_UNSUPPORTED, "hnsw_search: query (%u B) + ef %u need %zu B of shared memory", p.q_bytes, ef, smem);
    // threads per CTA: 256 = one 8-lane group per level-0 link (m0 = 32), fewer queries in flight per SM; 128 (default) = two scoring rounds
    // per hop, twice the resident queries.  The traversal is a chain of dependent memory round trips, so queries in flight is what hides them.
    const int nt = qb_opt().hnsw_threads == 256 ? 256 : (qb_opt().hnsw_threads == 64 ? 64 : 128);
    const int per_sm = nt == 128 ? occupancy_dispatch<128>(kind, metric, smem) : (nt == 64 ? occupancy_dispatch<64>(kind, metric, smem) : occupancy_dispatch<256>(kind, metric, smem));
    p.prefetch = qb_opt().hnsw_no_prefetch ? 0 : 1;
    const unsigned max_grid = (unsigned)s->sm_count * (unsigned)per_sm;
    const unsigned grid = std::min<unsigned>(max_grid, nq);
    // per-CTA visited bitmaps + logs (grown on demand, zeroed once: the kernel leaves them clean)
    const uint64_t words = ceil_div_u64(g->n_points, 32);
    if (g->visited_slots < grid || g->visited_words != words) {
        cudaFree(g->d_visited); cudaFree(g->d_vlog); g->d_visited = nullptr; g->d_vlog = nullptr; g->visited_slots = 0;
        g->vlog_cap = 32768;
        QB_CUDA(cudaMalloc(&g->d_visited, std::max<size_t>((size_t)max_grid * words * 4, 256)));
        QB_CUDA(cudaMalloc(&g->d_vlog, (size_t)max_grid * g->vlog_cap * 4));
        QB_CUDA(cudaMemsetAsync(g->d_visited, 0, std::max<size_t>((size_t)max_grid * words * 4, 256), stream));
        g->visited_slots = max_grid; g->visited_words = words;
    }
    p.visited = g->d_visited; p.visited_words = words; p.vlog = g->d_vlog; p.vlog_cap = g->vlog_cap; p.work = g->d_work;
    QB_CUDA(cudaMemsetAsync(g->d_work, 0, 4, stream));
    return nt == 128 ? launch_dispatch<128>(kind, metric, p, grid, smem, stream)
                     : (nt == 64 ? launch_dispatch<64>(kind, metric, p, grid, smem, stream) : launch_dispatch<256>(kind, metric, p, grid, smem, stream));
}

qb_status qb_hnsw_read_stats(qb_hnsw* g, cudaStream_t stream) {
    unsigned long long h[2] = {0, 0};
    QB_CUDA(cudaMemcpyAsync(h, g->d_stats, 16, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaStreamSynchronize(stream));
    QB_CUDA(cudaMemsetAsync(g->d_stats, 0, 16, stream));
    g->hops += h[0]; g->evals += h[1];
    return QB_OK;
}
