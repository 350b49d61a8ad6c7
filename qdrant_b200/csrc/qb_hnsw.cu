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
// The compressed `links.bin` every current index is written in (GraphLinksFormatParam::Compressed, hnsw/build.rs:548-562) is
// decoded on the device into exactly those arrays (qb_hnsw_create_compressed, below), so one traversal serves both formats.
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "qb_fold.cuh"
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
constexpr uint32_t HNSW_CUSTOM_SMEM = 48 * 1024;   // custom queries: examples up to this size are staged in shared memory

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
    // ACORN only (appended so the HNSW kernels' parameter offsets stay as they were)
    uint32_t hop_cap;                            // per-hop buffers: a power of two >= m0 * m0
    // custom queries only (appended likewise).  Query q's examples are encoded queries ex_first .. ex_first + n_ex of the
    // ex_stride that q_enc / q_off hold per query (discover's context stage skips the target: ex_first = 1)
    int ckind; uint32_t n_a, n_b;                // qb_query_kind and its shape (qbf::fold)
    uint32_t n_ex, ex_first, ex_stride;
    uint32_t ex_smem;                            // 1: the examples are staged in shared memory, 0: read from q_enc (too large)
    uint32_t q_smem;                             // bytes of shared memory the query / examples take
    const float* coef; uint32_t n_coef;          // feedback: [a, partial...] per query
    const qb_scored_point* cep; const uint32_t* cep_counts; uint32_t n_cep;   // custom_entry_points: [nq][n_cep], .idx used
    uint64_t lo_end;                             // level_offsets[levels] (point_level, view.rs:354-369)
};

struct HnswSmem {
    unsigned long long* keys[2];
    uint8_t* flags[2];
    unsigned long long* newk;   // [HNSW_MAX_LINKS] (ACORN: [hop_cap])
    uint32_t* ids;              // [HNSW_MAX_LINKS] (ACORN: [hop_cap])
    float* sc;                  // [HNSW_MAX_LINKS] (ACORN: [hop_cap])
    const uint8_t* q;           // query (custom: the first example, in shared or global memory; example e at q + e * q_bytes)
};

enum { ALGO_HNSW = 0, ALGO_ACORN = 1 };   // qb_hnsw_algorithm

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

// a nearest query: the similarity; a custom query: Query::score_by over the E examples (qb_fold.cuh), each similarity by the same
// chain as a nearest query's, so a score equals qb_score_points on a qb_scorer_create_custom / _feedback scorer.  The fold asks for
// every example exactly once, at points every lane of a group reaches together (its branches on similarities are group-uniform),
// so the shuffles of score_one stay converged.
// q = the query's index: its q_off / coefficients are found from it
template <int KIND, int METRIC, int CUSTOM>
__device__ __forceinline__ float score_q(const HnswParams& p, const HnswSmem& sm, float q_off, uint32_t id, int t, uint32_t q) {
    if constexpr (CUSTOM) {
        const float* off = p.q_off ? p.q_off + (size_t)q * p.ex_stride + p.ex_first : nullptr;
        return qbf::fold(p.ckind, p.n_a, p.n_b, p.coef ? p.coef + (size_t)q * p.n_coef : nullptr, [&](uint32_t e) {
            return score_one<KIND, METRIC>(p, sm.q + (size_t)e * p.q_bytes, off ? off[e] : 0.0f, id, t);
        });
    } else {
        return score_one<KIND, METRIC>(p, sm.q, q_off, id, t);
    }
}

// scores ids[0..n) into sc[0..n): one 8-lane group per id (dense small dims: one thread per id)
template <int KIND, int METRIC, int NT, int CUSTOM>
__device__ __forceinline__ void score_list(const HnswParams& p, const HnswSmem& sm, float q_off, uint32_t n, uint32_t q) {
    constexpr int HNSW_GROUPS = NT / 8;
    const int tid = threadIdx.x;
    if (KIND == HK_DENSE_SMALL) {
        if ((uint32_t)tid < n) sm.sc[tid] = score_q<KIND, METRIC, CUSTOM>(p, sm, q_off, sm.ids[tid], 0, q);
    } else {
        const int g = tid >> 3, t = tid & 7;
        for (uint32_t i = g; i < ((n + HNSW_GROUPS - 1) / HNSW_GROUPS) * HNSW_GROUPS; i += HNSW_GROUPS) {   // whole warps stay converged for the shuffles
            const uint32_t id = sm.ids[i < n ? i : 0];
            const float s = score_q<KIND, METRIC, CUSTOM>(p, sm, q_off, id, t, q);
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

// GraphLinksView::point_level (view.rs:354-369): the first level whose point count the point's reindex reaches, minus one
__device__ __forceinline__ uint32_t hnsw_point_level(const HnswParams& p, uint32_t id) {
    const uint64_t r = p.reindex[id];
    for (uint32_t l = 1; l < p.levels; ++l) {
        const uint64_t a = p.level_offsets[l], b = l + 1 < p.levels ? p.level_offsets[l + 1] : p.lo_end;
        if (r >= b - a) return l - 1;
    }
    return p.levels ? p.levels - 1 : 0;
}

// GraphLayers::get_entry_point (graph_layers.rs:506-528) for query q: of its custom entry points that pass the filter, the one with the
// highest level, the LAST of equal maxima (Iterator::max_by_key); none -> the caller's entry point
__device__ __forceinline__ void hnsw_custom_entry(const HnswParams& p, uint32_t q, uint32_t& entry, uint32_t& level) {
    entry = p.entry; level = p.entry_level;
    if (!p.cep) return;
    const uint32_t nc = min(p.cep_counts[q], p.n_cep);
    bool found = false;
    for (uint32_t i = 0; i < nc; ++i) {
        const uint32_t id = p.cep[(size_t)q * p.n_cep + i].idx;
        if (id >= p.n_points || hnsw_filtered_out(p, id)) continue;
        const uint32_t l = hnsw_point_level(p, id);
        if (!found || l >= level) { found = true; entry = id; level = l; }
    }
}

// ---- ACORN-1 level-0 step (search_on_level_acorn, graph_layers.rs:154-243) for the candidate `cand` = keys[best].
// The reference's order-dependent loops reduce to set operations here because a links0 row holds at most m0 ids:
//  * 1-hop: the loop breaks once to_score.len() >= m0, which only the m0-th link of a row of m0 fresh passing links can reach, so
//    the break never skips a link.  Every fresh link is marked in hop1 (test-and-set); passing ones go to to_score, the rest to
//    to_explore.
//  * 2-hop: a list breaks once it has added m0 points to to_score, again only at its last link, so every list is read to the end.
//    A passing link is scored the first time the pass meets it if it was not in hop1 before: test-and-set on hop1 finds that
//    first meeting, so all lists are processed at once by the whole CTA.
//  * hop2_visited_list cannot change what is scored, so it is not kept.  A passing link enters hop2 only on the step that also marks
//    it in hop1 (hop1 marks are never undone), so for a passing link `hop1.check || hop2.check_and_update` is the hop1 check; a
//    filtered-out 2-hop link is neither scored nor marked in hop1 whatever that test returns.  The reference's hop2 only saves
//    filter lookups; here it would cost a second bitmap per CTA and an atomic per filtered-out 2-hop link.
//  * to_score's order only decides the merge order of distinct keys, which the sorted merge does not depend on.
// Leaves s_n = |to_score| with the ids in sm.ids, and the marks logged.
template <int KIND, int NT>
__device__ __forceinline__ void acorn_collect(const HnswParams& p, const HnswSmem& sm, uint32_t* xids, uint32_t cand, uint32_t* visited, uint32_t* vlog,
                                              unsigned int& s_n, unsigned int& s_nx, unsigned int& s_nlog, unsigned int* s_warp_cnt) {
    const int tid = threadIdx.x;
    if (tid < 64) {
        const uint32_t l = (uint32_t)tid < p.m0 ? p.links0[(size_t)cand * p.m0 + tid] : HNSW_EMPTY;
        const bool fresh = l < p.n_points && ((atomicOr(&visited[l >> 5], 1u << (l & 31)) >> (l & 31)) & 1u) == 0u;
        const bool pass = fresh && !hnsw_filtered_out(p, l);
        const unsigned int bs = __ballot_sync(0xFFFFFFFFu, pass), bx = __ballot_sync(0xFFFFFFFFu, fresh && !pass);
        if ((tid & 31) == 0) { s_warp_cnt[tid >> 5] = __popc(bs); s_warp_cnt[2 + (tid >> 5)] = __popc(bx); }
        __syncwarp();
        asm volatile("bar.sync 1, 64;" ::: "memory");
        const unsigned int lt = (1u << (tid & 31)) - 1u;
        const uint32_t ps = ((tid >> 5) ? s_warp_cnt[0] : 0u) + __popc(bs & lt);
        const uint32_t px = ((tid >> 5) ? s_warp_cnt[2] : 0u) + __popc(bx & lt);
        if (pass) {
            if (p.prefetch) prefetch_point<KIND>(p, l);
            sm.ids[ps] = l;
        } else if (fresh) {
            xids[px] = l;
        }
        if (fresh) {
            const uint32_t lp = s_nlog + ps + px;
            if (lp < p.vlog_cap) vlog[lp] = l;
        }
        asm volatile("bar.sync 1, 64;" ::: "memory");
        if (tid == 0) {
            s_n = s_warp_cnt[0] + s_warp_cnt[1]; s_nx = s_warp_cnt[2] + s_warp_cnt[3];
            s_nlog += s_n + s_nx;
        }
    }
    __syncthreads();
    const uint32_t nx = s_nx, m0 = p.m0;
    for (uint32_t e = tid; e < nx * m0; e += NT) {
        const uint32_t h1 = xids[e / m0];
        const uint32_t l = p.links0[(size_t)h1 * m0 + (e % m0)];
        if (l >= p.n_points) continue;
        if (hnsw_filtered_out(p, l)) continue;
        const uint32_t bit = 1u << (l & 31);
        if (atomicOr(&visited[l >> 5], bit) & bit) continue;                // hop1_visited_list.check, then marked on acceptance
        if (p.prefetch) prefetch_point<KIND>(p, l);
        sm.ids[atomicAdd(&s_n, 1u)] = l;
        const uint32_t lp = atomicAdd(&s_nlog, 1u);
        if (lp < p.vlog_cap) vlog[lp] = l;
    }
    __syncthreads();
}

// descending bitonic sort of newk[0 .. n) (n <= hop_cap), padded with empty keys (0) to a power of two
template <int NT>
__device__ __forceinline__ void acorn_sort_desc(unsigned long long* newk, uint32_t n) {
    uint32_t P = 1;
    while (P < n) P <<= 1;
    for (uint32_t i = n + threadIdx.x; i < P; i += NT) newk[i] = 0ull;
    __syncthreads();
    for (uint32_t k = 2; k <= P; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < P; i += NT) {
                const uint32_t o = i ^ j;
                if (o > i) {
                    const unsigned long long a = newk[i], b = newk[o];
                    if (((i & k) == 0) ? (a < b) : (a > b)) { newk[i] = b; newk[o] = a; }
                }
            }
            __syncthreads();
        }
    }
}

// number of keys in keys[0 .. len) (distinct, descending) greater than k
__device__ __forceinline__ uint32_t count_greater(const unsigned long long* keys, uint32_t len, unsigned long long k) {
    uint32_t lo = 0, hi = len;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (keys[mid] > k) lo = mid + 1; else hi = mid; }
    return lo;
}

// CUSTOM = 1: a custom query (recommend / discover / context / feedback) scored through qbf::fold, with per-query custom entry points
template <int KIND, int METRIC, int NT, int ALGO, int CUSTOM>
__global__ void __launch_bounds__(NT) hnsw_search_kernel(const HnswParams p) {
    constexpr int HNSW_THREADS = NT;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ unsigned int s_q, s_best, s_n, s_nvalid, s_len, s_nlog, s_cur, s_changed, s_warp_cnt[ALGO == ALGO_ACORN ? 4 : 2];
    __shared__ float s_cur_score;
    __shared__ unsigned int s_nx;   // ACORN: |to_explore|
    __shared__ unsigned int s_entry, s_entry_level;   // CUSTOM: get_entry_point of this query
    const int tid = threadIdx.x;
    const uint32_t ef = p.ef;
    HnswSmem sm;
    uint32_t* xids = nullptr;   // ACORN: to_explore [HNSW_MAX_LINKS]
    {
        const uint32_t hop = ALGO == ALGO_ACORN ? p.hop_cap : HNSW_MAX_LINKS;
        uint8_t* b = smem_raw;
        sm.q = b; b += ((CUSTOM ? p.q_smem : p.q_bytes) + 15u) & ~15u;
        sm.keys[0] = reinterpret_cast<unsigned long long*>(b); b += (size_t)ef * 8;
        sm.keys[1] = reinterpret_cast<unsigned long long*>(b); b += (size_t)ef * 8;
        sm.newk = reinterpret_cast<unsigned long long*>(b); b += (size_t)hop * 8;
        sm.ids = reinterpret_cast<uint32_t*>(b); b += (size_t)hop * 4;
        sm.sc = reinterpret_cast<float*>(b); b += (size_t)hop * 4;
        sm.flags[0] = b; b += (ef + 15u) & ~15u;
        sm.flags[1] = b;
        if (ALGO == ALGO_ACORN) { b += (ef + 15u) & ~15u; xids = reinterpret_cast<uint32_t*>(b); }
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
        if constexpr (!CUSTOM) {
            const uint4* src = reinterpret_cast<const uint4*>(p.q_enc + (size_t)q * p.q_bytes);
            uint4* dst = reinterpret_cast<uint4*>(const_cast<uint8_t*>(sm.q));
            for (uint32_t i = tid; i < (p.q_bytes + 15u) / 16u; i += HNSW_THREADS) dst[i] = src[i];
        } else {
            // the examples: into shared memory when they fit, else read where they are (the same arithmetic either way)
            const size_t first = (size_t)q * p.ex_stride + p.ex_first;
            const uint8_t* src = p.q_enc + first * p.q_bytes;
            if (p.ex_smem) {
                const uint4* s4 = reinterpret_cast<const uint4*>(src);
                uint4* dst = reinterpret_cast<uint4*>(smem_raw);   // the query region of the layout above
                for (uint32_t i = tid; i < (p.n_ex * p.q_bytes) / 16u; i += HNSW_THREADS) dst[i] = s4[i];
                sm.q = smem_raw;
            } else {
                sm.q = src;
            }
        }
        const float q_off = (!CUSTOM && p.q_off) ? p.q_off[q] : 0.0f;
        if (tid == 0) {
            s_nlog = 0;
            if constexpr (CUSTOM) {
                uint32_t e, l;
                hnsw_custom_entry(p, q, e, l);
                s_entry = e; s_entry_level = l; sm.ids[0] = e;
            } else {
                sm.ids[0] = p.entry;
            }
        }
        __syncthreads();
        // `CUSTOM ? s_entry : p.entry` is written out at each use, not bound to a local, so the nearest-query kernels compile as before

        // ---- search_entry: greedy descent from the entry point's level to level 1 (graph_layers.rs:247-316)
        score_list<KIND, METRIC, NT, CUSTOM>(p, sm, q_off, 1, q);      // score_point(entry)
        __syncthreads();
        if (tid == 0) { s_cur = CUSTOM ? s_entry : p.entry; s_cur_score = sm.sc[0]; ++hops; ++evals; }
        __syncthreads();
        for (uint32_t lvl = CUSTOM ? s_entry_level : p.entry_level; lvl >= 1; --lvl) {
            // search_entry_on_level re-scores its entry point on every level (graph_layers.rs:298-301): same value, but the scorer call
            // and the scored point are metered, so they are counted here too
            if (tid == 0 && lvl != (CUSTOM ? s_entry_level : p.entry_level)) { ++hops; ++evals; }
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
                score_list<KIND, METRIC, NT, CUSTOM>(p, sm, q_off, n, q);
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
            if constexpr (ALGO == ALGO_ACORN) {
                if (tid == 0) flags[best] = 1;
                acorn_collect<KIND, NT>(p, sm, xids, cand, visited, vlog, s_n, s_nx, s_nlog, s_warp_cnt);
                const uint32_t n = s_n;
                if (tid == 0) { if (n) { ++hops; evals += n; } s_nvalid = 0; }
                if (n == 0) { __syncthreads(); continue; }
                // score_points_unfiltered(to_score)
                if (KIND == HK_DENSE_SMALL) {
                    for (uint32_t i = tid; i < n; i += HNSW_THREADS) sm.sc[i] = score_q<KIND, METRIC, CUSTOM>(p, sm, q_off, sm.ids[i], 0, q);
                } else {
                    score_list<KIND, METRIC, NT, CUSTOM>(p, sm, q_off, n, q);
                }
                __syncthreads();
                // keys that can enter `nearest`, compacted, sorted, at most ef of them
                const unsigned long long lower = (len == ef) ? keys[ef - 1] : 0ull;
                for (uint32_t i = tid; i < n; i += HNSW_THREADS) {
                    const unsigned long long k = qb_pack_key(sm.sc[i], sm.ids[i]);
                    if (k > lower) sm.newk[atomicAdd(&s_nvalid, 1u)] = k;
                }
                __syncthreads();
                const uint32_t nv = s_nvalid;
                if (nv == 0) continue;
                acorn_sort_desc<NT>(sm.newk, nv);
                const uint32_t nk_len = min(nv, ef);
                // merge: rank = own index + number of greater keys in the other list (both sorted: binary search)
                unsigned long long* nk = sm.keys[cb ^ 1];
                uint8_t* nf = sm.flags[cb ^ 1];
                for (uint32_t i = tid; i < len; i += HNSW_THREADS) {
                    const unsigned long long k = keys[i];
                    const uint32_t r = i + count_greater(sm.newk, nk_len, k);
                    if (r < ef) { nk[r] = k; nf[r] = flags[i]; }
                }
                for (uint32_t j = tid; j < nk_len; j += HNSW_THREADS) {
                    const unsigned long long k = sm.newk[j];
                    const uint32_t r = j + count_greater(keys, len, k);
                    if (r < ef) {
                        nk[r] = k; nf[r] = 0;
                        if (QB_HNSW_LINK_PREFETCH && p.prefetch) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.links0 + (size_t)qb_key_id(k) * p.m0));
                    }
                }
                __syncthreads();
                if (tid == 0) s_len = min(len + nk_len, ef);
                cb ^= 1;
                __syncthreads();
                continue;
            }
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
            score_list<KIND, METRIC, NT, CUSTOM>(p, sm, q_off, n, q);
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

template <int KIND, int NT, int ALGO, int CUSTOM>
qb_status launch_kind(int metric, const HnswParams& p, unsigned grid, size_t smem, cudaStream_t stream) {
#define QB_HNSW_LAUNCH(M)                                                                                              \
    do {                                                                                                               \
        QB_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<KIND, M, NT, ALGO, CUSTOM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        hnsw_search_kernel<KIND, M, NT, ALGO, CUSTOM><<<grid, NT, smem, stream>>>(p);                                          \
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

template <int KIND, int METRIC, int NT, int ALGO, int CUSTOM>
int occupancy_of(size_t smem) {
    int nb = 0;
    cudaFuncSetAttribute(hnsw_search_kernel<KIND, METRIC, NT, ALGO, CUSTOM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, hnsw_search_kernel<KIND, METRIC, NT, ALGO, CUSTOM>, NT, smem) != cudaSuccess) nb = 1;
    return nb < 1 ? 1 : nb;
}
template <int NT, int ALGO, int CUSTOM>
int occupancy_dispatch(int kind, int metric, size_t smem) {
    switch (kind) {
        case HK_DENSE_AVX: return metric == M_EUCLID ? occupancy_of<HK_DENSE_AVX, M_EUCLID, NT, ALGO, CUSTOM>(smem) : metric == M_MANHATTAN ? occupancy_of<HK_DENSE_AVX, M_MANHATTAN, NT, ALGO, CUSTOM>(smem) : occupancy_of<HK_DENSE_AVX, M_DOT, NT, ALGO, CUSTOM>(smem);
        case HK_DENSE_SMALL: return metric == M_EUCLID ? occupancy_of<HK_DENSE_SMALL, M_EUCLID, NT, ALGO, CUSTOM>(smem) : metric == M_MANHATTAN ? occupancy_of<HK_DENSE_SMALL, M_MANHATTAN, NT, ALGO, CUSTOM>(smem) : occupancy_of<HK_DENSE_SMALL, M_DOT, NT, ALGO, CUSTOM>(smem);
        case HK_SQ8: return occupancy_of<HK_SQ8, M_DOT, NT, ALGO, CUSTOM>(smem);
        default: return occupancy_of<HK_SQ8_LANEX, M_DOT, NT, ALGO, CUSTOM>(smem);
    }
}
template <int NT, int ALGO, int CUSTOM>
qb_status launch_dispatch(int kind, int metric, const HnswParams& p, unsigned grid, size_t smem, cudaStream_t stream) {
    switch (kind) {
        case HK_DENSE_AVX: return launch_kind<HK_DENSE_AVX, NT, ALGO, CUSTOM>(metric, p, grid, smem, stream);
        case HK_DENSE_SMALL: return launch_kind<HK_DENSE_SMALL, NT, ALGO, CUSTOM>(metric, p, grid, smem, stream);
        case HK_SQ8: return launch_kind<HK_SQ8, NT, ALGO, CUSTOM>(metric, p, grid, smem, stream);
        default: return launch_kind<HK_SQ8_LANEX, NT, ALGO, CUSTOM>(metric, p, grid, smem, stream);
    }
}
template <int ALGO>
int occupancy_nt(int nt, int kind, int metric, size_t smem) {
    return nt == 128 ? occupancy_dispatch<128, ALGO, 0>(kind, metric, smem) : (nt == 64 ? occupancy_dispatch<64, ALGO, 0>(kind, metric, smem) : occupancy_dispatch<256, ALGO, 0>(kind, metric, smem));
}
template <int ALGO>
qb_status launch_nt(int nt, int kind, int metric, const HnswParams& p, unsigned grid, size_t smem, cudaStream_t stream) {
    return nt == 128 ? launch_dispatch<128, ALGO, 0>(kind, metric, p, grid, smem, stream)
                     : (nt == 64 ? launch_dispatch<64, ALGO, 0>(kind, metric, p, grid, smem, stream) : launch_dispatch<256, ALGO, 0>(kind, metric, p, grid, smem, stream));
}

}  // namespace

// ------------------------------------------------------------------------------------------------ host side
static size_t hnsw_smem_bytes(uint32_t q_bytes, uint32_t ef) {
    return (size_t)((q_bytes + 15u) & ~15u) + (size_t)ef * 16 + HNSW_MAX_LINKS * 16 + 2 * (size_t)((ef + 15u) & ~15u);
}
// ACORN: to_score holds up to m0 * m0 ids (a passing 1-hop links and at most m0 - a explored lists of m0), its keys sorted in a
// power-of-two buffer; plus to_explore
static uint32_t acorn_hop_cap(uint32_t m0) {
    uint32_t c = HNSW_MAX_LINKS;
    while (c < m0 * m0) c <<= 1;
    return c;
}
static size_t acorn_smem_bytes(uint32_t q_bytes, uint32_t ef, uint32_t hop_cap) {
    return (size_t)((q_bytes + 15u) & ~15u) + (size_t)ef * 16 + (size_t)hop_cap * 16 + 2 * (size_t)((ef + 15u) & ~15u) + HNSW_MAX_LINKS * 4;
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
    std::vector<uint64_t> lo(levels + 1);
    {   // level offsets index the offsets table: validate before the device ever follows them
        memcpy(lo.data(), p_lo, 8 * levels);
        for (uint64_t l = 0; l < levels; ++l) QB_CHECK(lo[l] < n_off, QB_ERR_INVALID, "hnsw_create_plain: level offset %llu out of range", (unsigned long long)l);
        lo[levels] = n_off - 1;
    }
    cudaError_t ce = cudaSetDevice(s->device);
    if (ce != cudaSuccess) { qb_set_error("hnsw_create_plain: %s", cudaGetErrorString(ce)); return QB_ERR_CUDA; }
    qb_hnsw* g = new qb_hnsw();
    g->st = s; g->n_points = (uint32_t)n; g->m = m; g->m0 = m0; g->levels = (uint32_t)levels;
    g->level_offsets_ext = std::move(lo); g->n_offsets = n_off; g->n_neighbors = n_nb;
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

// ------------------------------------------------------------------------------------------------ compressed links.bin
// GraphLinksFormat::Compressed (graph_links/header.rs:22-34, view.rs:137-163, serializer.rs:62-194):
//   HeaderCompressed, 64 B little-endian, nothing after byte 32 aligned:
//     0 point_count | 8 version 0xFFFF_FFFF_FFFF_FF01 | 16 levels_count | 24 total_neighbors_bytes | 32 offsets length (u64) |
//     40 base_bits, 41 delta_bits, 42 chunk_len_log2 (u8 each) | 43 m (u64) | 51 m0 (u64) | 59 five zero bytes
//   then levels_count u64 level offsets, point_count u32 reindex, total_neighbors_bytes of packed links, the compressed offsets.
// Offsets (common/src/bitpacking_ordered.rs:12-39, 165-197, 292-315): chunks of 2^chunk_len_log2 values — a base_bits base,
// then delta_bits deltas from that base, byte-padded — and a 7-byte 0xFF tail.  The values are BYTE offsets into the packed
// links, in the plain format's index space (view.rs:209-218).
// Links of one (node, level) (bitpacking_links.rs:23-133; bit I/O bitpacking.rs:14-186, LSB first): the first
// min(count, level_m) are sorted and delta-coded (wrapping u32 sums) after a 5-bit header `bits_per_sorted - 8`; the rest are
// raw, bits_per_unsorted = max(8, packed_bits(point_count - 1)) bits each (view.rs:155-159).  The count is implicit in the byte
// length L: ns = min(level_m, (8L - 5) / bps), nu = (8L - 5 - ns * bps) / bits_per_unsorted; L == 0: no links.
// Ids may repeat and may be >= point_count (graph_links/tests.rs:59-80); the traversal skips the latter, as for plain graphs.
namespace {

constexpr uint64_t HNSW_VERSION_COMPRESSED = 0xFFFFFFFFFFFFFF01ull;
constexpr uint64_t HNSW_VERSION_COMPRESSED_WITH_VECTORS = 0xFFFFFFFFFFFFFF02ull;
constexpr uint64_t HC_PAD = 16;   // the device copy of the file is padded so the funnel-shift load below never leaves the allocation
enum : uint32_t { HC_OFFSET_PAST_END = 1u, HC_OFFSETS_DECREASE = 2u, HC_REINDEX = 4u };

__device__ __forceinline__ uint64_t hc_min(uint64_t a, uint64_t b) { return a < b ? a : b; }
__device__ __forceinline__ uint64_t hc_mask(uint32_t bits) { return bits >= 64 ? ~0ull : ((1ull << bits) - 1ull); }

// little-endian u64 at any byte address: two aligned 8-byte loads and a funnel shift
__device__ __forceinline__ uint64_t hc_load_le64(const uint8_t* p) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint64_t* w = reinterpret_cast<const uint64_t*>(a & ~uintptr_t(7));
    const uint32_t sh = (uint32_t)(a & 7) * 8;
    const uint64_t lo = __ldg(w);
    return sh ? (lo >> sh) | (__ldg(w + 1) << (64 - sh)) : lo;
}

// BitReader::read::<u32> of a `bits`-wide value at bit `bitpos` (bits <= 39, so bitpos % 8 + bits fits one 8-byte word)
__device__ __forceinline__ uint32_t hc_bits(const uint8_t* base, uint64_t bitpos, uint32_t bits) {
    return (uint32_t)((hc_load_le64(base + (bitpos >> 3)) >> (bitpos & 7)) & hc_mask(bits));
}

struct HcOffsets {
    const uint8_t* data;          // compressed offsets
    uint64_t length, chunk_bytes, limit;   // limit = total_neighbors_bytes
    uint32_t base_bits, delta_bits, log2;
};

// Reader::decode_chunk (bitpacking_ordered.rs:292-315), one thread per value; the 7-byte tail keeps every 8-byte read in the data
__global__ void hnsw_c_offsets_kernel(const HcOffsets p, uint64_t* __restrict__ out, uint32_t* __restrict__ flag) {
    const uint64_t base_mask = hc_mask(p.base_bits), delta_mask = hc_mask(p.delta_bits), in_chunk = (1ull << p.log2) - 1ull;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.length; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint8_t* c = p.data + (i >> p.log2) * p.chunk_bytes;
        uint64_t v = hc_load_le64(c) & base_mask;
        const uint64_t j = i & in_chunk;
        if (j) {
            const uint64_t bit = p.base_bits + (j - 1) * p.delta_bits;
            v += (hc_load_le64(c + (bit >> 3)) >> (bit & 7)) & delta_mask;
        }
        if (v > p.limit) atomicOr(flag, HC_OFFSET_PAST_END);
        out[i] = v;
    }
}

struct HcLinks {
    const uint8_t* links;         // packed links
    const uint64_t* byte_off;     // decoded offsets [n_entries + 1]
    uint64_t n_entries, limit;
    uint32_t n_points, m, m0, bits_unsorted;
};

// the implicit shape of entry e (iterate_packed_links, bitpacking_links.rs:75-107); entries [0, n_points) are level 0 (view.rs:205-206)
__device__ __forceinline__ void hc_shape(const HcLinks& p, uint64_t e, uint64_t s, uint64_t t, uint32_t& bps, uint64_t& ns, uint64_t& nu) {
    ns = nu = 0; bps = 8;
    if (t == s) return;
    bps = (p.links[s] & 31u) + 8u;
    const uint64_t bits = 8 * (t - s) - 5;
    ns = hc_min(e < p.n_points ? p.m0 : p.m, bits / bps);
    nu = (bits - ns * bps) / p.bits_unsorted;
}

// links per entry (counts[n_entries] = 0, so the exclusive scan ends on the total), and the file's checks that need the device
__global__ void hnsw_c_counts_kernel(const HcLinks p, const uint32_t* __restrict__ reindex, uint64_t* __restrict__ counts, uint32_t* __restrict__ flag) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e <= p.n_entries; e += stride) {
        uint64_t c = 0;
        if (e < p.n_entries) {
            const uint64_t s = p.byte_off[e], t = p.byte_off[e + 1];
            if (t < s) atomicOr(flag, HC_OFFSETS_DECREASE);
            else if (t <= p.limit) { uint32_t bps; uint64_t ns, nu; hc_shape(p, e, s, t, bps, ns, nu); c = ns + nu; }
        }
        counts[e] = c;
    }
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n_points; i += stride)
        if (reindex[i] >= p.n_points) atomicOr(flag, HC_REINDEX);
}

// one warp per entry: lane j decodes value j (j + 32, ...) at its own bit position; the sorted part is a warp inclusive scan of
// the deltas (wrapping u32 adds, PackedLinksIterator::next_sorted) with a carry across passes of 32
__global__ void hnsw_c_links_kernel(const HcLinks p, const uint64_t* __restrict__ offsets, uint32_t* __restrict__ neighbors) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t e = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < p.n_entries; e += n_warps) {
        const uint64_t s = p.byte_off[e], t = p.byte_off[e + 1];
        uint32_t bps; uint64_t ns, nu;
        hc_shape(p, e, s, t, bps, ns, nu);
        uint32_t* out = neighbors + offsets[e];
        const uint64_t bit0 = 8 * s + 5;
        uint32_t carry = 0;
        for (uint64_t k0 = 0; k0 < ns; k0 += 32) {
            const uint64_t k = k0 + lane;
            uint32_t v = k < ns ? hc_bits(p.links, bit0 + k * bps, bps) : 0u;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, v, d);
                if (lane >= (uint32_t)d) v += o;
            }
            v += carry;
            if (k < ns) out[k] = v;
            carry = __shfl_sync(0xFFFFFFFFu, v, 31);
        }
        const uint64_t bit1 = bit0 + ns * bps;
        for (uint64_t k = lane; k < nu; k += 32) out[ns + k] = hc_bits(p.links, bit1 + k * p.bits_unsorted, p.bits_unsorted);
    }
}

// offsets[length .. length + n) = total: an upper-level lookup level_offsets[l] + reindex[p] stays inside the table (and reads an
// empty list) even when a link leads to a point that is not on that level
__global__ void hnsw_c_pad_kernel(uint64_t* offsets, uint64_t length, uint64_t n) {
    const uint64_t total = offsets[length - 1];
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) offsets[length + i] = total;
}

// qb_hnsw_links: GraphLinks::links (view.rs:238-263) for a batch of points on one level, from the traversal's own arrays
__global__ void hnsw_links_gather_kernel(const uint32_t* __restrict__ ids, uint32_t n_ids, uint32_t level, uint64_t level_base, uint64_t on_level,
                                         const uint32_t* __restrict__ reindex, const uint64_t* __restrict__ offsets, uint64_t n_offsets,
                                         const uint32_t* __restrict__ neighbors, uint64_t n_neighbors, uint32_t cap, uint32_t* __restrict__ out,
                                         uint32_t* __restrict__ counts, uint32_t* __restrict__ flag) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_ids; i += gridDim.x * blockDim.x) {
        const uint32_t id = ids[i];
        counts[i] = 0;
        uint64_t idx = id;
        if (level) {
            const uint32_t r = reindex[id];
            if (r >= on_level) { atomicOr(flag, 1u); continue; }   // point_level(id) < level (view.rs:354-369)
            idx = level_base + r;
        }
        if (idx + 1 >= n_offsets) { atomicOr(flag, 2u); continue; }
        const uint64_t b = offsets[idx], e = offsets[idx + 1];
        if (b > e || e > n_neighbors) { atomicOr(flag, 2u); continue; }
        counts[i] = (uint32_t)hc_min(e - b, 0xFFFFFFFFull);
        const uint64_t n = hc_min(e - b, cap);
        for (uint64_t k = 0; k < n; ++k) out[(size_t)i * cap + k] = neighbors[b + k];
    }
}

// device temporaries of one call, freed on every exit path
struct HcScratch {
    std::vector<void*> bufs;
    cudaError_t alloc(void** p, size_t bytes) {
        *p = nullptr;
        const cudaError_t e = cudaMalloc(p, std::max<size_t>(bytes, 256));
        if (e == cudaSuccess) bufs.push_back(*p);
        return e;
    }
    ~HcScratch() { for (void* b : bufs) cudaFree(b); }
};

inline unsigned hc_grid(uint64_t items, uint64_t per_block, uint64_t max_blocks) {
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(ceil_div_u64(items, per_block), max_blocks));
}

}  // namespace

extern "C" qb_status qb_hnsw_create_compressed(qb_storage* s, const uint8_t* bytes, uint64_t n_bytes, qb_hnsw** out) {
    QB_CHECK(s && bytes && out, QB_ERR_INVALID, "hnsw_create_compressed: null argument");
    *out = nullptr;
    QB_CHECK(n_bytes >= 64, QB_ERR_INVALID, "hnsw_create_compressed: %llu bytes is smaller than HeaderCompressed", (unsigned long long)n_bytes);
    auto u64_at = [&](uint64_t o) { uint64_t v; memcpy(&v, bytes + o, 8); return v; };   // the file is little-endian, like every host this builds for
    const uint64_t n = u64_at(0), version = u64_at(8), levels = u64_at(16), nb_bytes = u64_at(24), length = u64_at(32), m = u64_at(43), m0 = u64_at(51);
    const uint32_t base_bits = bytes[40], delta_bits = bytes[41], log2 = bytes[42];
    QB_CHECK(version != HNSW_VERSION_COMPRESSED_WITH_VECTORS, QB_ERR_UNSUPPORTED,
             "hnsw_create_compressed: CompressedWithVectors (inline storage) graphs are searched from the quantized vectors stored with the links "
             "(graph_layers.rs:336-388), a different algorithm; this loader takes GraphLinksFormat::Compressed");
    QB_CHECK(version == HNSW_VERSION_COMPRESSED, QB_ERR_INVALID, "hnsw_create_compressed: version word %016llx is not HEADER_VERSION_COMPRESSED (a plain links.bin?)",
             (unsigned long long)version);
    QB_CHECK(n == s->count, QB_ERR_INVALID, "hnsw_create_compressed: graph has %llu points, storage %llu", (unsigned long long)n, (unsigned long long)s->count);
    QB_CHECK(n <= 0xFFFFFFFFull, QB_ERR_INVALID, "hnsw_create_compressed: %llu points", (unsigned long long)n);
    QB_CHECK(m >= 1 && m0 >= 1, QB_ERR_INVALID, "hnsw_create_compressed: m %llu / m0 %llu", (unsigned long long)m, (unsigned long long)m0);
    QB_CHECK(m <= HNSW_MAX_LINKS && m0 <= HNSW_MAX_LINKS, QB_ERR_UNSUPPORTED, "hnsw_create_compressed: m %llu / m0 %llu outside [1,%u]", (unsigned long long)m,
             (unsigned long long)m0, HNSW_MAX_LINKS);
    QB_CHECK(levels <= 64 && (levels >= 1 || n == 0), QB_ERR_INVALID, "hnsw_create_compressed: %llu levels", (unsigned long long)levels);
    // Parameters::validate (bitpacking_ordered.rs:165-180)
    QB_CHECK(base_bits >= 1 && base_bits <= 64 && delta_bits >= 1 && delta_bits <= 56 && log2 <= 7, QB_ERR_INVALID,
             "hnsw_create_compressed: offsets parameters base_bits %u delta_bits %u chunk_len_log2 %u", base_bits, delta_bits, log2);
    const uint64_t body = 64 + 8 * levels + 4 * n;
    QB_CHECK(body <= n_bytes && nb_bytes <= n_bytes - body, QB_ERR_INVALID, "hnsw_create_compressed: %llu bytes, header describes %llu before the offsets",
             (unsigned long long)n_bytes, (unsigned long long)(body + nb_bytes));
    const uint64_t rest = n_bytes - body - nb_bytes;
    const uint64_t chunk_bytes = ceil_div_u64(base_bits + (uint64_t)delta_bits * ((1ull << log2) - 1), 8);
    const uint64_t chunks = length / (1ull << log2) + ((length & ((1ull << log2) - 1)) ? 1 : 0);
    QB_CHECK(length >= 1 && chunks <= rest / chunk_bytes && chunks * chunk_bytes + 7 <= rest, QB_ERR_INVALID,
             "hnsw_create_compressed: %llu offsets do not fit the %llu bytes after the links", (unsigned long long)length, (unsigned long long)rest);
    const uint64_t used = body + nb_bytes + chunks * chunk_bytes + 7;
    // level offsets with the extra last element (read_level_offsets, view.rs:381-393): level 0 is the first n entries, every level's
    // range inside the table
    std::vector<uint64_t> lo(levels + 1);
    memcpy(lo.data(), bytes + 64, 8 * levels);
    lo[levels] = length - 1;
    for (uint64_t l = 0; l < levels; ++l)
        QB_CHECK(lo[l] <= lo[l + 1] && (l != 0 || (lo[0] == 0 && lo[1] == n)), QB_ERR_INVALID, "hnsw_create_compressed: level offset %llu (%llu) out of range",
                 (unsigned long long)l, (unsigned long long)lo[l]);
    const uint32_t bits_unsorted = std::max<uint32_t>(8, n > 1 ? 64 - __builtin_clzll(n - 1) : 0);

    cudaError_t ce = cudaSetDevice(s->device);
    if (ce != cudaSuccess) { qb_set_error("hnsw_create_compressed: %s", cudaGetErrorString(ce)); return QB_ERR_CUDA; }
    qb_hnsw* g = new qb_hnsw();
    g->st = s; g->n_points = (uint32_t)n; g->m = (uint32_t)m; g->m0 = (uint32_t)m0; g->levels = (uint32_t)levels;
    g->level_offsets_ext = lo; g->n_offsets = length;
    auto fail = [&](qb_status st, const char* what, cudaError_t e) {
        qb_set_error("hnsw_create_compressed: %s: %s", what, cudaGetErrorString(e));
        qb_hnsw_destroy(g);
        return st;
    };
    HcScratch tmp;
    uint8_t* d_file = nullptr; uint64_t* d_byte_off = nullptr; uint64_t* d_counts = nullptr; uint32_t* d_flag = nullptr;
    bool ok = cudaMalloc(&g->d_links0, std::max<size_t>((size_t)n * m0 * 4, 256)) == cudaSuccess &&
              cudaMalloc(&g->d_level_offsets, std::max<size_t>(8 * levels, 256)) == cudaSuccess &&
              cudaMalloc(&g->d_reindex, std::max<size_t>(4 * n, 256)) == cudaSuccess &&
              cudaMalloc(&g->d_offsets, 8 * (length + n) + 256) == cudaSuccess && cudaMalloc(&g->d_work, 256) == cudaSuccess &&
              cudaMalloc(&g->d_stats, 256) == cudaSuccess &&
              tmp.alloc((void**)&d_file, used + HC_PAD) == cudaSuccess && tmp.alloc((void**)&d_byte_off, 8 * length) == cudaSuccess &&
              tmp.alloc((void**)&d_counts, 8 * length) == cudaSuccess && tmp.alloc((void**)&d_flag, 4) == cudaSuccess;
    if (!ok) return fail(QB_ERR_OOM, "cudaMalloc failed", cudaGetLastError());
    // the file goes to HBM once; everything below reads it there
    ce = cudaMemcpy(d_file, bytes, used, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemset(d_file + used, 0, HC_PAD);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_level_offsets, d_file + 64, 8 * levels, cudaMemcpyDeviceToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_reindex, d_file + 64 + 8 * levels, 4 * n, cudaMemcpyDeviceToDevice);
    if (ce == cudaSuccess) ce = cudaMemset(g->d_stats, 0, 256);
    if (ce == cudaSuccess) ce = cudaMemset(d_flag, 0, 4);
    if (ce != cudaSuccess) return fail(QB_ERR_CUDA, "upload", ce);

    HcOffsets po{d_file + body + nb_bytes, length, chunk_bytes, nb_bytes, base_bits, delta_bits, log2};
    hnsw_c_offsets_kernel<<<hc_grid(length, 256, 132 * 16), 256>>>(po, d_byte_off, d_flag);
    QB_LAUNCHED();
    HcLinks pl{d_file + body, d_byte_off, length - 1, nb_bytes, (uint32_t)n, (uint32_t)m, (uint32_t)m0, bits_unsorted};
    hnsw_c_counts_kernel<<<hc_grid(std::max<uint64_t>(length, n), 256, 132 * 16), 256>>>(pl, g->d_reindex, d_counts, d_flag);
    QB_LAUNCHED();
    // plain element offsets = exclusive scan of the counts
    size_t scan_bytes = 0;
    ce = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, d_counts, g->d_offsets, (int64_t)length);
    void* d_scan = nullptr;
    if (ce == cudaSuccess) ce = tmp.alloc(&d_scan, scan_bytes);
    if (ce == cudaSuccess) ce = cub::DeviceScan::ExclusiveSum(d_scan, scan_bytes, d_counts, g->d_offsets, (int64_t)length);
    QB_LAUNCHED();
    uint32_t flag = 0;
    uint64_t total = 0;
    if (ce == cudaSuccess) ce = cudaMemcpy(&flag, d_flag, 4, cudaMemcpyDeviceToHost);
    if (ce == cudaSuccess) ce = cudaMemcpy(&total, g->d_offsets + (length - 1), 8, cudaMemcpyDeviceToHost);
    if (ce != cudaSuccess) return fail(QB_ERR_CUDA, "decode", ce);
    if (flag) {
        qb_set_error("hnsw_create_compressed: %s", (flag & HC_OFFSET_PAST_END) ? "a links offset lies past total_neighbors_bytes"
                                                   : (flag & HC_OFFSETS_DECREASE) ? "links offsets decrease"
                                                                                  : "a reindex entry is >= point_count");
        qb_hnsw_destroy(g);
        return QB_ERR_INVALID;
    }
    g->n_neighbors = total;
    g->hbm_bytes = (uint64_t)n * m0 * 4 + 8 * levels + 4 * n + 4 * total + 8 * (length + n);
    if (cudaMalloc(&g->d_neighbors, std::max<size_t>(4 * total, 256)) != cudaSuccess) return fail(QB_ERR_OOM, "cudaMalloc failed", cudaGetLastError());
    hnsw_c_links_kernel<<<hc_grid(length - 1, 8, 132 * 32), 256>>>(pl, g->d_offsets, g->d_neighbors);
    QB_LAUNCHED();
    hnsw_c_pad_kernel<<<hc_grid(n, 256, 132 * 4), 256>>>(g->d_offsets, length, n);
    QB_LAUNCHED();
    if (n) {
        hnsw_links0_kernel<<<hc_grid(n * m0, 256, 132 * 16), 256>>>(g->d_neighbors, g->d_offsets, (uint32_t)n, (uint32_t)m0, g->d_links0);
        QB_LAUNCHED();
    }
    ce = cudaDeviceSynchronize();
    if (ce == cudaSuccess) ce = cudaGetLastError();
    if (ce != cudaSuccess) return fail(QB_ERR_CUDA, "decode", ce);
    *out = g;
    return QB_OK;
}

extern "C" qb_status qb_hnsw_links(const qb_hnsw* g, uint32_t level, const uint32_t* ids, uint32_t n_ids, uint32_t cap, uint32_t* out, uint32_t* counts) {
    QB_CHECK(g && (ids || n_ids == 0) && (counts || n_ids == 0) && (out || cap == 0 || n_ids == 0), QB_ERR_INVALID, "hnsw_links: null argument");
    QB_CHECK(level < g->levels, QB_ERR_INVALID, "hnsw_links: level %u but the graph has %u levels", level, g->levels);
    for (uint32_t i = 0; i < n_ids; ++i) QB_CHECK(ids[i] < g->n_points, QB_ERR_INVALID, "hnsw_links: point %u out of range", ids[i]);
    if (n_ids == 0) return QB_OK;
    // a point is on `level` iff its reindex is below every level's point count up to there (point_level, view.rs:354-369)
    const std::vector<uint64_t>& lo = g->level_offsets_ext;
    uint64_t on_level = ~0ull;
    for (uint32_t l = 1; l <= level; ++l) on_level = std::min<uint64_t>(on_level, lo[l + 1] >= lo[l] ? lo[l + 1] - lo[l] : 0);
    QB_CUDA(cudaSetDevice(g->st->device));
    HcScratch tmp;
    uint32_t *d_ids = nullptr, *d_out = nullptr, *d_counts = nullptr, *d_flag = nullptr;
    QB_CUDA(tmp.alloc((void**)&d_ids, 4ull * n_ids));
    QB_CUDA(tmp.alloc((void**)&d_out, 4ull * n_ids * cap));
    QB_CUDA(tmp.alloc((void**)&d_counts, 4ull * n_ids));
    QB_CUDA(tmp.alloc((void**)&d_flag, 4));
    QB_CUDA(cudaMemcpy(d_ids, ids, 4ull * n_ids, cudaMemcpyHostToDevice));
    QB_CUDA(cudaMemset(d_flag, 0, 4));
    hnsw_links_gather_kernel<<<hc_grid(n_ids, 128, 132 * 8), 128>>>(d_ids, n_ids, level, level ? lo[level] : 0, on_level, g->d_reindex, g->d_offsets, g->n_offsets,
                                                                    g->d_neighbors, g->n_neighbors, cap, d_out, d_counts, d_flag);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    uint32_t flag = 0;
    QB_CUDA(cudaMemcpy(&flag, d_flag, 4, cudaMemcpyDeviceToHost));
    QB_CHECK(!(flag & 1u), QB_ERR_INVALID, "hnsw_links: a point's top level is below %u", level);
    QB_CHECK(!(flag & 2u), QB_ERR_INVALID, "hnsw_links: the graph's offsets point outside its tables");
    QB_CUDA(cudaMemcpy(counts, d_counts, 4ull * n_ids, cudaMemcpyDeviceToHost));
    if (cap) QB_CUDA(cudaMemcpy(out, d_out, 4ull * n_ids * cap, cudaMemcpyDeviceToHost));
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
                         const uint32_t* d_deleted2, qb_scored_point* d_out, uint32_t* d_counts, cudaStream_t stream, int algo, const QbHnswCustom* custom) {
    qb_storage* s = g->st;
    QB_CHECK(algo == ALGO_HNSW || algo == ALGO_ACORN, QB_ERR_INVALID, "hnsw_search: algorithm %d is neither QB_HNSW_ALGO_HNSW nor QB_HNSW_ALGO_ACORN", algo);
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
    const bool acorn = algo == ALGO_ACORN;
    p.hop_cap = acorn ? acorn_hop_cap(g->m0) : HNSW_MAX_LINKS;
    uint32_t q_smem = p.q_bytes;
    if (custom) {
        p.ckind = custom->kind; p.n_a = custom->n_a; p.n_b = custom->n_b;
        p.n_ex = custom->n_ex; p.ex_first = custom->ex_first; p.ex_stride = custom->ex_stride;
        p.coef = custom->d_coef; p.n_coef = custom->n_coef;
        p.cep = custom->d_cep; p.cep_counts = custom->d_cep_counts; p.n_cep = custom->n_cep;
        p.lo_end = g->level_offsets_ext.empty() ? 0 : g->level_offsets_ext.back();
        p.stats = g->d_stats + 2 * custom->stats_slot;
        if (custom->internal_out) p.id_base = 0;
        // the examples are staged in shared memory when they fit in HNSW_CUSTOM_SMEM, which keeps several queries in flight per SM;
        // larger sets are read from global memory (L1 / L2) by the same chains
        const uint64_t ex_bytes = (uint64_t)p.n_ex * p.q_bytes;
        p.ex_smem = ex_bytes <= HNSW_CUSTOM_SMEM ? 1u : 0u;
        q_smem = p.ex_smem ? (uint32_t)ex_bytes : 0u;
        p.q_smem = q_smem;
    }
    const size_t smem = acorn ? acorn_smem_bytes(q_smem, ef, p.hop_cap) : hnsw_smem_bytes(q_smem, ef);
    QB_CHECK(smem <= 200 * 1024, QB_ERR_UNSUPPORTED, "hnsw_search: query (%u B) + ef %u need %zu B of shared memory", q_smem, ef, smem);
    // threads per CTA: 256 = one 8-lane group per level-0 link (m0 = 32), fewer queries in flight per SM; 128 (default) = two scoring rounds
    // per hop, twice the resident queries.  The traversal is a chain of dependent memory round trips, so queries in flight is what hides them.
    // Custom queries are instantiated for 128 threads only.
    const int nt = custom ? 128 : (qb_opt().hnsw_threads == 256 ? 256 : (qb_opt().hnsw_threads == 64 ? 64 : 128));
    const int per_sm = custom ? (acorn ? occupancy_dispatch<128, ALGO_ACORN, 1>(kind, metric, smem) : occupancy_dispatch<128, ALGO_HNSW, 1>(kind, metric, smem))
                              : (acorn ? occupancy_nt<ALGO_ACORN>(nt, kind, metric, smem) : occupancy_nt<ALGO_HNSW>(nt, kind, metric, smem));
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
    if (custom)
        return acorn ? launch_dispatch<128, ALGO_ACORN, 1>(kind, metric, p, grid, smem, stream) : launch_dispatch<128, ALGO_HNSW, 1>(kind, metric, p, grid, smem, stream);
    return acorn ? launch_nt<ALGO_ACORN>(nt, kind, metric, p, grid, smem, stream) : launch_nt<ALGO_HNSW>(nt, kind, metric, p, grid, smem, stream);
}

qb_status qb_hnsw_read_stats(qb_hnsw* g, cudaStream_t stream, uint64_t* evals_by_slot) {
    unsigned long long h[4] = {0, 0, 0, 0};
    QB_CUDA(cudaMemcpyAsync(h, g->d_stats, 32, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaStreamSynchronize(stream));
    QB_CUDA(cudaMemsetAsync(g->d_stats, 0, 32, stream));
    g->hops += h[0] + h[2]; g->evals += h[1] + h[3];
    if (evals_by_slot) { evals_by_slot[0] = h[1]; evals_by_slot[1] = h[3]; }
    return QB_OK;
}
