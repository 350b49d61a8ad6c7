// qb_hnsw_traverse.cuh — the device HNSW traversal (hnsw_search_kernel) and the pieces it is made of: the kernel parameters, the
// per-hop scoring, the ACORN-1 step, the beam search.  qb_hnsw.cu instantiates it for searches, qb_hnsw_build.cu for the inserts of a
// graph build (ALGO_BUILD), so both run the same beam search.  The design notes are in qb_hnsw.cu's header.
#pragma once
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
constexpr uint32_t HNSW_MAX_LIST = 128;      // widest level list of a graph with inline vectors (qb_hnsw_create_with_vectors)

// HK_U8 / HK_U8_SMALL: Uint8 storages (rows / stride / dim as dense f32), dim >= 32 in 8-lane groups (GPU lane t = AVX lane t) and dim < 32
// one thread per id, integer-exact; appended so the other kinds' values stay as they were
enum { HK_DENSE_AVX = 0, HK_DENSE_SMALL = 1, HK_SQ8 = 2, HK_SQ8_LANEX = 3, HK_U8 = 4, HK_U8_SMALL = 5 };
// kinds whose rows are dense rows of `stride` bytes, and kinds that score one id per thread rather than per 8-lane group
__host__ __device__ constexpr bool hk_rows(int kind) { return kind == HK_DENSE_AVX || kind == HK_DENSE_SMALL || kind == HK_U8 || kind == HK_U8_SMALL; }
__host__ __device__ constexpr bool hk_one_thread(int kind) { return kind == HK_DENSE_SMALL || kind == HK_U8_SMALL; }

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
    // ALGO_BUILD only (appended likewise): one launch inserts (b_insert = 1) or greedily descends (0) the points b_pts[0 .. nq) on one
    // level whose rows are links0 [rows][m0] (m0 = that level's m), row of a point = b_remap[id] (null: the id).  b_entry[i] is point
    // i's entry, replaced by the best point found.  An insert writes its point's row and its backlinks (target << 32 | i, source) to
    // b_tkey / b_tval [nq][m0] (~0 = none).
    const uint32_t* b_pts; uint32_t* b_entry; const uint32_t* b_remap; uint32_t b_insert;
    unsigned long long* b_tkey; uint32_t* b_tval;
};
// Multivector MaxSim queries (CUSTOM == HC_MAXSIM) reuse fields that only graph builds and custom queries read, so HnswParams, and with it
// the code of every other instantiation, stays as it was.  Point p = token rows mv_tok(p)[p] .. [p + 1) of the storage; query q = encoded
// query vectors mv_qoff(p)[q] .. [q + 1) of q_enc / q_off, clamped to mv_nv(p); a query of at most mv_stage_q(p) vectors is staged in
// shared memory (q_smem bytes), a larger one is read where it is.
__host__ __device__ __forceinline__ const uint32_t*& mv_tok(HnswParams& p) { return p.b_pts; }
__host__ __device__ __forceinline__ const uint32_t*& mv_qoff(HnswParams& p) { return p.b_remap; }
__host__ __device__ __forceinline__ uint32_t& mv_nv(HnswParams& p) { return p.n_ex; }
__host__ __device__ __forceinline__ uint32_t& mv_stage_q(HnswParams& p) { return p.ex_smem; }
__device__ __forceinline__ const uint32_t* mv_tok(const HnswParams& p) { return p.b_pts; }
__device__ __forceinline__ const uint32_t* mv_qoff(const HnswParams& p) { return p.b_remap; }
__device__ __forceinline__ uint32_t mv_nv(const HnswParams& p) { return p.n_ex; }
__device__ __forceinline__ uint32_t mv_stage_q(const HnswParams& p) { return p.ex_smem; }
// A multivector graph build (qb_hnsw_build_multivector) reads every ALGO_BUILD field as well as the token offsets, so its inserts
// (hnsw_build_mv_kernel, qb_hnsw_build.cu) take HnswParams plus the offsets.  The pieces below that read the offsets are templated on the
// parameter type P and call mv_tok(p), which picks the right field by overload.  The inserted point's token rows are the query; they are
// staged in the first q_smem bytes of shared memory when they fit there, as a MaxSim search stages its query.
struct HnswMvBuildParams : HnswParams {
    const uint32_t* tok;   // point p = token rows tok[p] .. tok[p + 1) of the storage
};
__device__ __forceinline__ const uint32_t* mv_tok(const HnswMvBuildParams& p) { return p.tok; }
// A custom query whose examples are multivectors, over a graph of multivector points (CUSTOM == HC_MAXSIM_CUSTOM, hnsw_mv_custom_kernel in
// qb_hnsw_mv_custom.cu).  Every custom-query field of HnswParams keeps its meaning (kind and shape, n_ex / ex_first / ex_stride, coef,
// custom entry points), counted in examples rather than encoded vectors: example e of query q is the encoded vectors
// ex_off[q * ex_stride + ex_first + e] .. [+ 1) of q_enc / q_off.  ex_smem = 1: all of a query's examples are staged in shared memory
// (q_smem bytes); 0: they are read where they are.
struct HnswMvCustomParams : HnswParams {
    const uint32_t* tok;      // point p = token rows tok[p] .. tok[p + 1) of the storage
    const uint32_t* ex_off;   // [nq * ex_stride + 1] example offsets, ascending
};
__device__ __forceinline__ const uint32_t* mv_tok(const HnswMvCustomParams& p) { return p.tok; }
// the example offsets, named through CUSTOM so that only the HC_MAXSIM_CUSTOM instantiations of the search body read the field
template <int CUSTOM, class P>
__device__ __forceinline__ const uint32_t* mv_ex_off(const P& p) { return p.ex_off; }

struct HnswSmem {
    unsigned long long* keys[2];
    uint8_t* flags[2];
    unsigned long long* newk;   // [HNSW_MAX_LINKS] (ACORN: [hop_cap])
    uint32_t* ids;              // [HNSW_MAX_LINKS] (ACORN: [hop_cap])
    float* sc;                  // [HNSW_MAX_LINKS] (ACORN: [hop_cap])
    const uint8_t* q;           // query (custom: the first example, in shared or global memory; example e at q + e * q_bytes)
};

enum { ALGO_HNSW = 0, ALGO_ACORN = 1 };   // qb_hnsw_algorithm
// hnsw_search_kernel's CUSTOM: what a query is.  HC_MAXSIM_CUSTOM: a custom query with multivector examples (HnswMvCustomParams)
enum { HC_NEAREST = 0, HC_CUSTOM = 1, HC_MAXSIM = 2, HC_MAXSIM_CUSTOM = 3 };
// queries that take custom entry points (get_entry_point), and queries scored by MaxSim over multivector points
__host__ __device__ constexpr bool hc_entry_points(int custom) { return custom == HC_CUSTOM || custom == HC_MAXSIM_CUSTOM; }
__host__ __device__ constexpr bool hc_multivector(int custom) { return custom == HC_MAXSIM || custom == HC_MAXSIM_CUSTOM; }
enum { ALGO_BUILD = 2 };                  // an insert of qb_hnsw_build: HNSW level search of a stored point, then its links (qb_hnsw_build.cu)

// ALGO_BUILD: a point's row in its level's table
__device__ __forceinline__ uint32_t hnsw_build_row(const HnswParams& p, uint32_t id) { return p.b_remap ? p.b_remap[id] : id; }

template <int KIND, int METRIC>
__device__ __forceinline__ float score_one(const HnswParams& p, const uint8_t* q_smem, float q_off, uint32_t id, int t) {
    if (KIND == HK_DENSE_AVX) {
        return score_avx_group8<METRIC>(reinterpret_cast<const float*>(p.rows + (size_t)id * p.stride), reinterpret_cast<const float*>(q_smem), p.dim, t);
    } else if (KIND == HK_DENSE_SMALL) {
        return score_small<METRIC>(reinterpret_cast<const float*>(p.rows + (size_t)id * p.stride), reinterpret_cast<const float*>(q_smem), p.dim);
    } else if (KIND == HK_U8) {
        return u8_score_avx_group8(METRIC, p.rows + (size_t)id * p.stride, q_smem, p.dim, t);
    } else if (KIND == HK_U8_SMALL) {
        return u8_score_small(METRIC, p.rows + (size_t)id * p.stride, q_smem, p.dim);
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

// ---- multivector MaxSim (score_max_similarity, query_scorer/mod.rs:77-98; QuantizedMultivectorStorage::score_point_max_similarity,
// quantized_multivector_storage/mod.rs:328-352).  A point's score is, summed sequentially in query-vector order from +0.0, the maximum
// over its token rows of each query vector's similarity, that maximum being the sequential `if sim > max` fold from -inf.  The CTA
// scores the hop's (point, token row) items in parallel, so the fold is restated as a max over keys (mv_key) that picks exactly the
// value the sequential fold keeps: NaN and -inf never win, -0.0 and +0.0 are equal and the earlier token keeps its own bits.
constexpr uint32_t MV_PTS = 64;   // points per scoring batch
constexpr uint32_t MV_NQ = 8;     // query vectors per chunk (score_avx_group8_multi accumulators)

struct MvShared {
    unsigned long long key[MV_PTS * MV_NQ];   // [point][query vector of the chunk] max keys, 0 = none (-inf)
    float sum[MV_PTS];                         // running sums over the chunks
    uint32_t pre[MV_PTS + 1];                  // token-row prefix of the batch's points
    uint32_t q0, nqv;                          // the query's first encoded vector and its vector count
    unsigned long long rows;                   // token rows the query scored (the counters)
};
// one per CTA; only the MaxSim instantiations reference it
__device__ __forceinline__ MvShared& mv_shared() {
    __shared__ MvShared s;
    return s;
}

// (canonical value, earliest token) -> an ordered key, with the winner's sign of zero in bit 0
__device__ __forceinline__ unsigned long long mv_key(float v, uint32_t tok) {
    if (!(v > __int_as_float(0xff800000))) return 0ull;
    const uint32_t b = __float_as_uint(v == 0.0f ? 0.0f : v);
    const uint32_t ord = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    const uint32_t neg0 = (v == 0.0f) ? (__float_as_uint(v) >> 31) : 0u;
    return ((unsigned long long)ord << 32) | ((unsigned long long)(0x7FFFFFFFu - tok) << 1) | neg0;
}
__device__ __forceinline__ float mv_value(unsigned long long key) {
    if (!key) return __int_as_float(0xff800000);
    if (key & 1ull) return -0.0f;
    const uint32_t ord = (uint32_t)(key >> 32);
    return __uint_as_float((ord & 0x80000000u) ? (ord & 0x7FFFFFFFu) : ~ord);
}

// the batch point whose token rows hold item k: pre[i] <= k < pre[i + 1]
__device__ __forceinline__ uint32_t mv_find(const uint32_t* pre, uint32_t ns, uint32_t k) {
    uint32_t lo = 0, hi = ns - 1;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (pre[mid + 1] > k) hi = mid; else lo = mid + 1; }
    return lo;
}

// The two halves of a MaxSim scoring batch, shared by maxsim_list and maxsim_custom_list as macros, so that maxsim_list expands to the
// code it had before the custom queries with multivector examples were added.  In scope: p, sm, tid, ms (MvShared&), GROUPS (NT / 8).
// QB_MV_BATCH(S0, NS): the batch ids[S0 .. S0 + NS): its token-row prefix into ms.pre, its rows counted in ms.rows, ms.sum zeroed.
#define QB_MV_BATCH(S0, NS)                                                  \
    if ((uint32_t)tid < (NS)) {                                             \
        const uint32_t id = sm.ids[(S0) + tid];                             \
        ms.pre[tid + 1] = mv_tok(p)[id + 1] - mv_tok(p)[id];                \
        ms.sum[tid] = 0.0f;                                                 \
    }                                                                       \
    __syncthreads();                                                        \
    if (tid == 0) {                                                         \
        ms.pre[0] = 0;                                                      \
        for (uint32_t i = 0; i < (NS); ++i) ms.pre[i + 1] += ms.pre[i];     \
        ms.rows += ms.pre[NS];                                              \
    }                                                                       \
    __syncthreads();
// QB_MV_CHUNKS(Q, QOFF, NQV, S0, NS, ITEMS): the batch's MaxSim against the NQV query vectors at Q (their SQ8 offsets at QOFF, or null)
// added to ms.sum in vector order: chunks of MV_NQ vectors; every (point, token row) item of the batch goes to one 8-lane group (dense
// small dims: one thread), which scores the row against the chunk's vectors by the storage's own chain and folds each similarity into its
// (point, vector) key.  One thread per point then adds the chunk's maxima in order.
#define QB_MV_CHUNKS(Q, QOFF, NQV, S0, NS, ITEMS)                                                                                         \
    for (uint32_t c0 = 0; c0 < (NQV); c0 += MV_NQ) {                                                                                      \
        const uint32_t nc = min((NQV) - c0, MV_NQ);                                                                                       \
        for (uint32_t i = tid; i < (NS) * MV_NQ; i += NT) ms.key[i] = 0ull;                                                               \
        __syncthreads();                                                                                                                  \
        const uint8_t* qc = (Q) + (size_t)c0 * p.q_bytes;                                                                                 \
        if (KIND == HK_DENSE_SMALL) {                                                                                                     \
            for (uint32_t k = tid; k < (ITEMS); k += NT) {                                                                                \
                const uint32_t i = mv_find(ms.pre, (NS), k), tok = k - ms.pre[i], row = mv_tok(p)[sm.ids[(S0) + i]] + tok;                \
                for (uint32_t j = 0; j < nc; ++j)                                                                                         \
                    atomicMax(&ms.key[i * MV_NQ + j], mv_key(score_one<KIND, METRIC>(p, qc + (size_t)j * p.q_bytes, 0.0f, row, 0), tok)); \
            }                                                                                                                             \
        } else {                                                                                                                          \
            const int g = tid >> 3, t = tid & 7;                                                                                          \
            for (uint32_t k = g; k < (((ITEMS) + GROUPS - 1) / GROUPS) * GROUPS; k += GROUPS) { /* whole warps stay converged */         \
                const uint32_t kk = k < (ITEMS) ? k : 0;                                                                                  \
                const uint32_t i = mv_find(ms.pre, (NS), kk), tok = kk - ms.pre[i], row = mv_tok(p)[sm.ids[(S0) + i]] + tok;              \
                float v[MV_NQ];                                                                                                           \
                if (KIND == HK_DENSE_AVX && nc == MV_NQ) {                                                                                \
                    score_avx_group8_multi<METRIC, MV_NQ>(reinterpret_cast<const float*>(p.rows + (size_t)row * p.stride),                \
                                                          reinterpret_cast<const float*>(qc), p.q_bytes / 4, p.dim, t, v);                \
                } else {                                                                                                                  \
                    _Pragma("unroll") for (uint32_t j = 0; j < MV_NQ; ++j)                                                                \
                        if (j < nc) v[j] = score_one<KIND, METRIC>(p, qc + (size_t)j * p.q_bytes, (QOFF) ? (QOFF)[c0 + j] : 0.0f, row, t);\
                }                                                                                                                         \
                if (k < (ITEMS) && t == 0) {                                                                                              \
                    _Pragma("unroll") for (uint32_t j = 0; j < MV_NQ; ++j)                                                                \
                        if (j < nc) atomicMax(&ms.key[i * MV_NQ + j], mv_key(v[j], tok));                                                 \
                }                                                                                                                         \
            }                                                                                                                             \
        }                                                                                                                                 \
        __syncthreads();                                                                                                                  \
        if ((uint32_t)tid < (NS)) {                                                                                                       \
            float s = ms.sum[tid];                                                                                                        \
            for (uint32_t j = 0; j < nc; ++j) s = __fadd_rn(s, mv_value(ms.key[tid * MV_NQ + j]));                                        \
            ms.sum[tid] = s;                                                                                                              \
        }                                                                                                                                 \
        __syncthreads();                                                                                                                  \
    }

// MaxSim scores of the points ids[0 .. n) into sc[0 .. n), in batches of MV_PTS points
template <int KIND, int METRIC, int NT, class P>
__device__ __forceinline__ void maxsim_list(const P& p, const HnswSmem& sm, uint32_t n) {
    constexpr uint32_t GROUPS = NT / 8;
    MvShared& ms = mv_shared();
    const int tid = threadIdx.x;
    const uint32_t nqv = ms.nqv;
    const float* qoff = p.q_off ? p.q_off + ms.q0 : nullptr;
    for (uint32_t s0 = 0; s0 < n; s0 += MV_PTS) {
        const uint32_t ns = min(n - s0, MV_PTS);
        QB_MV_BATCH(s0, ns)
        const uint32_t items = ms.pre[ns];
        QB_MV_CHUNKS(sm.q, qoff, nqv, s0, ns, items)
        if ((uint32_t)tid < ns) sm.sc[s0 + tid] = ms.sum[tid];
        __syncthreads();
    }
}

// ---- custom queries with multivector examples (MultiCustomQueryScorer, multi_custom_query_scorer.rs:88-104): a point's similarity to
// example e is the MaxSim of e's vectors against its token rows, exactly as maxsim_list computes it; Query::score_by folds the E values
// (qbf::fold).  A batch keeps every point's E MaxSims in mv_custom_tab() as [point][e], so it holds at most MV_TAB / E points.
constexpr uint32_t MV_TAB = 4096;   // floats of the [point][example] table: 16 KB, one point at E = 4096
__host__ __device__ constexpr uint32_t mv_custom_batch(uint32_t n_ex) { return n_ex * MV_PTS <= MV_TAB ? MV_PTS : MV_TAB / n_ex; }
// one per CTA; only the HC_MAXSIM_CUSTOM instantiations reference it
__device__ __forceinline__ float* mv_custom_tab() {
    __shared__ float tab[MV_TAB];
    return tab;
}

// the scores of the points ids[0 .. n) for custom query q into sc[0 .. n); sm.q holds the query's first example from its first vector on
template <int KIND, int METRIC, int NT>
__device__ __forceinline__ void maxsim_custom_list(const HnswMvCustomParams& p, const HnswSmem& sm, uint32_t n, uint32_t q) {
    constexpr uint32_t GROUPS = NT / 8;
    MvShared& ms = mv_shared();
    float* tab = mv_custom_tab();
    const int tid = threadIdx.x;
    const uint32_t ne = p.n_ex, bp = mv_custom_batch(ne);
    const uint32_t* eo = p.ex_off + (size_t)q * p.ex_stride + p.ex_first;
    const uint32_t v0 = eo[0];
    for (uint32_t s0 = 0; s0 < n; s0 += bp) {
        const uint32_t ns = min(n - s0, bp);
        QB_MV_BATCH(s0, ns)
        const uint32_t items = ms.pre[ns];
        for (uint32_t e = 0; e < ne; ++e) {
            const uint32_t a = eo[e], nv = eo[e + 1] - a;
            const uint8_t* qe = sm.q + (size_t)(a - v0) * p.q_bytes;
            const float* qoff = p.q_off ? p.q_off + a : nullptr;
            if ((uint32_t)tid < ns) ms.sum[tid] = 0.0f;   // ordered before the sums by the chunks' first barrier
            QB_MV_CHUNKS(qe, qoff, nv, s0, ns, items)
            if ((uint32_t)tid < ns) tab[tid * ne + e] = ms.sum[tid];
        }
        if ((uint32_t)tid < ns) {
            const float* row = tab + tid * ne;
            sm.sc[s0 + tid] = qbf::fold(p.ckind, p.n_a, p.n_b, p.coef ? p.coef + (size_t)q * p.n_coef : nullptr, [&](uint32_t e) { return row[e]; });
        }
        __syncthreads();
    }
}

// scores ids[0..n) into sc[0..n): one 8-lane group per id (dense small dims: one thread per id)
template <int KIND, int METRIC, int NT, int CUSTOM, class P>
__device__ __forceinline__ void score_list(const P& p, const HnswSmem& sm, float q_off, uint32_t n, uint32_t q) {
    constexpr int HNSW_GROUPS = NT / 8;
    const int tid = threadIdx.x;
    if constexpr (CUSTOM == HC_MAXSIM) {
        maxsim_list<KIND, METRIC, NT>(p, sm, n);
    } else if constexpr (CUSTOM == HC_MAXSIM_CUSTOM) {
        maxsim_custom_list<KIND, METRIC, NT>(p, sm, n, q);
    } else if (hk_one_thread(KIND)) {
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

// scores the stored rows ids[0 .. n) against the stored row `qrow` (global memory) with GROUPS 8-lane groups of the calling lanes
// lid = 0 .. GROUPS * 8 - 1 (dense small dims: one lane per id), so every score is the chain score_list uses; f(j, score) runs on one
// lane per id.  All GROUPS * 8 lanes must call it (the groups' shuffles span whole warps).
template <int KIND, int METRIC, int GROUPS, class F>
__device__ __forceinline__ void hnsw_score_rows(const HnswParams& p, const uint8_t* qrow, const uint32_t* ids, uint32_t n, int lid, F f) {
    if (hk_one_thread(KIND)) {
        for (uint32_t j = lid; j < n; j += GROUPS * 8) f(j, score_one<KIND, METRIC>(p, qrow, 0.0f, ids[j], 0));
    } else {
        const int g = lid >> 3, t = lid & 7;
        for (uint32_t j = g; j < ((n + GROUPS - 1) / GROUPS) * GROUPS; j += GROUPS) {
            const float s = score_one<KIND, METRIC>(p, qrow, 0.0f, ids[j < n ? j : 0], t);
            if (j < n && t == 0) f(j, s);
        }
    }
}

// one TMA-engine instruction pulls a whole vector (dim * 4 bytes) from HBM into L2, so that the group's demand loads — which the
// compiler keeps only 3-4 deep — are L2 hits instead of HBM round trips
__device__ __forceinline__ void prefetch_row_l2(const void* p, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
// MV: a multivector point, whose token rows are consecutive
template <int KIND, int MV = 0, class P>
__device__ __forceinline__ void prefetch_point(const P& p, uint32_t id) {
    if constexpr (MV) {
        const uint32_t r0 = mv_tok(p)[id], r1 = mv_tok(p)[id + 1];
        if (r1 <= r0) return;
        if (KIND == HK_DENSE_AVX || KIND == HK_DENSE_SMALL) prefetch_row_l2(p.rows + (size_t)r0 * p.stride, (r1 - r0) * p.stride);
        else prefetch_row_l2(p.codes + (size_t)r0 * p.ad, (r1 - r0) * p.ad);
    } else if (hk_rows(KIND)) {
        prefetch_row_l2(p.rows + (size_t)id * p.stride, p.stride);
    } else {
        prefetch_row_l2(p.codes + (size_t)id * p.ad, p.ad);
    }
}

// ScorerFilters::check_vector fails: the resident deleted flags or the per-call bitmap (either may be null); P = HnswParams or the
// inline-vector search's parameters (qb_hnsw_inline.cu)
template <class P>
__device__ __forceinline__ bool hnsw_filtered_out(const P& p, uint32_t id) {
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
template <int KIND, int NT, int MV = 0, class P>
__device__ __forceinline__ void acorn_collect(const P& p, const HnswSmem& sm, uint32_t* xids, uint32_t cand, uint32_t* visited, uint32_t* vlog,
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
            if (p.prefetch) prefetch_point<KIND, MV>(p, l);
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
        if (p.prefetch) prefetch_point<KIND, MV>(p, l);
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

// a MaxSim build's query: the token rows r0 .. r1 of the storage (the inserted point, or a candidate of the heuristic), copied into the
// query region of shared memory when they fit in its q_smem bytes, else read where they are (the same arithmetic either way).  The
// caller synchronises before the region is read.
template <int NT, class P>
__device__ __forceinline__ void mv_stage_rows(const P& p, HnswSmem& sm, uint8_t* region, uint32_t r0, uint32_t r1) {
    const uint8_t* src = p.rows + (size_t)r0 * p.stride;
    if ((uint64_t)(r1 - r0) * p.stride <= p.q_smem) {
        const uint4* s4 = reinterpret_cast<const uint4*>(src);
        uint4* dst = reinterpret_cast<uint4*>(region);
        for (uint32_t i = threadIdx.x; i < (r1 - r0) * p.stride / 16u; i += NT) dst[i] = s4[i];
        sm.q = region;
    } else {
        sm.q = src;
    }
    if (threadIdx.x == 0) { MvShared& ms = mv_shared(); ms.q0 = 0; ms.nqv = r1 - r0; ms.rows = 0; }
}

// CUSTOM = HC_CUSTOM: a custom query (recommend / discover / context / feedback) scored through qbf::fold, with per-query custom entry
// points; HC_MAXSIM: a multivector query over a graph of multivector points, scored by maxsim_list (128 threads).  The body is shared
// with the inserts of a multivector build (ALGO_BUILD with HC_MAXSIM), whose kernel takes HnswMvBuildParams (qb_hnsw_build_mv.cu).
template <int KIND, int METRIC, int NT, int ALGO, int CUSTOM>
__global__ void __launch_bounds__(NT) hnsw_search_kernel(const HnswParams p) {
#include "qb_hnsw_search_body.cuh"
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
    else if constexpr (KIND == HK_U8 || KIND == HK_U8_SMALL) { if (metric == M_COSINE) QB_HNSW_LAUNCH(M_COSINE); else QB_HNSW_LAUNCH(M_DOT); }
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
// the u8 kinds have a fourth metric (M_COSINE); they are not instantiated for MaxSim (qb_hnsw_mv_check rejects u8 token storages)
template <int KIND, int NT, int ALGO, int CUSTOM>
int occupancy_u8(int metric, size_t smem) {
    switch (metric) {
        case M_EUCLID: return occupancy_of<KIND, M_EUCLID, NT, ALGO, CUSTOM>(smem);
        case M_MANHATTAN: return occupancy_of<KIND, M_MANHATTAN, NT, ALGO, CUSTOM>(smem);
        case M_COSINE: return occupancy_of<KIND, M_COSINE, NT, ALGO, CUSTOM>(smem);
        default: return occupancy_of<KIND, M_DOT, NT, ALGO, CUSTOM>(smem);
    }
}
template <int NT, int ALGO, int CUSTOM>
int occupancy_dispatch(int kind, int metric, size_t smem) {
    if (kind == HK_U8 || kind == HK_U8_SMALL) {
        if constexpr (CUSTOM == HC_MAXSIM) return 1;
        else return kind == HK_U8 ? occupancy_u8<HK_U8, NT, ALGO, CUSTOM>(metric, smem) : occupancy_u8<HK_U8_SMALL, NT, ALGO, CUSTOM>(metric, smem);
    }
    switch (kind) {
        case HK_DENSE_AVX: return metric == M_EUCLID ? occupancy_of<HK_DENSE_AVX, M_EUCLID, NT, ALGO, CUSTOM>(smem) : metric == M_MANHATTAN ? occupancy_of<HK_DENSE_AVX, M_MANHATTAN, NT, ALGO, CUSTOM>(smem) : occupancy_of<HK_DENSE_AVX, M_DOT, NT, ALGO, CUSTOM>(smem);
        case HK_DENSE_SMALL: return metric == M_EUCLID ? occupancy_of<HK_DENSE_SMALL, M_EUCLID, NT, ALGO, CUSTOM>(smem) : metric == M_MANHATTAN ? occupancy_of<HK_DENSE_SMALL, M_MANHATTAN, NT, ALGO, CUSTOM>(smem) : occupancy_of<HK_DENSE_SMALL, M_DOT, NT, ALGO, CUSTOM>(smem);
        case HK_SQ8: return occupancy_of<HK_SQ8, M_DOT, NT, ALGO, CUSTOM>(smem);
        default: return occupancy_of<HK_SQ8_LANEX, M_DOT, NT, ALGO, CUSTOM>(smem);
    }
}
template <int NT, int ALGO, int CUSTOM>
qb_status launch_dispatch(int kind, int metric, const HnswParams& p, unsigned grid, size_t smem, cudaStream_t stream) {
    if (kind == HK_U8 || kind == HK_U8_SMALL) {
        if constexpr (CUSTOM == HC_MAXSIM) {
            qb_set_error("hnsw_search_maxsim: MaxSim over Uint8 token storages is not supported");
            return QB_ERR_UNSUPPORTED;
        } else {
            return kind == HK_U8 ? launch_kind<HK_U8, NT, ALGO, CUSTOM>(metric, p, grid, smem, stream) : launch_kind<HK_U8_SMALL, NT, ALGO, CUSTOM>(metric, p, grid, smem, stream);
        }
    }
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


// the METRIC a storage's rows are scored with: f32 cosine rows are normalised (M_DOT), Uint8 cosine is its own chain
inline int hnsw_metric(const qb_storage* s) {
    switch (s->distance) {
        case QB_DIST_EUCLID: return M_EUCLID;
        case QB_DIST_MANHATTAN: return M_MANHATTAN;
        case QB_DIST_COSINE: return (s->kind == QB_KIND_DENSE && s->dtype == QB_DT_U8) ? M_COSINE : M_DOT;
        default: return M_DOT;
    }
}

// shared memory of one CTA of hnsw_search_kernel with HNSW level 0 (also ALGO_BUILD): query, two key buffers, the hop's lists, two flag buffers
inline size_t hnsw_smem_bytes(uint32_t q_bytes, uint32_t ef) {
    return (size_t)((q_bytes + 15u) & ~15u) + (size_t)ef * 16 + HNSW_MAX_LINKS * 16 + 2 * (size_t)((ef + 15u) & ~15u);
}

}  // namespace

// The custom queries with multivector examples (qb_hnsw_mv_custom.cu): `params` is qb_hnsw_launch's HnswParams in this header's layout,
// passed untyped because the type has internal linkage; the kernel's HnswMvCustomParams add d_tok and d_ex_off to it.  per_sm != null:
// nothing is launched, *per_sm receives the kernel's resident CTAs per SM at smem bytes of dynamic shared memory.
qb_status qb_hnsw_mv_custom_launch(const void* params, const uint32_t* d_tok, const uint32_t* d_ex_off, int kind, int metric, int algo, unsigned grid,
                                   size_t smem, cudaStream_t stream, int* per_sm);
