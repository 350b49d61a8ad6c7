// qb_sparse_custom.cu — recommend / discover / context / feedback queries over sparse vectors: the reference's brute-force
// search_scored (sparse_vector_index/read_view/search.rs:302-341), BatchFilteredSearcher::peek_top_iter over every live or
// prefiltered point driven by SparseCustomQueryScorer (vector_storage/query_scorer/sparse_custom_query_scorer.rs).
//
// Storage (qb_sparse_storage_create): the points' CSR rows in USER dims, each row sorted by dim with the row build of the inverted
// index (qb_sparse_sort_rows in qb_sparse.cu).  The index's rows are in internal dims, whose order is the tracker's first-appearance
// order; a merge-join in that order sums the products in a different order, so the custom scan keeps its own rows.
//
// Scan: a query's examples are sorted by dim on the host; queries are packed into groups (at most 64 queries, at most 512 example
// similarities and a bounded staging size per group).  A group's examples are staged in shared memory as the sorted union of their
// dims, each union dim with the list of (query * E + example, weight) entries that contain it.  One CTA (8 warps) per (group, slice
// of points); one warp per point at a time:
//   - the row is read once for the whole group, 32 elements per step; each lane binary-searches its element's dim in the union;
//   - the hits are applied in lane order (ballot, then the lanes one after another), each hit's entries in parallel over the lanes:
//     an example holds a dim at most once, so the entries of one dim are distinct accumulators, and every accumulator receives its
//     products in ascending dim order, 0 + p1 + p2 + ... with every product and sum rounded (score_vectors, sparse_vector.rs:66-90);
//     a point that shares no dim with an example keeps +0.0, the reference's unwrap_or(0.0);
//   - lane l folds queries l, l + 32, ... through qbf::fold (Query::score_by) from the warp's accumulators in shared memory, so no
//     similarity matrix leaves the SM, and stores the (score, id) key in a shared tile of 32 points;
//   - the CTA writes the tile coalesced into each query's dense key list, which the top-k selection (qb_topk.cu) reduces.
// Deleted points get the empty key.  Queries are processed in chunks whose key lists fit a fixed scratch budget.
#include <algorithm>
#include <cfloat>
#include <tuple>

#include "qb_fold.cuh"
#include "qb_internal.h"

namespace {

constexpr uint32_t SC_THREADS = 256;
constexpr uint32_t SC_WARPS = SC_THREADS / 32;
constexpr uint32_t SC_TILE = 32;                    // points per CTA round
constexpr uint32_t SC_SLOTS = 512;                  // similarity accumulators per warp: group queries x E
constexpr uint32_t SC_MAX_GROUP = 64;               // queries per group
constexpr uint32_t SC_STAGE_BYTES = 72 * 1024;      // a group's staged examples: union dims, their offsets, entries
constexpr uint32_t SC_FIXED_SMEM = SC_MAX_GROUP * SC_TILE * 8 + SC_WARPS * SC_SLOTS * 4;
constexpr uint64_t SC_KEY_BUDGET = 1ull << 30;      // bytes of key lists per chunk of queries

struct ScGroup { uint32_t q0, nq, u0, nu, e0; };    // queries [q0, q0 + nq); union dims [u0, u0 + nu), offsets [u0 + g, .. + nu], entries from e0

struct ScParams {
    const uint64_t* rptr; const uint32_t* rdims; const float* rw;
    const uint32_t* ids;         // the scored points: ids[k], or point k when null
    uint64_t n;                  // scored slots
    const uint32_t* deleted;     // 32-bit words, bit = 1 deleted, or null (ids == null only)
    const ScGroup* groups; const uint32_t* u_dims; const uint32_t* u_off; const uint2* ent;
    int kind; uint32_t n_a, n_b, E;
    const float* coef;           // [query][1 + n_a] for feedback, else null
    uint32_t cq0;                // the chunk's first query: query q's keys at cand[(q - cq0) * n]
    unsigned long long* cand;
    float* scores;               // score mode (one query): scores[k] instead of keys
};

__global__ void __launch_bounds__(SC_THREADS) sparse_custom_kernel(const ScParams p) {
    extern __shared__ __align__(16) unsigned char sc_smem[];
    unsigned long long* s_keys = reinterpret_cast<unsigned long long*>(sc_smem);
    float* s_acc = reinterpret_cast<float*>(sc_smem + SC_MAX_GROUP * SC_TILE * 8);
    uint2* s_ent = reinterpret_cast<uint2*>(sc_smem + SC_FIXED_SMEM);
    const ScGroup g = p.groups[blockIdx.y];
    const uint32_t* g_off = p.u_off + g.u0 + blockIdx.y;
    const uint32_t ne = g_off[g.nu];
    uint32_t* s_dims = reinterpret_cast<uint32_t*>(s_ent + ne);
    uint32_t* s_off = s_dims + g.nu;
    for (uint32_t i = threadIdx.x; i < ne; i += blockDim.x) s_ent[i] = p.ent[g.e0 + i];
    for (uint32_t i = threadIdx.x; i < g.nu; i += blockDim.x) s_dims[i] = p.u_dims[g.u0 + i];
    for (uint32_t i = threadIdx.x; i <= g.nu; i += blockDim.x) s_off[i] = g_off[i];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, E = p.E, nu = g.nu;
    float* acc = s_acc + warp * SC_SLOTS;
    for (uint32_t i = lane; i < g.nq * E; i += 32) acc[i] = 0.0f;
    __syncthreads();
    const float* coef = p.coef ? p.coef + (size_t)g.q0 * (1 + p.n_a) : nullptr;
    for (uint64_t t0 = (uint64_t)blockIdx.x * SC_TILE; t0 < p.n; t0 += (uint64_t)gridDim.x * SC_TILE) {
        for (uint32_t j = warp; j < SC_TILE; j += SC_WARPS) {
            const uint64_t k = t0 + j;
            bool live = k < p.n;
            uint32_t id = 0;
            if (live) {
                id = p.ids ? p.ids[k] : (uint32_t)k;
                live = !(p.deleted && ((p.deleted[id >> 5] >> (id & 31)) & 1u));
            }
            if (live) {
                const uint64_t r0 = p.rptr[id], r1 = p.rptr[id + 1];
                for (uint64_t c = r0; c < r1; c += 32) {
                    const uint64_t e = c + lane;
                    uint32_t lo = 0, hi = 0;
                    float v = 0.0f;
                    if (e < r1) {
                        const uint32_t d = p.rdims[e];
                        v = p.rw[e];
                        uint32_t a = 0, b = nu;
                        while (a < b) { const uint32_t m = (a + b) >> 1; if (s_dims[m] < d) a = m + 1; else b = m; }
                        if (a < nu && s_dims[a] == d) { lo = s_off[a]; hi = s_off[a + 1]; }
                    }
                    unsigned mask = __ballot_sync(0xFFFFFFFFu, hi > lo);
                    while (mask) {
                        const int b = __ffs(mask) - 1;
                        const uint32_t blo = __shfl_sync(0xFFFFFFFFu, lo, b), bhi = __shfl_sync(0xFFFFFFFFu, hi, b);
                        const float bv = __shfl_sync(0xFFFFFFFFu, v, b);
                        for (uint32_t i = blo + lane; i < bhi; i += 32) {
                            const uint2 en = s_ent[i];
                            acc[en.x] = __fadd_rn(acc[en.x], __fmul_rn(__uint_as_float(en.y), bv));
                        }
                        __syncwarp();
                        mask &= mask - 1;
                    }
                }
            }
            for (uint32_t ql = lane; ql < g.nq; ql += 32) {
                float* a = acc + ql * E;
                unsigned long long key = 0ull;
                if (live) {
                    const float s = qbf::fold(p.kind, p.n_a, p.n_b, coef ? coef + (size_t)ql * (1 + p.n_a) : nullptr, [&](uint32_t x) { return a[x]; });
                    key = p.scores ? (unsigned long long)__float_as_uint(s) : qb_pack_key(s, id);
                    for (uint32_t x = 0; x < E; ++x) a[x] = 0.0f;
                }
                s_keys[ql * SC_TILE + j] = key;
            }
            __syncwarp();
        }
        __syncthreads();
        if (p.scores) {
            for (uint32_t j = threadIdx.x; j < SC_TILE; j += blockDim.x)
                if (t0 + j < p.n) p.scores[t0 + j] = __uint_as_float((uint32_t)s_keys[j]);
        } else {
            for (uint32_t i = threadIdx.x; i < g.nq * SC_TILE; i += blockDim.x) {
                const uint32_t ql = i / SC_TILE, j = i % SC_TILE;
                if (t0 + j < p.n) p.cand[(uint64_t)(g.q0 + ql - p.cq0) * p.n + t0 + j] = s_keys[i];
            }
        }
        __syncthreads();
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------ the handle (qb_internal.h)
static void sc_free(qb_sparse_storage* x) {
    if (!x) return;
    cudaSetDevice(x->device);
    if (x->stream) cudaStreamSynchronize(x->stream);
    cudaFree(x->d_rptr); cudaFree(x->d_rdims); cudaFree(x->d_rw); cudaFree(x->d_scratch);
    if (x->stream) cudaStreamDestroy(x->stream);
    delete x;
}

template <typename T>
static qb_status sc_alloc(qb_sparse_storage* x, T** p, size_t elems) {
    const size_t b = std::max<size_t>(elems * sizeof(T), 16);
    QB_CUDA(cudaMalloc(reinterpret_cast<void**>(p), b));
    x->hbm_bytes += b;
    return QB_OK;
}

static qb_status sc_build(qb_sparse_storage* x, const uint64_t* indptr, const uint32_t* dims, const float* weights) {
    const uint64_t n = x->nnz;
    cudaStream_t st = x->stream;
    QB_TRY(sc_alloc(x, &x->d_rptr, (size_t)x->n_points + 1));
    QB_TRY(sc_alloc(x, &x->d_rdims, n));
    QB_TRY(sc_alloc(x, &x->d_rw, n));
    QB_CUDA(cudaMemcpyAsync(x->d_rptr, indptr, ((size_t)x->n_points + 1) * 8, cudaMemcpyHostToDevice, st));
    unsigned long long* post = nullptr;   // the row build's (dim, id) keys: not used here
    if (n) QB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&post), n * 8, st));
    unsigned int flags = 0;
    const qb_status rc = qb_sparse_sort_rows(st, x->n_points, n, x->d_rptr, dims, weights, 0, true, x->d_rdims, x->d_rw, post, &flags);
    cudaFreeAsync(post, st);
    const cudaError_t e = cudaStreamSynchronize(st);
    QB_TRY(rc);
    QB_CHECK(e == cudaSuccess, QB_ERR_CUDA, "sparse_storage_create: %s", cudaGetErrorString(e));
    QB_CHECK(!(flags & 2u), QB_ERR_INVALID, "sparse_storage_create: a weight is not finite");
    QB_CHECK(!(flags & 4u), QB_ERR_INVALID, "sparse_storage_create: a dim is repeated within a row");
    x->h_rptr.assign(indptr, indptr + (size_t)x->n_points + 1);
    return QB_OK;
}

extern "C" qb_status qb_sparse_storage_create(int32_t device, uint32_t n_points, const uint64_t* indptr, const uint32_t* dims, const float* weights,
                                              int32_t on_disk, qb_sparse_storage** out) {
    QB_CHECK(out && indptr, QB_ERR_INVALID, "sparse_storage_create: null argument");
    *out = nullptr;
    QB_CHECK(indptr[0] == 0, QB_ERR_INVALID, "sparse_storage_create: indptr[0] must be 0");
    for (uint32_t r = 0; r < n_points; ++r)
        QB_CHECK(indptr[r + 1] >= indptr[r], QB_ERR_INVALID, "sparse_storage_create: indptr descends at row %u", r);
    const uint64_t nnz = indptr[n_points];
    QB_CHECK(nnz == 0 || (dims && weights), QB_ERR_INVALID, "sparse_storage_create: null argument");
    QB_CHECK(nnz < 0xFFFFFFFFull, QB_ERR_UNSUPPORTED, "sparse_storage_create: %llu elements (32-bit positions)", (unsigned long long)nnz);
    QB_TRY(qb_use_device(device));
    qb_sparse_storage* x = new qb_sparse_storage();
    x->device = device; x->n_points = n_points; x->nnz = nnz; x->on_disk = on_disk ? 1 : 0;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) x->sm_count = prop.multiProcessorCount;
    qb_status rc = cudaStreamCreateWithFlags(&x->stream, cudaStreamNonBlocking) == cudaSuccess ? QB_OK : QB_ERR_CUDA;
    if (rc != QB_OK) qb_set_error("sparse_storage_create: cudaStreamCreate failed");
    if (rc == QB_OK) rc = sc_build(x, indptr, dims, weights);
    if (rc != QB_OK) { sc_free(x); return rc; }
    *out = x;
    return QB_OK;
}

extern "C" void qb_sparse_storage_destroy(qb_sparse_storage* s) { sc_free(s); }

extern "C" qb_status qb_sparse_storage_info(const qb_sparse_storage* s, uint32_t* n_points, uint64_t* n_elements, uint64_t* hbm_bytes) {
    QB_CHECK(s, QB_ERR_INVALID, "sparse_storage_info: null storage");
    if (n_points) *n_points = s->n_points;
    if (n_elements) *n_elements = s->nnz;
    if (hbm_bytes) *hbm_bytes = s->hbm_bytes;
    return QB_OK;
}

// ------------------------------------------------------------------------------------------------ the queries
constexpr uint32_t QB_SPARSE_CUSTOM_MAX_TOP = 4096;
constexpr uint32_t QB_SPARSE_CUSTOM_MAX_NNZ = 4096;        // example non-zeros per query
constexpr uint32_t QB_SPARSE_CUSTOM_MAX_EXAMPLES = 256;    // E

// a batch's examples checked, sorted by dim and packed into groups with their staged unions
struct ScPrep {
    uint32_t E = 0;
    std::vector<uint64_t> ex_nnz;       // per query: the example elements as given
    std::vector<ScGroup> groups;
    std::vector<uint32_t> u_dims, u_off;
    std::vector<uint2> ent;
    size_t max_stage = 0;               // bytes of the largest group's staging
};

static qb_status sc_prepare(int kind, uint32_t n_a, uint32_t n_b, const uint64_t* ex_indptr, const uint32_t* ex_dims, const float* ex_weights, const float* coef,
                            uint32_t nq, uint32_t max_group, ScPrep& pp, const char* who) {
    QB_CHECK(kind >= QB_QUERY_RECO_BEST_SCORE && kind <= QB_QUERY_FEEDBACK_NAIVE, QB_ERR_INVALID, "%s: unknown kind %d", who, kind);
    QB_CHECK((kind != QB_QUERY_DISCOVER && kind != QB_QUERY_CONTEXT && kind != QB_QUERY_FEEDBACK_NAIVE) || n_b == 0, QB_ERR_INVALID,
             "%s: n_b must be 0 for discover / context / feedback (n_a = pairs)", who);
    const uint32_t E = qb_custom_examples(kind, n_a, n_b);
    QB_CHECK(E >= 1 && E <= 4096, QB_ERR_INVALID, "%s: %u examples (need 1..4096)", who, E);
    QB_CHECK(kind != QB_QUERY_FEEDBACK_NAIVE || coef || nq == 0, QB_ERR_INVALID, "%s: feedback needs coef", who);
    QB_CHECK(nq == 0 || ex_indptr, QB_ERR_INVALID, "%s: null argument", who);
    const uint64_t n_ex = (uint64_t)nq * E;
    if (nq) {
        QB_CHECK(ex_indptr[0] == 0, QB_ERR_INVALID, "%s: ex_indptr[0] must be 0", who);
        for (uint64_t j = 0; j < n_ex; ++j) QB_CHECK(ex_indptr[j + 1] >= ex_indptr[j], QB_ERR_INVALID, "%s: ex_indptr descends at example %llu", who, (unsigned long long)j);
        QB_CHECK(ex_indptr[n_ex] == 0 || (ex_dims && ex_weights), QB_ERR_INVALID, "%s: null argument", who);
    }
    QB_CHECK(E <= QB_SPARSE_CUSTOM_MAX_EXAMPLES, QB_ERR_UNSUPPORTED, "%s: %u examples > %u", who, E, QB_SPARSE_CUSTOM_MAX_EXAMPLES);
    pp.E = E;
    pp.ex_nnz.assign(nq, 0);
    // every example sorted by dim (the scorer's sort_by_indices); a repeated dim fails SparseVector validation
    std::vector<std::pair<uint32_t, float>> v;
    std::vector<std::tuple<uint32_t, uint32_t, float>> tri;   // (dim, slot, weight) of the group being built
    const uint32_t g_cap = std::min(std::min(SC_MAX_GROUP, SC_SLOTS / E), std::max(max_group, 1u));
    auto close = [&](uint32_t q0, uint32_t q1) {
        std::sort(tri.begin(), tri.end(), [](const auto& a, const auto& b) { return std::get<0>(a) != std::get<0>(b) ? std::get<0>(a) < std::get<0>(b) : std::get<1>(a) < std::get<1>(b); });
        ScGroup g{q0, q1 - q0, (uint32_t)pp.u_dims.size(), 0, (uint32_t)pp.ent.size()};
        for (size_t i = 0; i < tri.size(); ++i) {
            if (i == 0 || std::get<0>(tri[i]) != std::get<0>(tri[i - 1])) { pp.u_dims.push_back(std::get<0>(tri[i])); pp.u_off.push_back((uint32_t)i); ++g.nu; }
            uint32_t wb;
            memcpy(&wb, &std::get<2>(tri[i]), 4);
            pp.ent.push_back(make_uint2(std::get<1>(tri[i]), wb));
        }
        pp.u_off.push_back((uint32_t)tri.size());
        pp.groups.push_back(g);
        pp.max_stage = std::max(pp.max_stage, (size_t)tri.size() * 8 + (size_t)g.nu * 8 + 4);
        tri.clear();
    };
    uint32_t gq0 = 0;
    for (uint32_t q = 0; q < nq; ++q) {
        const uint64_t qn = ex_indptr[(uint64_t)(q + 1) * E] - ex_indptr[(uint64_t)q * E];
        QB_CHECK(qn <= QB_SPARSE_CUSTOM_MAX_NNZ, QB_ERR_UNSUPPORTED, "%s: query %u has %llu example non-zeros > %u", who, q, (unsigned long long)qn,
                 QB_SPARSE_CUSTOM_MAX_NNZ);
        pp.ex_nnz[q] = qn;
        // a group ends at g_cap queries or when its staging could outgrow the budget (16 bytes per entry bounds it)
        if (q > gq0 && (q - gq0 == g_cap || (tri.size() + qn) * 16 + 8 > SC_STAGE_BYTES)) { close(gq0, q); gq0 = q; }
        for (uint32_t j = 0; j < E; ++j) {
            const uint64_t x = (uint64_t)q * E + j;
            v.clear();
            for (uint64_t e = ex_indptr[x]; e < ex_indptr[x + 1]; ++e) v.emplace_back(ex_dims[e], ex_weights[e]);
            std::sort(v.begin(), v.end(), [](const std::pair<uint32_t, float>& a, const std::pair<uint32_t, float>& b) { return a.first < b.first; });
            for (size_t i = 1; i < v.size(); ++i)
                QB_CHECK(v[i].first != v[i - 1].first, QB_ERR_INVALID, "%s: dim %u repeated in example %u of query %u", who, v[i].first, j, q);
            for (const auto& e : v) tri.emplace_back(e.first, (q - gq0) * E + j, e.second);
        }
    }
    if (nq) close(gq0, nq);
    return QB_OK;
}

// the scored points' element total (Σ|v|) for the counters
static uint64_t sc_elements(const qb_sparse_storage* s, const uint32_t* ids, uint64_t n) {
    uint64_t t = 0;
    for (uint64_t k = 0; k < n; ++k) t += s->h_rptr[ids[k] + 1] - s->h_rptr[ids[k]];
    return t;
}

static void sc_count(const qb_sparse_storage* s, const ScPrep& pp, uint64_t n_scored, uint64_t elems, qb_hw_counters* counters) {
    if (!counters) return;
    // per scored point and example: cpu += 4 * (|v| + |example|); per scored point: vector_io_read += 2 |v| * (4 on disk, else 0)
    for (uint64_t qn : pp.ex_nnz) {
        counters->cpu += 4 * ((uint64_t)pp.E * elems + n_scored * qn);
        counters->vector_io_read += s->on_disk ? 2 * elems * 4 : 0;
    }
}

// stage the examples, launch the scan over the scored slots for the groups [g0, g1) of queries [cq0, ..)
static qb_status sc_launch(qb_sparse_storage* s, const ScPrep& pp, int kind, uint32_t n_a, uint32_t n_b, const ScGroup* d_groups, const uint32_t* d_u_dims,
                           const uint32_t* d_u_off, const uint2* d_ent, const float* d_coef, const uint32_t* d_ids, uint64_t n, const uint32_t* d_deleted,
                           uint32_t g0, uint32_t g1, unsigned long long* d_cand, float* d_scores) {
    const size_t smem = SC_FIXED_SMEM + pp.max_stage;
    QB_CUDA(cudaFuncSetAttribute(sparse_custom_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 1;
    QB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sparse_custom_kernel, SC_THREADS, smem));
    const uint64_t tiles = (n + SC_TILE - 1) / SC_TILE;
    const uint64_t want = (uint64_t)s->sm_count * std::max(per_sm, 1) * 4;
    const unsigned gx = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(tiles, (want + (g1 - g0) - 1) / (g1 - g0)));
    // the offsets of group g start at u_off[u0 + g]: the kernel adds its group's local index to u0, so the table is shifted by g0
    const ScParams p{s->d_rptr, s->d_rdims, s->d_rw, d_ids, n, d_deleted, d_groups + g0, d_u_dims, d_u_off + g0, d_ent, kind, n_a, n_b, pp.E,
                     d_coef, pp.groups[g0].q0, d_cand, d_scores};
    sparse_custom_kernel<<<dim3(gx, g1 - g0), SC_THREADS, smem, s->stream>>>(p);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

static qb_status sc_check_ids(const qb_sparse_storage* s, const uint32_t* ids, uint64_t n, const char* who) {
    std::vector<uint32_t> sid(ids, ids + n);
    for (uint32_t id : sid) QB_CHECK(id < s->n_points, QB_ERR_INVALID, "%s: id %u >= n_points %u", who, id, s->n_points);
    std::sort(sid.begin(), sid.end());
    for (size_t i = 1; i < sid.size(); ++i) QB_CHECK(sid[i] != sid[i - 1], QB_ERR_INVALID, "%s: id %u repeated", who, sid[i]);
    return QB_OK;
}

extern "C" qb_status qb_sparse_search_custom_batch(qb_sparse_storage* s, qb_query_kind kind, uint32_t n_a, uint32_t n_b, const uint64_t* ex_indptr,
                                                   const uint32_t* ex_dims, const float* ex_weights, const float* coef, uint32_t n_queries, uint32_t top,
                                                   const uint64_t* deleted_bitmap, const uint32_t* id_list, uint64_t n_ids, const volatile int32_t* is_stopped,
                                                   qb_scored_point* out, uint32_t* out_counts, qb_hw_counters* counters) {
    const char* who = "sparse_search_custom_batch";
    QB_CHECK(s && out_counts && (out || n_queries == 0), QB_ERR_INVALID, "%s: null argument", who);
    QB_CHECK(id_list || n_ids == 0, QB_ERR_INVALID, "%s: null argument", who);
    QB_CHECK(top >= 1, QB_ERR_INVALID, "%s: top must be >= 1", who);
    if (id_list) QB_TRY(sc_check_ids(s, id_list, n_ids, who));
    // the scored points (peek_top_iter): the listed ids that are not deleted, or every point not deleted (keys of deleted points are empty)
    auto is_del = [&](uint32_t id) { return deleted_bitmap && ((deleted_bitmap[id >> 6] >> (id & 63)) & 1ull); };
    std::vector<uint32_t> ids;
    if (id_list)
        for (uint64_t k = 0; k < n_ids; ++k) if (!is_del(id_list[k])) ids.push_back(id_list[k]);
    const uint64_t n = id_list ? ids.size() : s->n_points;
    const uint64_t max_group = std::min<uint64_t>(65535, std::max<uint64_t>(1, SC_KEY_BUDGET / std::max<uint64_t>(n * 8, 1)));
    ScPrep pp;
    QB_TRY(sc_prepare((int)kind, n_a, n_b, ex_indptr, ex_dims, ex_weights, coef, n_queries, (uint32_t)max_group, pp, who));
    QB_CHECK(top <= QB_SPARSE_CUSTOM_MAX_TOP, QB_ERR_UNSUPPORTED, "%s: top %u > %u", who, top, QB_SPARSE_CUSTOM_MAX_TOP);
    if (n_queries == 0) return QB_OK;
    QB_CHECK(!(is_stopped && *is_stopped), QB_ERR_CANCELLED, "%s: cancelled", who);
    if (counters) {
        uint64_t elems = 0, live = n;
        if (id_list) elems = sc_elements(s, ids.data(), ids.size());
        else if (!deleted_bitmap) elems = s->nnz;
        else {
            live = 0;
            for (uint32_t id = 0; id < s->n_points; ++id) if (!is_del(id)) { ++live; elems += s->h_rptr[id + 1] - s->h_rptr[id]; }
        }
        sc_count(s, pp, live, elems, counters);
    }
    if (n == 0) {
        memset(out_counts, 0, (size_t)n_queries * 4);
        return QB_OK;
    }
    QB_TRY(qb_use_device(s->device));
    std::lock_guard<std::mutex> lk(s->mu);
    const size_t ng = pp.groups.size(), words = ((size_t)s->n_points + 63) / 64, ncoef = coef ? (size_t)n_queries * (1 + n_a) : 0;
    const uint64_t qc = max_group;   // queries per chunk
    // scratch = [groups | union dims | offsets | entries | coef | ids | deleted words | out | counts | keys]
    const size_t ud_at = round_up_u64(ng * sizeof(ScGroup), 16), uo_at = round_up_u64(ud_at + pp.u_dims.size() * 4, 16);
    const size_t en_at = round_up_u64(uo_at + pp.u_off.size() * 4, 16), cf_at = round_up_u64(en_at + pp.ent.size() * 8, 16);
    const size_t id_at = round_up_u64(cf_at + ncoef * 4, 16), del_at = round_up_u64(id_at + ids.size() * 4, 16);
    const size_t out_at = round_up_u64(del_at + (deleted_bitmap && !id_list ? words * 8 : 0), 16), cnt_at = out_at + (size_t)n_queries * top * 8;
    const size_t cand_at = round_up_u64(cnt_at + (size_t)n_queries * 4, 16), bytes = cand_at + std::min<uint64_t>(qc, n_queries) * n * 8;
    QB_TRY(qb_ensure_device(&s->d_scratch, &s->scratch_bytes, bytes));
    std::vector<uint8_t> h(out_at, 0);
    memcpy(h.data(), pp.groups.data(), ng * sizeof(ScGroup));
    memcpy(h.data() + ud_at, pp.u_dims.data(), pp.u_dims.size() * 4);
    memcpy(h.data() + uo_at, pp.u_off.data(), pp.u_off.size() * 4);
    memcpy(h.data() + en_at, pp.ent.data(), pp.ent.size() * 8);
    if (ncoef) memcpy(h.data() + cf_at, coef, ncoef * 4);
    if (!ids.empty()) memcpy(h.data() + id_at, ids.data(), ids.size() * 4);
    if (deleted_bitmap && !id_list) memcpy(h.data() + del_at, deleted_bitmap, words * 8);
    uint8_t* d = reinterpret_cast<uint8_t*>(s->d_scratch);
    QB_CUDA(cudaMemcpyAsync(d, h.data(), out_at, cudaMemcpyHostToDevice, s->stream));
    const ScGroup* d_groups = reinterpret_cast<const ScGroup*>(d);
    for (uint32_t g0 = 0; g0 < ng;) {
        // a chunk: the groups whose queries fit the key budget
        uint32_t g1 = g0 + 1;
        while (g1 < ng && pp.groups[g1].q0 + pp.groups[g1].nq - pp.groups[g0].q0 <= qc) ++g1;
        const uint32_t cq0 = pp.groups[g0].q0, cnq = pp.groups[g1 - 1].q0 + pp.groups[g1 - 1].nq - cq0;
        unsigned long long* cand = reinterpret_cast<unsigned long long*>(d + cand_at);
        QB_TRY(sc_launch(s, pp, (int)kind, n_a, n_b, d_groups, reinterpret_cast<const uint32_t*>(d + ud_at), reinterpret_cast<const uint32_t*>(d + uo_at),
                         reinterpret_cast<const uint2*>(d + en_at), ncoef ? reinterpret_cast<const float*>(d + cf_at) : nullptr,
                         id_list ? reinterpret_cast<const uint32_t*>(d + id_at) : nullptr, n,
                         deleted_bitmap && !id_list ? reinterpret_cast<const uint32_t*>(d + del_at) : nullptr, g0, g1, cand, nullptr));
        QB_TRY(qb_launch_select(cand, nullptr, n, n, cnq, top, 0, reinterpret_cast<qb_scored_point*>(d + out_at) + (size_t)cq0 * top,
                                reinterpret_cast<uint32_t*>(d + cnt_at) + cq0, nullptr, nullptr, s->stream));
        g0 = g1;
    }
    QB_CUDA(cudaMemcpyAsync(out, d + out_at, (size_t)n_queries * top * 8, cudaMemcpyDeviceToHost, s->stream));
    QB_CUDA(cudaMemcpyAsync(out_counts, d + cnt_at, (size_t)n_queries * 4, cudaMemcpyDeviceToHost, s->stream));
    QB_CUDA(cudaStreamSynchronize(s->stream));
    return QB_OK;
}

extern "C" qb_status qb_sparse_score_custom(qb_sparse_storage* s, qb_query_kind kind, uint32_t n_a, uint32_t n_b, const uint64_t* ex_indptr, const uint32_t* ex_dims,
                                            const float* ex_weights, const float* coef, const uint32_t* ids, uint64_t n, float* scores, qb_hw_counters* counters) {
    const char* who = "sparse_score_custom";
    QB_CHECK(s && ex_indptr && (n == 0 || (ids && scores)), QB_ERR_INVALID, "%s: null argument", who);
    QB_TRY(sc_check_ids(s, ids, n, who));
    ScPrep pp;
    QB_TRY(sc_prepare((int)kind, n_a, n_b, ex_indptr, ex_dims, ex_weights, coef, 1, 1, pp, who));
    if (counters) sc_count(s, pp, n, sc_elements(s, ids, n), counters);
    if (n == 0) return QB_OK;
    QB_TRY(qb_use_device(s->device));
    std::lock_guard<std::mutex> lk(s->mu);
    const size_t ncoef = coef ? 1 + (size_t)n_a : 0;
    // scratch = [group | union dims | offsets | entries | coef | ids | scores]
    const size_t ud_at = round_up_u64(sizeof(ScGroup), 16), uo_at = round_up_u64(ud_at + pp.u_dims.size() * 4, 16);
    const size_t en_at = round_up_u64(uo_at + pp.u_off.size() * 4, 16), cf_at = round_up_u64(en_at + pp.ent.size() * 8, 16);
    const size_t id_at = round_up_u64(cf_at + ncoef * 4, 16), sc_at = round_up_u64(id_at + n * 4, 16), bytes = sc_at + n * 4;
    QB_TRY(qb_ensure_device(&s->d_scratch, &s->scratch_bytes, bytes));
    std::vector<uint8_t> h(sc_at, 0);
    memcpy(h.data(), pp.groups.data(), sizeof(ScGroup));
    memcpy(h.data() + ud_at, pp.u_dims.data(), pp.u_dims.size() * 4);
    memcpy(h.data() + uo_at, pp.u_off.data(), pp.u_off.size() * 4);
    memcpy(h.data() + en_at, pp.ent.data(), pp.ent.size() * 8);
    if (ncoef) memcpy(h.data() + cf_at, coef, ncoef * 4);
    memcpy(h.data() + id_at, ids, n * 4);
    uint8_t* d = reinterpret_cast<uint8_t*>(s->d_scratch);
    QB_CUDA(cudaMemcpyAsync(d, h.data(), sc_at, cudaMemcpyHostToDevice, s->stream));
    QB_TRY(sc_launch(s, pp, (int)kind, n_a, n_b, reinterpret_cast<const ScGroup*>(d), reinterpret_cast<const uint32_t*>(d + ud_at),
                     reinterpret_cast<const uint32_t*>(d + uo_at), reinterpret_cast<const uint2*>(d + en_at),
                     ncoef ? reinterpret_cast<const float*>(d + cf_at) : nullptr, reinterpret_cast<const uint32_t*>(d + id_at), n, nullptr, 0, 1, nullptr,
                     reinterpret_cast<float*>(d + sc_at)));
    QB_CUDA(cudaMemcpyAsync(scores, d + sc_at, n * 4, cudaMemcpyDeviceToHost, s->stream));
    QB_CUDA(cudaStreamSynchronize(s->stream));
    return QB_OK;
}
