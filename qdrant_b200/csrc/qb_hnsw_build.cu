// qb_hnsw_build.cu — HNSW graph construction on the device for dense f32 storages (qb_hnsw_build), and the plain `links.bin` export.
//
// Schedule: the reference's GPU builder (gpu/gpu_graph_builder.rs:19-101, gpu_level_builder.rs:12-96, batched_points.rs:36-163).
// Points sorted by level descending, then id; the first is the entry point.  The rest are cut into batches of at most `batch` points,
// cut again where the level changes; the first serial_points - 1 of them are batches of one (the reference links them on the CPU
// one by one; level-major with one point per batch is the same graph).  Then level by level from the top: a batch whose level is >= l
// inserts its points at l; the points below l only move their entry by greedy descent, in one launch per level (they come after every
// insert at l in the order, so one launch gives what a launch per batch gives).
// Each insert is the CPU builder's arithmetic: search_on_level with ef = max(ef_construct, m0) (gpu_graph_builder.rs:38) from the
// point's entry, fill_from_sorted_with_heuristic over the sorted result (links_container.rs:47-71), and connect_with_heuristic on
// every selected neighbour (links_container.rs:139-...).
// One deliberate deviation from run_insert_vector.comp:68-124, which updates backlinks under racing per-point locks and skips a
// neighbour another subgroup holds (a nondeterministic graph that can drop backlinks): a batch runs in two phases.
//   1. every point searches the level as it was before the batch and writes its own row (no batch point can reach another: nothing
//      links to a point before phase 2), with the (target << 32 | position in batch, source) pairs of its links;
//   2. the pairs are radix-sorted and one warp per target applies connect_with_heuristic for its sources in batch order.
// Different targets commute, so phase 2 equals applying source 1's backlinks, then source 2's, ...: the graph is a pure function of
// (rows, levels, m, m0, ef_construct, batch, serial_points), restated on the CPU by tests/hnsw_build_ref.c.
//
// Tables while building: level l has one row per point whose level is >= l, level_m ids padded with HNSW_EMPTY (the links are the
// prefix before the first HNSW_EMPTY).  Level 0 is [n][m0] by id, level l >= 1 [N_l][m] by position in the sorted order (the
// reference's remap), which is also the plain format's row order, so the finish is a count, a scan and a copy.
// The insert is hnsw_search_kernel<..., ALGO_BUILD> (qb_hnsw_traverse.cuh): the search kernel's beam search on the level's rows.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <vector>

#include "qb_hnsw_traverse.cuh"

namespace {

constexpr int HB_THREADS = 128;       // insert kernel: threads per CTA (one point per CTA at a time)
constexpr int HB_WARPS = 4;           // backlink kernel: warps per CTA (one target per warp at a time)
constexpr uint32_t HB_MAX_LEVEL = 30; // the highest level a point may have (levels are u8; 30 keeps the per-level tables small)

// connect_with_heuristic (links_container.rs:139-...) of every target in keys[0 .. n) (sorted; key = target << 32 | position, ~0 = none)
// with its sources vals[] in position order, one warp per target.  A short list appends; a full one is re-scored against the target
// with its new point, sorted (score desc, id asc) and refilled by the heuristic.
template <int KIND, int METRIC>
__global__ void __launch_bounds__(HB_WARPS * 32) hnsw_backlink_kernel(const HnswParams p, const unsigned long long* __restrict__ keys,
                                                                      const uint32_t* __restrict__ vals, uint32_t n) {
    __shared__ unsigned long long s_key[HB_WARPS][HNSW_MAX_LINKS + 1], s_sorted[HB_WARPS][HNSW_MAX_LINKS + 1];
    __shared__ uint32_t s_ids[HB_WARPS][HNSW_MAX_LINKS + 1];
    const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31u, lm = p.m0;
    unsigned long long* wkey = s_key[w];
    unsigned long long* wsorted = s_sorted[w];
    uint32_t* wids = s_ids[w];
    for (uint32_t e = blockIdx.x * HB_WARPS + w; e < n; e += gridDim.x * HB_WARPS) {
        const uint32_t t = (uint32_t)(keys[e] >> 32);
        if (t == HNSW_EMPTY) break;                                      // the empty slots sort last
        if (e > 0 && (uint32_t)(keys[e - 1] >> 32) == t) continue;       // not the target's first pair
        uint32_t* row = const_cast<uint32_t*>(p.links0) + (size_t)hnsw_build_row(p, t) * lm;
        const uint8_t* trow = p.rows + (size_t)t * p.stride;
        for (uint32_t e2 = e; e2 < n && (uint32_t)(keys[e2] >> 32) == t; ++e2) {
            const uint32_t src = vals[e2];
            const uint32_t a = lane < lm ? row[lane] : HNSW_EMPTY, b = lane + 32 < lm ? row[lane + 32] : HNSW_EMPTY;
            const uint32_t cnt = __popc(__ballot_sync(0xFFFFFFFFu, a != HNSW_EMPTY)) + __popc(__ballot_sync(0xFFFFFFFFu, b != HNSW_EMPTY));
            if (cnt < lm) {
                if (lane == 0) row[cnt] = src;
                __syncwarp();
                continue;
            }
            if (lane < lm) wids[lane] = a;
            if (lane + 32 < lm) wids[lane + 32] = b;
            if (lane == 0) wids[lm] = src;
            __syncwarp();
            hnsw_score_rows<KIND, METRIC, HB_WARPS>(p, trow, wids, lm + 1, (int)lane, [&](uint32_t j, float s) { wkey[j] = qb_pack_key(s, wids[j]); });
            __syncwarp();
            for (uint32_t j = lane; j <= lm; j += 32) {   // rank sort of distinct keys, descending
                const unsigned long long k = wkey[j];
                uint32_t r = 0;
                for (uint32_t i = 0; i <= lm; ++i) r += wkey[i] > k ? 1u : 0u;
                wsorted[r] = k;
            }
            __syncwarp();
            // fill_from_sorted_with_heuristic: the kept links go to wids[0 .. nsel)
            uint32_t nsel = 0;
            for (uint32_t c = 0; c <= lm && nsel < lm; ++c) {
                const uint32_t cid = qb_key_id(wsorted[c]);
                const float cs = qb_key_score(wsorted[c]);
                bool beat = false;
                hnsw_score_rows<KIND, METRIC, HB_WARPS>(p, p.rows + (size_t)cid * p.stride, wids, nsel, (int)lane, [&](uint32_t, float s) { beat |= s > cs; });
                beat = __any_sync(0xFFFFFFFFu, beat);
                if (!beat) {
                    if (lane == 0) wids[nsel] = cid;
                    ++nsel;
                }
                __syncwarp();
            }
            for (uint32_t j = lane; j < lm; j += 32) row[j] = j < nsel ? wids[j] : HNSW_EMPTY;
            __syncwarp();
        }
    }
}

// the build tables of every level, for the finish
struct HbTables {
    const uint32_t* t[HB_MAX_LEVEL + 1];
    uint64_t lo[HB_MAX_LEVEL + 2];   // first row of each level in the plain order; lo[levels] = rows
    uint32_t levels, m, m0;
};
__device__ __forceinline__ const uint32_t* hb_row(const HbTables& tb, uint64_t r, uint32_t& lm) {
    uint32_t l = 0;
    while (l + 1 < tb.levels && r >= tb.lo[l + 1]) ++l;
    lm = l ? tb.m : tb.m0;
    return tb.t[l] + (r - tb.lo[l]) * lm;
}
// links per row (counts[rows] = 0, so the exclusive scan ends on the total)
__global__ void hnsw_build_counts_kernel(const HbTables tb, uint64_t* __restrict__ counts) {
    const uint64_t rows = tb.lo[tb.levels];
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= rows; r += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t c = 0;
        if (r < rows) {
            uint32_t lm;
            const uint32_t* row = hb_row(tb, r, lm);
            while (c < lm && row[c] != HNSW_EMPTY) ++c;
        }
        counts[r] = c;
    }
}
__global__ void hnsw_build_neighbors_kernel(const HbTables tb, const uint64_t* __restrict__ offsets, uint32_t* __restrict__ neighbors) {
    const uint64_t rows = tb.lo[tb.levels];
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t lm;
        const uint32_t* row = hb_row(tb, r, lm);
        const uint64_t b = offsets[r], e = offsets[r + 1];
        for (uint64_t k = 0; k < e - b; ++k) neighbors[b + k] = row[k];
    }
}

// device temporaries of one call, freed on every exit path
struct HbScratch {
    std::vector<void*> bufs;
    cudaError_t alloc(void** p, size_t bytes) {
        *p = nullptr;
        const cudaError_t e = cudaMalloc(p, std::max<size_t>(bytes, 256));
        if (e == cudaSuccess) bufs.push_back(*p);
        return e;
    }
    ~HbScratch() { cudaDeviceSynchronize(); for (void* b : bufs) cudaFree(b); }
};

inline unsigned hb_grid(uint64_t items, uint64_t per_block, uint64_t max_blocks) {
    return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(ceil_div_u64(items, per_block), max_blocks));
}

template <int KIND, int METRIC>
struct HbKernels {
    static qb_status insert(const HnswParams& p, unsigned grid, size_t smem) {
        hnsw_search_kernel<KIND, METRIC, HB_THREADS, ALGO_BUILD, 0><<<grid, HB_THREADS, smem>>>(p);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
    static qb_status backlinks(const HnswParams& p, const unsigned long long* keys, const uint32_t* vals, uint32_t n) {
        hnsw_backlink_kernel<KIND, METRIC><<<hb_grid(n, HB_WARPS, 132 * 16), HB_WARPS * 32>>>(p, keys, vals, n);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
    static qb_status prepare(size_t smem, int* per_sm) {
        QB_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<KIND, METRIC, HB_THREADS, ALGO_BUILD, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        QB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, hnsw_search_kernel<KIND, METRIC, HB_THREADS, ALGO_BUILD, 0>, HB_THREADS, smem));
        if (*per_sm < 1) *per_sm = 1;
        return QB_OK;
    }
};

// the host-side schedule
struct HbPlan {
    std::vector<uint32_t> rest;                       // inserted points after the entry, in the sorted order
    std::vector<std::pair<uint32_t, uint32_t>> batches;   // [begin, end) in rest
    std::vector<uint8_t> level_of_rest;
    uint32_t entry_level = 0, max_batch = 1;
};

template <int KIND, int METRIC>
qb_status hb_levels(HnswParams p, const HbPlan& plan, uint32_t m, uint32_t m0, uint32_t* const* tables, const uint32_t* d_remap, uint32_t* d_pts,
                    uint32_t* d_entry, unsigned long long* d_tkey, uint32_t* d_tval, unsigned long long* d_tkey2, uint32_t* d_tval2, void* d_sort,
                    size_t sort_bytes, unsigned max_grid, size_t smem, int key_bits) {
    const uint32_t nr = (uint32_t)plan.rest.size();
    p.b_tkey = d_tkey; p.b_tval = d_tval;
    for (int l = (int)plan.entry_level; l >= 0; --l) {
        const uint32_t lm = l ? m : m0;
        p.links0 = tables[l]; p.m = lm; p.m0 = lm; p.b_remap = l ? d_remap : nullptr;
        for (const auto& bt : plan.batches) {
            if (plan.level_of_rest[bt.first] < (uint32_t)l) continue;
            const uint32_t np = bt.second - bt.first;
            p.b_pts = d_pts + bt.first; p.b_entry = d_entry + bt.first; p.nq = np; p.b_insert = 1;
            QB_CUDA(cudaMemsetAsync(p.work, 0, 4));
            QB_TRY((HbKernels<KIND, METRIC>::insert(p, std::min<unsigned>(np, max_grid), smem)));
            size_t bytes = sort_bytes;
            QB_CUDA(cub::DeviceRadixSort::SortPairs(d_sort, bytes, d_tkey, d_tkey2, d_tval, d_tval2, (int)(np * lm), 0, key_bits));
            QB_LAUNCHED();
            QB_TRY((HbKernels<KIND, METRIC>::backlinks(p, d_tkey2, d_tval2, np * lm)));
        }
        if (l == 0) break;
        // the points below l: greedy descent on l, one launch (they follow every insert at l)
        const uint32_t g0 = (uint32_t)(std::find_if(plan.level_of_rest.begin(), plan.level_of_rest.end(), [&](uint8_t v) { return v < (uint32_t)l; }) -
                                       plan.level_of_rest.begin());
        if (g0 < nr) {
            p.b_pts = d_pts + g0; p.b_entry = d_entry + g0; p.nq = nr - g0; p.b_insert = 0;
            QB_CUDA(cudaMemsetAsync(p.work, 0, 4));
            QB_TRY((HbKernels<KIND, METRIC>::insert(p, std::min<unsigned>(nr - g0, max_grid), smem)));
        }
    }
    return QB_OK;
}

// resident CTAs per SM of the insert kernel
inline qb_status hb_occupancy(int kind, int metric, size_t smem, int* per_sm) {
    if (kind == HK_DENSE_AVX)
        return metric == M_EUCLID ? HbKernels<HK_DENSE_AVX, M_EUCLID>::prepare(smem, per_sm)
                                  : metric == M_MANHATTAN ? HbKernels<HK_DENSE_AVX, M_MANHATTAN>::prepare(smem, per_sm) : HbKernels<HK_DENSE_AVX, M_DOT>::prepare(smem, per_sm);
    return metric == M_EUCLID ? HbKernels<HK_DENSE_SMALL, M_EUCLID>::prepare(smem, per_sm)
                              : metric == M_MANHATTAN ? HbKernels<HK_DENSE_SMALL, M_MANHATTAN>::prepare(smem, per_sm) : HbKernels<HK_DENSE_SMALL, M_DOT>::prepare(smem, per_sm);
}

}  // namespace

extern "C" qb_status qb_hnsw_build(qb_storage* s, uint32_t m, uint32_t m0, uint32_t ef_construct, const uint8_t* levels, uint32_t batch, uint32_t serial_points,
                                   qb_hnsw** out, uint32_t* entry_point, uint32_t* entry_level) {
    QB_CHECK(s && levels && out, QB_ERR_INVALID, "hnsw_build: null argument");
    *out = nullptr;
    QB_CHECK(s->kind == QB_KIND_DENSE && s->dtype == QB_DT_F32, QB_ERR_UNSUPPORTED,
             "hnsw_build: graphs are built over dense f32 storages only (build over the original vectors, then bind the graph to the quantized storage)");
    QB_CHECK(s->count >= 1, QB_ERR_INVALID, "hnsw_build: empty storage");
    QB_CHECK(s->count < 0xFFFFFFFFull, QB_ERR_UNSUPPORTED, "hnsw_build: %llu points", (unsigned long long)s->count);
    QB_CHECK(m >= 1 && m0 >= 1, QB_ERR_INVALID, "hnsw_build: m %u / m0 %u", m, m0);
    QB_CHECK(m <= HNSW_MAX_LINKS && m0 <= HNSW_MAX_LINKS, QB_ERR_UNSUPPORTED, "hnsw_build: m %u / m0 %u outside [1,%u]", m, m0, HNSW_MAX_LINKS);
    const uint32_t ef = std::max(ef_construct, m0);   // gpu_graph_builder.rs:38
    QB_CHECK(ef <= HNSW_MAX_EF, QB_ERR_UNSUPPORTED, "hnsw_build: ef %u > %u", ef, HNSW_MAX_EF);
    const uint32_t n = (uint32_t)s->count;
    uint32_t top_level = 0;
    for (uint32_t i = 0; i < n; ++i) {
        QB_CHECK(levels[i] <= HB_MAX_LEVEL, QB_ERR_INVALID, "hnsw_build: levels[%u] = %u > %u", i, (unsigned)levels[i], HB_MAX_LEVEL);
        top_level = std::max<uint32_t>(top_level, levels[i]);
    }
    if (batch == 0) batch = 512;               // GPU_GROUPS_COUNT_DEFAULT, gpu/mod.rs:34
    if (serial_points == 0) serial_points = 256;   // SINGLE_THREADED_HNSW_BUILD_THRESHOLD
    QB_CUDA(cudaSetDevice(s->device));

    // ---- order, rows per level, the schedule
    const uint32_t L = top_level + 1;
    std::vector<uint32_t> deleted;
    if (s->d_deleted) {
        deleted.resize(ceil_div_u64(n, 32));
        QB_CUDA(cudaMemcpy(deleted.data(), s->d_deleted, 4 * deleted.size(), cudaMemcpyDeviceToHost));
    }
    std::vector<uint64_t> per_level(L + 1, 0), start(L + 1, 0);
    for (uint32_t i = 0; i < n; ++i) per_level[levels[i]]++;
    for (int l = (int)L - 2; l >= 0; --l) start[l] = start[l + 1] + per_level[l + 1];   // level desc, then id (a stable counting sort)
    std::vector<uint32_t> order(n), pos(n);
    for (uint32_t i = 0; i < n; ++i) { pos[i] = (uint32_t)start[levels[i]]++; order[pos[i]] = i; }
    std::vector<uint64_t> rows_on(L);   // N_l: points whose level is >= l = the first N_l of the order
    for (uint32_t l = 0; l < L; ++l) { uint64_t c = 0; for (uint32_t k = l; k < L; ++k) c += per_level[k]; rows_on[l] = c; }
    HbPlan plan;
    uint32_t entry = HNSW_EMPTY;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t id = order[i];
        if (!deleted.empty() && ((deleted[id >> 5] >> (id & 31)) & 1u)) continue;   // iter_internal_excluding(deleted)
        if (entry == HNSW_EMPTY) entry = id;
        else plan.rest.push_back(id);
    }
    QB_CHECK(entry != HNSW_EMPTY, QB_ERR_INVALID, "hnsw_build: every point is deleted");
    plan.entry_level = levels[entry];
    const uint32_t nr = (uint32_t)plan.rest.size();
    plan.level_of_rest.resize(nr);
    for (uint32_t i = 0; i < nr; ++i) plan.level_of_rest[i] = levels[plan.rest[i]];
    {
        uint32_t k = 0;
        for (; k < std::min(serial_points - 1, nr); ++k) plan.batches.push_back({k, k + 1});
        while (k < nr) {   // build_initial_batches: chunks of `batch` from the first point after the entry, cut where the level changes
            uint32_t e = (uint32_t)std::min<uint64_t>((uint64_t)(k / batch + 1) * batch, nr);
            for (uint32_t j = k + 1; j < e; ++j) if (plan.level_of_rest[j] != plan.level_of_rest[k]) { e = j; break; }
            plan.batches.push_back({k, e});
            plan.max_batch = std::max(plan.max_batch, e - k);
            k = e;
        }
    }

    // ---- device state
    const int kind = s->dim >= 32 ? HK_DENSE_AVX : HK_DENSE_SMALL;
    const int metric = s->distance == QB_DIST_EUCLID ? M_EUCLID : (s->distance == QB_DIST_MANHATTAN ? M_MANHATTAN : M_DOT);
    HbScratch tmp;
    std::vector<uint32_t*> tables(L, nullptr);
    for (uint32_t l = 0; l < L; ++l) {
        const size_t bytes = (size_t)rows_on[l] * (l ? m : m0) * 4;
        QB_CUDA(tmp.alloc((void**)&tables[l], bytes));
        QB_CUDA(cudaMemset(tables[l], 0xFF, bytes));
    }
    uint32_t *d_remap = nullptr, *d_pts = nullptr, *d_entry = nullptr, *d_tval = nullptr, *d_tval2 = nullptr;
    unsigned long long *d_tkey = nullptr, *d_tkey2 = nullptr;
    unsigned int* d_work = nullptr;
    const size_t trip = (size_t)plan.max_batch * m0;
    QB_CUDA(tmp.alloc((void**)&d_remap, 4ull * n));
    QB_CUDA(tmp.alloc((void**)&d_pts, 4ull * nr));
    QB_CUDA(tmp.alloc((void**)&d_entry, 4ull * nr));
    QB_CUDA(tmp.alloc((void**)&d_tkey, 8 * trip));
    QB_CUDA(tmp.alloc((void**)&d_tkey2, 8 * trip));
    QB_CUDA(tmp.alloc((void**)&d_tval, 4 * trip));
    QB_CUDA(tmp.alloc((void**)&d_tval2, 4 * trip));
    QB_CUDA(tmp.alloc((void**)&d_work, 4));
    QB_CUDA(cudaMemcpy(d_remap, pos.data(), 4ull * n, cudaMemcpyHostToDevice));
    if (nr) QB_CUDA(cudaMemcpy(d_pts, plan.rest.data(), 4ull * nr, cudaMemcpyHostToDevice));
    {
        std::vector<uint32_t> ent(nr, entry);   // PointLinkingData::entry starts at the first point
        if (nr) QB_CUDA(cudaMemcpy(d_entry, ent.data(), 4ull * nr, cudaMemcpyHostToDevice));
    }
    const int key_bits = 64;   // target << 32 | position; an empty slot (~0) sorts last
    size_t sort_bytes = 0;
    QB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, d_tkey, d_tkey2, d_tval, d_tval2, (int)trip, 0, (int)key_bits));
    void* d_sort = nullptr;
    QB_CUDA(tmp.alloc(&d_sort, sort_bytes));

    HnswParams p{};
    p.n_points = n; p.levels = L;
    p.rows = reinterpret_cast<const uint8_t*>(s->d_rows); p.stride = s->row_stride; p.dim = s->dim;
    p.q_bytes = s->row_stride; p.ef = ef; p.top = 0; p.entry = 0; p.entry_level = 0;
    p.prefetch = qb_opt().hnsw_no_prefetch ? 0 : 1;
    p.work = d_work;
    const size_t smem = hnsw_smem_bytes(p.q_bytes, ef);
    QB_CHECK(smem <= 200 * 1024, QB_ERR_UNSUPPORTED, "hnsw_build: a row (%u B) + ef %u need %zu B of shared memory", p.q_bytes, ef, smem);
    // grid: the resident CTAs, at most one per point of the largest launch; per-CTA visited bitmaps (the kernel leaves them clean) and logs
    int per_sm = 1;
    QB_TRY(hb_occupancy(kind, metric, smem, &per_sm));
    const unsigned grid = std::min<unsigned>((unsigned)s->sm_count * (unsigned)per_sm, std::max<uint32_t>(1, std::max(plan.max_batch, nr)));
    const uint64_t words = ceil_div_u64(n, 32);
    p.visited_words = words; p.vlog_cap = 32768;
    QB_CUDA(tmp.alloc((void**)&p.visited, (size_t)grid * words * 4));
    QB_CUDA(tmp.alloc((void**)&p.vlog, (size_t)grid * p.vlog_cap * 4));
    QB_CUDA(cudaMemset(p.visited, 0, (size_t)grid * words * 4));
#define QB_HB_LEVELS(K, M) hb_levels<K, M>(p, plan, m, m0, tables.data(), d_remap, d_pts, d_entry, d_tkey, d_tval, d_tkey2, d_tval2, d_sort, sort_bytes, grid, smem, key_bits)
    if (kind == HK_DENSE_AVX) QB_TRY(metric == M_EUCLID ? QB_HB_LEVELS(HK_DENSE_AVX, M_EUCLID) : metric == M_MANHATTAN ? QB_HB_LEVELS(HK_DENSE_AVX, M_MANHATTAN) : QB_HB_LEVELS(HK_DENSE_AVX, M_DOT));
    else QB_TRY(metric == M_EUCLID ? QB_HB_LEVELS(HK_DENSE_SMALL, M_EUCLID) : metric == M_MANHATTAN ? QB_HB_LEVELS(HK_DENSE_SMALL, M_MANHATTAN) : QB_HB_LEVELS(HK_DENSE_SMALL, M_DOT));
#undef QB_HB_LEVELS

    // ---- finish: the plain arrays (level offsets, reindex, neighbours, offsets), then the handle as qb_hnsw_create_plain makes it
    HbTables tb{};
    tb.levels = L; tb.m = m; tb.m0 = m0;
    std::vector<uint64_t> lo(L + 1, 0);
    for (uint32_t l = 0; l < L; ++l) { tb.t[l] = tables[l]; lo[l + 1] = lo[l] + rows_on[l]; }
    for (uint32_t l = 0; l <= L; ++l) tb.lo[l] = lo[l];
    const uint64_t rows = lo[L], n_off = rows + 1;
    uint64_t* d_counts = nullptr;
    QB_CUDA(tmp.alloc((void**)&d_counts, 8 * n_off));
    hnsw_build_counts_kernel<<<hb_grid(n_off, 256, 132 * 16), 256>>>(tb, d_counts);
    QB_LAUNCHED();
    qb_hnsw* g = new qb_hnsw();
    g->st = s; g->n_points = n; g->m = m; g->m0 = m0; g->levels = L;
    g->level_offsets_ext = lo; g->n_offsets = n_off;
    auto fail = [&](qb_status st, const char* what, cudaError_t e) {
        qb_set_error("hnsw_build: %s: %s", what, cudaGetErrorString(e));
        qb_hnsw_destroy(g);
        return st;
    };
    bool ok = cudaMalloc(&g->d_level_offsets, std::max<size_t>(8 * L, 256)) == cudaSuccess && cudaMalloc(&g->d_reindex, std::max<size_t>(4ull * n, 256)) == cudaSuccess &&
              cudaMalloc(&g->d_offsets, 8 * n_off + 256) == cudaSuccess;
    if (!ok) return fail(QB_ERR_OOM, "cudaMalloc failed", cudaGetLastError());
    size_t scan_bytes = 0;
    cudaError_t ce = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, d_counts, g->d_offsets, (int64_t)n_off);
    void* d_scan = nullptr;
    if (ce == cudaSuccess) ce = tmp.alloc(&d_scan, scan_bytes);
    if (ce == cudaSuccess) ce = cub::DeviceScan::ExclusiveSum(d_scan, scan_bytes, d_counts, g->d_offsets, (int64_t)n_off);
    QB_LAUNCHED();
    uint64_t total = 0;
    if (ce == cudaSuccess) ce = cudaMemcpy(&total, g->d_offsets + rows, 8, cudaMemcpyDeviceToHost);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_level_offsets, lo.data(), 8 * L, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_reindex, d_remap, 4ull * n, cudaMemcpyDeviceToDevice);
    if (ce != cudaSuccess) return fail(QB_ERR_CUDA, "build", ce);
    g->n_neighbors = total;
    if (cudaMalloc(&g->d_neighbors, std::max<size_t>(4 * total, 256)) != cudaSuccess) return fail(QB_ERR_OOM, "cudaMalloc failed", cudaGetLastError());
    hnsw_build_neighbors_kernel<<<hb_grid(rows, 256, 132 * 16), 256>>>(tb, g->d_offsets, g->d_neighbors);
    QB_LAUNCHED();
    ce = cudaGetLastError();
    if (ce != cudaSuccess) return fail(QB_ERR_CUDA, "build", ce);
    const qb_status st = qb_hnsw_finish_plain(g, "hnsw_build");
    if (st != QB_OK) { qb_hnsw_destroy(g); return st; }
    *out = g;
    if (entry_point) *entry_point = entry;
    if (entry_level) *entry_level = plan.entry_level;
    return QB_OK;
}

// the plain links.bin (graph_links/header.rs:9-20, serializer.rs:53-200) of any handle, from its device arrays
extern "C" qb_status qb_hnsw_export_plain(const qb_hnsw* g, uint8_t* out, uint64_t cap, uint64_t* n_bytes) {
    QB_CHECK(g && (out || n_bytes), QB_ERR_INVALID, "hnsw_export_plain: null argument");
    const uint64_t n = g->n_points, L = g->levels, n_nb = g->n_neighbors, n_off = g->n_offsets;
    const uint64_t pos = 64 + 8 * L + 4 * n + 4 * n_nb, pad = (8 - pos % 8) % 8, total = pos + pad + 8 * n_off;
    if (n_bytes) *n_bytes = total;
    if (!out) return QB_OK;
    QB_CHECK(cap >= total, QB_ERR_INVALID, "hnsw_export_plain: %llu bytes of room, the graph needs %llu", (unsigned long long)cap, (unsigned long long)total);
    QB_CUDA(cudaSetDevice(g->st->device));
    memset(out, 0, 64);
    const uint64_t hdr[5] = {n, L, n_nb, n_off, pad};   // HeaderPlain
    memcpy(out, hdr, sizeof(hdr));
    memcpy(out + 64, g->level_offsets_ext.data(), 8 * L);
    QB_CUDA(cudaMemcpy(out + 64 + 8 * L, g->d_reindex, 4 * n, cudaMemcpyDeviceToHost));
    QB_CUDA(cudaMemcpy(out + 64 + 8 * L + 4 * n, g->d_neighbors, 4 * n_nb, cudaMemcpyDeviceToHost));
    memset(out + pos, 0, pad);
    QB_CUDA(cudaMemcpy(out + pos + pad, g->d_offsets, 8 * n_off, cudaMemcpyDeviceToHost));
    return QB_OK;
}
