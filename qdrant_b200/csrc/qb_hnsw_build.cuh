// qb_hnsw_build.cuh — the host side of a device graph build, shared by qb_hnsw_build (qb_hnsw_build.cu) and qb_hnsw_build_multivector
// (qb_hnsw_build_mv.cu): the schedule (hb_plan), the level loop (hb_levels) and the finish into a plain-format handle (hb_run).  The
// inserts and backlinks are the kernels K of the caller: K::Params, K::insert, K::backlinks, K::prepare.  The schedule is described
// in qb_hnsw_build.cu's header.
#pragma once
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <functional>
#include <memory>
#include <vector>

#include "qb_hnsw_host.cuh"

namespace {

constexpr int HB_THREADS = 128;       // insert kernel: threads per CTA (one point per CTA at a time)
constexpr int HB_WARPS = 4;           // backlink kernel: warps per CTA (one target per warp at a time)
constexpr uint32_t HB_MAX_LEVEL = 30; // the highest level a point may have (levels are u8; 30 keeps the per-level tables small)

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

// the host-side schedule
struct HbPlan {
    std::vector<uint32_t> rest;                       // inserted points after the entry, in the sorted order
    std::vector<std::pair<uint32_t, uint32_t>> batches;   // [begin, end) in rest
    std::vector<uint8_t> level_of_rest;
    std::vector<uint32_t> pos;                        // each point's position in the sorted order (its row on the levels >= 1)
    std::vector<uint64_t> rows_on;                    // N_l: points whose level is >= l = the first N_l of the order
    uint32_t entry = HNSW_EMPTY, entry_level = 0, levels = 1, max_batch = 1;
    // an incremental build whose first new point is above the graph's top level (link_new_point, graph_layers_builder.rs:417-475):
    // rest[0] links on the levels <= entry_level from `entry`, then it is the entry of every later point, from its own level
    bool lead = false;
};

// the schedule of n points with these levels; deleted: 32-bit words, bit = 1: not inserted (null: none).  An incremental build passes
// the points its graph already holds as `given` (same layout; they are not inserted either) and that graph's entry; rest is then every
// other point, the first serial_points of them one at a time.  Without a given entry the first point of the order is the entry and the
// first serial_points - 1 after it go one at a time.
qb_status hb_plan(const uint8_t* levels, uint32_t n, const uint32_t* deleted, uint32_t batch, uint32_t serial_points, const char* who, HbPlan* out,
                  const uint32_t* given = nullptr, uint32_t entry = HNSW_EMPTY) {
    HbPlan& plan = *out;
    uint32_t top_level = 0;
    for (uint32_t i = 0; i < n; ++i) {
        QB_CHECK(levels[i] <= HB_MAX_LEVEL, QB_ERR_INVALID, "%s: levels[%u] = %u > %u", who, i, (unsigned)levels[i], HB_MAX_LEVEL);
        top_level = std::max<uint32_t>(top_level, levels[i]);
    }
    const uint32_t L = plan.levels = top_level + 1;
    std::vector<uint64_t> per_level(L + 1, 0), start(L + 1, 0);
    for (uint32_t i = 0; i < n; ++i) per_level[levels[i]]++;
    for (int l = (int)L - 2; l >= 0; --l) start[l] = start[l + 1] + per_level[l + 1];   // level desc, then id (a stable counting sort)
    std::vector<uint32_t> order(n);
    plan.pos.resize(n);
    for (uint32_t i = 0; i < n; ++i) { plan.pos[i] = (uint32_t)start[levels[i]]++; order[plan.pos[i]] = i; }
    plan.rows_on.resize(L);
    for (uint32_t l = 0; l < L; ++l) { uint64_t c = 0; for (uint32_t k = l; k < L; ++k) c += per_level[k]; plan.rows_on[l] = c; }
    plan.entry = entry;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t id = order[i];
        if (deleted && ((deleted[id >> 5] >> (id & 31)) & 1u)) continue;   // iter_internal_excluding(deleted)
        if (given && ((given[id >> 5] >> (id & 31)) & 1u)) continue;
        if (plan.entry == HNSW_EMPTY) plan.entry = id;
        else plan.rest.push_back(id);
    }
    QB_CHECK(plan.entry != HNSW_EMPTY, QB_ERR_INVALID, "%s: every point is deleted", who);
    plan.entry_level = levels[plan.entry];
    const uint32_t nr = (uint32_t)plan.rest.size();
    plan.level_of_rest.resize(nr);
    for (uint32_t i = 0; i < nr; ++i) plan.level_of_rest[i] = levels[plan.rest[i]];
    plan.lead = entry != HNSW_EMPTY && nr && plan.level_of_rest[0] > plan.entry_level;
    uint32_t k = 0;
    for (; k < std::min(entry != HNSW_EMPTY ? serial_points : serial_points - 1, nr); ++k) plan.batches.push_back({k, k + 1});
    while (k < nr) {   // build_initial_batches: chunks of `batch` from the first point after the entry, cut where the level changes
        uint32_t e = (uint32_t)std::min<uint64_t>((uint64_t)(k / batch + 1) * batch, nr);
        for (uint32_t j = k + 1; j < e; ++j) if (plan.level_of_rest[j] != plan.level_of_rest[k]) { e = j; break; }
        plan.batches.push_back({k, e});
        plan.max_batch = std::max(plan.max_batch, e - k);
        k = e;
    }
    return QB_OK;
}

template <class K>
qb_status hb_levels(typename K::Params p, const HbPlan& plan, uint32_t m, uint32_t m0, uint32_t* const* tables, const uint32_t* d_remap, uint32_t* d_pts,
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
            QB_TRY(K::insert(p, std::min<unsigned>(np, max_grid), smem));
            size_t bytes = sort_bytes;
            QB_CUDA(cub::DeviceRadixSort::SortPairs(d_sort, bytes, d_tkey, d_tkey2, d_tval, d_tval2, (int)(np * lm), 0, key_bits));
            QB_LAUNCHED();
            QB_TRY(K::backlinks(p, d_tkey2, d_tval2, np * lm));
        }
        if (l == 0) break;
        // the points below l: greedy descent on l, one launch (they follow every insert at l)
        const uint32_t g0 = (uint32_t)(std::find_if(plan.level_of_rest.begin(), plan.level_of_rest.end(), [&](uint8_t v) { return v < (uint32_t)l; }) -
                                       plan.level_of_rest.begin());
        if (g0 < nr) {
            p.b_pts = d_pts + g0; p.b_entry = d_entry + g0; p.nq = nr - g0; p.b_insert = 0;
            QB_CUDA(cudaMemsetAsync(p.work, 0, 4));
            QB_TRY(K::insert(p, std::min<unsigned>(nr - g0, max_grid), smem));
        }
    }
    return QB_OK;
}

// fills the build tables of an incremental build before its inserts: tables[l] as hb_run lays them out, d_remap = the plan's pos
using HbPrefill = std::function<qb_status(uint32_t* const* tables, const uint32_t* d_remap)>;

// the build of `plan` with the kernels K, then the handle as qb_hnsw_create_plain makes it from the plain arrays.  p: the storage and
// query fields (and K's own); smem: the insert kernel's shared memory; prefill: the rows the graph already has (null: none).
template <class K>
qb_status hb_run(qb_storage* s, typename K::Params p, const HbPlan& plan, uint32_t n, uint32_t m, uint32_t m0, size_t smem, const char* who, qb_hnsw** out,
                 const HbPrefill& prefill = nullptr) {
    const uint32_t L = plan.levels, nr = (uint32_t)plan.rest.size();
    HnswScratch tmp;
    std::vector<uint32_t*> tables(L, nullptr);
    for (uint32_t l = 0; l < L; ++l) {
        const size_t bytes = (size_t)plan.rows_on[l] * (l ? m : m0) * 4;
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
    QB_CUDA(cudaMemcpy(d_remap, plan.pos.data(), 4ull * n, cudaMemcpyHostToDevice));
    if (nr) QB_CUDA(cudaMemcpy(d_pts, plan.rest.data(), 4ull * nr, cudaMemcpyHostToDevice));
    {
        std::vector<uint32_t> ent(nr, plan.lead ? plan.rest[0] : plan.entry);   // PointLinkingData::entry starts at the first point
        if (plan.lead) ent[0] = plan.entry;
        if (nr) QB_CUDA(cudaMemcpy(d_entry, ent.data(), 4ull * nr, cudaMemcpyHostToDevice));
    }
    const int key_bits = 64;   // target << 32 | position; an empty slot (~0) sorts last
    size_t sort_bytes = 0;
    QB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, d_tkey, d_tkey2, d_tval, d_tval2, (int)trip, 0, (int)key_bits));
    void* d_sort = nullptr;
    QB_CUDA(tmp.alloc(&d_sort, sort_bytes));

    p.n_points = n; p.levels = L;
    p.prefetch = qb_opt().hnsw_no_prefetch ? 0 : 1;
    p.work = d_work;
    // grid: the resident CTAs, at most one per point of the largest launch; per-CTA visited bitmaps (the kernel leaves them clean) and logs
    int per_sm = 1;
    QB_TRY(K::prepare(p, smem, &per_sm));
    const unsigned grid = std::min<unsigned>((unsigned)s->sm_count * (unsigned)per_sm, std::max<uint32_t>(1, std::max(plan.max_batch, nr)));
    const uint64_t words = ceil_div_u64(n, 32);
    p.visited_words = words; p.vlog_cap = 32768;
    QB_CUDA(tmp.alloc((void**)&p.visited, (size_t)grid * words * 4));
    QB_CUDA(tmp.alloc((void**)&p.vlog, (size_t)grid * p.vlog_cap * 4));
    QB_CUDA(cudaMemset(p.visited, 0, (size_t)grid * words * 4));
    if (prefill) QB_TRY(prefill(tables.data(), d_remap));
    if (plan.lead) {   // rest[0] on the levels <= entry_level, then the others from it
        HbPlan one, others;
        one.rest = {plan.rest[0]}; one.batches = {{0, 1}}; one.level_of_rest = {plan.level_of_rest[0]}; one.entry_level = plan.entry_level;
        others.rest = plan.rest; others.level_of_rest = plan.level_of_rest; others.entry_level = plan.level_of_rest[0];
        others.batches.assign(plan.batches.begin() + 1, plan.batches.end());
        QB_TRY(hb_levels<K>(p, one, m, m0, tables.data(), d_remap, d_pts, d_entry, d_tkey, d_tval, d_tkey2, d_tval2, d_sort, sort_bytes, grid, smem, key_bits));
        QB_TRY(hb_levels<K>(p, others, m, m0, tables.data(), d_remap, d_pts, d_entry, d_tkey, d_tval, d_tkey2, d_tval2, d_sort, sort_bytes, grid, smem, key_bits));
    } else {
        QB_TRY(hb_levels<K>(p, plan, m, m0, tables.data(), d_remap, d_pts, d_entry, d_tkey, d_tval, d_tkey2, d_tval2, d_sort, sort_bytes, grid, smem, key_bits));
    }

    // ---- finish: the plain arrays (level offsets, reindex, neighbours, offsets), then the handle as qb_hnsw_create_plain makes it
    HbTables tb{};
    tb.levels = L; tb.m = m; tb.m0 = m0;
    std::vector<uint64_t> lo(L + 1, 0);
    for (uint32_t l = 0; l < L; ++l) { tb.t[l] = tables[l]; lo[l + 1] = lo[l] + plan.rows_on[l]; }
    for (uint32_t l = 0; l <= L; ++l) tb.lo[l] = lo[l];
    const uint64_t rows = lo[L], n_off = rows + 1;
    uint64_t* d_counts = nullptr;
    QB_CUDA(tmp.alloc((void**)&d_counts, 8 * n_off));
    hnsw_build_counts_kernel<<<hnsw_grid(n_off, 256, 132 * 16), 256>>>(tb, d_counts);
    QB_LAUNCHED();
    qb_hnsw* g = nullptr;
    QB_TRY(qb_hnsw_new(s, n, m, m0, std::move(lo), n_off, 0, who, &g));
    std::unique_ptr<qb_hnsw, decltype(&qb_hnsw_destroy)> guard(g, qb_hnsw_destroy);
    cudaError_t ce = cudaMemcpy(g->d_level_offsets, g->level_offsets_ext.data(), 8 * L, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(g->d_reindex, d_remap, 4ull * n, cudaMemcpyDeviceToDevice);
    if (ce != cudaSuccess) { qb_set_error("%s: build: %s", who, cudaGetErrorString(ce)); return QB_ERR_CUDA; }
    QB_TRY(hnsw_link_offsets(g, d_counts, n_off, tmp, who, "build", nullptr, nullptr, [&](const uint64_t* d_offsets, uint32_t* d_neighbors) {
        hnsw_build_neighbors_kernel<<<hnsw_grid(rows, 256, 132 * 16), 256>>>(tb, d_offsets, d_neighbors);
        QB_LAUNCHED();
    }));
    ce = cudaGetLastError();
    if (ce != cudaSuccess) { qb_set_error("%s: build: %s", who, cudaGetErrorString(ce)); return QB_ERR_CUDA; }
    QB_TRY(qb_hnsw_finish_plain(g, who));
    *out = guard.release();
    return QB_OK;
}

}  // namespace

// qb_hnsw_build's plan and inserts over a dense f32 or Uint8 storage (qb_hnsw_build.cu), with hb_plan's `given` points and entry and hb_run's
// prefill: qb_hnsw_build passes none, qb_hnsw_build_incremental (qb_hnsw_heal.cu) the healed graph.  Checks nothing the callers check.
qb_status qb_hnsw_build_dense(qb_storage* s, uint32_t m, uint32_t m0, uint32_t ef, const uint8_t* levels, const uint32_t* given, uint32_t entry, uint32_t batch,
                              uint32_t serial_points, const HbPrefill& prefill, const char* who, qb_hnsw** out, uint32_t* entry_point, uint32_t* entry_level);
