// qb_hnsw_build.cu — HNSW graph construction on the device for dense f32 and Uint8 storages (qb_hnsw_build), and the plain `links.bin` export.
// A Uint8 storage's inserts and backlinks are the same kernels instantiated for the u8 kinds (HK_U8, HK_U8_SMALL; DESIGN §3.13d).
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
// The host side (the plan, the level loop, the finish) is in qb_hnsw_build.cuh, shared with the multivector build (qb_hnsw_build_mv.cu).
#include "qb_hnsw_build.cuh"

namespace {

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

template <int KIND, int METRIC>
struct HbKernels {
    using Params = HnswParams;
    static qb_status insert(const HnswParams& p, unsigned grid, size_t smem) {
        hnsw_search_kernel<KIND, METRIC, HB_THREADS, ALGO_BUILD, 0><<<grid, HB_THREADS, smem>>>(p);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
    static qb_status backlinks(const HnswParams& p, const unsigned long long* keys, const uint32_t* vals, uint32_t n) {
        hnsw_backlink_kernel<KIND, METRIC><<<hnsw_grid(n, HB_WARPS, 132 * 16), HB_WARPS * 32>>>(p, keys, vals, n);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
    static qb_status prepare(const HnswParams&, size_t smem, int* per_sm) {
        QB_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<KIND, METRIC, HB_THREADS, ALGO_BUILD, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        QB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, hnsw_search_kernel<KIND, METRIC, HB_THREADS, ALGO_BUILD, 0>, HB_THREADS, smem));
        if (*per_sm < 1) *per_sm = 1;
        return QB_OK;
    }
};

// hb_run over a Uint8 storage, with its four metrics
template <int KIND>
qb_status hb_run_u8(int metric, qb_storage* s, const HnswParams& p, const HbPlan& plan, uint32_t n, uint32_t m, uint32_t m0, size_t smem, const char* who,
                    qb_hnsw** out, const HbPrefill& prefill) {
    switch (metric) {
        case M_EUCLID: return hb_run<HbKernels<KIND, M_EUCLID>>(s, p, plan, n, m, m0, smem, who, out, prefill);
        case M_MANHATTAN: return hb_run<HbKernels<KIND, M_MANHATTAN>>(s, p, plan, n, m, m0, smem, who, out, prefill);
        case M_COSINE: return hb_run<HbKernels<KIND, M_COSINE>>(s, p, plan, n, m, m0, smem, who, out, prefill);
        default: return hb_run<HbKernels<KIND, M_DOT>>(s, p, plan, n, m, m0, smem, who, out, prefill);
    }
}

}  // namespace

extern "C" qb_status qb_hnsw_build(qb_storage* s, uint32_t m, uint32_t m0, uint32_t ef_construct, const uint8_t* levels, uint32_t batch, uint32_t serial_points,
                                   qb_hnsw** out, uint32_t* entry_point, uint32_t* entry_level) {
    QB_CHECK(s && levels && out, QB_ERR_INVALID, "hnsw_build: null argument");
    *out = nullptr;
    QB_CHECK(s->kind == QB_KIND_DENSE && (s->dtype == QB_DT_F32 || s->dtype == QB_DT_U8), QB_ERR_UNSUPPORTED,
             "hnsw_build: graphs are built over dense f32 and Uint8 storages only (build over the original vectors, then bind the graph to the quantized "
             "storage)");
    QB_CHECK(s->count >= 1, QB_ERR_INVALID, "hnsw_build: empty storage");
    QB_CHECK(s->count < 0xFFFFFFFFull, QB_ERR_UNSUPPORTED, "hnsw_build: %llu points", (unsigned long long)s->count);
    QB_CHECK(m >= 1 && m0 >= 1, QB_ERR_INVALID, "hnsw_build: m %u / m0 %u", m, m0);
    QB_CHECK(m <= HNSW_MAX_LINKS && m0 <= HNSW_MAX_LINKS, QB_ERR_UNSUPPORTED, "hnsw_build: m %u / m0 %u outside [1,%u]", m, m0, HNSW_MAX_LINKS);
    const uint32_t ef = std::max(ef_construct, m0);   // gpu_graph_builder.rs:38
    QB_CHECK(ef <= HNSW_MAX_EF, QB_ERR_UNSUPPORTED, "hnsw_build: ef %u > %u", ef, HNSW_MAX_EF);
    return qb_hnsw_build_dense(s, m, m0, ef, levels, nullptr, HNSW_EMPTY, batch, serial_points, nullptr, "hnsw_build", out, entry_point, entry_level);
}

qb_status qb_hnsw_build_dense(qb_storage* s, uint32_t m, uint32_t m0, uint32_t ef, const uint8_t* levels, const uint32_t* given, uint32_t entry, uint32_t batch,
                              uint32_t serial_points, const HbPrefill& prefill, const char* who, qb_hnsw** out, uint32_t* entry_point, uint32_t* entry_level) {
    const uint32_t n = (uint32_t)s->count;
    if (batch == 0) batch = 512;               // GPU_GROUPS_COUNT_DEFAULT, gpu/mod.rs:34
    if (serial_points == 0) serial_points = 256;   // SINGLE_THREADED_HNSW_BUILD_THRESHOLD
    QB_CUDA(cudaSetDevice(s->device));

    std::vector<uint32_t> deleted;
    if (s->d_deleted) {
        deleted.resize(ceil_div_u64(n, 32));
        QB_CUDA(cudaMemcpy(deleted.data(), s->d_deleted, 4 * deleted.size(), cudaMemcpyDeviceToHost));
    }
    HbPlan plan;
    QB_TRY(hb_plan(levels, n, deleted.empty() ? nullptr : deleted.data(), batch, serial_points, who, &plan, given, entry));

    const bool u8 = s->dtype == QB_DT_U8;
    const int kind = s->dim >= 32 ? (u8 ? HK_U8 : HK_DENSE_AVX) : (u8 ? HK_U8_SMALL : HK_DENSE_SMALL);
    const int metric = hnsw_metric(s);
    HnswParams p{};
    p.rows = reinterpret_cast<const uint8_t*>(s->d_rows); p.stride = s->row_stride; p.dim = s->dim;
    p.q_bytes = s->row_stride; p.ef = ef;
    const size_t smem = hnsw_smem_bytes(p.q_bytes, ef);
    QB_CHECK(smem <= 200 * 1024, QB_ERR_UNSUPPORTED, "%s: a row (%u B) + ef %u need %zu B of shared memory", who, p.q_bytes, ef, smem);
#define QB_HB_RUN(K, M) hb_run<HbKernels<K, M>>(s, p, plan, n, m, m0, smem, who, out, prefill)
    if (kind == HK_DENSE_AVX) QB_TRY(metric == M_EUCLID ? QB_HB_RUN(HK_DENSE_AVX, M_EUCLID) : metric == M_MANHATTAN ? QB_HB_RUN(HK_DENSE_AVX, M_MANHATTAN) : QB_HB_RUN(HK_DENSE_AVX, M_DOT));
    else if (kind == HK_DENSE_SMALL) QB_TRY(metric == M_EUCLID ? QB_HB_RUN(HK_DENSE_SMALL, M_EUCLID) : metric == M_MANHATTAN ? QB_HB_RUN(HK_DENSE_SMALL, M_MANHATTAN) : QB_HB_RUN(HK_DENSE_SMALL, M_DOT));
    else if (kind == HK_U8) QB_TRY(hb_run_u8<HK_U8>(metric, s, p, plan, n, m, m0, smem, who, out, prefill));
    else QB_TRY(hb_run_u8<HK_U8_SMALL>(metric, s, p, plan, n, m, m0, smem, who, out, prefill));
#undef QB_HB_RUN
    const uint32_t e = plan.lead ? plan.rest[0] : plan.entry;   // entry_points.rs new_point: a new point strictly above the top
    if (entry_point) *entry_point = e;
    if (entry_level) *entry_level = levels[e];
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
