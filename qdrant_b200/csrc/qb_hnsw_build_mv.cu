// qb_hnsw_build_mv.cu — the graph of a multivector collection's POINTS built on the device (qb_hnsw_build_multivector): qb_hnsw_build's
// schedule (qb_hnsw_build.cuh) with MaxSim scores.  Its kernels live in their own object so that the machine code of qb_hnsw_build.o
// stays as it was.
#include <memory>

#include "qb_hnsw_build.cuh"

namespace {
// the inserts of a multivector build: the search kernel's body with MaxSim scores (ALGO_BUILD, HC_MAXSIM) and the token offsets in
// HnswMvBuildParams; the inserted point's token rows are the query
template <int KIND, int METRIC>
__global__ void __launch_bounds__(HB_THREADS, 1) hnsw_build_mv_kernel(const HnswMvBuildParams p) {
    constexpr int NT = HB_THREADS, ALGO = ALGO_BUILD, CUSTOM = HC_MAXSIM;
#include "qb_hnsw_search_body.cuh"
}

// hnsw_backlink_kernel's connect_with_heuristic with MaxSim scores: a full list is re-scored with the target's token rows as the query,
// and each candidate of the heuristic with its own token rows as the query against the kept links.  A list of m0 + 1 MaxSim scores is
// too much work for a warp, so one CTA takes a target and scores the list with maxsim_list's item-parallel layout.
template <int KIND, int METRIC>
__global__ void __launch_bounds__(HB_THREADS, 1) hnsw_backlink_mv_kernel(const HnswMvBuildParams p, const unsigned long long* __restrict__ keys,
                                                                      const uint32_t* __restrict__ vals, uint32_t n) {
    extern __shared__ __align__(16) uint8_t smem_raw[];   // the staged query, p.q_smem bytes
    __shared__ unsigned long long s_key[HNSW_MAX_LINKS + 1], s_sorted[HNSW_MAX_LINKS + 1];
    __shared__ uint32_t s_ids[HNSW_MAX_LINKS + 1];
    __shared__ float s_sc[HNSW_MAX_LINKS + 1];
    const uint32_t tid = threadIdx.x, lm = p.m0;
    HnswSmem sm{};
    sm.ids = s_ids; sm.sc = s_sc;
    for (uint32_t e = blockIdx.x; e < n; e += gridDim.x) {
        const uint32_t t = (uint32_t)(keys[e] >> 32);
        if (t == HNSW_EMPTY) break;                                      // the empty slots sort last
        if (e > 0 && (uint32_t)(keys[e - 1] >> 32) == t) continue;       // not the target's first pair
        uint32_t* row = const_cast<uint32_t*>(p.links0) + (size_t)hnsw_build_row(p, t) * lm;
        for (uint32_t e2 = e; e2 < n && (uint32_t)(keys[e2] >> 32) == t; ++e2) {
            const uint32_t src = vals[e2];
            const uint32_t cnt = (uint32_t)__syncthreads_count(tid < lm && row[tid] != HNSW_EMPTY);
            if (cnt < lm) {
                if (tid == 0) row[cnt] = src;
                __syncthreads();
                continue;
            }
            if (tid < lm) s_ids[tid] = row[tid];
            if (tid == 0) s_ids[lm] = src;
            mv_stage_rows<HB_THREADS>(p, sm, smem_raw, p.tok[t], p.tok[t + 1]);
            __syncthreads();
            maxsim_list<KIND, METRIC, HB_THREADS>(p, sm, lm + 1);
            if (tid <= lm) s_key[tid] = qb_pack_key(s_sc[tid], s_ids[tid]);
            __syncthreads();
            if (tid <= lm) {   // rank sort of distinct keys, descending
                const unsigned long long k = s_key[tid];
                uint32_t r = 0;
                for (uint32_t i = 0; i <= lm; ++i) r += s_key[i] > k ? 1u : 0u;
                s_sorted[r] = k;
            }
            __syncthreads();
            // fill_from_sorted_with_heuristic: the kept links go to s_ids[0 .. nsel)
            uint32_t nsel = 0;
            for (uint32_t c = 0; c <= lm && nsel < lm; ++c) {
                const uint32_t cid = qb_key_id(s_sorted[c]);
                const float cs = qb_key_score(s_sorted[c]);
                bool beat = false;
                if (nsel) {
                    mv_stage_rows<HB_THREADS>(p, sm, smem_raw, p.tok[cid], p.tok[cid + 1]);
                    __syncthreads();
                    maxsim_list<KIND, METRIC, HB_THREADS>(p, sm, nsel);
                    beat = __syncthreads_or(tid < nsel && s_sc[tid] > cs) != 0;
                }
                if (!beat) {
                    if (tid == 0) s_ids[nsel] = cid;
                    ++nsel;
                }
                __syncthreads();
            }
            if (tid < lm) row[tid] = tid < nsel ? s_ids[tid] : HNSW_EMPTY;
            __syncthreads();
        }
    }
}

// the same for a multivector build: MaxSim inserts and backlinks, both staging a query of p.q_smem bytes
template <int KIND, int METRIC>
struct HbMvKernels {
    using Params = HnswMvBuildParams;
    static qb_status insert(const HnswMvBuildParams& p, unsigned grid, size_t smem) {
        hnsw_build_mv_kernel<KIND, METRIC><<<grid, HB_THREADS, smem>>>(p);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
    static qb_status backlinks(const HnswMvBuildParams& p, const unsigned long long* keys, const uint32_t* vals, uint32_t n) {
        hnsw_backlink_mv_kernel<KIND, METRIC><<<hnsw_grid(n, 1, 132 * 16), HB_THREADS, p.q_smem>>>(p, keys, vals, n);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
    static qb_status prepare(const HnswMvBuildParams& p, size_t smem, int* per_sm) {
        QB_CUDA(cudaFuncSetAttribute(hnsw_backlink_mv_kernel<KIND, METRIC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.q_smem));
        QB_CUDA(cudaFuncSetAttribute(hnsw_build_mv_kernel<KIND, METRIC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        QB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, hnsw_build_mv_kernel<KIND, METRIC>, HB_THREADS, smem));
        if (*per_sm < 1) *per_sm = 1;
        return QB_OK;
    }
};

}  // namespace

// The graph of a multivector collection's POINTS, built with qb_hnsw_build's schedule; every score is MaxSim between two stored points
// (MultiMetricQueryScorer::score_internal, multi_metric_query_scorer.rs:64-121), the first point's token rows being the query.
extern "C" qb_status qb_hnsw_build_multivector(qb_storage* tokens, const uint32_t* point_offsets, uint32_t n_points, uint32_t m, uint32_t m0,
                                               uint32_t ef_construct, const uint8_t* levels, const uint64_t* deleted_points, uint32_t batch,
                                               uint32_t serial_points, qb_hnsw** out, uint32_t* entry_point, uint32_t* entry_level) {
    const char* who = "hnsw_build_multivector";
    QB_CHECK(tokens && point_offsets && levels && out, QB_ERR_INVALID, "%s: null argument", who);
    *out = nullptr;
    QB_CHECK(tokens->kind == QB_KIND_DENSE && tokens->dtype == QB_DT_F32, QB_ERR_UNSUPPORTED,
             "%s: graphs are built over dense f32 token storages only (build over the original vectors, then bind the graph to the quantized storage)", who);
    QB_CHECK(n_points >= 1, QB_ERR_INVALID, "%s: no points", who);
    QB_TRY(qb_hnsw_mv_check(tokens, point_offsets, n_points, who));
    QB_CHECK(m >= 1 && m0 >= 1, QB_ERR_INVALID, "%s: m %u / m0 %u", who, m, m0);
    QB_CHECK(m <= HNSW_MAX_LINKS && m0 <= HNSW_MAX_LINKS, QB_ERR_UNSUPPORTED, "%s: m %u / m0 %u outside [1,%u]", who, m, m0, HNSW_MAX_LINKS);
    const uint32_t ef = std::max(ef_construct, m0);   // gpu_graph_builder.rs:38
    QB_CHECK(ef <= HNSW_MAX_EF, QB_ERR_UNSUPPORTED, "%s: ef %u > %u", who, ef, HNSW_MAX_EF);
    if (batch == 0) batch = 512;
    if (serial_points == 0) serial_points = 256;
    QB_CUDA(cudaSetDevice(tokens->device));
    // a bitmap over points; read as 32-bit words (little-endian), as the plan takes it.  The token storage's resident flags are per row.
    HbPlan plan;
    QB_TRY(hb_plan(levels, n_points, reinterpret_cast<const uint32_t*>(deleted_points), batch, serial_points, who, &plan));

    HnswMvBuildParams p{};
    p.rows = reinterpret_cast<const uint8_t*>(tokens->d_rows); p.stride = tokens->row_stride; p.dim = tokens->dim;
    p.q_bytes = tokens->row_stride; p.ef = ef;
    // a query (an inserted point or a heuristic candidate) is staged in shared memory when its rows fit in HNSW_CUSTOM_SMEM
    uint32_t max_run = 0;
    for (uint32_t i = 0; i < n_points; ++i) max_run = std::max(max_run, point_offsets[i + 1] - point_offsets[i]);
    p.q_smem = std::min(max_run, HNSW_CUSTOM_SMEM / p.stride) * p.stride;
    const size_t smem = hnsw_smem_bytes(p.q_smem, ef);
    QB_CHECK(smem <= 200 * 1024, QB_ERR_UNSUPPORTED, "%s: a query (%u B) + ef %u need %zu B of shared memory", who, p.q_smem, ef, smem);
    // the token offsets, kept by the handle (d_mv_tok) once the build succeeds
    uint32_t* d_tok = nullptr;
    QB_TRY(qb_hnsw_mv_upload(point_offsets, n_points, who, &d_tok));
    std::unique_ptr<uint32_t, decltype(&cudaFree)> tok_guard(d_tok, cudaFree);
    p.tok = d_tok;

    const int kind = tokens->dim >= 32 ? HK_DENSE_AVX : HK_DENSE_SMALL;
    const int metric = hnsw_metric(tokens);
    qb_hnsw* g = nullptr;
#define QB_HB_RUN(K, M) hb_run<HbMvKernels<K, M>>(tokens, p, plan, n_points, m, m0, smem, who, &g)
    if (kind == HK_DENSE_AVX) QB_TRY(metric == M_EUCLID ? QB_HB_RUN(HK_DENSE_AVX, M_EUCLID) : metric == M_MANHATTAN ? QB_HB_RUN(HK_DENSE_AVX, M_MANHATTAN) : QB_HB_RUN(HK_DENSE_AVX, M_DOT));
    else QB_TRY(metric == M_EUCLID ? QB_HB_RUN(HK_DENSE_SMALL, M_EUCLID) : metric == M_MANHATTAN ? QB_HB_RUN(HK_DENSE_SMALL, M_MANHATTAN) : QB_HB_RUN(HK_DENSE_SMALL, M_DOT));
#undef QB_HB_RUN
    qb_hnsw_mv_attach(g, tok_guard.release(), n_points);
    *out = g;
    if (entry_point) *entry_point = plan.entry;
    if (entry_level) *entry_level = plan.entry_level;
    return QB_OK;
}

