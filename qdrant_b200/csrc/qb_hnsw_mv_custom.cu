// qb_hnsw_mv_custom.cu — custom queries (recommend / discover / context / feedback) whose examples are multivectors, through the device
// traversal of a graph over multivector points (qb_hnsw_search_maxsim_custom_batch / _discover_batch).  The search kernel's body with
// MaxSim scores per example folded by Query::score_by (HC_MAXSIM_CUSTOM, HnswMvCustomParams); qb_hnsw_launch (qb_hnsw.cu) fills the
// parameters.  Its kernels live in their own object so that the machine code of qb_hnsw.o stays as it was.
#include "qb_hnsw_traverse.cuh"

namespace {

template <int KIND, int METRIC, int ALGO>
__global__ void __launch_bounds__(128) hnsw_mv_custom_kernel(const HnswMvCustomParams p) {
    constexpr int NT = 128, CUSTOM = HC_MAXSIM_CUSTOM;
#include "qb_hnsw_search_body.cuh"
}

// per_sm != null: the kernel's resident CTAs per SM at smem bytes of dynamic shared memory; else the launch
template <int KIND, int METRIC, int ALGO>
qb_status mvc_run(const HnswMvCustomParams& p, unsigned grid, size_t smem, cudaStream_t stream, int* per_sm) {
    QB_CUDA(cudaFuncSetAttribute(hnsw_mv_custom_kernel<KIND, METRIC, ALGO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (per_sm) {
        QB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, hnsw_mv_custom_kernel<KIND, METRIC, ALGO>, 128, smem));
        if (*per_sm < 1) *per_sm = 1;
        return QB_OK;
    }
    hnsw_mv_custom_kernel<KIND, METRIC, ALGO><<<grid, 128, smem, stream>>>(p);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

template <int ALGO>
qb_status mvc_dispatch(int kind, int metric, const HnswMvCustomParams& p, unsigned grid, size_t smem, cudaStream_t stream, int* per_sm) {
#define QB_MVC(K) (metric == M_EUCLID ? mvc_run<K, M_EUCLID, ALGO>(p, grid, smem, stream, per_sm)            \
                   : metric == M_MANHATTAN ? mvc_run<K, M_MANHATTAN, ALGO>(p, grid, smem, stream, per_sm) \
                                           : mvc_run<K, M_DOT, ALGO>(p, grid, smem, stream, per_sm))
    switch (kind) {
        case HK_DENSE_AVX: return QB_MVC(HK_DENSE_AVX);
        case HK_DENSE_SMALL: return QB_MVC(HK_DENSE_SMALL);
        case HK_SQ8: return mvc_run<HK_SQ8, M_DOT, ALGO>(p, grid, smem, stream, per_sm);
        case HK_SQ8_LANEX: return mvc_run<HK_SQ8_LANEX, M_DOT, ALGO>(p, grid, smem, stream, per_sm);
        default:
            qb_set_error("hnsw_search_maxsim_custom: dense f32 and SQ8 token storages only");
            return QB_ERR_UNSUPPORTED;
    }
#undef QB_MVC
}

}  // namespace

qb_status qb_hnsw_mv_custom_launch(const void* params, const uint32_t* d_tok, const uint32_t* d_ex_off, int kind, int metric, int algo, unsigned grid,
                                   size_t smem, cudaStream_t stream, int* per_sm) {
    HnswMvCustomParams p{};
    static_cast<HnswParams&>(p) = *static_cast<const HnswParams*>(params);
    p.tok = d_tok;
    p.ex_off = d_ex_off;
    return algo == ALGO_ACORN ? mvc_dispatch<ALGO_ACORN>(kind, metric, p, grid, smem, stream, per_sm)
                              : mvc_dispatch<ALGO_HNSW>(kind, metric, p, grid, smem, stream, per_sm);
}
