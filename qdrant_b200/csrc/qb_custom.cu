// qb_custom.cu — the custom-query combinators (recommend / discover / context) on top of the per-example similarities.
//
// In the reference a custom query is a set of example vectors plus `Query::score_by(similarity)`: the scorer evaluates the
// ordinary similarity of the stored vector against EVERY example and folds the results
// (vector_storage/query_scorer/custom_query_scorer.rs:78-122, quantized/quantized_custom_query_scorer.rs).  Here the E
// similarities of a candidate come from the same kernels as plain queries (one launch per example, each bit-exact), and
// this file is the fold: one thread per candidate, f32 operations in the reference's order.
//   RecoBestScore  query/reco_query.rs:64-90     max over positives / negatives (total_cmp), scaled_fast_sigmoid of the winner
//   RecoSumScores  query/reco_query.rs:116-133   sequential f32 sums, positives minus negatives
//   Discover       query/discover_query.rs:16-76 rank = sum of total_cmp(positive, negative) per pair, + sigmoid(target)
//   Context        query/context_query.rs:52-62,111-119   sum over pairs of fast_sigmoid(min(p - n - EPSILON, 0))
//   Feedback       query/feedback_query.rs:204-226 a * sim(target) + sum over pairs of partial_computation * (sim(pos) - sim(neg))
//   MaxSim         query_scorer/mod.rs:77-98     multivectors: sum over query tokens of the best similarity to a point's tokens
// fast_sigmoid = x / (1 + |x|), scaled_fast_sigmoid = 0.5 * (fast_sigmoid(x) + 1)   (lib/common/common/src/math.rs:7-18)
#include "qb_internal.h"
#include "qb_fold.cuh"

namespace {

__global__ void custom_combine_kernel(int kind, uint32_t n_a, uint32_t n_b, const float* __restrict__ coef, const float* __restrict__ sims, uint64_t stride, uint64_t n, float* __restrict__ scores,
                                      const uint32_t* __restrict__ ids, QbEmit emit, int to_keys) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const float sc = qbf::fold(kind, n_a, n_b, coef, [&](uint32_t e) { return sims[(uint64_t)e * stride + i]; });
        if (to_keys) qb_emit(emit, 0, i, ids ? ids[i] : (uint32_t)i, sc);
        else scores[i] = sc;
    }
}

// Multivector MaxSim (score_max_similarity, vector_storage/query_scorer/mod.rs:77-98): a point is a run of consecutive token rows,
// score = sum over query tokens (sequential f32, from 0.0) of the maximum similarity to any of the point's tokens
// (`if sim > max_sim` starting from -inf).  sims: [n_query_tokens][stride] per-row similarities; one thread per point.
__global__ void maxsim_fold_kernel(const float* __restrict__ sims, uint64_t stride, uint32_t n_query_tokens, const uint32_t* __restrict__ row_offsets,
                                   const uint32_t* __restrict__ point_ids, uint64_t n_points, float* __restrict__ scores, QbEmit emit, int to_keys) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_points; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t r0 = row_offsets[i], r1 = row_offsets[i + 1];
        float sum = 0.0f;
        for (uint32_t e = 0; e < n_query_tokens; ++e) {
            const float* col = sims + (uint64_t)e * stride;
            float mx = __int_as_float(0xff800000);
            for (uint32_t r = r0; r < r1; ++r) { const float v = col[r]; if (v > mx) mx = v; }
            sum = __fadd_rn(sum, mx);
        }
        const uint32_t id = point_ids ? point_ids[i] : (uint32_t)i;
        if (to_keys) qb_emit(emit, 0, i, id, sum);
        else scores[i] = sum;
    }
}

__global__ void iota_kernel(uint32_t* p, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = (uint32_t)i;
}

}  // namespace

uint32_t qb_custom_examples(int kind, uint32_t n_a, uint32_t n_b) {
    switch (kind) {
        case QB_QUERY_RECO_BEST_SCORE:
        case QB_QUERY_RECO_SUM_SCORES: return n_a + n_b;
        case QB_QUERY_DISCOVER:
        case QB_QUERY_FEEDBACK_NAIVE: return 1 + 2 * n_a;
        case QB_QUERY_CONTEXT: return 2 * n_a;
        default: return 0;
    }
}

// scores (to_keys = 0) or dense-mode candidate keys for query slot 0 of `emit` (to_keys = 1; ids = null means row i)
qb_status qb_launch_custom_combine(int kind, uint32_t n_a, uint32_t n_b, const float* d_coef, const float* d_sims, uint64_t stride, uint64_t n, float* d_scores, const uint32_t* d_ids,
                                   const QbEmit* emit, cudaStream_t stream) {
    if (n == 0) return QB_OK;
    QbEmit e{};
    if (emit) e = *emit;
    const unsigned grid = (unsigned)std::min<uint64_t>(ceil_div_u64(n, 256), 132ull * 16);
    custom_combine_kernel<<<grid, 256, 0, stream>>>(kind, n_a, n_b, d_coef, d_sims, stride, n, d_scores, d_ids, e, emit ? 1 : 0);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

// row_offsets: n_points + 1 entries indexing the columns of d_sims; scores (emit = null) or dense-mode keys for query slot 0
qb_status qb_launch_maxsim_fold(const float* d_sims, uint64_t stride, uint32_t n_query_tokens, const uint32_t* d_row_offsets, const uint32_t* d_point_ids,
                                uint64_t n_points, float* d_scores, const QbEmit* emit, cudaStream_t stream) {
    if (n_points == 0) return QB_OK;
    QbEmit e{};
    if (emit) e = *emit;
    const unsigned grid = (unsigned)std::min<uint64_t>(ceil_div_u64(n_points, 128), 132ull * 16);
    maxsim_fold_kernel<<<grid, 128, 0, stream>>>(d_sims, stride, n_query_tokens, d_row_offsets, d_point_ids, n_points, d_scores, e, emit ? 1 : 0);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

qb_status qb_launch_iota(uint32_t* d, uint64_t n, cudaStream_t stream) {
    if (n == 0) return QB_OK;
    iota_kernel<<<(unsigned)std::min<uint64_t>(ceil_div_u64(n, 256), 132ull * 16), 256, 0, stream>>>(d, n);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}
