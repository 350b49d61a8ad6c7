/*
 * hnsw_build_mv_ref.c — the CPU restatement of the device graph build over multivector points (qb_hnsw_build_multivector), the
 * checker its graphs are compared with.
 *
 * It is tests/hnsw_build_ref.c — the oracle's link_new_point, search_on_level, heuristics and the serial and batched two-phase
 * schedules — compiled once more with one pair score in place of the oracle's f32 similarity; the oracle's sources are not changed.
 * The oracle's HNSW scores two stored points a, b as qo_similarity_f32(distance, base + a * dim, base + b * dim, dim), and an insert's
 * search scores the internal query base + p * dim against base + id * dim.  A multivector graph is built with dim = 1 over a `base`
 * holding one float per point (its values are not read), so the two addresses name the points, and the score is S(a, b) =
 * qo_maxsim_f32 with point a's token rows as the query against point b's rows (MultiMetricQueryScorer::score_internal,
 * multi_metric_query_scorer.rs:64-121).  qo_mv_bind names the token rows before a build; one build runs at a time.
 */
#define _GNU_SOURCE   /* before any system header, as oracle/hnsw.c needs it */
#include <stddef.h>
#include <stdint.h>

float qo_maxsim_f32(int distance, const float* a, uint32_t na, const float* b, uint32_t nb, uint32_t dim);

static struct {
    const float* base;        /* the graph's base: one float per point */
    const float* tokens;      /* token rows, dim floats each */
    const uint32_t* offsets;  /* point p = rows offsets[p] .. offsets[p + 1) */
    uint32_t dim;
} mv;

static float mv_pair_score(int distance, const float* a, const float* b, size_t n) {
    (void)n;
    const size_t pa = (size_t)(a - mv.base), pb = (size_t)(b - mv.base);
    const uint32_t a0 = mv.offsets[pa], b0 = mv.offsets[pb];
    return qo_maxsim_f32(distance, mv.tokens + (size_t)a0 * mv.dim, mv.offsets[pa + 1] - a0, mv.tokens + (size_t)b0 * mv.dim, mv.offsets[pb + 1] - b0, mv.dim);
}

#define qo_similarity_f32 mv_pair_score
#include "hnsw_build_ref.c"

/* the token rows of the points the next qo_hnsw_build_levels / qo_hnsw_build_batched call (base = `base`, dim = 1) links */
API void qo_mv_bind(const float* base, const float* tokens, const uint32_t* offsets, uint32_t dim) {
    mv.base = base; mv.tokens = tokens; mv.offsets = offsets; mv.dim = dim;
}
