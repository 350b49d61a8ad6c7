/* The checker of qb_mmr_maxsim_batch: maximal marginal relevance over multivector candidates, restated over the oracle's MaxSim
 * (qo_maxsim_f32 / qo_preprocess_f32, passed in as function pointers), one query at a time, single-threaded, the way the reference runs it:
 *   - unique_by(id), first occurrence kept; fewer than two left: returned as they are, nothing scored;
 *   - rel[i] = MaxSim(preprocess(Q), P_i) for every candidate (one MultiMetricQueryScorer over the volatile storage);
 *   - a lazily filled matrix: pair(c, s) = MaxSim(preprocess(P_c), P_s) (candidate c's scorer: c's vectors are the query side), scored
 *     on first use and counted then;
 *   - the remaining candidates as an explicit position array; a pick is swap-removed (the last position moves into its place);
 *   - every max / argmax keeps the LAST maximal element under OrderedFloat (NaN above everything and equal to NaN, -0.0 == +0.0);
 *   - mmr = lambda * rel - (1 - lambda) * maxsim, four separately rounded f32 operations (compiled without contraction).
 * Counters: cpu += dim * 4 per vector pair of each MaxSim (T_a * T_b), as MultiMetricQueryScorer meters them; vector_io_read stays 0. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define API __attribute__((visibility("default")))

typedef struct { uint32_t idx; float score; } scored;
typedef float (*maxsim_fn)(int distance, const float* a, uint32_t na, const float* b, uint32_t nb, uint32_t dim);
typedef void (*pre_fn)(int distance, const float* v, float* out, size_t n);

/* OrderedFloat's Ord: NaN == NaN and above everything; otherwise IEEE order, so -0.0 == +0.0 */
static int ocmp(float a, float b) {
    const int na = a != a, nb = b != b;
    if (na || nb) return na - nb;
    return (a > b) - (a < b);
}

/* one query.  rows: the token storage, dim f32 per row; point p = rows [offsets[p], offsets[p+1]).  query: n_qv raw vectors.
 * cand: n_cand candidates (point ids with token rows).  out: up to max(limit, 1) entries; returns how many.  cpu / io: added to. */
API uint32_t qmm_mmr(maxsim_fn maxsim, pre_fn pre, int distance, const float* rows, const uint32_t* offsets, uint32_t dim, const float* query,
                     uint32_t n_qv, float lambda, const scored* cand, uint32_t n_cand, uint32_t limit, scored* out, uint64_t* cpu, uint64_t* io) {
    (void)io;   /* the volatile storage is never on disk */
    uint32_t* uniq = malloc(sizeof(uint32_t) * (n_cand + 1));
    uint32_t n = 0;
    for (uint32_t i = 0; i < n_cand; i++) {
        int dup = 0;
        for (uint32_t j = 0; j < n && !dup; j++) dup = cand[uniq[j]].idx == cand[i].idx;
        if (!dup) uniq[n++] = i;
    }
    if (n < 2) {
        for (uint32_t k = 0; k < n; k++) out[k] = cand[uniq[k]];
        free(uniq);
        return n;
    }
    const uint64_t units = (uint64_t)dim * 4;
    float* qp = malloc(sizeof(float) * (size_t)n_qv * dim);
    for (uint32_t v = 0; v < n_qv; v++) pre(distance, query + (size_t)v * dim, qp + (size_t)v * dim, dim);   /* MultiMetricQueryScorer::new */
    const float** vec = malloc(sizeof(float*) * n);
    float** vpre = malloc(sizeof(float*) * n);
    uint32_t* nt = malloc(sizeof(uint32_t) * n);
    float* rel = malloc(sizeof(float) * n);
    const uint32_t cap = limit < n ? limit : n;   /* the matrix's columns are the picks, in pick order: pair(c, pick k) at c * cap + k */
    float* mat = malloc(sizeof(float) * (size_t)n * (cap ? cap : 1));
    unsigned char* have = calloc((size_t)n * (cap ? cap : 1), 1);
    uint32_t* pos = malloc(sizeof(uint32_t) * n);
    uint32_t* sel = malloc(sizeof(uint32_t) * n);
    for (uint32_t c = 0; c < n; c++) {
        const uint32_t p = cand[uniq[c]].idx;
        vec[c] = rows + (size_t)offsets[p] * dim;
        nt[c] = offsets[p + 1] - offsets[p];
        rel[c] = maxsim(distance, qp, n_qv, vec[c], nt[c], dim);
        *cpu += units * n_qv * nt[c];
        /* LazyMatrix::new: one scorer per candidate, its vectors preprocessed */
        vpre[c] = malloc(sizeof(float) * ((size_t)nt[c] * dim + 1));
        for (uint32_t t = 0; t < nt[c]; t++) pre(distance, vec[c] + (size_t)t * dim, vpre[c] + (size_t)t * dim, dim);
        pos[c] = c;
    }
    uint32_t len = n, n_sel = 0;
    if (limit > 0) {
        uint32_t best = 0;
        for (uint32_t p = 1; p < len; p++)
            if (ocmp(rel[pos[p]], rel[pos[best]]) >= 0) best = p;
        sel[n_sel++] = pos[best];
        pos[best] = pos[--len];
    }
    while (n_sel < limit && len > 0) {
        uint32_t best = 0;
        float best_mmr = 0.0f;
        for (uint32_t p = 0; p < len; p++) {
            const uint32_t c = pos[p];
            float maxsim_v = 0.0f;
            for (uint32_t k = 0; k < n_sel; k++) {
                const uint32_t s = sel[k];
                const size_t at = (size_t)c * cap + k;
                if (!have[at]) {
                    mat[at] = maxsim(distance, vpre[c], nt[c], vec[s], nt[s], dim);
                    have[at] = 1;
                    *cpu += units * nt[c] * nt[s];
                }
                if (k == 0 || ocmp(mat[at], maxsim_v) >= 0) maxsim_v = mat[at];
            }
            const float a = lambda * rel[c];
            const float b = 1.0f - lambda;
            const float d = b * maxsim_v;
            const float mmr = a - d;
            if (p == 0 || ocmp(mmr, best_mmr) >= 0) { best = p; best_mmr = mmr; }
        }
        sel[n_sel++] = pos[best];
        pos[best] = pos[--len];
    }
    for (uint32_t k = 0; k < n_sel; k++) out[k] = cand[uniq[sel[k]]];
    for (uint32_t c = 0; c < n; c++) free(vpre[c]);
    free(qp); free(vec); free(vpre); free(nt); free(rel); free(mat); free(have); free(pos); free(sel); free(uniq);
    return n_sel;
}
