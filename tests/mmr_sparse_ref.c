/* The checker of qb_mmr_sparse_batch: maximal marginal relevance over sparse vector candidates, one query at a time, single-threaded,
 * the way the reference runs it:
 *   - unique_by(id), first occurrence kept; fewer than two left: returned as they are, nothing scored or counted;
 *   - every vector sorted by dim (the volatile storage's insert, VectorInternal::preprocess for the query);
 *   - score_vectors(a, b): a sum from 0.0 of a_w * b_w over the shared dims in ascending dim order, every product and sum rounded
 *     (compiled without contraction); +0.0 when no dim is shared (unwrap_or_default);
 *   - rel[i] = score_vectors(q, v_i);
 *   - a lazily filled matrix: pair(c, s) = score_vectors(v_c, v_s) (candidate c's scorer), scored on first use and counted then;
 *   - the remaining candidates as an explicit position array; a pick is swap-removed (the last position moves into its place);
 *   - every max / argmax keeps the LAST maximal element under OrderedFloat (NaN above everything and equal to NaN, -0.0 == +0.0);
 *   - mmr = lambda * rel - (1 - lambda) * maxsim, four separately rounded f32 operations.
 * Counters: cpu += min(|a|, |b|) per scored pair (SparseMetricQueryScorer, multiplier 1); vector_io_read stays 0. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define API __attribute__((visibility("default")))

typedef struct { uint32_t idx; float score; } scored;
typedef struct { uint32_t d; float w; } elem;

static int ocmp(float a, float b) {
    const int na = a != a, nb = b != b;
    if (na || nb) return na - nb;
    return (a > b) - (a < b);
}

static int by_dim(const void* a, const void* b) {
    const uint32_t x = ((const elem*)a)->d, y = ((const elem*)b)->d;
    return (x > y) - (x < y);
}

/* a vector's elements sorted by dim */
static elem* sorted(const uint32_t* dims, const float* w, uint64_t n) {
    elem* e = malloc(sizeof(elem) * (n + 1));
    for (uint64_t i = 0; i < n; i++) { e[i].d = dims[i]; e[i].w = w[i]; }
    qsort(e, n, sizeof(elem), by_dim);
    return e;
}

/* score_vectors over two dim-sorted vectors: self's weight times other's */
static float score_sorted(const elem* a, uint64_t na, const elem* b, uint64_t nb) {
    float s = 0.0f;
    uint64_t i = 0, j = 0;
    while (i < na && j < nb) {
        if (a[i].d < b[j].d) i++;
        else if (a[i].d > b[j].d) j++;
        else { const float p = a[i].w * b[j].w; s = s + p; i++; j++; }
    }
    return s;
}

API float qms_score(const uint32_t* ad, const float* aw, uint64_t na, const uint32_t* bd, const float* bw, uint64_t nb) {
    elem* a = sorted(ad, aw, na);
    elem* b = sorted(bd, bw, nb);
    const float s = score_sorted(a, na, b, nb);
    free(a); free(b);
    return s;
}

/* one query.  indptr / dims / weights: the storage's CSR rows (any order within a row).  q: the query's q_n elements (any order).
 * cand: n_cand candidates, ids < n_points.  out: up to max(n_cand, 1) entries; returns how many.  cpu / io: added to. */
API uint32_t qms_mmr(const uint64_t* indptr, const uint32_t* dims, const float* weights, const uint32_t* q_dims, const float* q_w, uint64_t q_n,
                     float lambda, const scored* cand, uint32_t n_cand, uint32_t limit, scored* out, uint64_t* cpu, uint64_t* io) {
    (void)io;   /* the volatile storage is in memory */
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
    elem* q = sorted(q_dims, q_w, q_n);
    elem** vec = malloc(sizeof(elem*) * n);
    uint64_t* len = malloc(sizeof(uint64_t) * n);
    float* rel = malloc(sizeof(float) * n);
    const uint32_t cap = limit < n ? limit : n;   /* the matrix's columns are the picks, in pick order: pair(c, pick k) at c * cap + k */
    float* mat = malloc(sizeof(float) * (size_t)n * (cap ? cap : 1));
    unsigned char* have = calloc((size_t)n * (cap ? cap : 1), 1);
    uint32_t* pos = malloc(sizeof(uint32_t) * n);
    uint32_t* sel = malloc(sizeof(uint32_t) * n);
    for (uint32_t c = 0; c < n; c++) {
        const uint32_t p = cand[uniq[c]].idx;
        len[c] = indptr[p + 1] - indptr[p];
        vec[c] = sorted(dims + indptr[p], weights + indptr[p], len[c]);
        rel[c] = score_sorted(q, q_n, vec[c], len[c]);
        *cpu += q_n < len[c] ? q_n : len[c];
        pos[c] = c;
    }
    uint32_t cnt = n, n_sel = 0;
    if (limit > 0) {
        uint32_t best = 0;
        for (uint32_t p = 1; p < cnt; p++)
            if (ocmp(rel[pos[p]], rel[pos[best]]) >= 0) best = p;
        sel[n_sel++] = pos[best];
        pos[best] = pos[--cnt];
    }
    while (n_sel < limit && cnt > 0) {
        uint32_t best = 0;
        float best_mmr = 0.0f;
        for (uint32_t p = 0; p < cnt; p++) {
            const uint32_t c = pos[p];
            float maxsim = 0.0f;
            for (uint32_t k = 0; k < n_sel; k++) {
                const uint32_t s = sel[k];
                const size_t at = (size_t)c * cap + k;
                if (!have[at]) {
                    mat[at] = score_sorted(vec[c], len[c], vec[s], len[s]);
                    have[at] = 1;
                    *cpu += len[c] < len[s] ? len[c] : len[s];
                }
                if (k == 0 || ocmp(mat[at], maxsim) >= 0) maxsim = mat[at];
            }
            const float a = lambda * rel[c];
            const float b = 1.0f - lambda;
            const float d = b * maxsim;
            const float mmr = a - d;
            if (p == 0 || ocmp(mmr, best_mmr) >= 0) { best = p; best_mmr = mmr; }
        }
        sel[n_sel++] = pos[best];
        pos[best] = pos[--cnt];
    }
    for (uint32_t k = 0; k < n_sel; k++) out[k] = cand[uniq[sel[k]]];
    for (uint32_t c = 0; c < n; c++) free(vec[c]);
    free(q); free(vec); free(len); free(rel); free(mat); free(have); free(pos); free(sel); free(uniq);
    return n_sel;
}
