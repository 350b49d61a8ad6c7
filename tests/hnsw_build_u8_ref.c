/*
 * hnsw_build_u8_ref.c — the CPU restatements of the device graph builds over Uint8 storages (qb_hnsw_build, qb_hnsw_build_incremental),
 * the checkers their graphs are compared with.
 *
 * It is tests/hnsw_build_incr_ref.c, and with it tests/hnsw_build_ref.c and the oracle's HNSW, compiled once more with one pair score in
 * place of the oracle's f32 similarity, as tests/hnsw_build_mv_ref.c does for MaxSim.  A graph is built with dim = 1 over a `base` holding
 * one float per point (its values are not read), so the two addresses name the points, and the score is Metric<u8>::similarity of their
 * stored rows, the first point's row as the query (the oracle's qo_u8_*: the avx2 chains for dim >= 32, the integer-exact scalar tier
 * below).  The inserts' query is the stored row itself, as FilteredScorer::new_internal gives it for u8 (f32 -> identity preprocess ->
 * `as u8`).  qo_u8_bind names the rows before a build; one build runs at a time.  tests/hnsw_build_keyed_ref.py
 * also compiles it over tests/hnsw_keyed_oracle.c, the device's tie order.
 */
#define _GNU_SOURCE   /* before any system header, as oracle/hnsw.c needs it */
#include <stddef.h>
#include <stdint.h>

float qo_u8_dot_avx(const uint8_t* v1, const uint8_t* v2, size_t len);
float qo_u8_cosine_avx(const uint8_t* v1, const uint8_t* v2, size_t len);
float qo_u8_euclid_avx(const uint8_t* v1, const uint8_t* v2, size_t len);
float qo_u8_manhattan_avx(const uint8_t* v1, const uint8_t* v2, size_t len);
float qo_u8_dot_scalar(const uint8_t* a, const uint8_t* b, size_t n);
float qo_u8_euclid_scalar(const uint8_t* a, const uint8_t* b, size_t n);
float qo_u8_manhattan_scalar(const uint8_t* a, const uint8_t* b, size_t n);
float qo_u8_cosine_scalar(const uint8_t* a, const uint8_t* b, size_t n);

static struct {
    const float* base;     /* the graph's base: one float per point */
    const uint8_t* rows;   /* the stored rows, dim bytes each */
    uint32_t dim;
} u8;

/* Metric<u8>::similarity (the oracle's u8_similarity dispatch); the distance codes are the oracle's (QO_COSINE 0, QO_EUCLID 1, QO_DOT 2,
   QO_MANHATTAN 3) */
static float u8_pair_score(int distance, const float* a, const float* b, size_t n) {
    (void)n;
    const uint8_t* x = u8.rows + (size_t)(a - u8.base) * u8.dim;
    const uint8_t* y = u8.rows + (size_t)(b - u8.base) * u8.dim;
    const int avx = u8.dim >= 32;
    switch (distance) {
        case 0: return avx ? qo_u8_cosine_avx(x, y, u8.dim) : qo_u8_cosine_scalar(x, y, u8.dim);
        case 1: return avx ? qo_u8_euclid_avx(x, y, u8.dim) : qo_u8_euclid_scalar(x, y, u8.dim);
        case 3: return avx ? qo_u8_manhattan_avx(x, y, u8.dim) : qo_u8_manhattan_scalar(x, y, u8.dim);
        default: return avx ? qo_u8_dot_avx(x, y, u8.dim) : qo_u8_dot_scalar(x, y, u8.dim);
    }
}

#define qo_similarity_f32 u8_pair_score
#include "hnsw_build_incr_ref.c"

/* the rows of the points the next build (base = `base`, dim = 1) links */
API void qo_u8_bind(const float* base, const uint8_t* rows, uint32_t dim) {
    u8.base = base; u8.rows = rows; u8.dim = dim;
}
