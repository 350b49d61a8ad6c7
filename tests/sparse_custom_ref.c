/* sparse_custom_ref.c — the checker of the device's custom queries over a sparse vector storage: the reference's search_scored
 * (sparse_vector_index/read_view/search.rs:302-341) with a SparseCustomQueryScorer (query_scorer/sparse_custom_query_scorer.rs),
 * restated on the CPU in the parts that are not the fold:
 *   - score_vectors (lib/sparse/src/common/sparse_vector.rs:66-90): both vectors sorted by dim, a merge-join summing example weight x
 *     stored weight from 0.0 in ascending dim order, None (0.0 after unwrap_or) when no dim is shared;
 *   - the points BatchFilteredSearcher::peek_top_iter scores: every point not deleted, or the listed ids that are not deleted;
 *   - the top-k under the project's (score desc, id asc) keys, NaN above everything;
 *   - the HardwareCounterCell units: cpu 4 x (|v| + |example|) per point and example, vector_io_read 2 |v| x (4 on disk, else 0) per point.
 * The per-example similarities leave as an E x N matrix; the fold (Query::score_by) is the oracle's, pinned elsewhere.
 * Compiled with -ffp-contract=off: every product and sum rounds as in the reference. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define API __attribute__((visibility("default")))

typedef struct { uint32_t d; float w; } Elem;

typedef struct {
    uint32_t n_points;
    uint64_t* ptr;
    Elem* el;      /* rows sorted by dim */
    int on_disk;
} Storage;

static int by_dim(const void* a, const void* b) {
    const uint32_t x = ((const Elem*)a)->d, y = ((const Elem*)b)->d;
    return (x > y) - (x < y);
}

API void* scr_storage_new(uint32_t n_points, const uint64_t* indptr, const uint32_t* dims, const float* weights, int on_disk) {
    Storage* s = (Storage*)calloc(1, sizeof(Storage));
    const uint64_t n = indptr[n_points];
    s->n_points = n_points;
    s->on_disk = on_disk;
    s->ptr = (uint64_t*)malloc((n_points + 1) * sizeof(uint64_t));
    memcpy(s->ptr, indptr, (n_points + 1) * sizeof(uint64_t));
    s->el = (Elem*)malloc((n ? n : 1) * sizeof(Elem));
    for (uint64_t e = 0; e < n; e++) { s->el[e].d = dims[e]; s->el[e].w = weights[e]; }
    for (uint32_t r = 0; r < n_points; r++) qsort(s->el + indptr[r], indptr[r + 1] - indptr[r], sizeof(Elem), by_dim);   /* distinct dims: any sort */
    return s;
}

API void scr_storage_free(void* p) {
    Storage* s = (Storage*)p;
    if (!s) return;
    free(s->ptr);
    free(s->el);
    free(s);
}

/* score_vectors(example, stored).unwrap_or(0.0) over sorted sides */
static float score_vectors(const Elem* a, uint64_t na, const Elem* b, uint64_t nb) {
    float score = 0.0f;
    uint64_t i = 0, j = 0;
    while (i < na && j < nb) {
        if (a[i].d < b[j].d) i++;
        else if (a[i].d > b[j].d) j++;
        else { score += a[i].w * b[j].w; i++; j++; }
    }
    return score;   /* no overlap: the 0.0 it started from, which is unwrap_or's 0.0 */
}

/* one vector's score for a plain (dims, weights) pair, both given in any order: for the reference's unit cases */
API float scr_score(const uint32_t* ad, const float* aw, uint32_t na, const uint32_t* bd, const float* bw, uint32_t nb, int* overlap) {
    Elem* a = (Elem*)malloc((na + 1) * sizeof(Elem));
    Elem* b = (Elem*)malloc((nb + 1) * sizeof(Elem));
    for (uint32_t i = 0; i < na; i++) { a[i].d = ad[i]; a[i].w = aw[i]; }
    for (uint32_t i = 0; i < nb; i++) { b[i].d = bd[i]; b[i].w = bw[i]; }
    qsort(a, na, sizeof(Elem), by_dim);
    qsort(b, nb, sizeof(Elem), by_dim);
    int ov = 0;
    for (uint32_t i = 0, j = 0; i < na && j < nb;) {
        if (a[i].d < b[j].d) i++;
        else if (a[i].d > b[j].d) j++;
        else { ov = 1; break; }
    }
    const float s = score_vectors(a, na, b, nb);
    free(a);
    free(b);
    *overlap = ov;
    return s;
}

/* sims[e * n + k] = similarity of point ids[k] to example e; example e = entries [ex_ptr[e], ex_ptr[e + 1]) in any order */
API void scr_sims(const void* p, uint32_t E, const uint64_t* ex_ptr, const uint32_t* ex_dims, const float* ex_w, const uint32_t* ids, uint64_t n, float* sims) {
    const Storage* s = (const Storage*)p;
    for (uint32_t e = 0; e < E; e++) {
        const uint64_t m = ex_ptr[e + 1] - ex_ptr[e];
        Elem* x = (Elem*)malloc((m + 1) * sizeof(Elem));
        for (uint64_t i = 0; i < m; i++) { x[i].d = ex_dims[ex_ptr[e] + i]; x[i].w = ex_w[ex_ptr[e] + i]; }
        qsort(x, m, sizeof(Elem), by_dim);   /* sort_by_indices */
        for (uint64_t k = 0; k < n; k++) {
            const uint32_t id = ids[k];
            sims[(uint64_t)e * n + k] = score_vectors(x, m, s->el + s->ptr[id], s->ptr[id + 1] - s->ptr[id]);
        }
        free(x);
    }
}

/* the points peek_top_iter scores, in order: the listed ids that are not deleted, or every point that is not */
API uint64_t scr_points(const void* p, const uint64_t* deleted, const uint32_t* id_list, uint64_t n_ids, uint32_t* out) {
    const Storage* s = (const Storage*)p;
    uint64_t n = 0;
    const uint64_t m = id_list ? n_ids : s->n_points;
    for (uint64_t k = 0; k < m; k++) {
        const uint32_t id = id_list ? id_list[k] : (uint32_t)k;
        if (deleted && ((deleted[id >> 6] >> (id & 63)) & 1ull)) continue;
        out[n++] = id;
    }
    return n;
}

/* counters of scoring `ids` with one query of E examples */
API void scr_counters(const void* p, const uint32_t* ids, uint64_t n, uint32_t E, const uint64_t* ex_ptr, uint64_t* cpu, uint64_t* io) {
    const Storage* s = (const Storage*)p;
    for (uint64_t k = 0; k < n; k++) {
        const uint64_t v = s->ptr[ids[k] + 1] - s->ptr[ids[k]];
        for (uint32_t e = 0; e < E; e++) *cpu += 4 * (v + (ex_ptr[e + 1] - ex_ptr[e]));   /* set_cpu_multiplier(size_of::<DimWeight>()) */
        *io += (2 * v) * (s->on_disk ? 4 : 0);                                              /* indices + values, size_of::<DimId>() on disk */
    }
}

/* (score desc, id asc) keys: -0.0 just below +0.0, every NaN one key above +inf */
static uint32_t orderable(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    if ((u & 0x7FFFFFFFu) > 0x7F800000u) return 0xFFC00000u;
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
static float unorderable(uint32_t o) {
    const uint32_t u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
    float f;
    memcpy(&f, &u, 4);
    return f;
}
static int key_desc(const void* a, const void* b) {
    const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
    return (x < y) - (x > y);
}

/* the best `top` of (ids[k], scores[k]) in (score desc, id asc) order; the scores come back as the keys carry them */
API uint64_t scr_topk(const uint32_t* ids, const float* scores, uint64_t n, uint32_t top, uint32_t* out_ids, float* out_scores) {
    uint64_t* keys = (uint64_t*)malloc((n + 1) * sizeof(uint64_t));
    for (uint64_t k = 0; k < n; k++) keys[k] = ((uint64_t)orderable(scores[k]) << 32) | (uint64_t)(0xFFFFFFFFu - ids[k]);
    qsort(keys, n, sizeof(uint64_t), key_desc);
    const uint64_t m = n < top ? n : top;
    for (uint64_t i = 0; i < m; i++) {
        out_ids[i] = 0xFFFFFFFFu - (uint32_t)keys[i];
        out_scores[i] = unorderable((uint32_t)(keys[i] >> 32));
    }
    free(keys);
    return m;
}
