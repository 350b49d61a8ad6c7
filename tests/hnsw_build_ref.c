/*
 * hnsw_build_ref.c — the CPU restatement of the device graph build (qb_hnsw_build), the checker its graphs are compared with.
 *
 * It compiles the oracle's HNSW (oracle/hnsw.c) into itself, so every insert below is the oracle's own search_on_level,
 * search_entry_on_level, fill_with_heuristic, connect_with_heuristic and link_new_point; this file adds only the schedules:
 *   - qo_hnsw_build_levels: link_new_point in a given order with given levels (the serial builder);
 *   - qo_hnsw_build_batched: the reference GPU builder's schedule (gpu_graph_builder.rs:19-101, gpu_level_builder.rs:12-96,
 *     batched_points.rs:36-163) with two-phase batches: every point of a batch searches the level as it stood before the batch and
 *     selects its links, then the backlinks are applied target by target, each target's sources in batch order.  Single-threaded,
 *     so deterministic.  `shuffle` != 0 processes the targets in a shuffled order (the rule does not depend on it).
 *   - qo_hnsw_levels: the levels a graph was built with (those qo_hnsw_build drew).
 */
#include "../oracle/hnsw.c"

static hnsw_t* hb_new(const float* base, uint32_t n, uint32_t dim, int distance, uint32_t m, uint32_t m0, uint32_t ef, const uint8_t* levels) {
    hnsw_t* h = (hnsw_t*)calloc(1, sizeof(hnsw_t));
    h->n = n; h->dim = dim; h->m = m; h->m0 = m0; h->ef_construct = ef; h->distance = distance; h->base = base;
    pthread_mutex_init(&h->entry_mu, NULL);
    h->level = (uint8_t*)calloc(n ? n : 1, 1);
    h->lock = (atomic_uchar*)calloc(n ? n : 1, 1);
    h->links = (uint32_t***)calloc(n ? n : 1, sizeof(uint32_t**));
    for (uint32_t p = 0; p < n; p++) {
        h->level[p] = levels[p];
        h->links[p] = (uint32_t**)calloc((size_t)levels[p] + 1, sizeof(uint32_t*));
        for (uint32_t l = 0; l <= levels[p]; l++) h->links[p][l] = (uint32_t*)calloc(level_m(h, l) + 2, sizeof(uint32_t));
    }
    return h;
}

API void* qo_hnsw_build_levels(const float* base, uint32_t n, uint32_t dim, int distance, uint32_t m, uint32_t m0, uint32_t ef_construct, const uint8_t* levels,
                               const uint32_t* order) {
    hnsw_t* h = hb_new(base, n, dim, distance, m, m0, ef_construct, levels);
    tctx_t t; tctx_init(&t, n, ef_construct);
    sp_t* sorted = (sp_t*)malloc(sizeof(sp_t) * (ef_construct + 1));
    for (uint32_t i = 0; i < n; i++) link_new_point(h, &t, order ? order[i] : i, sorted);
    free(sorted); tctx_free(&t);
    h->n_score_calls = h->n_scored = 0;
    return h;
}

API void qo_hnsw_levels(void* hp, uint8_t* out) {
    hnsw_t* h = (hnsw_t*)hp;
    memcpy(out, h->level, h->n);
}

typedef struct { uint32_t target, pos, source; } trip_t;
static int cmp_trip(const void* a, const void* b) {
    const trip_t* x = (const trip_t*)a; const trip_t* y = (const trip_t*)b;
    if (x->target != y->target) return x->target < y->target ? -1 : 1;
    return (x->pos > y->pos) - (x->pos < y->pos);
}
static const uint8_t* g_levels;
static int cmp_order(const void* a, const void* b) {   /* level descending, then id (BatchedPoints::sort_points_by_level) */
    const uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b;
    if (g_levels[x] != g_levels[y]) return g_levels[x] > g_levels[y] ? -1 : 1;
    return (x > y) - (x < y);
}

/* deleted: optional bitmap (bit = 1: not inserted).  batch, serial_points >= 1.  Returns the graph; its entry is the first inserted point. */
API void* qo_hnsw_build_batched(const float* base, uint32_t n, uint32_t dim, int distance, uint32_t m, uint32_t m0, uint32_t ef_construct, const uint8_t* levels,
                                const uint64_t* deleted, uint32_t batch, uint32_t serial_points, uint64_t shuffle) {
    const uint32_t ef = ef_construct > m0 ? ef_construct : m0;   /* gpu_graph_builder.rs:38 */
    hnsw_t* h = hb_new(base, n, dim, distance, m, m0, ef, levels);
    uint32_t* order = (uint32_t*)malloc(sizeof(uint32_t) * (n ? n : 1));
    uint32_t n_ins = 0;
    for (uint32_t p = 0; p < n; p++) if (!deleted || !((deleted[p >> 6] >> (p & 63)) & 1)) order[n_ins++] = p;
    g_levels = levels;
    qsort(order, n_ins, sizeof(uint32_t), cmp_order);
    tctx_t t; tctx_init(&t, n, ef);
    sp_t* sorted = (sp_t*)malloc(sizeof(sp_t) * (ef + 1));
    /* the serial prefix, the entry point first (link_new_point, point by point) */
    const uint32_t sp = serial_points < n_ins ? serial_points : n_ins;
    for (uint32_t i = 0; i < sp; i++) link_new_point(h, &t, order[i], sorted);
    if (n_ins > sp) {
        const uint32_t* rest = order + 1;
        const uint32_t nr = n_ins - 1, first = sp - 1;
        uint32_t* ent = (uint32_t*)malloc(sizeof(uint32_t) * nr);
        for (uint32_t i = 0; i < nr; i++) ent[i] = order[0];          /* PointLinkingData::entry starts at the first point */
        /* batches: chunks of `batch` from the first point after the entry, cut where the level changes, from `first` on */
        uint32_t* bb = (uint32_t*)malloc(sizeof(uint32_t) * (nr + 1));
        uint32_t nb = 0;
        for (uint32_t k = first; k < nr;) {
            uint32_t e = (k / batch + 1) * batch;
            if (e > nr) e = nr;
            for (uint32_t j = k + 1; j < e; j++) if (levels[rest[j]] != levels[rest[k]]) { e = j; break; }
            bb[nb++] = k;
            k = e;
        }
        bb[nb] = nr;
        trip_t* tr = (trip_t*)malloc(sizeof(trip_t) * ((size_t)batch * (m0 > m ? m0 : m) + 1));
        uint32_t* grp = (uint32_t*)malloc(sizeof(uint32_t) * ((size_t)batch * (m0 > m ? m0 : m) + 2));
        uint64_t rs = shuffle;
        for (int l = (int)h->entry_level; l >= 0; l--) {
            const uint32_t lm = level_m(h, (uint32_t)l);
            for (uint32_t b = 0; b < nb; b++) {
                const uint32_t k0 = bb[b], k1 = bb[b + 1];
                if (levels[rest[k0]] < (uint32_t)l) continue;
                /* phase 1: search the level as it was before the batch, select the point's links */
                uint32_t nt = 0;
                for (uint32_t i = k0; i < k1; i++) {
                    const uint32_t p = rest[i];
                    scorer_t s = { h, &t, NULL, NULL, h->base + (size_t)p * h->dim, NULL };
                    sp_t le; le.idx = ent[i]; le.score = score_internal(h, p, ent[i]);
                    search_on_level(h, &s, le, (uint32_t)l, ef);
                    memcpy(sorted, t.nearest.d, t.nearest.len * sizeof(sp_t));
                    qsort(sorted, t.nearest.len, sizeof(sp_t), cmp_desc);
                    ent[i] = sorted[0].idx;
                    fill_with_heuristic(h, h->links[p][l], sorted, t.nearest.len, lm);
                    for (uint32_t j = 0; j < h->links[p][l][0]; j++) { tr[nt].target = h->links[p][l][1 + j]; tr[nt].pos = i - k0; tr[nt].source = p; nt++; }
                }
                /* phase 2: the backlinks, target by target, each target's sources in batch order */
                qsort(tr, nt, sizeof(trip_t), cmp_trip);
                uint32_t ng = 0;
                for (uint32_t i = 0; i < nt; i++) if (i == 0 || tr[i].target != tr[i - 1].target) grp[ng++] = i;
                grp[ng] = nt;
                uint32_t* go = (uint32_t*)malloc(sizeof(uint32_t) * (ng ? ng : 1));
                for (uint32_t g = 0; g < ng; g++) go[g] = g;
                if (shuffle) for (uint32_t g = ng; g > 1; g--) { uint32_t j = (uint32_t)(splitmix(&rs) % g), x = go[g - 1]; go[g - 1] = go[j]; go[j] = x; }
                for (uint32_t gi = 0; gi < ng; gi++) {
                    const uint32_t g = go[gi];
                    for (uint32_t i = grp[g]; i < grp[g + 1]; i++) connect_with_heuristic(h, h->links[tr[i].target][l], tr[i].source, tr[i].target, lm);
                }
                free(go);
            }
            if (l == 0) break;
            /* the points below l: greedy descent on l (search_entry_on_level) */
            for (uint32_t i = first; i < nr; i++) {
                if (levels[rest[i]] >= (uint32_t)l) continue;
                const uint32_t p = rest[i];
                scorer_t s = { h, &t, NULL, NULL, h->base + (size_t)p * h->dim, NULL };
                ent[i] = search_entry_on_level(h, &s, ent[i], (uint32_t)l).idx;
            }
        }
        free(tr); free(grp); free(bb); free(ent);
    }
    free(sorted); tctx_free(&t); free(order);
    h->n_score_calls = h->n_scored = 0;
    return h;
}
