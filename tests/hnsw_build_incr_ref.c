/*
 * hnsw_build_incr_ref.c — the CPU restatement of the incremental device graph build (qb_hnsw_build_incremental), the checker its graphs
 * are compared with.
 *
 * It compiles the build restatement (tests/hnsw_build_ref.c) and with it the oracle's HNSW (oracle/hnsw.c) into itself, so every score,
 * heuristic and insert below is the oracle's own (score_internal, fill_with_heuristic, connect_with_heuristic, link_new_point,
 * search_on_level); this file adds the steps of the reference's old-index path (hnsw/build.rs:225-357):
 *   - qo_hnsw_from_plain: a graph from a plain links.bin, each list cut to its first level_m links (GraphLayersHealer::new, :33-47);
 *   - qo_hnsw_heal: the to-heal items (point ascending, then level, unmapped points included), then per level the two-phase heal:
 *     every item runs search_shortcuts_on_level (:82-158) over the lists as loaded and writes its own list (heal_point_on_level,
 *     :160-191), then the backlinks in (target, item) order, each skipped when the target's list holds the item at that moment;
 *   - qo_hnsw_renumber: save_into_builder (:236-256) into a graph over the new rows, a repeated link kept once, the entry by
 *     EntryPoints::new_point in old-offset order;
 *   - qo_hnsw_insert_new: the new points with qb_hnsw_build's schedule (serial prefix, then level-major batches with two-phase
 *     backlinks), or serial link_new_point of each in the order (serial != 0).
 */
#include "hnsw_build_ref.c"

/* a plain links.bin (graph_links/header.rs:9-20) as a graph over `base`; a list longer than level_m keeps its first level_m links */
API void* qo_hnsw_from_plain(const float* base, uint32_t dim, int distance, uint32_t m, uint32_t m0, uint32_t ef, const uint8_t* blob) {
    const uint64_t* hdr = (const uint64_t*)blob;
    const uint32_t n = (uint32_t)hdr[0], L = (uint32_t)hdr[1];
    const uint64_t n_nb = hdr[2], n_off = hdr[3], pad = hdr[4];
    const uint64_t* lo = (const uint64_t*)(blob + 64);
    const uint32_t* reindex = (const uint32_t*)(blob + 64 + 8ull * L);
    const uint32_t* nb = reindex + n;
    const uint64_t* offs = (const uint64_t*)(blob + 64 + 8ull * L + 4ull * n + 4ull * n_nb + pad);
    uint8_t* levels = (uint8_t*)calloc(n ? n : 1, 1);
    for (uint32_t p = 0; p < n; p++) {
        uint32_t l = 0;
        while (l + 1 < L && reindex[p] < (l + 2 < L ? lo[l + 2] : n_off - 1) - lo[l + 1]) l++;
        levels[p] = (uint8_t)l;
    }
    hnsw_t* h = hb_new(base, n, dim, distance, m, m0, ef, levels);
    free(levels);
    for (uint32_t p = 0; p < n; p++)
        for (uint32_t l = 0; l <= h->level[p]; l++) {
            const uint64_t r = lo[l] + (l ? reindex[p] : p), b = offs[r], e = offs[r + 1];
            const uint32_t lm = level_m(h, l);
            uint32_t* lk = h->links[p][l];
            lk[0] = 0;
            for (uint64_t k = b; k < e && lk[0] < lm; k++) lk[1 + lk[0]++] = nb[k];
        }
    return h;
}

#define GONE(o2n, x) ((o2n)[x] == 0xFFFFFFFFu)

typedef struct { sp_t* d; size_t len, cap; } stack_t_;
static void st_push(stack_t_* s, sp_t v) { if (s->len == s->cap) { s->cap = s->cap * 2 + 64; s->d = (sp_t*)realloc(s->d, s->cap * sizeof(sp_t)); } s->d[s->len++] = v; }

/* search_shortcuts_on_level (graph_layers_healer.rs:82-158) over the lists `old` of one level; the result is left in t->nearest */
static void search_shortcuts(hnsw_t* h, tctx_t* t, uint32_t*** old, uint32_t p, uint32_t l, const uint32_t* o2n, uint32_t ef, stack_t_* pending) {
    t->stamp++;
    if (t->stamp == 0) { memset(t->visited, 0, sizeof(uint32_t) * h->n); t->stamp = 1; }
    flpq_t* nearest = &t->nearest;
    nearest->len = 0; nearest->cap = ef;
    pending->len = 0;
    t->visited[p] = t->stamp;
    const uint32_t* lk = old[p][l];
    for (uint32_t j = 0; j < lk[0]; j++) {
        const uint32_t x = lk[1 + j];
        if (!GONE(o2n, x)) t->visited[x] = t->stamp;
        else { sp_t v = { x, score_internal(h, p, x) }; st_push(pending, v); }
    }
    while (pending->len) {
        const sp_t c = pending->d[--pending->len];
        if (nearest->len == nearest->cap && c.score < nearest->d[0].score) continue;
        if (t->visited[c.idx] == t->stamp) continue;
        t->visited[c.idx] = t->stamp;
        const uint32_t* cl = old[c.idx][l];
        uint32_t ids[514], n = 0;
        for (uint32_t j = 0; j < cl[0]; j++) if (t->visited[cl[1 + j]] != t->stamp) ids[n++] = cl[1 + j];
        for (uint32_t j = 0; j < n; j++) {
            sp_t v = { ids[j], score_internal(h, p, ids[j]) };
            if (!GONE(o2n, ids[j])) flpq_push(nearest, v);
            else st_push(pending, v);
        }
    }
}

typedef struct { uint32_t target, item, source; } hpair_t;
static int cmp_hpair(const void* a, const void* b) {
    const hpair_t* x = (const hpair_t*)a; const hpair_t* y = (const hpair_t*)b;
    if (x->target != y->target) return x->target < y->target ? -1 : 1;
    return (x->item > y->item) - (x->item < y->item);
}

/* heals h (a graph over the OLD rows) in place; o2n: old_to_new (0xFFFFFFFF = not carried over); returns the number of items.
   only_item >= 0 heals that item alone (its index in the to-heal order), a check of the single-item case. */
API uint32_t qo_hnsw_heal(void* hp, const uint32_t* o2n, uint32_t ef_construct, int64_t only_item) {
    hnsw_t* h = (hnsw_t*)hp;
    const uint32_t n = h->n;
    uint32_t top = 0;
    for (uint32_t p = 0; p < n; p++) if (h->level[p] > top) top = h->level[p];
    /* the to-heal items in to_edges_impl's order: (point, level), point ascending, then level */
    uint32_t *ip = (uint32_t*)malloc(sizeof(uint32_t) * ((size_t)n * (top + 1) + 1)), *il = (uint32_t*)malloc(sizeof(uint32_t) * ((size_t)n * (top + 1) + 1));
    uint32_t ni = 0;
    for (uint32_t p = 0; p < n; p++)
        for (uint32_t l = 0; l <= h->level[p]; l++) {
            const uint32_t* lk = h->links[p][l];
            int gone = 0;
            for (uint32_t j = 0; j < lk[0]; j++) gone |= GONE(o2n, lk[1 + j]);
            if (gone) { ip[ni] = p; il[ni] = l; ni++; }
        }
    /* the lists as loaded, read by phase 1 */
    uint32_t*** old = (uint32_t***)calloc(n ? n : 1, sizeof(uint32_t**));
    for (uint32_t p = 0; p < n; p++) {
        old[p] = (uint32_t**)calloc((size_t)h->level[p] + 1, sizeof(uint32_t*));
        for (uint32_t l = 0; l <= h->level[p]; l++) {
            old[p][l] = (uint32_t*)malloc(sizeof(uint32_t) * (level_m(h, l) + 2));
            memcpy(old[p][l], h->links[p][l], sizeof(uint32_t) * (h->links[p][l][0] + 1));
        }
    }
    tctx_t t; tctx_init(&t, n, ef_construct);
    stack_t_ pending = { NULL, 0, 0 };
    sp_t* sorted = (sp_t*)malloc(sizeof(sp_t) * (ef_construct + 1));
    hpair_t* pr = (hpair_t*)malloc(sizeof(hpair_t) * ((size_t)ni * (h->m0 > h->m ? h->m0 : h->m) + 1));
    for (uint32_t l = 0; l <= top; l++) {
        const uint32_t lm = level_m(h, l);
        uint32_t np = 0;
        for (uint32_t i = 0; i < ni; i++) {   /* phase 1 */
            if (il[i] != l || (only_item >= 0 && (int64_t)i != only_item)) continue;
            const uint32_t p = ip[i];
            search_shortcuts(h, &t, old, p, l, o2n, ef_construct, &pending);
            memcpy(sorted, t.nearest.d, t.nearest.len * sizeof(sp_t));
            qsort(sorted, t.nearest.len, sizeof(sp_t), cmp_desc);
            uint32_t valid[514], nv = 0;
            for (uint32_t j = 0; j < old[p][l][0]; j++) if (!GONE(o2n, old[p][l][1 + j])) valid[nv++] = old[p][l][1 + j];
            uint32_t* lk = h->links[p][l];
            fill_with_heuristic(h, lk, sorted, t.nearest.len, lm - nv);
            for (uint32_t j = 0; j < nv; j++) lk[1 + lk[0]++] = valid[j];
            for (uint32_t j = 0; j < lk[0]; j++) { pr[np].target = lk[1 + j]; pr[np].item = i; pr[np].source = p; np++; }
        }
        qsort(pr, np, sizeof(hpair_t), cmp_hpair);   /* phase 2 */
        for (uint32_t k = 0; k < np; k++) {
            uint32_t* tl = h->links[pr[k].target][l];
            int has = 0;
            for (uint32_t j = 0; j < tl[0]; j++) has |= tl[1 + j] == pr[k].source;
            if (!has) connect_with_heuristic(h, tl, pr[k].source, pr[k].target, lm);
        }
    }
    for (uint32_t p = 0; p < n; p++) { for (uint32_t l = 0; l <= h->level[p]; l++) free(old[p][l]); free(old[p]); }
    free(old); free(ip); free(il); free(pr); free(sorted); free(pending.d); tctx_free(&t);
    return ni;
}

/* save_into_builder: a graph over the new rows whose mapped points hold their healed lists, renamed, unmapped links dropped.  levels: one
   per new point (a mapped point's = its old level); ef: the inserts' ef (max(ef_construct, m0)). */
API void* qo_hnsw_renumber(void* hp, const uint32_t* o2n, const float* new_base, uint32_t n_new, const uint8_t* levels, uint32_t ef) {
    hnsw_t* h = (hnsw_t*)hp;
    hnsw_t* g = hb_new(new_base, n_new, h->dim, h->distance, h->m, h->m0, ef, levels);
    for (uint32_t o = 0; o < h->n; o++) {
        const uint32_t t = o2n[o];
        if (t == 0xFFFFFFFFu) continue;
        for (uint32_t l = 0; l <= h->level[o]; l++) {
            const uint32_t* src = h->links[o][l];
            uint32_t* dst = g->links[t][l];
            dst[0] = 0;
            for (uint32_t j = 0; j < src[0]; j++) {   /* a repeated link (Dot scores can keep a shortcut twice) is kept once */
                int seen = 0;
                for (uint32_t i = 0; i < j; i++) seen |= src[1 + i] == src[1 + j];
                if (!GONE(o2n, src[1 + j]) && !seen) dst[1 + dst[0]++] = o2n[src[1 + j]];
            }
        }
        if (!g->has_entry || g->level[t] > g->entry_level) { g->entry = t; g->entry_level = g->level[t]; g->has_entry = 1; }   /* new_point */
    }
    return g;
}

/* inserts the points with is_new[p] != 0 into g (renumbered, with its entry), in the order level descending, then id.  serial != 0:
   link_new_point point by point; else qb_hnsw_build's schedule: the first serial_points one at a time, then batches of at most `batch`
   cut where the level changes, level by level from the entry's level, two-phase backlinks. */
API void qo_hnsw_insert_new(void* gp, const uint8_t* is_new, uint32_t batch, uint32_t serial_points, int serial) {
    hnsw_t* h = (hnsw_t*)gp;
    const uint32_t n = h->n;
    uint32_t* rest = (uint32_t*)malloc(sizeof(uint32_t) * (n ? n : 1));
    uint32_t nr = 0;
    for (uint32_t p = 0; p < n; p++) if (is_new[p]) rest[nr++] = p;
    g_levels = h->level;
    qsort(rest, nr, sizeof(uint32_t), cmp_order);
    tctx_t t; tctx_init(&t, n, h->ef_construct);
    sp_t* sorted = (sp_t*)malloc(sizeof(sp_t) * (h->ef_construct + 1));
    const uint32_t sp = serial ? nr : (serial_points < nr ? serial_points : nr);
    for (uint32_t i = 0; i < sp; i++) link_new_point(h, &t, rest[i], sorted);   /* a first point above the top becomes the entry here */
    if (nr > sp) {
        const uint32_t ef = h->ef_construct, first = sp;
        uint32_t* ent = (uint32_t*)malloc(sizeof(uint32_t) * nr);
        for (uint32_t i = 0; i < nr; i++) ent[i] = h->entry;
        uint32_t* bb = (uint32_t*)malloc(sizeof(uint32_t) * (nr + 1));
        uint32_t nb = 0;
        for (uint32_t k = first; k < nr;) {
            uint32_t e = (k / batch + 1) * batch;
            if (e > nr) e = nr;
            for (uint32_t j = k + 1; j < e; j++) if (h->level[rest[j]] != h->level[rest[k]]) { e = j; break; }
            bb[nb++] = k;
            k = e;
        }
        bb[nb] = nr;
        const uint32_t mm = h->m0 > h->m ? h->m0 : h->m;
        trip_t* tr = (trip_t*)malloc(sizeof(trip_t) * ((size_t)batch * mm + 1));
        for (int l = (int)h->entry_level; l >= 0; l--) {
            const uint32_t lm = level_m(h, (uint32_t)l);
            for (uint32_t b = 0; b < nb; b++) {
                const uint32_t k0 = bb[b], k1 = bb[b + 1];
                if (h->level[rest[k0]] < (uint32_t)l) continue;
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
                qsort(tr, nt, sizeof(trip_t), cmp_trip);
                for (uint32_t i = 0; i < nt; i++) connect_with_heuristic(h, h->links[tr[i].target][l], tr[i].source, tr[i].target, lm);
            }
            if (l == 0) break;
            for (uint32_t i = first; i < nr; i++) {
                if (h->level[rest[i]] >= (uint32_t)l) continue;
                const uint32_t p = rest[i];
                scorer_t s = { h, &t, NULL, NULL, h->base + (size_t)p * h->dim, NULL };
                ent[i] = search_entry_on_level(h, &s, ent[i], (uint32_t)l).idx;
            }
        }
        free(tr); free(bb); free(ent);
    }
    free(sorted); tctx_free(&t); free(rest);
    h->n_score_calls = h->n_scored = 0;
}
