/*
 * hnsw_keyed_oracle.c — the oracle's HNSW (oracle/hnsw.c) with the level-0 comparisons of an insert on the device's (score desc, id asc)
 * keys (qb_pack_key), for the checkers of the device builds over Uint8 storages, whose integer scores tie often.
 *
 * It stands in for oracle/hnsw.c when the build restatements (tests/hnsw_build_ref.c, tests/hnsw_build_incr_ref.c) are compiled in
 * keyed mode: tests/hnsw_build_keyed_ref.py compiles copies of them next to a copy of this file named oracle/hnsw.c, so their
 * `#include "../oracle/hnsw.c"` finds it, and this file includes the real oracle/hnsw.c (QB_ORACLE_HNSW, its path).  After the oracle's
 * definitions it defines keyed versions of
 *   - search_on_level: the candidate heap, the fixed-length `nearest` queue and the stop test on keys (a candidate below the worst key
 *     of `nearest` ends the search);
 *   - link_new_point: the oracle's, serial, with that search;
 *   - flpq_push: the fixed-length queue the heal's search_shortcuts fills;
 * and names them with the oracle's names for the code that follows, so the restatements run unchanged on them.  The greedy descent
 * through the upper levels (search_entry_on_level) and the heal's stack test stay score-only, as on the device.  The oracle's own
 * entry points, compiled before the renaming, are untouched.
 */
#include QB_ORACLE_HNSW

static uint64_t hk_key(sp_t v) {   /* qb_pack_key: orderable score bits, then the inverted id */
    uint32_t u; memcpy(&u, &v.score, 4);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ((uint64_t)u << 32) | (uint64_t)(0xFFFFFFFFu - v.idx);
}
static int hk_gt(sp_t a, sp_t b) { return hk_key(a) > hk_key(b); }

static void hk_maxheap_push(heap_t* h, sp_t v) {
    heap_reserve(h, h->len + 1);
    size_t i = h->len++;
    while (i > 0) { size_t p = (i - 1) / 2; if (!hk_gt(v, h->d[p])) break; h->d[i] = h->d[p]; i = p; }
    h->d[i] = v;
}
static sp_t hk_maxheap_pop(heap_t* h) {
    sp_t top = h->d[0], v = h->d[--h->len];
    size_t i = 0;
    for (;;) {
        size_t c = 2 * i + 1;
        if (c >= h->len) break;
        if (c + 1 < h->len && hk_gt(h->d[c + 1], h->d[c])) c++;
        if (!hk_gt(h->d[c], v)) break;
        h->d[i] = h->d[c]; i = c;
    }
    if (h->len) h->d[i] = v;
    return top;
}
static void hk_minheap_down(sp_t* d, size_t len, size_t i) {
    sp_t v = d[i];
    for (;;) {
        size_t c = 2 * i + 1;
        if (c >= len) break;
        if (c + 1 < len && hk_gt(d[c], d[c + 1])) c++;
        if (!hk_gt(v, d[c])) break;
        d[i] = d[c]; i = c;
    }
    d[i] = v;
}
/* FixedLengthPriorityQueue::push on keys; returns 1 if v was kept */
static int hk_flpq_push(flpq_t* q, sp_t v) {
    if (q->len < q->cap) {
        size_t i = q->len++;
        while (i > 0) { size_t p = (i - 1) / 2; if (!hk_gt(q->d[p], v)) break; q->d[i] = q->d[p]; i = p; }
        q->d[i] = v;
        return 1;
    }
    if (hk_gt(v, q->d[0])) { q->d[0] = v; hk_minheap_down(q->d, q->len, 0); return 1; }
    return 0;
}
/* search_on_level as oracle/hnsw.c states it, every comparison on keys */
static void hk_search_on_level(hnsw_t* h, scorer_t* s, sp_t level_entry, uint32_t lvl, uint32_t ef) {
    tctx_t* t = s->t;
    t->stamp++;
    if (t->stamp == 0) { memset(t->visited, 0, sizeof(uint32_t) * h->n); t->stamp = 1; }
    t->visited[level_entry.idx] = t->stamp;
    flpq_t* nearest = &t->nearest; heap_t* cand = &t->cand;
    nearest->len = 0; nearest->cap = ef; cand->len = 0;
    if (hk_flpq_push(nearest, level_entry)) hk_maxheap_push(cand, level_entry);
    uint32_t limit = level_m(h, lvl);
    uint32_t ids[512], lk[512]; float sc[512];
    while (cand->len) {
        sp_t c = hk_maxheap_pop(cand);
        if (nearest->len && hk_gt(nearest->d[0], c)) break;
        uint32_t nl = read_links(h, c.idx, lvl, lk), n = 0;
        for (uint32_t i = 0; i < nl; i++) if (t->visited[lk[i]] != t->stamp) ids[n++] = lk[i];
        n = filter_ids(s, ids, n, limit);
        if (n) score_points(s, ids, n, sc);
        for (uint32_t i = 0; i < n; i++) {
            sp_t p = { ids[i], sc[i] };
            if (hk_flpq_push(nearest, p)) hk_maxheap_push(cand, p);
            t->visited[ids[i]] = t->stamp;
        }
    }
}
/* link_new_point as oracle/hnsw.c states it (serial: no locks), with hk_search_on_level */
static void hk_link_new_point(hnsw_t* h, tctx_t* t, uint32_t p, sp_t* sorted) {
    const uint32_t level = h->level[p];
    scorer_t s = { h, t, NULL, NULL, h->base + (size_t)p * h->dim, NULL };
    if (!h->has_entry) { h->entry = p; h->entry_level = level; h->has_entry = 1; return; }
    const uint32_t entry = h->entry, entry_level = h->entry_level;
    sp_t level_entry;
    if (entry_level > level) level_entry = search_entry(h, &s, entry, entry_level, level);
    else { level_entry.idx = entry; level_entry.score = score_internal(h, p, entry); }
    const uint32_t linking = level < entry_level ? level : entry_level;
    for (int cl = (int)linking; cl >= 0; cl--) {
        hk_search_on_level(h, &s, level_entry, (uint32_t)cl, h->ef_construct);
        memcpy(sorted, t->nearest.d, t->nearest.len * sizeof(sp_t));
        qsort(sorted, t->nearest.len, sizeof(sp_t), cmp_desc);
        if (t->nearest.len) level_entry = sorted[0];
        const uint32_t lm = level_m(h, (uint32_t)cl);
        fill_with_heuristic(h, h->links[p][cl], sorted, t->nearest.len, lm);
        for (uint32_t i = 0; i < h->links[p][cl][0]; i++) { const uint32_t o = h->links[p][cl][1 + i]; connect_with_heuristic(h, h->links[o][cl], p, o, lm); }
    }
    if (level > entry_level) { h->entry = p; h->entry_level = level; }
}

#define search_on_level hk_search_on_level
#define link_new_point hk_link_new_point
#define flpq_push hk_flpq_push
