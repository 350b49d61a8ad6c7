/*
 * hnsw_custom_ref.c — the checker of the device traversal's custom queries (qb_hnsw_search_custom_batch,
 * qb_hnsw_search_discover_batch): GraphLayers::search (lib/segment/src/index/hnsw_index/graph_layers.rs:530-561) over a plain
 * `links.bin`, level 0 as search_on_level (:108-148, algo 0) or search_on_level_acorn (:154-243, algo 1), with
 *   - a custom scorer: a point's E similarities through `sim` (the oracle's qo_similarity_f32), folded by the oracle's qo_custom_score /
 *     qo_feedback_score (custom_query_scorer.rs:78-111), or a per-call callback (e.g. qb_score_points on a custom SQ8 scorer);
 *   - custom_entry_points restating get_entry_point (graph_layers.rs:506-528) over point_level (view.rs:354-369);
 *   - `keyed` = 1: every level-0 comparison (nearest insertion and eviction, candidate order, the stop test) on (score desc, id asc)
 *     keys, the device's tie order; keyed = 0 is the reference's score-only order.  The greedy descent is score-only either way, as on
 *     the device.
 * The traversal is the one of tests/hnsw_acorn_ref.c statement by statement, with the comparisons routed through gt / lt;
 * tests/test_hnsw_custom_cpu.py checks that, unkeyed and with a one-example query, both give the same lists, hops and scored points.
 * Filter: optional bitmap, bit = 1 -> the point fails ScorerFilters::check_vector.
 */
#define _GNU_SOURCE
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define API __attribute__((visibility("default")))

typedef struct { uint32_t idx; float score; } sp_t;
typedef float (*qc_sim_fn)(int distance, const float* q, const float* v, size_t n);
typedef void (*qc_score_cb)(void* user, const uint32_t* ids, uint32_t n, float* scores);
typedef float (*qc_custom_fn)(int kind, uint32_t n_a, uint32_t n_b, const float* sims, uint64_t stride);              /* qo_custom_score */
typedef float (*qc_feedback_fn)(uint32_t n_pairs, float a, const float* partial, const float* sims, uint64_t stride);  /* qo_feedback_score */

typedef struct {
    uint64_t n, levels, n_nb, n_off;
    uint64_t* level_offsets;
    uint32_t* reindex;
    uint32_t* neighbors;
    uint64_t* offsets;
    uint32_t m, m0;
} graph_t;

/* GraphLinks::links (view.rs:203-215): level 0 is indexed by point id, upper levels by level_offsets[l] + reindex[p] */
static uint32_t links_of(const graph_t* g, uint32_t p, uint32_t lvl, const uint32_t** out) {
    const uint64_t idx = lvl == 0 ? p : g->level_offsets[lvl] + g->reindex[p];
    const uint64_t b = g->offsets[idx], e = g->offsets[idx + 1];
    *out = g->neighbors + b;
    return (uint32_t)(e - b);
}

API void* qc_graph_load(const uint8_t* bin, uint64_t n_bytes, uint32_t m, uint32_t m0) {
    if (n_bytes < 64) return NULL;
    uint64_t hdr[5];
    memcpy(hdr, bin, sizeof(hdr));
    graph_t* g = (graph_t*)calloc(1, sizeof(graph_t));
    g->n = hdr[0]; g->levels = hdr[1]; g->n_nb = hdr[2]; g->n_off = hdr[3];
    const uint64_t pad = hdr[4];
    if (64 + 8 * g->levels + 4 * g->n + 4 * g->n_nb + pad + 8 * g->n_off > n_bytes) { free(g); return NULL; }
    g->m = m; g->m0 = m0;
    const uint8_t* p = bin + 64;
    g->level_offsets = (uint64_t*)malloc(8 * g->levels + 8); memcpy(g->level_offsets, p, 8 * g->levels); p += 8 * g->levels;
    g->reindex = (uint32_t*)malloc(4 * g->n + 4); memcpy(g->reindex, p, 4 * g->n); p += 4 * g->n;
    g->neighbors = (uint32_t*)malloc(4 * g->n_nb + 4); memcpy(g->neighbors, p, 4 * g->n_nb); p += 4 * g->n_nb + pad;
    g->offsets = (uint64_t*)malloc(8 * g->n_off + 8); memcpy(g->offsets, p, 8 * g->n_off);
    return g;
}

API void qc_graph_free(void* gp) {
    graph_t* g = (graph_t*)gp;
    if (!g) return;
    free(g->level_offsets); free(g->reindex); free(g->neighbors); free(g->offsets); free(g);
}

/* ---- per-search state ---------------------------------------------------------------------------------------- */
typedef struct {
    const graph_t* g;
    const float* base; uint32_t dim; int distance; qc_sim_fn sim;
    qc_score_cb cb; void* user;
    const uint64_t* filtered;
    uint32_t* hop1; uint32_t* hop2; uint32_t stamp;      /* visited lists: stamp == current search <=> visited */
    sp_t* nearest; size_t n_len, n_cap;                 /* FixedLengthPriorityQueue: min-heap on score */
    sp_t* cand; size_t c_len, c_cap;                    /* BinaryHeap: max-heap on score */
    uint32_t* to_score; uint32_t* to_explore; float* sc; size_t buf_cap;
    uint64_t calls, scored, marks1, marks2;             /* scorer calls with n > 0, scored points, visited-list entries */
    int keyed;                                          /* level-0 comparisons on (score desc, id asc) keys */
    const float* ex; uint32_t n_ex; int ckind; uint32_t n_a, n_b; const float* coef;   /* the query: n_ex examples */
    qc_custom_fn cfold; qc_feedback_fn ffold; float* sims;
    const uint32_t* cep; uint32_t n_cep;                /* custom entry points */
} ctx_t;

/* the device's key (qb_pack_key): orderable score bits, then the inverted id */
static uint64_t key_of(sp_t v) {
    uint32_t u; memcpy(&u, &v.score, 4);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ((uint64_t)u << 32) | (uint64_t)(0xFFFFFFFFu - v.idx);
}
static int gt(const ctx_t* c, sp_t a, sp_t b) { return c->keyed ? key_of(a) > key_of(b) : a.score > b.score; }
static int lt(const ctx_t* c, sp_t a, sp_t b) { return c->keyed ? key_of(a) < key_of(b) : a.score < b.score; }

static int passes(const ctx_t* c, uint32_t id) { return !c->filtered || !((c->filtered[id >> 6] >> (id & 63)) & 1u); }

/* VisitedList::check_and_update_visited: returns whether it was already set */
static int check_and_update(ctx_t* c, uint32_t* list, uint32_t id) {
    const int was = list[id] == c->stamp;
    if (!was) { list[id] = c->stamp; if (list == c->hop1) c->marks1++; else c->marks2++; }
    return was;
}

static void score(ctx_t* c, const uint32_t* ids, uint32_t n, float* out) {
    if (!n) return;                                     /* an empty call meters nothing */
    c->calls++; c->scored += n;
    if (c->cb) { c->cb(c->user, ids, n, out); return; }
    for (uint32_t i = 0; i < n; i++) {                  /* custom scorer: E similarities, then Query::score_by */
        const float* v = c->base + (size_t)ids[i] * c->dim;
        for (uint32_t e = 0; e < c->n_ex; e++) c->sims[e] = c->sim(c->distance, c->ex + (size_t)e * c->dim, v, c->dim);
        out[i] = c->ckind == 5 ? c->ffold(c->n_a, c->coef[0], c->coef + 1, c->sims, 1) : c->cfold(c->ckind, c->n_a, c->n_b, c->sims, 1);
    }
}

static void maxheap_push(ctx_t* c, sp_t v) {
    if (c->c_len == c->c_cap) { c->c_cap = c->c_cap * 2 + 16; c->cand = (sp_t*)realloc(c->cand, c->c_cap * sizeof(sp_t)); }
    size_t i = c->c_len++;
    while (i > 0) { size_t p = (i - 1) / 2; if (!gt(c, v, c->cand[p])) break; c->cand[i] = c->cand[p]; i = p; }
    c->cand[i] = v;
}
static sp_t maxheap_pop(ctx_t* c) {
    sp_t top = c->cand[0], v = c->cand[--c->c_len];
    size_t i = 0;
    for (;;) {
        size_t ch = 2 * i + 1;
        if (ch >= c->c_len) break;
        if (ch + 1 < c->c_len && gt(c, c->cand[ch + 1], c->cand[ch])) ch++;
        if (!gt(c, c->cand[ch], v)) break;
        c->cand[i] = c->cand[ch]; i = ch;
    }
    if (c->c_len) c->cand[i] = v;
    return top;
}
static void minheap_down(const ctx_t* c, sp_t* d, size_t len, size_t i) {
    sp_t v = d[i];
    for (;;) {
        size_t ch = 2 * i + 1;
        if (ch >= len) break;
        if (ch + 1 < len && lt(c, d[ch + 1], d[ch])) ch++;
        if (!lt(c, d[ch], v)) break;
        d[i] = d[ch]; i = ch;
    }
    d[i] = v;
}
/* SearchContext::process_candidate (search_context.rs:31-40) over FixedLengthPriorityQueue::push */
static void process_candidate(ctx_t* c, sp_t v) {
    int added;
    if (c->n_len < c->n_cap) {
        size_t i = c->n_len++;
        while (i > 0) { size_t p = (i - 1) / 2; if (!lt(c, v, c->nearest[p])) break; c->nearest[i] = c->nearest[p]; i = p; }
        c->nearest[i] = v;
        added = 1;
    } else if (lt(c, c->nearest[0], v)) {
        c->nearest[0] = v; minheap_down(c, c->nearest, c->n_len, 0);
        added = 1;
    } else {
        added = 0;
    }
    if (added) maxheap_push(c, v);
}
/* SearchContext::lower_bound (search_context.rs:23-28) */
static float lower_bound(const ctx_t* c) { return c->n_len ? c->nearest[0].score : -INFINITY; }
/* `candidate.score < lower_bound` (graph_layers.rs:118-120, :165-167), on keys in keyed mode */
static int below_lower_bound(const ctx_t* c, sp_t cand) { return c->keyed ? (c->n_len && lt(c, cand, c->nearest[0])) : cand.score < lower_bound(c); }

static void reserve(ctx_t* c, size_t n) {
    if (n <= c->buf_cap) return;
    c->buf_cap = n * 2;
    c->to_score = (uint32_t*)realloc(c->to_score, c->buf_cap * 4);
    c->to_explore = (uint32_t*)realloc(c->to_explore, c->buf_cap * 4);
    c->sc = (float*)realloc(c->sc, c->buf_cap * 4);
}

/* search_entry_on_level (graph_layers.rs:279-316): FilteredScorer::score_points filters, then keeps the first level_m */
static sp_t search_entry_on_level(ctx_t* c, uint32_t entry, uint32_t lvl) {
    const uint32_t limit = lvl == 0 ? c->g->m0 : c->g->m;
    sp_t cur; cur.idx = entry; score(c, &entry, 1, &cur.score);
    int changed = 1;
    while (changed) {
        changed = 0;
        const uint32_t* l; uint32_t nl = links_of(c->g, cur.idx, lvl, &l), n = 0;
        reserve(c, nl);
        for (uint32_t i = 0; i < nl; i++) if (passes(c, l[i])) c->to_score[n++] = l[i];
        if (n > limit) n = limit;
        score(c, c->to_score, n, c->sc);
        for (uint32_t i = 0; i < n; i++) if (c->sc[i] > cur.score) { changed = 1; cur.idx = c->to_score[i]; cur.score = c->sc[i]; }
    }
    return cur;
}

/* search_on_level (graph_layers.rs:108-148) */
static void search_on_level(ctx_t* c, sp_t level_entry, uint32_t ef) {
    const uint32_t limit = c->g->m0;
    check_and_update(c, c->hop1, level_entry.idx);
    process_candidate(c, level_entry);
    while (c->c_len) {
        const sp_t cand = maxheap_pop(c);
        if (below_lower_bound(c, cand)) break;
        const uint32_t* l; const uint32_t nl = links_of(c->g, cand.idx, 0, &l);
        reserve(c, nl);
        uint32_t n = 0;
        for (uint32_t i = 0; i < nl; i++) if (c->hop1[l[i]] != c->stamp) c->to_score[n++] = l[i];
        uint32_t k = 0;                                         /* score_points(points_ids, limit): filter, then truncate */
        for (uint32_t i = 0; i < n; i++) if (passes(c, c->to_score[i])) c->to_score[k++] = c->to_score[i];
        if (k > limit) k = limit;
        score(c, c->to_score, k, c->sc);
        for (uint32_t i = 0; i < k; i++) {
            sp_t p = { c->to_score[i], c->sc[i] };
            process_candidate(c, p);
            check_and_update(c, c->hop1, p.idx);
        }
    }
    (void)ef;
}

/* search_on_level_acorn (graph_layers.rs:154-243) */
static void search_on_level_acorn(ctx_t* c, sp_t level_entry) {
    const graph_t* g = c->g;
    check_and_update(c, c->hop1, level_entry.idx);          /* hop1_visited_list starts with the level entry */
    process_candidate(c, level_entry);                      /* hop2_visited_list starts empty */
    const uint32_t hop1_limit = g->m0, hop2_limit = g->m0;
    while (c->c_len) {
        const sp_t cand = maxheap_pop(c);
        if (below_lower_bound(c, cand)) break;
        size_t n_score = 0, n_explore = 0;
        /* 1-hop neighbours, stored order; break once to_score reaches hop1_limit */
        const uint32_t* l; const uint32_t nl = links_of(g, cand.idx, 0, &l);
        reserve(c, nl);
        for (uint32_t i = 0; i < nl; i++) {
            const uint32_t hop1 = l[i];
            if (check_and_update(c, c->hop1, hop1)) continue;
            if (passes(c, hop1)) {
                c->to_score[n_score++] = hop1;
                if (n_score >= hop1_limit) break;
            } else {
                c->to_explore[n_explore++] = hop1;
            }
        }
        /* 2-hop neighbours: each explored list until to_score has grown by hop2_limit during it */
        for (size_t x = 0; x < n_explore; x++) {
            const size_t total_limit = n_score + hop2_limit;
            const uint32_t* l2; const uint32_t nl2 = links_of(g, c->to_explore[x], 0, &l2);
            reserve(c, n_score + nl2);
            for (uint32_t i = 0; i < nl2; i++) {
                const uint32_t hop2 = l2[i];
                if (c->hop1[hop2] == c->stamp || check_and_update(c, c->hop2, hop2)) continue;
                if (passes(c, hop2)) {
                    check_and_update(c, c->hop1, hop2);
                    c->to_score[n_score++] = hop2;
                    if (n_score >= total_limit) break;
                }
            }
        }
        /* score_points_unfiltered: all of to_score, no filter, no limit */
        score(c, c->to_score, (uint32_t)n_score, c->sc);
        for (size_t i = 0; i < n_score; i++) { sp_t p = { c->to_score[i], c->sc[i] }; process_candidate(c, p); }
    }
}

static int cmp_desc(const void* a, const void* b) {
    const sp_t* x = (const sp_t*)a; const sp_t* y = (const sp_t*)b;
    if (x->score > y->score) return -1;
    if (x->score < y->score) return 1;
    return (x->idx > y->idx) - (x->idx < y->idx);
}

static void ctx_init(ctx_t* c, const graph_t* g) {
    memset(c, 0, sizeof(*c));
    c->g = g;
    c->hop1 = (uint32_t*)calloc(g->n ? g->n : 1, 4);
    c->hop2 = (uint32_t*)calloc(g->n ? g->n : 1, 4);
}
static void ctx_free(ctx_t* c) { free(c->hop1); free(c->hop2); free(c->nearest); free(c->cand); free(c->to_score); free(c->to_explore); free(c->sc); free(c->sims); }

/* GraphLinksView::point_level (view.rs:354-369); the plain format's last level offset is offsets.len() - 1 */
static uint32_t point_level(const graph_t* g, uint32_t p) {
    const uint64_t r = g->reindex[p];
    for (uint64_t l = 1; l < g->levels; l++) {
        const uint64_t a = g->level_offsets[l], b = l + 1 < g->levels ? g->level_offsets[l + 1] : g->n_off - 1;
        if (r >= b - a) return (uint32_t)(l - 1);
    }
    return g->levels ? (uint32_t)(g->levels - 1) : 0;
}

/* GraphLayers::get_entry_point (graph_layers.rs:506-528): the custom entry points that pass the filter, the highest point level,
   Iterator::max_by_key's LAST maximum; none -> the given entry point.  Returns whether a custom entry point was taken. */
static int get_entry_point(const ctx_t* c, const uint32_t* cep, uint32_t n, uint32_t* entry, uint32_t* entry_level) {
    int found = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (!passes(c, cep[i])) continue;
        const uint32_t l = point_level(c->g, cep[i]);
        if (!found || l >= *entry_level) { found = 1; *entry = cep[i]; *entry_level = l; }
    }
    return found;
}

/* GraphLayers::search (graph_layers.rs:530-561) from a given entry point; stats[0..4) += calls, scored points, max hop1 / hop2
   visited-list entries of one search */
static uint32_t search_one(ctx_t* c, int algo, uint32_t entry, uint32_t entry_level, uint32_t top, uint32_t ef, sp_t* out, uint64_t* stats) {
    c->stamp++;
    c->calls = c->scored = c->marks1 = c->marks2 = 0;
    c->n_len = 0; c->c_len = 0;
    const uint32_t e = ef > top ? ef : top;
    if (e > c->n_cap) { c->n_cap = e; c->nearest = (sp_t*)realloc(c->nearest, sizeof(sp_t) * (e + 1)); }
    c->n_cap = e;
    if (c->cep) get_entry_point(c, c->cep, c->n_cep, &entry, &entry_level);
    /* search_entry (graph_layers.rs:247-277) */
    sp_t zero; int have = 0; uint32_t cur = entry;
    for (uint32_t lvl = entry_level; lvl > 0; lvl--) { zero = search_entry_on_level(c, cur, lvl); cur = zero.idx; have = 1; }
    if (!have) { zero.idx = entry; score(c, &entry, 1, &zero.score); }
    if (algo == 1) search_on_level_acorn(c, zero);
    else search_on_level(c, zero, e);
    qsort(c->nearest, c->n_len, sizeof(sp_t), cmp_desc);   /* into_iter_sorted().take(top) */
    const uint32_t n = c->n_len < top ? (uint32_t)c->n_len : top;
    memcpy(out, c->nearest, n * sizeof(sp_t));
    __atomic_fetch_add(&stats[0], c->calls, __ATOMIC_RELAXED);
    __atomic_fetch_add(&stats[1], c->scored, __ATOMIC_RELAXED);
    uint64_t m1 = __atomic_load_n(&stats[2], __ATOMIC_RELAXED);
    while (c->marks1 > m1 && !__atomic_compare_exchange_n(&stats[2], &m1, c->marks1, 0, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    uint64_t m2 = __atomic_load_n(&stats[3], __ATOMIC_RELAXED);
    while (c->marks2 > m2 && !__atomic_compare_exchange_n(&stats[3], &m2, c->marks2, 0, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    return n;
}

/* get_entry_point alone: the chosen (entry, level) in out[0..2); returns 1 if a custom entry point was taken */
API int qc_get_entry_point(void* gp, const uint64_t* filtered, const uint32_t* cep, uint32_t n, uint32_t entry, uint32_t entry_level, uint32_t* out) {
    ctx_t c; memset(&c, 0, sizeof(c));
    c.g = (graph_t*)gp; c.filtered = filtered;
    const int r = get_entry_point(&c, cep, n, &entry, &entry_level);
    out[0] = entry; out[1] = entry_level;
    return r;
}

/* one search scored through `cb` */
API uint32_t qc_search_cb(void* gp, int algo, int keyed, uint32_t entry, uint32_t entry_level, const uint32_t* cep, uint32_t n_cep, qc_score_cb cb, void* user,
                             const uint64_t* filtered, uint32_t top, uint32_t ef, sp_t* out, uint64_t* stats) {
    graph_t* g = (graph_t*)gp;
    ctx_t c; ctx_init(&c, g);
    c.cb = cb; c.user = user; c.filtered = filtered; c.keyed = keyed; c.cep = cep; c.n_cep = n_cep;
    const uint32_t n = search_one(&c, algo, entry, entry_level, top, ef, out, stats);
    ctx_free(&c);
    return n;
}

typedef struct {
    graph_t* g; int algo, keyed; uint32_t entry, entry_level;
    const float* ex; uint32_t n_ex, nq; int ckind; uint32_t n_a, n_b; const float* coef; qc_custom_fn cfold; qc_feedback_fn ffold;
    const uint32_t* cep; const uint32_t* cep_counts; uint32_t n_cep;
    const float* base; uint32_t dim; int distance; qc_sim_fn sim;
    const uint64_t* filtered; uint32_t top, ef; sp_t* out; uint32_t* counts; uint64_t* stats; uint32_t* next;
} custom_batch_t;

static void* custom_worker(void* ap) {
    custom_batch_t* a = (custom_batch_t*)ap;
    ctx_t c; ctx_init(&c, a->g);
    c.base = a->base; c.dim = a->dim; c.distance = a->distance; c.sim = a->sim; c.filtered = a->filtered; c.keyed = a->keyed;
    c.n_ex = a->n_ex; c.ckind = a->ckind; c.n_a = a->n_a; c.n_b = a->n_b; c.cfold = a->cfold; c.ffold = a->ffold;
    c.sims = (float*)malloc(4 * (size_t)a->n_ex);
    for (;;) {
        const uint32_t i = __atomic_fetch_add(a->next, 1, __ATOMIC_RELAXED);
        if (i >= a->nq) break;
        c.ex = a->ex + (size_t)i * a->n_ex * a->dim;
        c.coef = a->coef ? a->coef + (size_t)i * (1 + a->n_a) : NULL;
        c.cep = a->cep ? a->cep + (size_t)i * a->n_cep : NULL;
        c.n_cep = a->cep ? a->cep_counts[i] : 0;
        a->counts[i] = search_one(&c, a->algo, a->entry, a->entry_level, a->top, a->ef, a->out + (size_t)i * a->top, a->stats);
    }
    ctx_free(&c);
    return NULL;
}

/* many custom searches: query i's n_ex preprocessed examples at ex + i * n_ex * dim (the qb_scorer_create_custom layout), feedback
   coefficients [a, partial...] at coef + i * (1 + n_a), custom entry points cep[i * n_cep ..] (cep_counts[i] of them) or none */
API void qc_search_custom_batch(void* gp, int algo, int keyed, uint32_t entry, uint32_t entry_level, const float* ex, uint32_t n_ex, uint32_t nq, int ckind,
                                uint32_t n_a, uint32_t n_b, const float* coef, qc_custom_fn cfold, qc_feedback_fn ffold, const uint32_t* cep,
                                const uint32_t* cep_counts, uint32_t n_cep, const float* base, uint32_t dim, int distance, qc_sim_fn sim,
                                const uint64_t* filtered, uint32_t top, uint32_t ef, uint32_t threads, sp_t* out, uint32_t* counts, uint64_t* stats) {
    if (threads < 1) threads = 1;
    if (threads > nq) threads = nq ? nq : 1;
    uint32_t next = 0;
    custom_batch_t a = { (graph_t*)gp, algo, keyed, entry, entry_level, ex, n_ex, nq, ckind, n_a, n_b, coef, cfold, ffold, cep, cep_counts, n_cep,
                         base, dim, distance, sim, filtered, top, ef, out, counts, stats, &next };
    pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * threads);
    for (uint32_t i = 0; i < threads; i++) pthread_create(&th[i], NULL, custom_worker, &a);
    for (uint32_t i = 0; i < threads; i++) pthread_join(th[i], NULL);
    free(th);
}
