/* sparse_ref.c — the checker of the device sparse index: a C restatement of the reference's inverted index and SearchContext.
 *   PostingBuilder::build      lib/sparse/src/index/posting_list.rs:140-170 (sorted by id, max_next_weight from the end, -inf last)
 *   TopK                       lib/common/common/src/top_k.rs:22-64 (threshold from f32::MIN, push when score > threshold, at 2k keep k)
 *   SearchContext::new/search  lib/sparse/src/index/search_context.rs:42-87, 146-414 (batches of 10 001 ids, retain, last list,
 *                              promote with max_by (the last longest list), prune)
 *   SearchContext::plain_search :92-143 with score_vectors (lib/sparse/src/common/sparse_vector.rs:66-90)
 * The query is a RemappedSparseVector: the caller has sorted it by dim and dropped the dims the index does not know.
 * TopK's kept entries order by (score desc, id asc) — the device's keys; `keyed = 0` breaks ties by id desc instead, another order the
 * reference's select_nth_unstable allows.  Compile with -ffp-contract=off: every product and sum rounds as in the reference. */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define EXPORT __attribute__((visibility("default")))
#define BATCH 10000u

typedef struct { uint32_t id; float w, mnw; } elem;
typedef struct { elem* e; uint32_t n; } plist;
typedef struct { uint32_t n_points, n_dims; plist* lists; } sr_index;

static uint32_t orderable(float s) {
    uint32_t u;
    memcpy(&u, &s, 4);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

EXPORT void* sr_index_new(uint32_t n_points, uint32_t n_dims, const uint64_t* indptr, const uint32_t* dims, const float* w) {
    sr_index* x = calloc(1, sizeof(sr_index));
    x->n_points = n_points; x->n_dims = n_dims;
    x->lists = calloc(n_dims ? n_dims : 1, sizeof(plist));
    uint32_t* cnt = calloc(n_dims ? n_dims : 1, 4);
    for (uint64_t e = 0; e < indptr[n_points]; ++e) cnt[dims[e]]++;
    for (uint32_t d = 0; d < n_dims; ++d) x->lists[d].e = malloc((cnt[d] ? cnt[d] : 1) * sizeof(elem));
    /* rows in id order: each list is already sorted by id */
    for (uint32_t r = 0; r < n_points; ++r)
        for (uint64_t e = indptr[r]; e < indptr[r + 1]; ++e) {
            plist* L = &x->lists[dims[e]];
            L->e[L->n++] = (elem){r, w[e], 0.0f};
        }
    for (uint32_t d = 0; d < n_dims; ++d) {
        float m = -INFINITY;
        for (uint32_t i = x->lists[d].n; i-- > 0;) {
            x->lists[d].e[i].mnw = m;
            m = fmaxf(m, x->lists[d].e[i].w);
        }
    }
    free(cnt);
    return x;
}

EXPORT void sr_index_free(void* p) {
    sr_index* x = p;
    for (uint32_t d = 0; d < x->n_dims; ++d) free(x->lists[d].e);
    free(x->lists);
    free(x);
}

/* ---- TopK */
typedef struct { uint64_t* e; uint32_t k, len; float thr; int keyed; } topk;

static uint64_t key_of(const topk* t, float s, uint32_t id) { return ((uint64_t)orderable(s) << 32) | (t->keyed ? 0xFFFFFFFFu - id : id); }
static float key_score(uint64_t k) {
    uint32_t o = (uint32_t)(k >> 32), u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
    float f;
    memcpy(&f, &u, 4);
    return f;
}
static uint32_t key_id(const topk* t, uint64_t k) { return t->keyed ? 0xFFFFFFFFu - (uint32_t)k : (uint32_t)k; }
static int desc(const void* a, const void* b) {
    const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
    return x < y ? 1 : (x > y ? -1 : 0);
}
static void topk_push(topk* t, float s, uint32_t id) {
    if (!(s > t->thr)) return;
    t->e[t->len++] = key_of(t, s, id);
    if (t->len == 2 * t->k) {
        qsort(t->e, t->len, 8, desc);
        t->thr = key_score(t->e[t->k - 1]);
        t->len = t->k;
    }
}

/* ---- SearchContext */
typedef struct { const elem* e; uint32_t n, pos, dim; float qw; } iter;
typedef struct {
    const sr_index* x;
    iter* it; uint32_t n_it;
    uint32_t qlen;
    int has_min; uint32_t min_id, max_id;
    int use_pruning;
    topk top;
} ctx;

EXPORT void* sr_ctx_new(const void* idx, const uint32_t* qd, const float* qw, uint32_t qn, uint32_t top, int reliable, int keyed) {
    const sr_index* x = idx;
    ctx* c = calloc(1, sizeof(ctx));
    c->x = x; c->qlen = qn;
    c->it = calloc(qn ? qn : 1, sizeof(iter));
    uint32_t mn = 0xFFFFFFFFu, mx = 0;
    int nonneg = 1;
    for (uint32_t i = 0; i < qn; ++i) {
        nonneg = nonneg && qw[i] >= 0.0f;
        if (qd[i] >= x->n_dims) continue;
        const plist* L = &x->lists[qd[i]];
        if (!L->n) continue;
        if (L->e[0].id < mn) mn = L->e[0].id;
        if (L->e[L->n - 1].id > mx) mx = L->e[L->n - 1].id;
        c->it[c->n_it++] = (iter){L->e, L->n, 0, qd[i], qw[i]};
    }
    c->has_min = 1; c->min_id = mn; c->max_id = mx;
    c->use_pruning = reliable && nonneg;
    c->top = (topk){calloc(2 * (size_t)top + 1, 8), top, 0, -FLT_MAX, keyed};
    return c;
}

EXPORT void sr_ctx_free(void* p) {
    ctx* c = p;
    free(c->it); free(c->top.e); free(c);
}

EXPORT uint32_t sr_ctx_list_len(const void* p, uint32_t i) { const ctx* c = p; return c->it[i].n - c->it[i].pos; }
EXPORT uint32_t sr_ctx_list_dim(const void* p, uint32_t i) { const ctx* c = p; return c->it[i].dim; }

static int next_min_id(const iter* it, uint32_t n, uint32_t* out) {
    int found = 0;
    for (uint32_t i = 0; i < n; ++i)
        if (it[i].pos < it[i].n && (!found || it[i].e[it[i].pos].id < *out)) { *out = it[i].e[it[i].pos].id; found = 1; }
    return found;
}

/* skip_to (posting_list.rs:268-290): binary search of [pos, n) for id; Ok -> its position, Err -> the insertion point */
static int skip_to(iter* t, uint32_t id, elem* found) {
    if (t->pos >= t->n) return 0;
    uint32_t lo = t->pos, hi = t->n;
    while (lo < hi) { const uint32_t m = lo + (hi - lo) / 2; if (t->e[m].id < id) lo = m + 1; else hi = m; }
    t->pos = lo;
    if (lo < t->n && t->e[lo].id == id) { if (found) *found = t->e[lo]; return 1; }
    return 0;
}

EXPORT void sr_ctx_promote(void* p) {
    ctx* c = p;
    if (!c->n_it) return;
    uint32_t best = 0;
    for (uint32_t i = 1; i < c->n_it; ++i)   /* max_by: the last maximum wins */
        if (c->it[i].n - c->it[i].pos >= c->it[best].n - c->it[best].pos) best = i;
    if (best != 0) { const iter t = c->it[0]; c->it[0] = c->it[best]; c->it[best] = t; }
}

EXPORT int sr_ctx_prune(void* p, float min_score) {
    ctx* c = p;
    if (!c->n_it) return 0;
    iter* L = &c->it[0];
    if (L->pos >= L->n) return 0;
    const elem el = L->e[L->pos];
    uint32_t nm = 0;
    const int some = next_min_id(c->it + 1, c->n_it - 1, &nm);
    const float contrib = fmaxf(el.w, el.mnw) * L->qw;
    if (some) {
        if (nm <= el.id) return 0;
        if (contrib <= min_score) {
            const uint32_t before = L->pos;
            skip_to(L, nm, NULL);
            return before != L->pos;
        }
    } else if (contrib <= min_score) {
        L->pos = L->n;
        return 1;
    }
    return 0;
}

static int is_deleted(const uint64_t* del, uint32_t id) { return del && ((del[id >> 6] >> (id & 63)) & 1u); }

static uint32_t finish(ctx* c, uint32_t* out_ids, float* out_scores) {
    topk* t = &c->top;
    qsort(t->e, t->len, 8, desc);
    const uint32_t n = t->len < t->k ? t->len : t->k;
    for (uint32_t i = 0; i < n; ++i) { out_ids[i] = key_id(t, t->e[i]); out_scores[i] = key_score(t->e[i]); }
    return n;
}

EXPORT uint32_t sr_ctx_search(void* p, const uint64_t* deleted, uint32_t* out_ids, float* out_scores, uint64_t* cpu) {
    ctx* c = p;
    if (!c->n_it) return 0;
    for (uint32_t i = 0; i < c->n_it; ++i) *cpu += (uint64_t)(c->it[i].n - c->it[i].pos) * 4;
    float* scores = malloc((BATCH + 1) * sizeof(float));
    float best_min = -FLT_MAX;
    for (;;) {
        if (!c->has_min) break;
        const uint32_t start = c->min_id;
        const uint32_t last = (uint64_t)start + BATCH < c->max_id ? start + BATCH : c->max_id;
        const uint32_t blen = last - start + 1;
        for (uint32_t i = 0; i < blen; ++i) scores[i] = 0.0f;
        for (uint32_t j = 0; j < c->n_it; ++j) {
            iter* t = &c->it[j];
            while (t->pos < t->n && t->e[t->pos].id <= last) {
                scores[t->e[t->pos].id - start] += t->e[t->pos].w * t->qw;
                t->pos++;
            }
        }
        for (uint32_t i = 0; i < blen; ++i)
            if (scores[i] != 0.0f && scores[i] > c->top.thr && !is_deleted(deleted, start + i)) topk_push(&c->top, scores[i], start + i);
        uint32_t n = 0;
        for (uint32_t j = 0; j < c->n_it; ++j) if (c->it[j].pos != c->it[j].n) c->it[n++] = c->it[j];
        c->n_it = n;
        c->has_min = next_min_id(c->it, c->n_it, &c->min_id);
        if (c->n_it == 0) break;
        if (c->n_it == 1) {
            iter* t = &c->it[0];
            for (; t->pos < t->n; ++t->pos)
                if (!is_deleted(deleted, t->e[t->pos].id)) topk_push(&c->top, t->e[t->pos].w * t->qw, t->e[t->pos].id);
            break;
        }
        if (c->use_pruning && c->top.len >= c->top.k) {
            const float nms = c->top.thr;
            if (nms == best_min) continue;
            best_min = nms;
            sr_ctx_promote(c);
            if (sr_ctx_prune(c, nms)) c->has_min = next_min_id(c->it, c->n_it, &c->min_id);
        }
    }
    free(scores);
    return finish(c, out_ids, out_scores);
}

static int cmp_u32(const void* a, const void* b) {
    const uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b;
    return x < y ? -1 : (x > y);
}

/* score_vectors over the matched (query dim, stored weight) pairs, both ascending: 0 + sum of stored * query */
EXPORT uint32_t sr_ctx_plain(void* p, const uint32_t* qd, const float* qw, const uint32_t* ids, uint32_t n_ids, uint32_t* out_ids, float* out_scores,
                             uint64_t* cpu) {
    ctx* c = p;
    uint32_t* s = malloc((n_ids ? n_ids : 1) * 4);
    memcpy(s, ids, (size_t)n_ids * 4);
    qsort(s, n_ids, 4, cmp_u32);
    uint32_t* md = malloc((c->n_it ? c->n_it : 1) * 4);
    float* mw = malloc((c->n_it ? c->n_it : 1) * 4);
    for (uint32_t k = 0; k < n_ids; ++k) {
        uint32_t nm = 0;
        for (uint32_t j = 0; j < c->n_it; ++j) {
            elem f;
            if (skip_to(&c->it[j], s[k], &f)) { md[nm] = c->it[j].dim; mw[nm++] = f.w; }
        }
        if (!nm) continue;
        *cpu += c->qlen + (uint64_t)nm * 4;
        float score = 0.0f;
        uint32_t i = 0, j = 0;
        while (i < nm && j < c->qlen) {
            if (md[i] < qd[j]) ++i;
            else if (md[i] > qd[j]) ++j;
            else { score += mw[i] * qw[j]; ++i; ++j; }
        }
        topk_push(&c->top, score, s[k]);
    }
    free(s); free(md); free(mw);
    return finish(c, out_ids, out_scores);
}
