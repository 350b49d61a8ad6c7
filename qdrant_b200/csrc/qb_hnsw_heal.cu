// qb_hnsw_heal.cu — incremental HNSW construction on the device (qb_hnsw_build_incremental): the old graph's lists that link to a point
// that has gone are healed, the lists are renumbered into the new storage's ids, and only the new points are inserted.
//
// The reference's path (hnsw/build.rs:225-357 with an old index): OldIndexCandidate::evaluate gives old_to_new (the caller's input
// here), GraphLayersHealer (graph_layers_healer.rs) heals, save_into_builder renumbers, then the points the old graph did not have are
// linked.  Restated in that order:
//   1. to-heal items: every (point, level) of the old graph whose first level_m links include an unmapped point, point ascending, then
//      level ascending (to_edges_impl, graph_links/links.rs:174-186), over every old point, unmapped ones included: the reference heals
//      points that are going away too, and their backlinks can displace live links that the renumbering then drops.  Kept as it is.
//   2. heal (heal_point_on_level, :160-207): the stack-based search through unmapped points (search_shortcuts_on_level, :82-158) fills
//      an ef_construct-sized `nearest` with the border points; fill_from_sorted_with_heuristic keeps up to level_m - |valid links| of
//      them and the valid links follow in their order; then a backlink to the item in each kept link's list unless it is there
//      already (connect_with_heuristic).  The query is the item's stored row (the reference preprocesses it once more, which leaves a
//      normalised cosine row as it is).
//   3. One deliberate deviation: the reference heals its items in parallel under per-list locks, so what an item reads depends on the
//      race.  Here every level heals in two phases.  Phase 1: every item searches the lists as loaded and writes only its own list
//      and its (target << 32 | item, item's point) backlink pairs.  Phase 2: the pairs are radix-sorted and each target applies its
//      sources in item order, testing "already linked" when the pair is applied (an earlier pair can evict the source).  The graph
//      is then a pure function of the inputs; tests/hnsw_build_incr_ref.c restates it on the CPU.
//   4. renumber (save_into_builder, :236-256): each mapped point's lists move to its new id without the unmapped links, straight into
//      qb_hnsw_build's tables (hb_run's layout); the entry is EntryPoints::new_point over the mapped points in old-offset order
//      (entry_points.rs:46-86): the first with the strictly highest level.
//   5. insert the new points with qb_hnsw_build's schedule (qb_hnsw_build.cuh, hb_plan with the mapped points given): the first
//      serial_points one at a time, then batches cut where the level changes.  A first new point above the old top links up to the
//      old top from the old entry and is the entry of every later point (link_new_point, graph_layers_builder.rs:417-475).
//
// Kernels: hnsw_heal_kernel (phase 1) gives each item one persistent 128-thread CTA (work stealing over the items).  The DFS stack is
// per-CTA global scratch; `nearest` is a sorted array of keys (score desc, id asc) in shared memory; each popped point's unvisited links
// are scored by the 8-lane chains (hnsw_score_rows) and the heuristic runs on the CTA's 16 groups as the insert kernel's does.  A stack
// that would overflow abandons its item; the host reruns those items with a larger stack (the count of reruns is reported under
// QB_VERBOSE).  hnsw_heal_backlink_kernel (phase 2) is the build's backlink kernel plus the membership test.  They live in this
// object of their own so that qb_hnsw_build.o keeps its machine code.
#include "qb_hnsw_build.cuh"

namespace {

constexpr uint32_t HEAL_STACK = 16384;   // DFS stack entries per CTA on the first run

// the old graph's lists while healing: level l's table [N_l][lm] in the plain format's row order (level 0 by id, level l >= 1 by the
// old reindex), HNSW_EMPTY padded
struct HealArgs {
    const uint32_t* old_tab;       // as loaded: the first lm links of each list (phase 1 reads these)
    uint32_t* tab;                 // healed (phase 1 writes its items' rows, phase 2 the backlinks)
    const uint32_t* remap;         // row of a point (null: the id)
    const uint32_t* o2n;           // old_to_new (HNSW_EMPTY: not carried over)
    const uint32_t* items;         // the level's to-heal points, in order
    const uint32_t* sel;           // a rerun: the item indices to heal (null: all n_items)
    uint32_t n_items, n_work, lm, ef;
    unsigned long long* stack; uint32_t stack_cap;    // [grid][stack_cap]: (score bits << 32 | id)
    uint32_t* visited; uint64_t visited_words;        // [grid][visited_words], left clean
    uint32_t* vlog; uint32_t vlog_cap;                // [grid][vlog_cap]
    unsigned int* work;
    unsigned long long* tkey; uint32_t* tval;         // [n_items][lm] backlink pairs (~0 = none)
    uint32_t* ovf; unsigned int* n_ovf;               // items whose stack overflowed
};

__device__ __forceinline__ uint32_t heal_row(const HealArgs& a, uint32_t id) { return a.remap ? a.remap[id] : id; }
__device__ __forceinline__ bool heal_gone(const HealArgs& a, uint32_t id) { return a.o2n[id] == HNSW_EMPTY; }

template <int KIND, int METRIC>
__global__ void __launch_bounds__(HB_THREADS) hnsw_heal_kernel(const HnswParams p, const HealArgs a) {
    extern __shared__ unsigned long long s_near[];   // [2][ef]: nearest, sorted desc, and the merge's target
    __shared__ uint32_t s_ids[HNSW_MAX_LINKS], s_valid[HNSW_MAX_LINKS], s_sel[HNSW_MAX_LINKS];
    __shared__ float s_sc[HNSW_MAX_LINKS];
    __shared__ unsigned long long s_new[HNSW_MAX_LINKS], s_newsorted[HNSW_MAX_LINKS];
    __shared__ uint32_t s_work, s_n, s_nnew, s_cnt, s_buf, s_nvalid, s_cand, s_ovf, s_nlog, s_top;
    const int tid = threadIdx.x;
    const uint32_t lm = a.lm, ef = a.ef;
    uint32_t* vis = a.visited + (size_t)blockIdx.x * a.visited_words;
    uint32_t* vlog = a.vlog + (size_t)blockIdx.x * a.vlog_cap;
    unsigned long long* stack = a.stack + (size_t)blockIdx.x * a.stack_cap;
    // check_and_update_visited, one thread
    auto visit = [&](uint32_t id) -> bool {
        const uint32_t w = id >> 5, b = 1u << (id & 31);
        if (vis[w] & b) return true;
        vis[w] |= b;
        if (s_nlog < a.vlog_cap) vlog[s_nlog] = id;
        ++s_nlog;
        return false;
    };
    auto push = [&](uint32_t id, float s) {
        if (s_top == a.stack_cap) { s_ovf = 1; return; }
        stack[s_top++] = ((unsigned long long)__float_as_uint(s) << 32) | id;
    };
    for (;;) {
        if (tid == 0) s_work = atomicAdd(a.work, 1u);
        __syncthreads();
        const uint32_t w = s_work;
        if (w >= a.n_work) break;
        const uint32_t it = a.sel ? a.sel[w] : w, pt = a.items[it];
        const uint8_t* qrow = p.rows + (size_t)pt * p.stride;
        const uint32_t* orow = a.old_tab + (size_t)heal_row(a, pt) * lm;
        // the item's links: the valid ones are visited (already linked), the others are scored onto the stack in link order
        if (tid == 0) {
            s_nlog = 0; s_top = 0; s_ovf = 0; s_cnt = 0; s_buf = 0;
            visit(pt);
            uint32_t nv = 0, n = 0;
            for (uint32_t j = 0; j < lm; ++j) {
                const uint32_t l = orow[j];
                if (l == HNSW_EMPTY) break;
                if (!heal_gone(a, l)) { visit(l); s_valid[nv++] = l; }
                else s_ids[n++] = l;
            }
            s_nvalid = nv; s_n = n;
        }
        __syncthreads();
        hnsw_score_rows<KIND, METRIC, HB_THREADS / 8>(p, qrow, s_ids, s_n, tid, [&](uint32_t j, float s) { s_sc[j] = s; });
        __syncthreads();
        if (tid == 0) for (uint32_t j = 0; j < s_n && !s_ovf; ++j) push(s_ids[j], s_sc[j]);
        __syncthreads();
        // search_shortcuts_on_level: pop, skip when not promising or visited, score the unvisited links of the rest
        for (;;) {
            if (tid == 0) {
                uint32_t cand = HNSW_EMPTY;
                while (s_top > 0 && !s_ovf) {
                    const unsigned long long e = stack[--s_top];
                    const uint32_t id = (uint32_t)e;
                    const float sc = __uint_as_float((uint32_t)(e >> 32));
                    if (s_cnt == ef && sc < qb_key_score(s_near[s_buf * ef + s_cnt - 1])) continue;
                    if (visit(id)) continue;
                    cand = id;
                    break;
                }
                uint32_t n = 0;
                if (cand != HNSW_EMPTY) {
                    const uint32_t* crow = a.old_tab + (size_t)heal_row(a, cand) * lm;
                    for (uint32_t j = 0; j < lm; ++j) {
                        const uint32_t l = crow[j];
                        if (l == HNSW_EMPTY) break;
                        if (!((vis[l >> 5] >> (l & 31)) & 1u)) s_ids[n++] = l;
                    }
                }
                s_cand = s_ovf ? HNSW_EMPTY : cand; s_n = n;
            }
            __syncthreads();
            if (s_cand == HNSW_EMPTY) break;
            hnsw_score_rows<KIND, METRIC, HB_THREADS / 8>(p, qrow, s_ids, s_n, tid, [&](uint32_t j, float s) { s_sc[j] = s; });
            __syncthreads();
            if (tid == 0) {   // border points to `nearest`, gone points onto the stack, in link order
                uint32_t nb = 0;
                for (uint32_t j = 0; j < s_n; ++j) {
                    if (!heal_gone(a, s_ids[j])) s_new[nb++] = qb_pack_key(s_sc[j], s_ids[j]);
                    else if (!s_ovf) push(s_ids[j], s_sc[j]);
                }
                s_nnew = nb;
            }
            __syncthreads();
            // FixedLengthPriorityQueue::push of each border point in turn keeps the ef best of the union: merge the sorted new keys
            const uint32_t nb = s_nnew, cnt = s_cnt;
            if (nb) {
                if ((uint32_t)tid < nb) {   // stable rank among the new keys (a point reached twice is kept twice, as the reference does)
                    const unsigned long long k = s_new[tid];
                    uint32_t r = 0;
                    for (uint32_t i = 0; i < nb; ++i) r += (s_new[i] > k || (s_new[i] == k && i < (uint32_t)tid)) ? 1u : 0u;
                    s_newsorted[r] = k;
                }
                __syncthreads();
                const unsigned long long* cur = s_near + (size_t)s_buf * ef;
                unsigned long long* nxt = s_near + (size_t)(s_buf ^ 1u) * ef;
                for (uint32_t i = tid; i < cnt; i += HB_THREADS) {   // an old key moves down by the new keys above it
                    const unsigned long long k = cur[i];
                    uint32_t lo = 0, hi = nb;
                    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (s_newsorted[mid] > k) lo = mid + 1; else hi = mid; }
                    if (i + lo < ef) nxt[i + lo] = k;
                }
                if ((uint32_t)tid < nb) {   // a new key goes below the old keys >= it
                    const unsigned long long k = s_newsorted[tid];
                    uint32_t lo = 0, hi = cnt;
                    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (cur[mid] >= k) lo = mid + 1; else hi = mid; }
                    if (tid + lo < ef) nxt[tid + lo] = k;
                }
                __syncthreads();
                if (tid == 0) { s_cnt = min(cnt + nb, ef); s_buf ^= 1u; }
            }
            __syncthreads();
        }
        if (s_ovf) {
            if (tid == 0) a.ovf[atomicAdd(a.n_ovf, 1u)] = it;
        } else {
            // fill_from_sorted_with_heuristic up to lm - |valid|, then the valid links
            const unsigned long long* near = s_near + (size_t)s_buf * ef;
            const uint32_t cnt = s_cnt, lim = lm - s_nvalid;
            uint32_t nsel = 0;
            for (uint32_t c = 0; c < cnt && nsel < lim; ++c) {
                const uint32_t cid = qb_key_id(near[c]);
                const float cs = qb_key_score(near[c]);
                bool beat = false;
                hnsw_score_rows<KIND, METRIC, HB_THREADS / 8>(p, p.rows + (size_t)cid * p.stride, s_sel, nsel, tid, [&](uint32_t, float s) { beat |= s > cs; });
                if (!__syncthreads_or(beat)) {
                    if (tid == 0) s_sel[nsel] = cid;
                    ++nsel;
                }
                __syncthreads();
            }
            uint32_t* row = a.tab + (size_t)heal_row(a, pt) * lm;
            const uint32_t total = nsel + s_nvalid;
            for (uint32_t j = tid; j < lm; j += HB_THREADS) {
                const uint32_t l = j < nsel ? s_sel[j] : (j < total ? s_valid[j - nsel] : HNSW_EMPTY);
                row[j] = l;
                a.tkey[(size_t)it * lm + j] = l != HNSW_EMPTY ? ((unsigned long long)l << 32) | it : ~0ull;
                a.tval[(size_t)it * lm + j] = pt;
            }
        }
        __syncthreads();
        // leave the bitmap clean
        if (s_nlog <= a.vlog_cap) {
            for (uint32_t i = tid; i < s_nlog; i += HB_THREADS) { const uint32_t id = vlog[i]; vis[id >> 5] = 0u; }
        } else {
            for (uint64_t i = tid; i < a.visited_words; i += HB_THREADS) vis[i] = 0u;
        }
        __syncthreads();
    }
}

// phase 2: connect_with_heuristic of every target in keys[0 .. n) (sorted; key = target << 32 | item, ~0 = none) with its sources in
// item order, one warp per target, unless the target's list holds the source when the pair is applied (heal_point_on_level, :193-206).
// The build's backlink kernel (hnsw_backlink_kernel, qb_hnsw_build.cu) with that test; links0 / m0 = the level's table and level_m,
// b_remap = its rows.
template <int KIND, int METRIC>
__global__ void __launch_bounds__(HB_WARPS * 32) hnsw_heal_backlink_kernel(const HnswParams p, const unsigned long long* __restrict__ keys,
                                                                           const uint32_t* __restrict__ vals, uint32_t n) {
    __shared__ unsigned long long s_key[HB_WARPS][HNSW_MAX_LINKS + 1], s_sorted[HB_WARPS][HNSW_MAX_LINKS + 1];
    __shared__ uint32_t s_ids[HB_WARPS][HNSW_MAX_LINKS + 1];
    const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31u, lm = p.m0;
    unsigned long long* wkey = s_key[w];
    unsigned long long* wsorted = s_sorted[w];
    uint32_t* wids = s_ids[w];
    for (uint32_t e = blockIdx.x * HB_WARPS + w; e < n; e += gridDim.x * HB_WARPS) {
        const uint32_t t = (uint32_t)(keys[e] >> 32);
        if (t == HNSW_EMPTY) break;
        if (e > 0 && (uint32_t)(keys[e - 1] >> 32) == t) continue;
        uint32_t* row = const_cast<uint32_t*>(p.links0) + (size_t)hnsw_build_row(p, t) * lm;
        const uint8_t* trow = p.rows + (size_t)t * p.stride;
        for (uint32_t e2 = e; e2 < n && (uint32_t)(keys[e2] >> 32) == t; ++e2) {
            const uint32_t src = vals[e2];
            const uint32_t a = lane < lm ? row[lane] : HNSW_EMPTY, b = lane + 32 < lm ? row[lane + 32] : HNSW_EMPTY;
            if (__any_sync(0xFFFFFFFFu, a == src || b == src)) continue;   // already linked
            const uint32_t cnt = __popc(__ballot_sync(0xFFFFFFFFu, a != HNSW_EMPTY)) + __popc(__ballot_sync(0xFFFFFFFFu, b != HNSW_EMPTY));
            if (cnt < lm) {
                if (lane == 0) row[cnt] = src;
                __syncwarp();
                continue;
            }
            if (lane < lm) wids[lane] = a;
            if (lane + 32 < lm) wids[lane + 32] = b;
            if (lane == 0) wids[lm] = src;
            __syncwarp();
            hnsw_score_rows<KIND, METRIC, HB_WARPS>(p, trow, wids, lm + 1, (int)lane, [&](uint32_t j, float s) { wkey[j] = qb_pack_key(s, wids[j]); });
            __syncwarp();
            for (uint32_t j = lane; j <= lm; j += 32) {   // stable rank: a healed list can hold a point twice (see the renumbering)
                const unsigned long long k = wkey[j];
                uint32_t r = 0;
                for (uint32_t i = 0; i <= lm; ++i) r += (wkey[i] > k || (wkey[i] == k && i < j)) ? 1u : 0u;
                wsorted[r] = k;
            }
            __syncwarp();
            uint32_t nsel = 0;
            for (uint32_t c = 0; c <= lm && nsel < lm; ++c) {
                const uint32_t cid = qb_key_id(wsorted[c]);
                const float cs = qb_key_score(wsorted[c]);
                bool beat = false;
                hnsw_score_rows<KIND, METRIC, HB_WARPS>(p, p.rows + (size_t)cid * p.stride, wids, nsel, (int)lane, [&](uint32_t, float s) { beat |= s > cs; });
                beat = __any_sync(0xFFFFFFFFu, beat);
                if (!beat) {
                    if (lane == 0) wids[nsel] = cid;
                    ++nsel;
                }
                __syncwarp();
            }
            for (uint32_t j = lane; j < lm; j += 32) row[j] = j < nsel ? wids[j] : HNSW_EMPTY;
            __syncwarp();
        }
    }
}

// the old graph's level table from its plain arrays: row r of level l = the first lm links of plain row lo + r
__global__ void hnsw_heal_table_kernel(const uint64_t* __restrict__ offsets, const uint32_t* __restrict__ neighbors, uint64_t lo, uint64_t rows, uint32_t lm,
                                       uint32_t* __restrict__ tab) {
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t b = offsets[lo + r], len = offsets[lo + r + 1] - b;
        for (uint32_t j = 0; j < lm; ++j) tab[r * lm + j] = j < len ? neighbors[b + j] : HNSW_EMPTY;
    }
}

// a bit per level whose list (its first lm links) holds an unmapped point: flags[p] bit l
__global__ void hnsw_heal_flags_kernel(const uint32_t* __restrict__ tab, uint64_t rows, uint32_t lm, const uint32_t* __restrict__ o2n, uint32_t* __restrict__ flags,
                                       uint32_t bit) {
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (uint64_t)gridDim.x * blockDim.x) {
        bool gone = false;
        for (uint32_t j = 0; j < lm; ++j) {
            const uint32_t l = tab[r * lm + j];
            if (l == HNSW_EMPTY) break;
            gone |= o2n[l] == HNSW_EMPTY;
        }
        if (gone) flags[r] |= bit;
    }
}

// save_into_builder: each mapped point's healed list on level l, unmapped links dropped and the rest renamed, into the build table's
// row of its new id (level 0: the id, else remap_new[id]).  A link the list holds twice is kept once: the shortcut search can reach a
// border point from two gone points, and with Dot scores the heuristic can keep both copies (score(c, c) <= score(item, c)); the
// reference keeps them, but the build's kernels that insert the new points take a list's links to be distinct.
__global__ void hnsw_heal_renumber_kernel(const uint32_t* __restrict__ tab, const uint32_t* __restrict__ remap_old, const uint8_t* __restrict__ old_level,
                                          const uint32_t* __restrict__ o2n, uint32_t n_old, uint32_t level, uint32_t lm, const uint32_t* __restrict__ remap_new,
                                          uint32_t* __restrict__ dst) {
    for (uint32_t o = blockIdx.x * blockDim.x + threadIdx.x; o < n_old; o += gridDim.x * blockDim.x) {
        const uint32_t t = o2n[o];
        if (t == HNSW_EMPTY || old_level[o] < level) continue;
        const uint32_t* src = tab + (size_t)(level ? remap_old[o] : o) * lm;
        uint32_t* out = dst + (size_t)(level ? remap_new[t] : t) * lm;
        uint32_t k = 0;
        for (uint32_t j = 0; j < lm; ++j) {
            const uint32_t l = src[j];
            if (l == HNSW_EMPTY) break;
            if (o2n[l] == HNSW_EMPTY) continue;
            bool seen = false;
            for (uint32_t i = 0; i < j; ++i) seen |= src[i] == l;
            if (!seen) out[k++] = o2n[l];
        }
    }
}

template <int KIND, int METRIC>
struct HealKernels {
    static qb_status heal(const HnswParams& p, const HealArgs& a, unsigned grid, size_t smem) {
        QB_CUDA(cudaFuncSetAttribute(hnsw_heal_kernel<KIND, METRIC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        hnsw_heal_kernel<KIND, METRIC><<<grid, HB_THREADS, smem>>>(p, a);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
    static qb_status backlinks(const HnswParams& p, const unsigned long long* keys, const uint32_t* vals, uint32_t n) {
        hnsw_heal_backlink_kernel<KIND, METRIC><<<hnsw_grid(n, HB_WARPS, 132 * 16), HB_WARPS * 32>>>(p, keys, vals, n);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    }
};

// the old graph, healed in place of its level tables (tabs[l], rows as in the plain format)
struct HealJob {
    const qb_hnsw* old;
    const uint32_t* d_o2n;
    std::vector<uint8_t> old_level;                 // per old point
    std::vector<std::vector<uint32_t>> items;       // per level: the to-heal points, ascending
    uint32_t ef_construct, m, m0;
    uint64_t n_gone;
};

template <int KIND, int METRIC>
qb_status heal_levels(HnswScratch& tmp, const HealJob& job, const std::vector<uint32_t*>& tabs, const std::vector<uint32_t*>& old_tabs, unsigned sm_count,
                      const char* who) {
    using K = HealKernels<KIND, METRIC>;
    const qb_hnsw* g = job.old;
    const qb_storage* s = g->st;
    const uint32_t n = g->n_points;
    HnswParams p{};
    p.rows = reinterpret_cast<const uint8_t*>(s->d_rows); p.stride = s->row_stride; p.dim = s->dim;
    uint32_t max_items = 0;
    for (const auto& v : job.items) max_items = std::max<uint32_t>(max_items, (uint32_t)v.size());
    if (!max_items) return QB_OK;
    const uint32_t lmax = std::max(job.m, job.m0);
    const size_t trip = (size_t)max_items * lmax;
    uint32_t *d_items = nullptr, *d_tval = nullptr, *d_tval2 = nullptr, *d_ovf = nullptr, *d_sel = nullptr;
    unsigned long long *d_tkey = nullptr, *d_tkey2 = nullptr;
    unsigned int *d_work = nullptr, *d_nov = nullptr;
    QB_CUDA(tmp.alloc((void**)&d_items, 4ull * max_items));
    QB_CUDA(tmp.alloc((void**)&d_ovf, 4ull * max_items));
    QB_CUDA(tmp.alloc((void**)&d_sel, 4ull * max_items));
    QB_CUDA(tmp.alloc((void**)&d_tkey, 8 * trip));
    QB_CUDA(tmp.alloc((void**)&d_tkey2, 8 * trip));
    QB_CUDA(tmp.alloc((void**)&d_tval, 4 * trip));
    QB_CUDA(tmp.alloc((void**)&d_tval2, 4 * trip));
    QB_CUDA(tmp.alloc((void**)&d_work, 4));
    QB_CUDA(tmp.alloc((void**)&d_nov, 4));
    size_t sort_bytes = 0;
    QB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, d_tkey, d_tkey2, d_tval, d_tval2, (int)trip, 0, 64));
    void* d_sort = nullptr;
    QB_CUDA(tmp.alloc(&d_sort, sort_bytes));
    const uint32_t ef = job.ef_construct;
    const size_t smem = 2ull * ef * 8;
    int per_sm = 1;
    QB_CUDA(cudaFuncSetAttribute(hnsw_heal_kernel<KIND, METRIC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    QB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hnsw_heal_kernel<KIND, METRIC>, HB_THREADS, smem));
    const unsigned grid = std::min<unsigned>(sm_count * (unsigned)std::max(per_sm, 1), max_items);
    HealArgs a{};
    a.visited_words = ceil_div_u64(n, 32); a.vlog_cap = 32768;
    QB_CUDA(tmp.alloc((void**)&a.visited, (size_t)grid * a.visited_words * 4));
    QB_CUDA(tmp.alloc((void**)&a.vlog, (size_t)grid * a.vlog_cap * 4));
    QB_CUDA(cudaMemset(a.visited, 0, (size_t)grid * a.visited_words * 4));
    // the first runs: a fixed stack per CTA; a rerun of the items that overflowed it: the bound lm * (gone points + 1) (a gone point is
    // expanded once and pushes at most lm links; the item pushes at most lm), or 16x the last size when that is smaller, with fewer CTAs
    uint32_t stack_cap = qb_opt().hnsw_heal_stack ? qb_opt().hnsw_heal_stack : HEAL_STACK;
    unsigned long long* d_stack = nullptr;
    QB_CUDA(tmp.alloc((void**)&d_stack, (size_t)grid * stack_cap * 8));
    uint64_t reruns = 0;
    for (uint32_t l = 0; l < (uint32_t)job.items.size(); ++l) {
        const uint32_t ni = (uint32_t)job.items[l].size();
        if (!ni) continue;
        const uint32_t lm = l ? job.m : job.m0;
        QB_CUDA(cudaMemcpy(d_items, job.items[l].data(), 4ull * ni, cudaMemcpyHostToDevice));
        a.old_tab = old_tabs[l]; a.tab = tabs[l]; a.remap = l ? g->d_reindex : nullptr; a.o2n = job.d_o2n;
        a.items = d_items; a.sel = nullptr; a.n_items = ni; a.n_work = ni; a.lm = lm; a.ef = ef;
        a.stack = d_stack; a.stack_cap = stack_cap; a.work = d_work; a.tkey = d_tkey; a.tval = d_tval; a.ovf = d_ovf; a.n_ovf = d_nov;
        unsigned run_grid = std::min<unsigned>(grid, ni);
        for (;;) {
            QB_CUDA(cudaMemsetAsync(d_work, 0, 4));
            QB_CUDA(cudaMemsetAsync(d_nov, 0, 4));
            QB_TRY(K::heal(p, a, run_grid, smem));
            uint32_t nov = 0;
            QB_CUDA(cudaMemcpy(&nov, d_nov, 4, cudaMemcpyDeviceToHost));
            if (!nov) break;
            ++reruns;
            const uint64_t bound = (uint64_t)lm * (job.n_gone + 1);
            QB_CHECK(a.stack_cap < bound, QB_ERR_CUDA, "%s: the heal stack of %u entries overflowed its bound %llu", who, a.stack_cap, (unsigned long long)bound);
            const uint64_t cap = std::min<uint64_t>(bound, (uint64_t)a.stack_cap * 16);
            run_grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>({(uint64_t)nov, (uint64_t)grid, (1ull << 30) / (cap * 8)}));
            unsigned long long* d_big = nullptr;
            QB_CUDA(tmp.alloc((void**)&d_big, (size_t)run_grid * cap * 8));
            QB_CUDA(cudaMemcpy(d_sel, d_ovf, 4ull * nov, cudaMemcpyDeviceToDevice));
            a.stack = d_big; a.stack_cap = (uint32_t)cap; a.sel = d_sel; a.n_work = nov;
        }
        size_t bytes = sort_bytes;
        QB_CUDA(cub::DeviceRadixSort::SortPairs(d_sort, bytes, d_tkey, d_tkey2, d_tval, d_tval2, (int)((size_t)ni * lm), 0, 64));
        QB_LAUNCHED();
        HnswParams q = p;
        q.links0 = tabs[l]; q.m = lm; q.m0 = lm; q.b_remap = l ? g->d_reindex : nullptr;
        QB_TRY(K::backlinks(q, d_tkey2, d_tval2, ni * lm));
    }
    if (qb_opt().verbose) {
        uint64_t lists = 0;
        for (const auto& v : job.items) lists += v.size();
        fprintf(stderr, "[qb200] %s: healed %llu lists, %llu stack reruns\n", who, (unsigned long long)lists, (unsigned long long)reruns);
    }
    return QB_OK;
}

// heal_levels over a Uint8 storage, with its four metrics
template <int KIND>
qb_status heal_levels_u8(int metric, HnswScratch& tmp, const HealJob& job, const std::vector<uint32_t*>& tabs, const std::vector<uint32_t*>& old_tabs,
                         unsigned sm_count, const char* who) {
    switch (metric) {
        case M_EUCLID: return heal_levels<KIND, M_EUCLID>(tmp, job, tabs, old_tabs, sm_count, who);
        case M_MANHATTAN: return heal_levels<KIND, M_MANHATTAN>(tmp, job, tabs, old_tabs, sm_count, who);
        case M_COSINE: return heal_levels<KIND, M_COSINE>(tmp, job, tabs, old_tabs, sm_count, who);
        default: return heal_levels<KIND, M_DOT>(tmp, job, tabs, old_tabs, sm_count, who);
    }
}

}  // namespace

extern "C" qb_status qb_hnsw_build_incremental(qb_storage* s, const qb_hnsw* old, const uint32_t* old_to_new, uint32_t ef_construct, const uint8_t* levels,
                                               uint32_t batch, uint32_t serial_points, qb_hnsw** out, uint32_t* entry_point, uint32_t* entry_level) {
    const char* who = "hnsw_build_incremental";
    QB_CHECK(s && old && old_to_new && levels && out, QB_ERR_INVALID, "%s: null argument", who);
    *out = nullptr;
    QB_CHECK(s->kind == QB_KIND_DENSE && (s->dtype == QB_DT_F32 || s->dtype == QB_DT_U8), QB_ERR_UNSUPPORTED,
             "%s: graphs are built over dense f32 and Uint8 storages only (build over the original vectors, then bind the graph to the quantized storage)",
             who);
    const qb_storage* os = old->st;
    QB_CHECK(os && os->kind == QB_KIND_DENSE && os->dtype == s->dtype, QB_ERR_UNSUPPORTED,
             "%s: the old graph is bound to a storage that is not dense of the new storage's datatype (f32 or Uint8)", who);
    QB_CHECK(os->dim == s->dim && os->distance == s->distance && os->device == s->device, QB_ERR_UNSUPPORTED,
             "%s: the old graph's storage has another dim, distance or device", who);
    QB_CHECK(!old->d_mv_tok, QB_ERR_UNSUPPORTED, "%s: the old graph is over multivector points", who);
    QB_CHECK(!old->d_blob, QB_ERR_UNSUPPORTED, "%s: the old graph holds inline vectors (CompressedWithVectors; old_index.rs:72-76)", who);
    QB_CHECK(s->count >= 1, QB_ERR_INVALID, "%s: empty storage", who);
    QB_CHECK(s->count < 0xFFFFFFFFull, QB_ERR_UNSUPPORTED, "%s: %llu points", who, (unsigned long long)s->count);
    const uint32_t m = old->m, m0 = old->m0, n = (uint32_t)s->count, n_old = old->n_points;
    QB_CHECK(m >= 1 && m0 >= 1 && m <= HNSW_MAX_LINKS && m0 <= HNSW_MAX_LINKS, QB_ERR_UNSUPPORTED, "%s: m %u / m0 %u outside [1,%u]", who, m, m0, HNSW_MAX_LINKS);
    const uint32_t ef = std::max(ef_construct, m0);
    QB_CHECK(ef <= HNSW_MAX_EF, QB_ERR_UNSUPPORTED, "%s: ef %u > %u", who, ef, HNSW_MAX_EF);
    QB_CHECK(ef_construct >= 1, QB_ERR_INVALID, "%s: ef_construct 0", who);
    QB_CUDA(cudaSetDevice(s->device));

    // the old points' levels (point_level, view.rs:354-369) and the new storage's deleted flags
    const uint32_t L_old = old->levels;
    std::vector<uint32_t> reindex(n_old);
    if (n_old) QB_CUDA(cudaMemcpy(reindex.data(), old->d_reindex, 4ull * n_old, cudaMemcpyDeviceToHost));
    std::vector<uint64_t> rows_old(L_old);
    for (uint32_t l = 0; l < L_old; ++l) rows_old[l] = (l + 1 < L_old ? old->level_offsets_ext[l + 1] : old->n_offsets - 1) - old->level_offsets_ext[l];
    HealJob job;
    job.old = old; job.ef_construct = ef_construct; job.m = m; job.m0 = m0;
    job.old_level.assign(n_old, 0);
    for (uint32_t o = 0; o < n_old; ++o) { uint32_t l = 0; while (l + 1 < L_old && reindex[o] < rows_old[l + 1]) ++l; job.old_level[o] = (uint8_t)l; }
    std::vector<uint32_t> deleted;
    if (s->d_deleted) {
        deleted.resize(ceil_div_u64(n, 32));
        QB_CUDA(cudaMemcpy(deleted.data(), s->d_deleted, 4 * deleted.size(), cudaMemcpyDeviceToHost));
    }
    std::vector<uint32_t> given(ceil_div_u64(n, 32), 0u);
    uint32_t entry = HNSW_EMPTY, n_mapped = 0;
    job.n_gone = 0;
    for (uint32_t o = 0; o < n_old; ++o) {
        const uint32_t t = old_to_new[o];
        if (t == HNSW_EMPTY) { ++job.n_gone; continue; }
        QB_CHECK(t < n, QB_ERR_INVALID, "%s: old_to_new[%u] = %u >= %u points", who, o, t, n);
        QB_CHECK(!((given[t >> 5] >> (t & 31)) & 1u), QB_ERR_INVALID, "%s: two old points map to %u", who, t);
        QB_CHECK(deleted.empty() || !((deleted[t >> 5] >> (t & 31)) & 1u), QB_ERR_INVALID, "%s: old point %u maps to %u, which is deleted", who, o, t);
        QB_CHECK(levels[t] <= HB_MAX_LEVEL, QB_ERR_INVALID, "%s: levels[%u] = %u > %u", who, t, (unsigned)levels[t], HB_MAX_LEVEL);
        QB_CHECK(levels[t] == job.old_level[o], QB_ERR_INVALID, "%s: levels[%u] = %u, its old point %u has level %u", who, t, (unsigned)levels[t], o,
                 (unsigned)job.old_level[o]);
        given[t >> 5] |= 1u << (t & 31);
        if (entry == HNSW_EMPTY || levels[t] > levels[entry]) entry = t;   // EntryPoints::new_point in old-offset order
        ++n_mapped;
    }
    QB_CHECK(n_mapped, QB_ERR_INVALID, "%s: no old point is carried over (build from scratch with qb_hnsw_build)", who);
    uint32_t top_new = 0;
    for (uint32_t i = 0; i < n; ++i) {
        QB_CHECK(levels[i] <= HB_MAX_LEVEL, QB_ERR_INVALID, "%s: levels[%u] = %u > %u", who, i, (unsigned)levels[i], HB_MAX_LEVEL);
        top_new = std::max<uint32_t>(top_new, levels[i]);
    }

    // the old graph's level tables, as loaded and to be healed; the to-heal items
    HnswScratch tmp;
    uint32_t* d_o2n = nullptr;
    QB_CUDA(tmp.alloc((void**)&d_o2n, 4ull * n_old));
    QB_CUDA(cudaMemcpy(d_o2n, old_to_new, 4ull * n_old, cudaMemcpyHostToDevice));
    job.d_o2n = d_o2n;
    std::vector<uint32_t*> tabs(L_old, nullptr), old_tabs(L_old, nullptr);
    uint32_t* d_flags = nullptr;
    QB_CUDA(tmp.alloc((void**)&d_flags, 4ull * n_old));
    QB_CUDA(cudaMemset(d_flags, 0, 4ull * n_old));
    for (uint32_t l = 0; l < L_old; ++l) {
        const uint32_t lm = l ? m : m0;
        const size_t bytes = (size_t)rows_old[l] * lm * 4;
        QB_CUDA(tmp.alloc((void**)&old_tabs[l], bytes));
        QB_CUDA(tmp.alloc((void**)&tabs[l], bytes));
        hnsw_heal_table_kernel<<<hnsw_grid(rows_old[l], 256, 132 * 16), 256>>>(old->d_offsets, old->d_neighbors, old->level_offsets_ext[l], rows_old[l], lm, old_tabs[l]);
        QB_LAUNCHED();
        QB_CUDA(cudaMemcpyAsync(tabs[l], old_tabs[l], bytes, cudaMemcpyDeviceToDevice));
        hnsw_heal_flags_kernel<<<hnsw_grid(rows_old[l], 256, 132 * 16), 256>>>(old_tabs[l], rows_old[l], lm, d_o2n, d_flags, 1u << l);
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
    }
    // flags[r] bit l: row r of level l.  Items: point ascending per level (rows of level l >= 1 are the old reindex)
    std::vector<uint32_t> flags(n_old);
    if (n_old) QB_CUDA(cudaMemcpy(flags.data(), d_flags, 4ull * n_old, cudaMemcpyDeviceToHost));
    job.items.assign(L_old, {});
    for (uint32_t o = 0; o < n_old; ++o)
        for (uint32_t l = 0; l <= job.old_level[o]; ++l)
            if ((flags[l ? reindex[o] : o] >> l) & 1u) job.items[l].push_back(o);

    const bool u8 = s->dtype == QB_DT_U8;
    const int kind = s->dim >= 32 ? (u8 ? HK_U8 : HK_DENSE_AVX) : (u8 ? HK_U8_SMALL : HK_DENSE_SMALL);
    const int metric = hnsw_metric(s);
    const unsigned sms = (unsigned)os->sm_count;
#define QB_HEAL(K, M) heal_levels<K, M>(tmp, job, tabs, old_tabs, sms, who)
    if (kind == HK_DENSE_AVX) QB_TRY(metric == M_EUCLID ? QB_HEAL(HK_DENSE_AVX, M_EUCLID) : metric == M_MANHATTAN ? QB_HEAL(HK_DENSE_AVX, M_MANHATTAN) : QB_HEAL(HK_DENSE_AVX, M_DOT));
    else if (kind == HK_DENSE_SMALL) QB_TRY(metric == M_EUCLID ? QB_HEAL(HK_DENSE_SMALL, M_EUCLID) : metric == M_MANHATTAN ? QB_HEAL(HK_DENSE_SMALL, M_MANHATTAN) : QB_HEAL(HK_DENSE_SMALL, M_DOT));
    else if (kind == HK_U8) QB_TRY(heal_levels_u8<HK_U8>(metric, tmp, job, tabs, old_tabs, sms, who));
    else QB_TRY(heal_levels_u8<HK_U8_SMALL>(metric, tmp, job, tabs, old_tabs, sms, who));
#undef QB_HEAL

    // renumber into the build's tables, then insert the new points
    uint8_t* d_old_level = nullptr;
    QB_CUDA(tmp.alloc((void**)&d_old_level, n_old));
    QB_CUDA(cudaMemcpy(d_old_level, job.old_level.data(), n_old, cudaMemcpyHostToDevice));
    auto prefill = [&](uint32_t* const* tables, const uint32_t* d_remap) -> qb_status {
        for (uint32_t l = 0; l < std::min(L_old, top_new + 1); ++l) {   // the mapped points keep their levels: none is above top_new
            hnsw_heal_renumber_kernel<<<hnsw_grid(n_old, 256, 132 * 16), 256>>>(tabs[l], old->d_reindex, d_old_level, d_o2n, n_old, l, l ? m : m0, d_remap, tables[l]);
            QB_LAUNCHED();
        }
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    };
    return qb_hnsw_build_dense(s, m, m0, ef, levels, given.data(), entry, batch, serial_points, prefill, who, out, entry_point, entry_level);
}
