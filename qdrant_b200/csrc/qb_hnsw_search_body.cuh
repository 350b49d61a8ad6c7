// qb_hnsw_search_body.cuh — the body of hnsw_search_kernel (qb_hnsw_traverse.cuh), included inside the braces of a kernel that defines
// KIND, METRIC, NT, ALGO and CUSTOM and takes its parameters as `p`: hnsw_search_kernel (p: HnswParams) and the inserts of a multivector
// build, hnsw_build_mv_kernel (qb_hnsw_build_mv.cu; p: HnswMvBuildParams), and the custom queries with multivector examples,
// hnsw_mv_custom_kernel (qb_hnsw_mv_custom.cu; p: HnswMvCustomParams).  Not a standalone header.  The kernels keep the body in their
// own braces, rather than calling a shared device function, so that every hnsw_search_kernel instantiation compiles to the machine
// code it had before the multivector build was added.
    constexpr int HNSW_THREADS = NT;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __shared__ unsigned int s_q, s_best, s_n, s_nvalid, s_len, s_nlog, s_cur, s_changed, s_warp_cnt[ALGO == ALGO_ACORN ? 4 : 2];
    __shared__ float s_cur_score;
    __shared__ unsigned int s_nx;   // ACORN: |to_explore|
    __shared__ unsigned int s_entry, s_entry_level;   // CUSTOM: get_entry_point of this query
    const int tid = threadIdx.x;
    const uint32_t ef = p.ef;
    HnswSmem sm;
    uint32_t* xids = nullptr;   // ACORN: to_explore [HNSW_MAX_LINKS]
    {
        const uint32_t hop = ALGO == ALGO_ACORN ? p.hop_cap : HNSW_MAX_LINKS;
        uint8_t* b = smem_raw;
        sm.q = b; b += ((CUSTOM ? p.q_smem : p.q_bytes) + 15u) & ~15u;
        sm.keys[0] = reinterpret_cast<unsigned long long*>(b); b += (size_t)ef * 8;
        sm.keys[1] = reinterpret_cast<unsigned long long*>(b); b += (size_t)ef * 8;
        sm.newk = reinterpret_cast<unsigned long long*>(b); b += (size_t)hop * 8;
        sm.ids = reinterpret_cast<uint32_t*>(b); b += (size_t)hop * 4;
        sm.sc = reinterpret_cast<float*>(b); b += (size_t)hop * 4;
        sm.flags[0] = b; b += (ef + 15u) & ~15u;
        sm.flags[1] = b;
        if (ALGO == ALGO_ACORN) { b += (ef + 15u) & ~15u; xids = reinterpret_cast<uint32_t*>(b); }
    }
    uint32_t* visited = p.visited + (size_t)blockIdx.x * p.visited_words;
    uint32_t* vlog = p.vlog + (size_t)blockIdx.x * p.vlog_cap;
    unsigned long long hops = 0, evals = 0;   // thread 0 only
    unsigned long long mv_rows = 0, mv_qrows = 0;   // MaxSim, thread 0: token rows scored, and times the query's (examples') vector count

    for (;;) {
        if (tid == 0) s_q = atomicAdd(p.work, 1u);
        __syncthreads();
        const uint32_t q = s_q;
        if (q >= p.nq) break;
        // ---- query into shared memory
        if constexpr (ALGO == ALGO_BUILD && CUSTOM == HC_MAXSIM) {
            // the multivector point being inserted: its stored token rows are the query (FilteredScorer::new_internal)
            const uint32_t pt = p.b_pts[q];
            mv_stage_rows<NT>(p, sm, smem_raw, mv_tok(p)[pt], mv_tok(p)[pt + 1]);
        } else if constexpr (ALGO == ALGO_BUILD) {
            // the point being inserted: its stored row is the query (FilteredScorer::new_internal)
            const uint4* src = reinterpret_cast<const uint4*>(p.rows + (size_t)p.b_pts[q] * p.stride);
            uint4* dst = reinterpret_cast<uint4*>(const_cast<uint8_t*>(sm.q));
            for (uint32_t i = tid; i < p.q_bytes / 16u; i += HNSW_THREADS) dst[i] = src[i];
        } else if constexpr (!CUSTOM) {
            const uint4* src = reinterpret_cast<const uint4*>(p.q_enc + (size_t)q * p.q_bytes);
            uint4* dst = reinterpret_cast<uint4*>(const_cast<uint8_t*>(sm.q));
            for (uint32_t i = tid; i < (p.q_bytes + 15u) / 16u; i += HNSW_THREADS) dst[i] = src[i];
        } else if constexpr (CUSTOM == HC_MAXSIM) {
            // the query's vectors: into shared memory when they fit, else read where they are (the same arithmetic either way)
            MvShared& ms = mv_shared();
            const uint32_t q1 = min(mv_qoff(p)[q + 1], mv_nv(p)), q0 = min(mv_qoff(p)[q], q1);
            const uint8_t* src = p.q_enc + (size_t)q0 * p.q_bytes;
            if (q1 - q0 <= mv_stage_q(p)) {
                const uint4* s4 = reinterpret_cast<const uint4*>(src);
                uint4* dst = reinterpret_cast<uint4*>(smem_raw);
                for (uint32_t i = tid; i < ((q1 - q0) * p.q_bytes) / 16u; i += HNSW_THREADS) dst[i] = s4[i];
                sm.q = smem_raw;
            } else {
                sm.q = src;
            }
            if (tid == 0) { ms.q0 = q0; ms.nqv = q1 - q0; ms.rows = 0; }
        } else if constexpr (CUSTOM == HC_MAXSIM_CUSTOM) {
            // all of the query's example vectors: into shared memory when they fit, else read where they are; ms.nqv = their count (the counters)
            MvShared& ms = mv_shared();
            const uint32_t* eo = mv_ex_off<CUSTOM>(p) + (size_t)q * p.ex_stride + p.ex_first;
            const uint32_t v0 = eo[0], v1 = eo[p.n_ex];
            const uint8_t* src = p.q_enc + (size_t)v0 * p.q_bytes;
            if (p.ex_smem) {
                const uint4* s4 = reinterpret_cast<const uint4*>(src);
                uint4* dst = reinterpret_cast<uint4*>(smem_raw);
                for (uint32_t i = tid; i < ((v1 - v0) * p.q_bytes) / 16u; i += HNSW_THREADS) dst[i] = s4[i];
                sm.q = smem_raw;
            } else {
                sm.q = src;
            }
            if (tid == 0) { ms.q0 = v0; ms.nqv = v1 - v0; ms.rows = 0; }
        } else {
            // the examples: into shared memory when they fit, else read where they are (the same arithmetic either way)
            const size_t first = (size_t)q * p.ex_stride + p.ex_first;
            const uint8_t* src = p.q_enc + first * p.q_bytes;
            if (p.ex_smem) {
                const uint4* s4 = reinterpret_cast<const uint4*>(src);
                uint4* dst = reinterpret_cast<uint4*>(smem_raw);   // the query region of the layout above
                for (uint32_t i = tid; i < (p.n_ex * p.q_bytes) / 16u; i += HNSW_THREADS) dst[i] = s4[i];
                sm.q = smem_raw;
            } else {
                sm.q = src;
            }
        }
        const float q_off = (!CUSTOM && p.q_off) ? p.q_off[q] : 0.0f;
        if (tid == 0) {
            s_nlog = 0;
            if constexpr (hc_entry_points(CUSTOM)) {
                uint32_t e, l;
                hnsw_custom_entry(p, q, e, l);
                s_entry = e; s_entry_level = l; sm.ids[0] = e;
            } else if constexpr (ALGO == ALGO_BUILD) {
                sm.ids[0] = p.b_entry[q];
            } else {
                sm.ids[0] = p.entry;
            }
        }
        __syncthreads();
        // `hc_entry_points(CUSTOM) ? s_entry : p.entry` is written out at each use, not bound to a local, so the nearest-query kernels compile as before

        // ---- search_entry: greedy descent from the entry point's level to level 1 (graph_layers.rs:247-316)
        score_list<KIND, METRIC, NT, CUSTOM>(p, sm, q_off, 1, q);      // score_point(entry)
        __syncthreads();
        if (tid == 0) { s_cur = hc_entry_points(CUSTOM) ? s_entry : (ALGO == ALGO_BUILD ? sm.ids[0] : p.entry); s_cur_score = sm.sc[0]; ++hops; ++evals; }
        __syncthreads();
        for (uint32_t lvl = hc_entry_points(CUSTOM) ? s_entry_level : p.entry_level; lvl >= 1; --lvl) {
            // search_entry_on_level re-scores its entry point on every level (graph_layers.rs:298-301): same value, but the scorer call
            // and the scored point are metered, so they are counted here too
            if (tid == 0 && lvl != (hc_entry_points(CUSTOM) ? s_entry_level : p.entry_level)) {
                ++hops; ++evals;
                if constexpr (hc_multivector(CUSTOM)) mv_shared().rows += mv_tok(p)[s_cur + 1] - mv_tok(p)[s_cur];
            }
            for (;;) {
                const uint32_t cur = s_cur;
                // links of `cur` on this level: neighbors[offsets[idx] .. offsets[idx + 1]), idx = level_offsets[lvl] + reindex[cur] (view.rs:203-215)
                if (tid < 32) {
                    const uint64_t idx = p.level_offsets[lvl] + p.reindex[cur];
                    const uint64_t b = p.offsets[idx], e = p.offsets[idx + 1];
                    uint32_t cnt = 0;
                    // filter (check_batched keeps matches in order), then truncate to level_m (point_scorer.rs:270-277)
                    for (uint64_t base = b; base < e && cnt < p.m; base += 32) {
                        const uint64_t i = base + tid;
                        const uint32_t l = i < e ? p.neighbors[i] : HNSW_EMPTY;
                        const bool keep = l != HNSW_EMPTY && l < p.n_points && !hnsw_filtered_out(p, l);
                        const unsigned int bal = __ballot_sync(0xFFFFFFFFu, keep);
                        const uint32_t pos = cnt + __popc(bal & ((1u << tid) - 1u));
                        if (keep && pos < p.m && pos < HNSW_MAX_LINKS) { sm.ids[pos] = l; if (p.prefetch) prefetch_point<KIND, hc_multivector(CUSTOM)>(p, l); }
                        cnt += __popc(bal);
                    }
                    if (tid == 0) s_n = min(min(cnt, p.m), HNSW_MAX_LINKS);
                }
                __syncthreads();
                const uint32_t n = s_n;
                score_list<KIND, METRIC, NT, CUSTOM>(p, sm, q_off, n, q);
                __syncthreads();
                if (tid == 0) {
                    bool changed = false;
                    uint32_t c = cur; float cs = s_cur_score;
                    for (uint32_t i = 0; i < n; ++i) if (sm.sc[i] > cs) { changed = true; c = sm.ids[i]; cs = sm.sc[i]; }
                    s_cur = c; s_cur_score = cs; s_changed = changed ? 1u : 0u;
                    if (n) { ++hops; evals += n; }
                }
                __syncthreads();
                if (!s_changed) break;
            }
        }

        if constexpr (ALGO == ALGO_BUILD) {
            // a point below this level: search_entry_on_level (graph_layers.rs:279-316) on the level's rows, a row's links being the
            // prefix before its first HNSW_EMPTY; the entry moves to a strictly better link, the first in link order
            if (!p.b_insert) {
                for (;;) {
                    const uint32_t cur = s_cur;
                    if (tid < 64) {
                        const uint32_t l = (uint32_t)tid < p.m0 ? p.links0[(size_t)hnsw_build_row(p, cur) * p.m0 + tid] : HNSW_EMPTY;
                        if (l != HNSW_EMPTY) sm.ids[tid] = l;
                        const unsigned int bal = __ballot_sync(0xFFFFFFFFu, l != HNSW_EMPTY);
                        if ((tid & 31) == 0) s_warp_cnt[tid >> 5] = __popc(bal);
                    }
                    __syncthreads();
                    const uint32_t n = s_warp_cnt[0] + s_warp_cnt[1];
                    score_list<KIND, METRIC, NT, CUSTOM>(p, sm, q_off, n, q);
                    __syncthreads();
                    if (tid == 0) {
                        bool changed = false;
                        uint32_t c = cur; float cs = s_cur_score;
                        for (uint32_t i = 0; i < n; ++i) if (sm.sc[i] > cs) { changed = true; c = sm.ids[i]; cs = sm.sc[i]; }
                        s_cur = c; s_cur_score = cs; s_changed = changed ? 1u : 0u;
                    }
                    __syncthreads();
                    if (!s_changed) break;
                }
                if (tid == 0) p.b_entry[q] = s_cur;
                __syncthreads();
                continue;
            }
        }

        // ---- search_on_level(level 0, ef): nearest = [level entry], entry visited
        if (tid == 0) {
            const uint32_t e0 = s_cur;
            sm.keys[0][0] = qb_pack_key(s_cur_score, e0);
            sm.flags[0][0] = 0;
            s_len = 1;
            atomicOr(&visited[e0 >> 5], 1u << (e0 & 31));
            vlog[0] = e0; s_nlog = 1;
        }
        __syncthreads();
        int cb = 0;   // current buffer
        for (;;) {
            unsigned long long* keys = sm.keys[cb];
            uint8_t* flags = sm.flags[cb];
            const uint32_t len = s_len;
            // 1. best not-yet-expanded entry
            if (tid == 0) s_best = 0xFFFFFFFFu;
            __syncthreads();
            for (uint32_t i = tid; i < len; i += HNSW_THREADS) if (!flags[i]) atomicMin(&s_best, i);
            __syncthreads();
            const uint32_t best = s_best;
            if (best == 0xFFFFFFFFu) break;
            const uint32_t cand = qb_key_id(keys[best]);
            if constexpr (ALGO == ALGO_ACORN) {
                if (tid == 0) flags[best] = 1;
                acorn_collect<KIND, NT, hc_multivector(CUSTOM)>(p, sm, xids, cand, visited, vlog, s_n, s_nx, s_nlog, s_warp_cnt);
                const uint32_t n = s_n;
                if (tid == 0) { if (n) { ++hops; evals += n; } s_nvalid = 0; }
                if (n == 0) { __syncthreads(); continue; }
                // score_points_unfiltered(to_score)
                if (hk_one_thread(KIND) && !hc_multivector(CUSTOM)) {
                    for (uint32_t i = tid; i < n; i += HNSW_THREADS) sm.sc[i] = score_q<KIND, METRIC, CUSTOM>(p, sm, q_off, sm.ids[i], 0, q);
                } else {
                    score_list<KIND, METRIC, NT, CUSTOM>(p, sm, q_off, n, q);
                }
                __syncthreads();
                // keys that can enter `nearest`, compacted, sorted, at most ef of them
                const unsigned long long lower = (len == ef) ? keys[ef - 1] : 0ull;
                for (uint32_t i = tid; i < n; i += HNSW_THREADS) {
                    const unsigned long long k = qb_pack_key(sm.sc[i], sm.ids[i]);
                    if (k > lower) sm.newk[atomicAdd(&s_nvalid, 1u)] = k;
                }
                __syncthreads();
                const uint32_t nv = s_nvalid;
                if (nv == 0) continue;
                acorn_sort_desc<NT>(sm.newk, nv);
                const uint32_t nk_len = min(nv, ef);
                // merge: rank = own index + number of greater keys in the other list (both sorted: binary search)
                unsigned long long* nk = sm.keys[cb ^ 1];
                uint8_t* nf = sm.flags[cb ^ 1];
                for (uint32_t i = tid; i < len; i += HNSW_THREADS) {
                    const unsigned long long k = keys[i];
                    const uint32_t r = i + count_greater(sm.newk, nk_len, k);
                    if (r < ef) { nk[r] = k; nf[r] = flags[i]; }
                }
                for (uint32_t j = tid; j < nk_len; j += HNSW_THREADS) {
                    const unsigned long long k = sm.newk[j];
                    const uint32_t r = j + count_greater(keys, len, k);
                    if (r < ef) {
                        nk[r] = k; nf[r] = 0;
                        if (QB_HNSW_LINK_PREFETCH && p.prefetch) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.links0 + (size_t)(ALGO == ALGO_BUILD ? hnsw_build_row(p, qb_key_id(k)) : qb_key_id(k)) * p.m0));
                    }
                }
                __syncthreads();
                if (tid == 0) s_len = min(len + nk_len, ef);
                cb ^= 1;
                __syncthreads();
                continue;
            }
            // 2. its level-0 links that pass the filter and were not visited (test-and-set), in link order
            if (tid < 64) {
                const uint32_t l = (uint32_t)tid < p.m0 ? p.links0[(size_t)(ALGO == ALGO_BUILD ? hnsw_build_row(p, cand) : cand) * p.m0 + tid] : HNSW_EMPTY;
                bool keep = l < p.n_points && !hnsw_filtered_out(p, l);
                if (keep) keep = ((atomicOr(&visited[l >> 5], 1u << (l & 31)) >> (l & 31)) & 1u) == 0u;
                const unsigned int bal = __ballot_sync(0xFFFFFFFFu, keep);
                if ((tid & 31) == 0) s_warp_cnt[tid >> 5] = __popc(bal);
                __syncwarp();
                // two warps: positions of warp 1 follow warp 0's
                asm volatile("bar.sync 1, 64;" ::: "memory");
                const uint32_t pos = ((tid >> 5) ? s_warp_cnt[0] : 0u) + __popc(bal & ((1u << (tid & 31)) - 1u));
                if (keep) {
                    if (p.prefetch) prefetch_point<KIND, hc_multivector(CUSTOM)>(p, l);          // HBM -> L2 for the whole vector, in flight while the list is published
                    sm.ids[pos] = l;
                    const uint32_t lp = s_nlog + pos;
                    if (lp < p.vlog_cap) vlog[lp] = l;
                }
                if (tid == 0) { flags[best] = 1; s_n = s_warp_cnt[0] + s_warp_cnt[1]; }
            }
            __syncthreads();
            const uint32_t n = s_n;
            if (tid == 0) { s_nlog += n; if (n) { ++hops; evals += n; } s_nvalid = 0; }
            if (n == 0) { __syncthreads(); continue; }
            // 3. score
            score_list<KIND, METRIC, NT, CUSTOM>(p, sm, q_off, n, q);
            __syncthreads();
            // 4. keys of the new points; the ones that cannot enter a full list are dropped here (key 0 = empty)
            const unsigned long long lower = (len == ef) ? keys[ef - 1] : 0ull;
            if ((uint32_t)tid < n) {
                unsigned long long k = qb_pack_key(sm.sc[tid], sm.ids[tid]);
                if (k <= lower) k = 0ull; else atomicAdd(&s_nvalid, 1u);
                sm.newk[tid] = k;
            }
            __syncthreads();
            const uint32_t nvalid = s_nvalid;
            if (nvalid == 0) continue;
            // 5. merge into the other buffer: rank = own index + number of greater keys in the other list
            unsigned long long* nk = sm.keys[cb ^ 1];
            uint8_t* nf = sm.flags[cb ^ 1];
            for (uint32_t i = tid; i < len; i += HNSW_THREADS) {
                const unsigned long long k = keys[i];
                uint32_t r = i;
                for (uint32_t j = 0; j < n; ++j) r += (sm.newk[j] > k) ? 1u : 0u;
                if (r < ef) { nk[r] = k; nf[r] = flags[i]; }
            }
            if ((uint32_t)tid >= HNSW_THREADS - HNSW_MAX_LINKS) {   // the last two warps place the new keys
                const uint32_t j = (uint32_t)tid - (HNSW_THREADS - HNSW_MAX_LINKS);
                const unsigned long long k = j < n ? sm.newk[j] : 0ull;
                if (k) {
                    uint32_t r = 0;
                    for (uint32_t j2 = 0; j2 < n; ++j2) r += (sm.newk[j2] > k) ? 1u : 0u;
                    uint32_t lo = 0, hi = len;   // first index with keys[idx] < k (keys are distinct and descending)
                    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (keys[mid] > k) lo = mid + 1; else hi = mid; }
                    r += lo;
                    if (r < ef) {
                        nk[r] = k; nf[r] = 0;
                        // every point that enters `nearest` is a future candidate: pull its level-0 link row (one 128-byte line at m0 = 32) into L2 now
                        if (QB_HNSW_LINK_PREFETCH && p.prefetch) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.links0 + (size_t)(ALGO == ALGO_BUILD ? hnsw_build_row(p, qb_key_id(k)) : qb_key_id(k)) * p.m0));
                    }
                }
            }
            __syncthreads();
            if (tid == 0) s_len = min(len + nvalid, ef);
            cb ^= 1;
            __syncthreads();
        }

        if constexpr (ALGO == ALGO_BUILD) {
            // the point's next entry is the best it found (link_new_point, graph_layers_builder.rs:417-475); its links are
            // fill_from_sorted_with_heuristic (links_container.rs:47-71) over `nearest`: candidate c is kept unless a kept link scores
            // higher against c than the point does.  The kept links go to sm.ids, their number to s_n.
            const unsigned long long* keys = sm.keys[cb];
            const uint32_t len = s_len, pt = p.b_pts[q];
            if (tid == 0) { p.b_entry[q] = qb_key_id(keys[0]); s_n = 0; }
            __syncthreads();
            for (uint32_t c = 0; c < len; ++c) {
                const uint32_t nsel = s_n;
                if (nsel >= p.m0) break;
                const uint32_t cid = qb_key_id(keys[c]);
                const float cs = qb_key_score(keys[c]);
                if (tid == 0) s_changed = 0;
                __syncthreads();
                if constexpr (CUSTOM == HC_MAXSIM) {
                    // MaxSim with the candidate's token rows as the query, against each kept link
                    if (nsel) {
                        mv_stage_rows<NT>(p, sm, smem_raw, mv_tok(p)[cid], mv_tok(p)[cid + 1]);
                        __syncthreads();
                        maxsim_list<KIND, METRIC, NT>(p, sm, nsel);
                        if ((uint32_t)tid < nsel && sm.sc[tid] > cs) s_changed = 1;
                    }
                } else {
                    hnsw_score_rows<KIND, METRIC, NT / 8>(p, p.rows + (size_t)cid * p.stride, sm.ids, nsel, tid, [&](uint32_t, float s) {
                        if (s > cs) s_changed = 1;
                    });
                }
                __syncthreads();
                if (tid == 0 && !s_changed) { sm.ids[nsel] = cid; s_n = nsel + 1; }
                __syncthreads();
            }
            // the point's row, and its backlinks for the backlink pass
            const uint32_t nsel = s_n;
            uint32_t* row = const_cast<uint32_t*>(p.links0) + (size_t)hnsw_build_row(p, pt) * p.m0;
            for (uint32_t j = tid; j < p.m0; j += HNSW_THREADS) {
                const uint32_t l = j < nsel ? sm.ids[j] : HNSW_EMPTY;
                row[j] = l;
                p.b_tkey[(size_t)q * p.m0 + j] = j < nsel ? (((unsigned long long)l << 32) | q) : ~0ull;
                p.b_tval[(size_t)q * p.m0 + j] = pt;
            }
        }
        // ---- results: into_iter_sorted().take(top) (graph_layers.rs:560)
        if constexpr (ALGO != ALGO_BUILD) {
            const unsigned long long* keys = sm.keys[cb];
            const uint32_t len = s_len, cnt = min(len, p.top);
            for (uint32_t i = tid; i < cnt; i += HNSW_THREADS) {
                qb_scored_point sp;
                sp.idx = qb_key_id(keys[i]) + p.id_base;
                sp.score = qb_key_score(keys[i]);
                p.out[(size_t)q * p.top + i] = sp;
            }
            if (tid == 0) p.out_counts[q] = cnt;
        }
        if constexpr (hc_multivector(CUSTOM)) {
            if (tid == 0) { const MvShared& ms = mv_shared(); mv_rows += ms.rows; mv_qrows += ms.rows * ms.nqv; }
        }
        // ---- un-set the visited bits this query set
        {
            const uint32_t nlog = s_nlog;
            if (nlog <= p.vlog_cap) {
                for (uint32_t i = tid; i < nlog; i += HNSW_THREADS) visited[vlog[i] >> 5] = 0u;
            } else {
                for (uint64_t i = tid; i < p.visited_words; i += HNSW_THREADS) visited[i] = 0u;
            }
        }
        __syncthreads();
    }
    if (tid == 0 && p.stats) { atomicAdd(&p.stats[0], hops); atomicAdd(&p.stats[1], evals); }
    if constexpr (hc_multivector(CUSTOM)) {
        if (tid == 0 && p.stats) { atomicAdd(&p.stats[2], mv_rows); atomicAdd(&p.stats[3], mv_qrows); }
    }
