// qb_mmr_maxsim.cu — maximal marginal relevance (MMR) reranking of multivector (MaxSim) candidate lists on the device.
//
// Replaces: mmr_from_points_with_vector (lib/shard/src/query/mmr/mod.rs:42-125) for a multivector named vector, whose candidates go into
// a volatile multi-dense f32 storage without preprocessing (volatile_multi_dense_vector_storage.rs:138-148), and LazyMatrix
// (lazy_matrix.rs), whose scorers are MultiMetricQueryScorer (ColBERT MaxSim).  Here that storage is a dense f32 token storage with
// point offsets: point p = token rows [tok[p], tok[p + 1]).
//   MaxSim(A, B) = sum over a in A, in order, from +0.0 (sequential f32) of max over b in B (`sim > max` from -inf) of sim(a, b)
//   rel[i]       = MaxSim(preprocess(Q), P_i)                  the query's vectors are the query side
//   pair(c, s)   = MaxSim(preprocess(P_c), P_s)                LazyMatrix::get_similarity(c, s): candidate c's scorer, so c's tokens are
//                                                              the query side and the pick's tokens the stored side.  Not symmetric.
// The selection is qb_mmr.cu's, with the same pieces (qb_mmr.cuh): one thread-block cluster per query, each CTA owning a slice of the
// candidates, replicated u16 position arrays, one DSMEM argmax per step and the same swap_remove.
//
// The unit of work is an item: (candidate, one of its tokens) in a step, (candidate, one query vector) in the relevance pass.  Items
// are numbered through a per-slice token prefix (the relevance pass: T_q items per candidate) and scored in batches of MMS_BATCH: an
// 8-lane group (one thread below dim 32) takes an item and folds `sim > max` over the stored side's vectors in order with the f32
// chains of qb_score.cuh, writing the item's maximum to shared memory; one thread per candidate then adds its items' maxima in token
// order.  The pick's token rows are staged in shared memory when they fit (MMS_STAGE_MAX_F floats), else read from global memory;
// the results are the same.  For Cosine the query side is preprocess(P_c): every candidate's token rows are gathered into scratch and
// normalised with qb_launch_preprocess_rows, the batch in chunks of queries within MMS_PRE_BUDGET.
#include "qb_mmr.cuh"

using namespace qb_mmr;

namespace {

constexpr uint32_t MMS_STAGE_MAX_F = 16384;           // pick tokens / query vectors of up to 64 KB are staged in shared memory
constexpr uint32_t MMS_BATCH = 2048;                  // items scored per batch, their maxima held in shared memory
constexpr size_t MMS_PRE_BUDGET = 512ull << 20;       // Cosine: preprocessed candidate token rows of one launch

// dynamic shared memory of one CTA: [stage | 2 step slots + one per warp (u64) | 4 u32 | item maxima | rel, maxsim, sum, point (per
// owned) | token prefix (per owned + 1) | rem, where]
struct MmsSmem {
    uint32_t stage_f, slice, n_cap;
    __host__ __device__ size_t slots_at() const { return (size_t)stage_f * 4; }
    __host__ __device__ size_t cnt_at() const { return slots_at() + (2 + MMR_WARPS) * 8; }
    __host__ __device__ size_t tmax_at() const { return cnt_at() + 16; }
    __host__ __device__ size_t rel_at() const { return tmax_at() + (size_t)MMS_BATCH * 4; }
    __host__ __device__ size_t tpre_at() const { return rel_at() + (size_t)slice * 16; }
    __host__ __device__ size_t pos_at() const { return (tpre_at() + ((size_t)slice + 1) * 4 + 15) & ~(size_t)15; }
    __host__ __device__ size_t bytes() const { return pos_at() + (size_t)n_cap * 4; }
};

struct MmsParams {
    const float* rows;                 // the token storage's rows, stride_f floats apart
    uint32_t stride_f, dim;
    const uint32_t* tok;               // [n_points + 1] point offsets
    uint32_t n_points;
    const float* q_pre;                // [n_qv][stride_f] preprocessed query vectors
    const uint32_t* q_off;             // [nq + 1]: query q = vectors [q_off[q], q_off[q + 1]), clamped to n_qv
    uint32_t n_qv;
    const float* lambdas;              // [nq]
    const qb_scored_point* cand;       // [nq][max_cand]
    const uint32_t* cand_counts;       // [nq]
    uint32_t max_cand;
    const float* pre;                  // Cosine: [launch queries][max_cand][pre_t][stride_f] preprocess(P_i) by input index; null: the rows
    uint32_t pre_t;
    uint32_t q0;                       // first query of this launch
    uint32_t limit;
    qb_scored_point* out;              // [nq][out_stride]
    uint32_t out_stride;
    uint32_t* out_counts;              // [nq]
    unsigned long long* pairs;         // [nq]: token-weighted pair count (the counters)
    MmsSmem sm;
};

template <int METRIC, bool SMALL>
__device__ __forceinline__ float pair_score(const float* row, const float* qry, uint32_t dim) {
    if (SMALL) return score_small<METRIC>(row, qry, dim);
    return score_avx_group8<METRIC>(row, qry, dim, threadIdx.x & 7);
}

// the slice candidate whose items hold item k: pre[j] <= k < pre[j + 1] (candidates without items are skipped)
__device__ __forceinline__ uint32_t item_owner(const uint32_t* pre, uint32_t ns, uint32_t k) {
    uint32_t lo = 0, hi = ns - 1;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (pre[mid + 1] > k) hi = mid; else lo = mid + 1; }
    return lo;
}

// Items [0, total) in batches: item(k) -> (ok, query-side vector, stored-side rows, their count) scores the fold; the maxima are added
// in item order to sum[owner].  owner(k) maps an item to its slice candidate, first(j) is candidate j's first item.  Every thread of the
// block calls it; on return sum[] is complete.
template <int METRIC, bool SMALL, class Owner, class First, class Item>
__device__ __forceinline__ void score_items(const MmsParams& p, uint32_t total, const uint16_t* where_s, float* tmax, float* sum, Owner owner, First first,
                                            Item item) {
    const uint32_t tid = threadIdx.x, unit = SMALL ? 1u : 8u, n_units = MMR_THREADS / unit, u = tid / unit;
    for (uint32_t b0 = 0; b0 < total; b0 += MMS_BATCH) {
        const uint32_t b1 = min(total, b0 + MMS_BATCH);
        for (uint32_t base = b0; base < b1; base += n_units) {   // the same trip count for every lane of a warp
            const uint32_t k = base + u;
            uint32_t j = 0;
            bool ok = k < b1;
            if (ok) j = owner(k);
            ok = ok && where_s[j] != MMR_GONE;
            if (!SMALL && !__any_sync(0xFFFFFFFFu, ok)) continue;
            if (SMALL && !ok) continue;
            const float* qc;
            const float* vs;
            uint32_t nv, stride;
            item(ok, j, k - (ok ? first(j) : 0u), qc, vs, nv, stride);
            const uint32_t nt = SMALL ? nv : __reduce_max_sync(0xFFFFFFFFu, nv);   // lanes past their own count score row 0 and drop it
            float m = __int_as_float(0xff800000);
            for (uint32_t t = 0; t < nt; ++t) {
                const float s = pair_score<METRIC, SMALL>(t < nv ? vs + (size_t)t * stride : p.rows, qc, p.dim);
                if (t < nv && s > m) m = s;
            }
            if (ok && (SMALL || (tid & 7) == 0)) tmax[k - b0] = m;
        }
        __syncthreads();
        const uint32_t j0 = owner(b0), j1 = owner(b1 - 1);
        for (uint32_t j = j0 + tid; j <= j1; j += MMR_THREADS) {
            if (where_s[j] == MMR_GONE) continue;
            const uint32_t a = max(first(j), b0), e = min(first(j + 1), b1);
            float s = sum[j];
            for (uint32_t i = a; i < e; ++i) s = __fadd_rn(s, tmax[i - b0]);
            sum[j] = s;
        }
        __syncthreads();
    }
}

template <int METRIC, bool SMALL>
__global__ void __launch_bounds__(MMR_THREADS, 1) mmr_maxsim_kernel(const MmsParams p) {
    cg::cluster_group cluster = cg::this_cluster();
    const uint32_t C = cluster.num_blocks(), rank = cluster.block_rank();
    const uint32_t ql = blockIdx.x / C, q = p.q0 + ql, tid = threadIdx.x;
    extern __shared__ __align__(16) unsigned char smem[];
    float* stage = reinterpret_cast<float*>(smem);
    unsigned long long* slot = reinterpret_cast<unsigned long long*>(smem + p.sm.slots_at());   // [2] this CTA's best of a step, by parity
    unsigned long long* wbest = slot + 2;                                                      // [MMR_WARPS]
    uint32_t* cnt = reinterpret_cast<uint32_t*>(smem + p.sm.cnt_at());                         // [0] kept candidates, [1] their tokens
    float* tmax = reinterpret_cast<float*>(smem + p.sm.tmax_at());
    float* rel = reinterpret_cast<float*>(smem + p.sm.rel_at());
    float* msim = rel + p.sm.slice;
    float* psum = msim + p.sm.slice;
    uint32_t* lpt = reinterpret_cast<uint32_t*>(psum + p.sm.slice);                            // point id, or ~0 when not kept
    uint32_t* tpre = reinterpret_cast<uint32_t*>(smem + p.sm.tpre_at());
    uint16_t* rem = reinterpret_cast<uint16_t*>(smem + p.sm.pos_at());
    uint16_t* where = rem + p.sm.n_cap;

    const qb_scored_point* cand = p.cand + (size_t)q * p.max_cand;
    const uint32_t n = min(p.cand_counts[q], p.max_cand);
    const uint32_t per = (n + C - 1) / C;
    const uint32_t lo = min(n, rank * per), hi = min(n, lo + per), sn = hi - lo;
    const uint16_t* where_s = where + lo;

    // 1. unique_by(id), first occurrence kept; ids outside the points and points without token rows are dropped
    mmr_dedup(tid, cand, lo, hi, lpt, [&](uint32_t id, uint32_t& local) {
        local = id;
        return id < p.n_points && p.tok[id + 1] > p.tok[id];
    });
    // the slice's token prefix over its kept candidates (warp 0: a contiguous run per lane, then a warp scan); cnt[1] = its total
    if (tid < 32) {
        const uint32_t run_len = (sn + 31) / 32, a = min(sn, tid * run_len), b = min(sn, a + run_len);
        uint32_t s = 0;
        for (uint32_t j = a; j < b; ++j) s += lpt[j] != 0xFFFFFFFFu ? p.tok[lpt[j] + 1] - p.tok[lpt[j]] : 0u;
        uint32_t incl = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
            if ((int)tid >= o) incl += v;
        }
        uint32_t r = incl - s;
        for (uint32_t j = a; j < b; ++j) {
            tpre[j] = r;
            r += lpt[j] != 0xFFFFFFFFu ? p.tok[lpt[j] + 1] - p.tok[lpt[j]] : 0u;
        }
        if (tid == 31) { tpre[sn] = incl; cnt[1] = incl; }
    }
    // 2. positions (psum holds each kept candidate's rank within the slice); its barriers publish tpre and cnt[1]
    const uint32_t n_keep = mmr_positions(tid, cluster, C, rank, lo, hi, lpt, reinterpret_cast<uint32_t*>(psum), wbest, cnt, rem, where);
    if (n_keep < 2) {   // mod.rs:77-80: returned as it is, no scoring
        if (rank == 0 && tid == 0) {
            if (n_keep == 1) p.out[(size_t)q * p.out_stride] = cand[rem[0]];
            p.out_counts[q] = n_keep;
            p.pairs[q] = 0;
        }
        return;
    }
    const uint32_t L = min(p.limit, n_keep);
    const uint32_t qa = min(p.q_off[q], p.n_qv), qb = min(max(p.q_off[q + 1], p.q_off[q]), p.n_qv), tq = qb - qa;
    unsigned long long tok_left = 0, pairs = 0;
    if (rank == 0 && tid == 0) {
        for (uint32_t r = 0; r < C; ++r) tok_left += cluster.map_shared_rank(cnt, r)[1];
        pairs = (unsigned long long)tq * tok_left;
    }

    // 3. relevance: item (j, v) = query vector v against candidate j's token rows
    const float* qv = p.q_pre + (size_t)qa * p.stride_f;
    if ((size_t)tq * p.stride_f <= p.sm.stage_f) {
        for (uint32_t f = tid; f < tq * p.stride_f; f += MMR_THREADS) stage[f] = qv[f];
        qv = stage;
    }
    for (uint32_t j = tid; j < sn; j += MMR_THREADS) psum[j] = 0.0f;
    __syncthreads();
    score_items<METRIC, SMALL>(
        p, sn * tq, where_s, tmax, psum, [&](uint32_t k) { return k / tq; }, [&](uint32_t j) { return j * tq; },
        [&](bool ok, uint32_t j, uint32_t v, const float*& qc, const float*& vs, uint32_t& nv, uint32_t& stride) {
            qc = ok ? qv + (size_t)v * p.stride_f : qv;
            vs = ok ? p.rows + (size_t)p.tok[lpt[j]] * p.stride_f : p.rows;
            nv = ok ? p.tok[lpt[j] + 1] - p.tok[lpt[j]] : 0u;
            stride = p.stride_f;
        });
    unsigned long long best = 0;
    for (uint32_t j = tid; j < sn; j += MMR_THREADS) {
        if (where_s[j] == MMR_GONE) continue;
        rel[j] = psum[j];
        const unsigned long long k = pos_key(psum[j], where_s[j]);
        best = k > best ? k : best;
    }

    const float lam = p.lambdas[q], one_minus = __fsub_rn(1.0f, lam);
    const float* pre = p.pre ? p.pre + (size_t)ql * p.max_cand * p.pre_t * p.stride_f : nullptr;
    uint32_t remaining = n_keep, par = 0;
    for (uint32_t k = 0;; ++k, par ^= 1u) {
        // 4. cluster argmax of this step
        best = mmr_cluster_best(tid, cluster, C, best, wbest, slot, par);
        const uint32_t pos = (uint32_t)(best & 0xFFFFFFFFu), sel = rem[pos];
        if (rank == 0 && tid == 0) p.out[(size_t)q * p.out_stride + k] = cand[sel];
        if (k + 1 == L) break;
        __syncthreads();   // every thread has read rem[pos]
        // 5. swap_remove; stage the pick's token rows
        if (tid == 0) mmr_swap_remove(rem, where, pos, sel, remaining);
        --remaining;
        const uint32_t pid = cand[sel].idx, t0 = p.tok[pid], tp = p.tok[pid + 1] - t0;
        if (rank == 0 && tid == 0) {
            tok_left -= tp;
            pairs += (unsigned long long)tp * tok_left;
        }
        const float* vs = p.rows + (size_t)t0 * p.stride_f;
        if ((size_t)tp * p.stride_f <= p.sm.stage_f) {
            for (uint32_t f = tid; f < tp * p.stride_f; f += MMR_THREADS) stage[f] = vs[f];
            vs = stage;
        }
        for (uint32_t j = tid; j < sn; j += MMR_THREADS) psum[j] = 0.0f;
        __syncthreads();
        // 6. pair(c, newest) = MaxSim(preprocess(P_c), P_pick): item (j, a) = candidate j's token a against the pick's token rows
        score_items<METRIC, SMALL>(
            p, tpre[sn], where_s, tmax, psum, [&](uint32_t i) { return item_owner(tpre, sn, i); }, [&](uint32_t j) { return tpre[j]; },
            [&](bool ok, uint32_t j, uint32_t a, const float*& qc, const float*& v, uint32_t& nv, uint32_t& stride) {
                qc = !ok ? p.rows : pre ? pre + ((size_t)(lo + j) * p.pre_t + a) * p.stride_f : p.rows + (size_t)(p.tok[lpt[j]] + a) * p.stride_f;
                v = vs;
                nv = tp;
                stride = p.stride_f;
            });
        // the running max (new value on >=), mmr and the local argmax
        best = 0;
        for (uint32_t j = tid; j < sn; j += MMR_THREADS) {
            if (where_s[j] == MMR_GONE) continue;
            const float m = psum[j], prev = msim[j];
            const float ms = (k == 0 || ord_key(m) >= ord_key(prev)) ? m : prev;
            msim[j] = ms;
            const float mmr = __fsub_rn(__fmul_rn(lam, rel[j]), __fmul_rn(one_minus, ms));
            const unsigned long long key = pos_key(mmr, where_s[j]);
            best = key > best ? key : best;
        }
    }
    if (rank == 0 && tid == 0) {
        p.out_counts[q] = L;
        p.pairs[q] = pairs;
    }
    cluster.sync();   // no CTA leaves while a peer may still read its slot or counts
}

// Cosine: rows[((q - q0) * max_cand + i) * pre_t + a] = token a of candidate i of query q (zeros past the count, past the point's tokens
// or for an id outside the points), to be preprocessed in place.  One warp per row.
__global__ void __launch_bounds__(256) mmr_maxsim_gather_kernel(const float* __restrict__ rows, uint32_t stride_f, const uint32_t* __restrict__ tok,
                                                                uint32_t n_points, const qb_scored_point* __restrict__ cand,
                                                                const uint32_t* __restrict__ cand_counts, uint32_t max_cand, uint32_t pre_t, uint32_t q0,
                                                                uint64_t n_rows, float* __restrict__ out) {
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    const uint32_t lane = threadIdx.x & 31;
    for (uint64_t r = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n_rows; r += warps) {
        const uint64_t slot = r / pre_t;
        const uint32_t a = (uint32_t)(r % pre_t), q = q0 + (uint32_t)(slot / max_cand), i = (uint32_t)(slot % max_cand);
        const uint32_t id = cand[(size_t)q * max_cand + i].idx;
        const bool ok = i < min(cand_counts[q], max_cand) && id < n_points && a < tok[id + 1] - tok[id];
        const float4* src = reinterpret_cast<const float4*>(rows + (size_t)(ok ? tok[id] + a : 0u) * stride_f);
        float4* dst = reinterpret_cast<float4*>(out + (size_t)r * stride_f);
        for (uint32_t f = lane; f < stride_f / 4; f += 32) dst[f] = ok ? src[f] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

template <int METRIC, bool SMALL>
qb_status launch_mms(const MmsParams& p, uint32_t nq, uint32_t C, cudaStream_t stream) {
    const size_t smem = p.sm.bytes();
    QB_CUDA(cudaFuncSetAttribute(mmr_maxsim_kernel<METRIC, SMALL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(nq * C);
    cfg.blockDim = dim3(MMR_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    QB_CUDA(cudaLaunchKernelEx(&cfg, mmr_maxsim_kernel<METRIC, SMALL>, p));
    QB_LAUNCHED();
    return QB_OK;
}

template <bool SMALL>
qb_status launch_metric(const qb_storage* s, const MmsParams& p, uint32_t nq, uint32_t C, cudaStream_t stream) {
    switch (s->distance) {
        case QB_DIST_EUCLID: return launch_mms<M_EUCLID, SMALL>(p, nq, C, stream);
        case QB_DIST_MANHATTAN: return launch_mms<M_MANHATTAN, SMALL>(p, nq, C, stream);
        default: return launch_mms<M_DOT, SMALL>(p, nq, C, stream);
    }
}

uint32_t pre_queries(const qb_storage* s, uint32_t nq, uint32_t max_cand, uint32_t max_tokens) {
    const size_t per_query = (size_t)max_cand * max_tokens * s->row_stride;
    if (s->distance != QB_DIST_COSINE || per_query == 0) return 0;
    return (uint32_t)std::min<size_t>(nq, std::max<size_t>(1, MMS_PRE_BUDGET / per_query));
}

}  // namespace

size_t qb_mmr_maxsim_scratch_bytes(const qb_storage* s, uint32_t nq, uint32_t max_cand, uint32_t max_tokens) {
    return (size_t)pre_queries(s, nq, max_cand, max_tokens) * max_cand * max_tokens * s->row_stride;
}

qb_status qb_mmr_maxsim_launch(const qb_storage* s, const uint32_t* d_tok, uint32_t n_points, uint32_t max_tokens, const float* d_q_pre,
                               const uint32_t* d_q_off, uint32_t n_qv, uint32_t max_qv, uint32_t nq, const float* d_lambdas, const qb_scored_point* d_cand,
                               const uint32_t* d_cand_counts, uint32_t max_cand, uint32_t n_max, uint32_t limit, qb_scored_point* d_out,
                               uint32_t out_stride, uint32_t* d_out_counts, unsigned long long* d_pairs, float* d_scratch, cudaStream_t stream) {
    if (nq == 0) return QB_OK;
    const uint32_t C = mmr_ctas(n_max);
    MmsParams p{};
    p.rows = reinterpret_cast<const float*>(s->d_rows);
    p.stride_f = s->row_stride / 4; p.dim = s->dim; p.tok = d_tok; p.n_points = n_points;
    p.q_pre = d_q_pre; p.q_off = d_q_off; p.n_qv = n_qv;
    p.lambdas = d_lambdas; p.cand = d_cand; p.cand_counts = d_cand_counts; p.max_cand = max_cand;
    p.limit = limit; p.out = d_out; p.out_stride = out_stride; p.out_counts = d_out_counts; p.pairs = d_pairs;
    p.sm.stage_f = (uint32_t)std::min<uint64_t>(MMS_STAGE_MAX_F, (uint64_t)std::max(max_tokens, max_qv) * p.stride_f);
    p.sm.slice = std::max<uint32_t>(1, (uint32_t)ceil_div_u64(n_max, C));
    p.sm.n_cap = (uint32_t)round_up_u64(std::max<uint32_t>(n_max, 1), 8);
    const bool small = s->dim < 32;
    const uint32_t chunk = pre_queries(s, nq, max_cand, max_tokens);
    for (uint32_t q0 = 0; q0 < nq; q0 += chunk ? chunk : nq) {
        const uint32_t nqc = chunk ? std::min(chunk, nq - q0) : nq;
        p.q0 = q0;
        if (chunk) {
            const uint64_t n_rows = (uint64_t)nqc * max_cand * max_tokens;
            const uint64_t blocks = std::min<uint64_t>(ceil_div_u64(n_rows, 8), (uint64_t)s->sm_count * 16);
            mmr_maxsim_gather_kernel<<<(unsigned)blocks, 256, 0, stream>>>(p.rows, p.stride_f, d_tok, n_points, d_cand, d_cand_counts, max_cand, max_tokens,
                                                                           q0, n_rows, d_scratch);
            QB_LAUNCHED();
            QB_CUDA(cudaGetLastError());
            QB_TRY(qb_launch_preprocess_rows(QB_DIST_COSINE, s->dim, n_rows, d_scratch, p.stride_f, d_scratch, p.stride_f, stream));
            p.pre = d_scratch;
            p.pre_t = max_tokens;
        }
        QB_TRY(small ? launch_metric<true>(s, p, nqc, C, stream) : launch_metric<false>(s, p, nqc, C, stream));
    }
    return QB_OK;
}
