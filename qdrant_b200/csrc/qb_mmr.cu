// qb_mmr.cu — maximal marginal relevance (MMR) reranking of candidate lists on the device.
//
// Replaces: mmr_from_points_with_vector + maximal_marginal_relevance (lib/shard/src/query/mmr/mod.rs:42-279) and LazyMatrix
// (lazy_matrix.rs) for dense vectors.  The reference puts the candidates' vectors into a volatile f32 storage without preprocessing
// (volatile_dense_vector_storage.rs:170-182); here that storage is any dense f32 qb_storage whose rows are those vectors.
//   rel[i]     = sim(preprocess(query), v_i)                    relevance_similarities, one RawScorer over every candidate
//   pair(c, s) = sim(preprocess(v_c), v_s)                      LazyMatrix::get_similarity(c, s): candidate c's scorer, point s
//   pick 1     = argmax rel over positions 0..n
//   pick k     = argmax over the remaining positions of λ·rel − (1 − λ)·max_{selected s, in selection order} pair(c, s)
// Every argmax / max is max_by_key(OrderedFloat): the LAST maximal element wins, NaN is above everything and equal to NaN, −0.0
// equals +0.0.  A pick is swap_remove-d from the IndexSet of remaining candidates, so ties are decided by current positions.
//
// One thread-block cluster per query does the whole selection.  The query's candidates (input indices 0..n) are split into C
// contiguous slices, one per CTA; a CTA keeps its slice's relevance, running max similarity and local row in shared memory, and
// every CTA keeps the same replicated position arrays (rem: position -> input index, where: input index -> position, u16).  Per
// step each CTA scores its remaining candidates against the newest pick (its stored row staged in shared memory), folds the running
// max, takes its local (mmr, position) argmax, and the CTAs reduce those through DSMEM after one cluster barrier; every CTA then
// applies the same swap_remove.  The scores are the f32 chains of qb_score.cuh that qb_score_points runs (score_avx_group8 for
// dim >= 32, score_small below), with the candidate's preprocessed row as the query side.  For Cosine, preprocess(v_c) is
// materialised by a gather + qb_launch_preprocess_rows into scratch; for the other distances it is the stored row itself.
#include "qb_mmr.cuh"

using namespace qb_mmr;

namespace {

constexpr uint32_t MMR_STAGE_MAX_F = 16384;           // stored rows of up to 64 KB are staged in shared memory, longer ones read from HBM
constexpr size_t MMR_PRE_BUDGET = 512ull << 20;       // Cosine: preprocessed candidate rows of one launch

// dynamic shared memory of one CTA: [staged row | 2 step slots + one per warp (u64) | 4 u32 | rel, maxsim, row (per owned) | rem, where]
struct MmrSmem {
    uint32_t stage_f, slice, n_cap;
    __host__ __device__ size_t slots_at() const { return (size_t)stage_f * 4; }
    __host__ __device__ size_t cnt_at() const { return slots_at() + (2 + MMR_WARPS) * 8; }
    __host__ __device__ size_t rel_at() const { return cnt_at() + 16; }
    __host__ __device__ size_t pos_at() const { return rel_at() + (size_t)slice * 12; }
    __host__ __device__ size_t bytes() const { return pos_at() + (size_t)n_cap * 4; }
};

struct MmrParams {
    const float* rows;                 // the storage's rows, stride_f floats apart
    uint32_t stride_f, dim;
    uint64_t count;
    uint32_t id_base;
    const float* q_pre;                // [nq][stride_f] preprocessed queries
    const float* lambdas;              // [nq]
    const qb_scored_point* cand;       // [nq][max_cand]
    const uint32_t* cand_counts;       // [nq]
    uint32_t max_cand;
    const float* pre;                  // Cosine: [launch queries][max_cand][stride_f] preprocess(v_i) by input index; null: the stored rows
    uint32_t q0;                       // first query of this launch
    uint32_t limit;
    qb_scored_point* out;              // [nq][out_stride]
    uint32_t out_stride;
    uint32_t* out_counts;              // [nq]
    uint32_t* n_unique;                // [nq]: candidates left after the dedup (for the counters)
    MmrSmem sm;
};

// score = sim(qry, row) by the chain qb_score_points runs: lanes of an 8-lane group (AVX tier) or one thread (dim < 32)
template <int METRIC, bool SMALL>
__device__ __forceinline__ float pair_score(const float* row, const float* qry, uint32_t dim) {
    if (SMALL) return score_small<METRIC>(row, qry, dim);
    return score_avx_group8<METRIC>(row, qry, dim, threadIdx.x & 7);
}

template <int METRIC, bool SMALL>
__global__ void __launch_bounds__(MMR_THREADS, 1) mmr_kernel(const MmrParams p) {
    cg::cluster_group cluster = cg::this_cluster();
    const uint32_t C = cluster.num_blocks(), rank = cluster.block_rank();
    const uint32_t ql = blockIdx.x / C, q = p.q0 + ql, tid = threadIdx.x;
    extern __shared__ __align__(16) unsigned char smem[];
    float* srow = reinterpret_cast<float*>(smem);
    unsigned long long* slot = reinterpret_cast<unsigned long long*>(smem + p.sm.slots_at());   // [2] this CTA's best of a step, by parity
    unsigned long long* wbest = slot + 2;                                                      // [MMR_WARPS]
    uint32_t* cnt = reinterpret_cast<uint32_t*>(smem + p.sm.cnt_at());                         // [0]: kept candidates of the slice
    float* rel = reinterpret_cast<float*>(smem + p.sm.rel_at());
    float* msim = rel + p.sm.slice;
    uint32_t* lrow = reinterpret_cast<uint32_t*>(msim + p.sm.slice);
    uint16_t* rem = reinterpret_cast<uint16_t*>(smem + p.sm.pos_at());
    uint16_t* where = rem + p.sm.n_cap;

    const qb_scored_point* cand = p.cand + (size_t)q * p.max_cand;
    const uint32_t n = min(p.cand_counts[q], p.max_cand);
    const uint32_t per = (n + C - 1) / C;
    const uint32_t lo = min(n, rank * per), hi = min(n, lo + per);
    const bool stage = p.sm.stage_f != 0;

    // 1. unique_by(id), first occurrence kept; ids outside the storage are dropped.  lrow = local row, or ~0 when not kept
    for (uint32_t i = lo + tid; i < hi; i += MMR_THREADS) {
        const uint32_t id = cand[i].idx, local = id - p.id_base;
        bool keep = id >= p.id_base && (uint64_t)local < p.count;
        for (uint32_t j = 0; keep && j < i; ++j) keep = __ldg(&cand[j].idx) != id;
        lrow[i - lo] = keep ? local : 0xFFFFFFFFu;
    }
    __syncthreads();
    // 2. positions: the kept candidates in input order, numbered across the cluster.  msim holds each one's rank within the slice
    uint32_t* kpos = reinterpret_cast<uint32_t*>(msim);
    uint32_t run = 0;
    for (uint32_t base = lo; base < hi; base += MMR_THREADS) {
        const uint32_t i = base + tid;
        const bool f = i < hi && lrow[i - lo] != 0xFFFFFFFFu;
        const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, f), lane = tid & 31, warp = tid >> 5;
        if (lane == 0) reinterpret_cast<uint32_t*>(wbest)[warp] = __popc(ballot);
        __syncthreads();
        uint32_t off = run, total = 0;
        for (uint32_t w = 0; w < MMR_WARPS; ++w) {
            const uint32_t c = reinterpret_cast<uint32_t*>(wbest)[w];
            if (w < warp) off += c;
            total += c;
        }
        if (f) kpos[i - lo] = off + __popc(ballot & ((1u << lane) - 1u));
        __syncthreads();
        run += total;
    }
    if (tid == 0) cnt[0] = run;
    cluster.sync();
    uint32_t offset = 0, n_keep = 0;
    for (uint32_t r = 0; r < C; ++r) {
        const uint32_t c = *cluster.map_shared_rank(cnt, r);
        if (r < rank) offset += c;
        n_keep += c;
    }
    for (uint32_t i = lo + tid; i < hi; i += MMR_THREADS) {
        const bool f = lrow[i - lo] != 0xFFFFFFFFu;
        const uint32_t pos = f ? offset + kpos[i - lo] : MMR_GONE;
        for (uint32_t r = 0; r < C; ++r) {
            cluster.map_shared_rank(where, r)[i] = (uint16_t)pos;
            if (f) cluster.map_shared_rank(rem, r)[pos] = (uint16_t)i;
        }
    }
    cluster.sync();   // every CTA's rem / where complete; the last remote access of the slot counts
    if (n_keep < 2) {   // mod.rs:77-80: returned as it is, no scoring
        if (rank == 0 && tid == 0) {
            if (n_keep == 1) p.out[(size_t)q * p.out_stride] = cand[rem[0]];
            p.out_counts[q] = n_keep;
            p.n_unique[q] = n_keep;
        }
        return;
    }
    const uint32_t L = min(p.limit, n_keep);

    // 3. relevance of the slice against the preprocessed query; the first pick's key
    const float* qry = p.q_pre + (size_t)q * p.stride_f;
    if (stage) {
        for (uint32_t f = tid; f < p.stride_f; f += MMR_THREADS) srow[f] = qry[f];
        __syncthreads();
        qry = srow;
    }
    const uint32_t unit = SMALL ? 1u : 8u, n_units = MMR_THREADS / unit, u = tid / unit;
    unsigned long long best = 0;
    for (uint32_t base = lo; base < hi; base += n_units) {
        const uint32_t i = base + u;
        const bool ok = i < hi && where[i] != MMR_GONE;
        if (!SMALL && !__any_sync(0xFFFFFFFFu, ok)) continue;
        if (SMALL && !ok) continue;
        const float* row = ok ? p.rows + (size_t)lrow[i - lo] * p.stride_f : p.rows;   // a lane without a candidate scores row 0 and drops it
        const float s = pair_score<METRIC, SMALL>(row, qry, p.dim);
        if (ok) {
            if (SMALL || (tid & 7) == 0) rel[i - lo] = s;
            const unsigned long long k = pos_key(s, where[i]);
            best = k > best ? k : best;
        }
    }

    const float lam = p.lambdas[q], one_minus = __fsub_rn(1.0f, lam);
    const float* pre = p.pre ? p.pre + (size_t)ql * p.max_cand * p.stride_f : nullptr;
    uint32_t remaining = n_keep, par = 0;
    for (uint32_t k = 0;; ++k, par ^= 1u) {
        // 4. cluster argmax of this step: every CTA reads every CTA's slot after one barrier, and takes the same pick
        best = mmr_cluster_best(tid, cluster, C, best, wbest, slot, par);
        const uint32_t pos = (uint32_t)(best & 0xFFFFFFFFu), sel = rem[pos];
        if (rank == 0 && tid == 0) p.out[(size_t)q * p.out_stride + k] = cand[sel];
        if (k + 1 == L) break;
        __syncthreads();   // every thread has read rem[pos]
        // 5. IndexSet::swap_remove on the replicated positions; stage the pick's stored row
        if (tid == 0) mmr_swap_remove(rem, where, pos, sel, remaining);
        --remaining;
        const float* srow_g = p.rows + (size_t)(cand[sel].idx - p.id_base) * p.stride_f;
        const float* vs = srow_g;
        if (stage) {
            for (uint32_t f = tid; f < p.stride_f; f += MMR_THREADS) srow[f] = srow_g[f];
            vs = srow;
        }
        __syncthreads();
        // 6. pair(c, newest) for the slice's remaining candidates, the running max (new value on >=), mmr and the local argmax
        best = 0;
        for (uint32_t base = lo; base < hi; base += n_units) {
            const uint32_t i = base + u;
            const bool ok = i < hi && where[i] != MMR_GONE;
            if (!SMALL && !__any_sync(0xFFFFFFFFu, ok)) continue;
            if (SMALL && !ok) continue;
            const uint32_t j = ok ? i - lo : 0;
            const float* qc = pre ? pre + (size_t)(lo + j) * p.stride_f : ok ? p.rows + (size_t)lrow[j] * p.stride_f : p.rows;
            const float m = pair_score<METRIC, SMALL>(vs, qc, p.dim);
            if (ok) {
                const float prev = msim[j];
                const float ms = (k == 0 || ord_key(m) >= ord_key(prev)) ? m : prev;
                if (SMALL || (tid & 7) == 0) msim[j] = ms;
                const float mmr = __fsub_rn(__fmul_rn(lam, rel[j]), __fmul_rn(one_minus, ms));
                const unsigned long long key = pos_key(mmr, where[i]);
                best = key > best ? key : best;
            }
        }
    }
    if (rank == 0 && tid == 0) {
        p.out_counts[q] = L;
        p.n_unique[q] = n_keep;
    }
    cluster.sync();   // no CTA leaves while a peer may still read its slot
}

// Cosine: rows[(q - q0) * max_cand + i] = the stored row of candidate i of query q (zeros past the count or for an id outside the
// storage), to be preprocessed in place.  One warp per row.
__global__ void __launch_bounds__(256) mmr_gather_kernel(const float* __restrict__ rows, uint32_t stride_f, uint64_t count, uint32_t id_base,
                                                         const qb_scored_point* __restrict__ cand, const uint32_t* __restrict__ cand_counts,
                                                         uint32_t max_cand, uint32_t q0, uint64_t n_rows, float* __restrict__ out) {
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    const uint32_t lane = threadIdx.x & 31;
    for (uint64_t r = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < n_rows; r += warps) {
        const uint32_t q = q0 + (uint32_t)(r / max_cand), i = (uint32_t)(r % max_cand);
        const uint32_t id = cand[(size_t)q * max_cand + i].idx, local = id - id_base;
        const bool ok = i < min(cand_counts[q], max_cand) && id >= id_base && (uint64_t)local < count;
        const float4* src = reinterpret_cast<const float4*>(rows + (size_t)local * stride_f);
        float4* dst = reinterpret_cast<float4*>(out + (size_t)r * stride_f);
        for (uint32_t f = lane; f < stride_f / 4; f += 32) dst[f] = ok ? src[f] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

template <int METRIC, bool SMALL>
qb_status launch_mmr(const MmrParams& p, uint32_t nq, uint32_t C, cudaStream_t stream) {
    const size_t smem = p.sm.bytes();
    QB_CUDA(cudaFuncSetAttribute(mmr_kernel<METRIC, SMALL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
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
    QB_CUDA(cudaLaunchKernelEx(&cfg, mmr_kernel<METRIC, SMALL>, p));
    QB_LAUNCHED();
    return QB_OK;
}

template <bool SMALL>
qb_status launch_metric(const qb_storage* s, const MmrParams& p, uint32_t nq, uint32_t C, cudaStream_t stream) {
    switch (s->distance) {
        case QB_DIST_EUCLID: return launch_mmr<M_EUCLID, SMALL>(p, nq, C, stream);
        case QB_DIST_MANHATTAN: return launch_mmr<M_MANHATTAN, SMALL>(p, nq, C, stream);
        default: return launch_mmr<M_DOT, SMALL>(p, nq, C, stream);
    }
}

uint32_t pre_queries(const qb_storage* s, uint32_t nq, uint32_t max_cand) {
    const size_t per_query = (size_t)max_cand * s->row_stride;
    if (s->distance != QB_DIST_COSINE || per_query == 0) return 0;
    return (uint32_t)std::min<size_t>(nq, std::max<size_t>(1, MMR_PRE_BUDGET / per_query));
}

}  // namespace

size_t qb_mmr_scratch_bytes(const qb_storage* s, uint32_t nq, uint32_t max_cand) {
    return (size_t)pre_queries(s, nq, max_cand) * max_cand * s->row_stride;
}

qb_status qb_mmr_launch(const qb_storage* s, const float* d_q_pre, uint32_t nq, const float* d_lambdas, const qb_scored_point* d_cand,
                        const uint32_t* d_cand_counts, uint32_t max_cand, uint32_t n_max, uint32_t limit, qb_scored_point* d_out, uint32_t out_stride,
                        uint32_t* d_out_counts, uint32_t* d_n_unique, float* d_scratch, cudaStream_t stream) {
    if (nq == 0) return QB_OK;
    const uint32_t C = mmr_ctas(n_max);
    MmrParams p{};
    p.rows = reinterpret_cast<const float*>(s->d_rows);
    p.stride_f = s->row_stride / 4; p.dim = s->dim; p.count = s->count; p.id_base = s->id_base;
    p.q_pre = d_q_pre; p.lambdas = d_lambdas; p.cand = d_cand; p.cand_counts = d_cand_counts; p.max_cand = max_cand;
    p.limit = limit; p.out = d_out; p.out_stride = out_stride; p.out_counts = d_out_counts; p.n_unique = d_n_unique;
    p.sm.stage_f = p.stride_f <= MMR_STAGE_MAX_F ? p.stride_f : 0;
    p.sm.slice = std::max<uint32_t>(1, (uint32_t)ceil_div_u64(n_max, C));
    p.sm.n_cap = (uint32_t)round_up_u64(std::max<uint32_t>(n_max, 1), 8);
    const bool small = s->dim < 32;
    const uint32_t chunk = pre_queries(s, nq, max_cand);
    for (uint32_t q0 = 0; q0 < nq; q0 += chunk ? chunk : nq) {
        const uint32_t nqc = chunk ? std::min(chunk, nq - q0) : nq;
        p.q0 = q0;
        if (chunk) {
            const uint64_t n_rows = (uint64_t)nqc * max_cand;
            const uint64_t blocks = std::min<uint64_t>(ceil_div_u64(n_rows, 8), (uint64_t)s->sm_count * 16);
            mmr_gather_kernel<<<(unsigned)blocks, 256, 0, stream>>>(p.rows, p.stride_f, s->count, s->id_base, d_cand, d_cand_counts, max_cand, q0, n_rows,
                                                                    d_scratch);
            QB_LAUNCHED();
            QB_CUDA(cudaGetLastError());
            QB_TRY(qb_launch_preprocess_rows(QB_DIST_COSINE, s->dim, n_rows, d_scratch, p.stride_f, d_scratch, p.stride_f, stream));
            p.pre = d_scratch;
        }
        QB_TRY(small ? launch_metric<true>(s, p, nqc, C, stream) : launch_metric<false>(s, p, nqc, C, stream));
    }
    return QB_OK;
}
