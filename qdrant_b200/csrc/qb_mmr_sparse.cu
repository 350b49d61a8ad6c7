// qb_mmr_sparse.cu — maximal marginal relevance (MMR) reranking of sparse vector candidate lists on the device.
//
// Replaces: mmr_from_points_with_vector (lib/shard/src/query/mmr/mod.rs:42-157) for a sparse named vector (mod.rs:130), whose candidates
// go into a VolatileSparseVectorStorage, each vector sorted by dim on insertion (volatile_sparse_vector_storage.rs:214-226), and LazyMatrix
// (lazy_matrix.rs:45-67), whose scorers are SparseMetricQueryScorer (query_scorer/sparse_metric_query_scorer.rs).  Here that storage is a
// qb_sparse_storage (qb_sparse_custom.cu), whose rows are sorted by dim already; candidate ids are its point ids.
//   score_vectors(a, b) = 0 + a_w * b_w over the shared dims in ascending dim order, every product and sum rounded; +0.0 when no dim is
//                         shared (sparse_vector.rs:66-90, unwrap_or_default in raw_scorer.rs:142-160)
//   rel[i]     = score_vectors(q, v_i)      the query sorted by dim on the host: VectorInternal::preprocess sorts a sparse vector
//                                           (vectors.rs:68-80), and the query of NearestWithMmr goes through it
//                                           (collection_query.rs:430) before it becomes MmrInternal's vector (collection_query.rs:472-480)
//   pair(c, s) = score_vectors(v_c, v_s)    symmetric bit for bit: the products commute and both orders sum in ascending dim order, so a
//                                           step scores every remaining candidate against the pick's row
// The selection is qb_mmr.cu's, with the same pieces (qb_mmr.cuh): one thread-block cluster per query, each CTA owning a slice of the
// candidates, replicated u16 position arrays, one DSMEM argmax per step and the same swap_remove.
//
// Scoring: one warp per remaining candidate of the slice reads the candidate's row 32 elements at a time; each lane binary-searches its
// element's dim in the other side's row (the sorted query in the relevance pass, the pick's row in a step) and the hits are added to a
// +0.0 accumulator in lane order with __fmul_rn / __fadd_rn, the ordered reduction of sparse_plain_kernel and sparse_custom_kernel, so
// every score sums in ascending dim order.  The other side is staged in shared memory up to MSP_STAGE_MAX elements and read from global
// memory past that; the bits are the same.  Counters: SparseMetricQueryScorer adds min(|a|, |b|) per scored pair (cpu multiplier 1);
// lane 0 of each warp sums its pairs and adds them to the query's u64 count.
#include <algorithm>

#include "qb_mmr.cuh"

using namespace qb_mmr;

namespace {

constexpr uint32_t MSP_STAGE_MAX = 4096;   // query / pick rows of up to 4096 elements (32 KB of dims and weights) are staged

// dynamic shared memory of one CTA: [stage dims | stage weights | 2 step slots + one per warp (u64) | 4 u32 | rel, maxsim, row start,
// row length (per owned) | rem, where]
struct MspSmem {
    uint32_t stage_e, slice, n_cap;                                    // stage_e even, so the slots start 16-byte aligned
    __host__ __device__ size_t slots_at() const { return (size_t)stage_e * 8; }
    __host__ __device__ size_t cnt_at() const { return slots_at() + (2 + MMR_WARPS) * 8; }
    __host__ __device__ size_t rel_at() const { return cnt_at() + 16; }
    __host__ __device__ size_t pos_at() const { return (rel_at() + (size_t)slice * 16 + 15) & ~(size_t)15; }
    __host__ __device__ size_t bytes() const { return pos_at() + (size_t)n_cap * 4; }
};

struct MspParams {
    const uint64_t* rptr; const uint32_t* rdims; const float* rw;   // the storage's rows, sorted by dim
    uint32_t n_points;
    const uint64_t* q_ptr; const uint32_t* q_dims; const float* q_w;   // [nq + 1] offsets; each query sorted by dim
    const float* lambdas;              // [nq]
    const qb_scored_point* cand;       // [nq][max_cand]
    const uint32_t* cand_counts;       // [nq]
    uint32_t max_cand, limit;
    qb_scored_point* out;              // [nq][out_stride]
    uint32_t out_stride;
    uint32_t* out_counts;              // [nq]
    unsigned long long* cpu;           // [nq], zeroed: the cpu counter
    MspSmem sm;
};

// score_vectors(candidate row cd / cw of n elements, other row od / ow of m elements), the same value in every lane of the warp
__device__ __forceinline__ float warp_score(const uint32_t* cd, const float* cw, uint32_t n, const uint32_t* od, const float* ow, uint32_t m, uint32_t lane) {
    float s = 0.0f;
    if (m == 0) return s;
    for (uint32_t c = 0; c < n; c += 32) {
        const uint32_t e = c + lane;
        bool hit = false;
        float prod = 0.0f;
        if (e < n) {
            const uint32_t d = cd[e];
            uint32_t a = 0, b = m;
            while (a < b) { const uint32_t mid = (a + b) >> 1; if (od[mid] < d) a = mid + 1; else b = mid; }
            if (a < m && od[a] == d) { hit = true; prod = __fmul_rn(ow[a], cw[e]); }
        }
        unsigned mask = __ballot_sync(0xFFFFFFFFu, hit);
        while (mask) {
            const int b = __ffs(mask) - 1;
            s = __fadd_rn(s, __shfl_sync(0xFFFFFFFFu, prod, b));
            mask &= mask - 1;
        }
    }
    return s;
}

// a row into the stage when it fits (every thread of the block calls it); *d / *w point at the row to read
__device__ __forceinline__ void stage_row(const MspParams& p, uint32_t* sdims, float* sw, uint32_t n, const uint32_t*& d, const float*& w) {
    if (n > p.sm.stage_e) return;
    for (uint32_t f = threadIdx.x; f < n; f += MMR_THREADS) {
        sdims[f] = d[f];
        sw[f] = w[f];
    }
    d = sdims;
    w = sw;
}

__global__ void __launch_bounds__(MMR_THREADS, 1) mmr_sparse_kernel(const MspParams p) {
    cg::cluster_group cluster = cg::this_cluster();
    const uint32_t C = cluster.num_blocks(), rank = cluster.block_rank();
    const uint32_t q = blockIdx.x / C, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    extern __shared__ __align__(16) unsigned char smem[];
    uint32_t* sdims = reinterpret_cast<uint32_t*>(smem);
    float* sw = reinterpret_cast<float*>(smem + (size_t)p.sm.stage_e * 4);
    unsigned long long* slot = reinterpret_cast<unsigned long long*>(smem + p.sm.slots_at());   // [2] this CTA's best of a step, by parity
    unsigned long long* wbest = slot + 2;                                                      // [MMR_WARPS]
    uint32_t* cnt = reinterpret_cast<uint32_t*>(smem + p.sm.cnt_at());                         // [0] kept candidates
    float* rel = reinterpret_cast<float*>(smem + p.sm.rel_at());
    float* msim = rel + p.sm.slice;
    uint32_t* r0 = reinterpret_cast<uint32_t*>(msim + p.sm.slice);                             // point id (~0 when not kept), then row start
    uint32_t* rn = r0 + p.sm.slice;                                                            // row length
    uint16_t* rem = reinterpret_cast<uint16_t*>(smem + p.sm.pos_at());
    uint16_t* where = rem + p.sm.n_cap;

    const qb_scored_point* cand = p.cand + (size_t)q * p.max_cand;
    const uint32_t n = min(p.cand_counts[q], p.max_cand);
    const uint32_t per = (n + C - 1) / C;
    const uint32_t lo = min(n, rank * per), hi = min(n, lo + per), sn = hi - lo;
    const uint16_t* where_s = where + lo;

    // 1. unique_by(id), first occurrence kept; ids outside the storage are dropped.  An empty row is a vector and stays
    mmr_dedup(tid, cand, lo, hi, r0, [&](uint32_t id, uint32_t& local) {
        local = id;
        return id < p.n_points;
    });
    // 2. positions (msim holds each kept candidate's rank within the slice)
    const uint32_t n_keep = mmr_positions(tid, cluster, C, rank, lo, hi, r0, reinterpret_cast<uint32_t*>(msim), wbest, cnt, rem, where);
    if (n_keep < 2) {   // mod.rs:77-80: returned as it is, no scoring
        if (rank == 0 && tid == 0) {
            if (n_keep == 1) p.out[(size_t)q * p.out_stride] = cand[rem[0]];
            p.out_counts[q] = n_keep;
        }
        return;
    }
    const uint32_t L = min(p.limit, n_keep);
    for (uint32_t j = tid; j < sn; j += MMR_THREADS) {
        if (where_s[j] == MMR_GONE) continue;
        const uint64_t a = p.rptr[r0[j]];
        rn[j] = (uint32_t)(p.rptr[r0[j] + 1] - a);
        r0[j] = (uint32_t)a;
    }

    // 3. relevance: score_vectors(q, v_j)
    const uint64_t qa = p.q_ptr[q];
    const uint32_t qn = (uint32_t)(p.q_ptr[q + 1] - qa);
    const uint32_t* od = p.q_dims + qa;
    const float* ow = p.q_w + qa;
    stage_row(p, sdims, sw, qn, od, ow);
    __syncthreads();
    unsigned long long best = 0, cpu = 0;
    for (uint32_t j = warp; j < sn; j += MMR_WARPS) {
        if (where_s[j] == MMR_GONE) continue;
        const float s = warp_score(p.rdims + r0[j], p.rw + r0[j], rn[j], od, ow, qn, lane);
        if (lane == 0) {
            rel[j] = s;
            cpu += min(rn[j], qn);
            const unsigned long long k = pos_key(s, where_s[j]);
            best = k > best ? k : best;
        }
    }

    const float lam = p.lambdas[q], one_minus = __fsub_rn(1.0f, lam);
    uint32_t remaining = n_keep, par = 0;
    for (uint32_t k = 0;; ++k, par ^= 1u) {
        // 4. cluster argmax of this step
        best = mmr_cluster_best(tid, cluster, C, best, wbest, slot, par);
        const uint32_t pos = (uint32_t)(best & 0xFFFFFFFFu), sel = rem[pos];
        if (rank == 0 && tid == 0) p.out[(size_t)q * p.out_stride + k] = cand[sel];
        if (k + 1 == L) break;
        __syncthreads();   // every thread has read rem[pos]
        // 5. swap_remove; stage the pick's row
        if (tid == 0) mmr_swap_remove(rem, where, pos, sel, remaining);
        --remaining;
        const uint32_t pid = cand[sel].idx;
        const uint64_t pa = p.rptr[pid];
        const uint32_t pn = (uint32_t)(p.rptr[pid + 1] - pa);
        const uint32_t* pd = p.rdims + pa;
        const float* pw = p.rw + pa;
        stage_row(p, sdims, sw, pn, pd, pw);
        __syncthreads();
        // 6. pair(c, pick) for every remaining candidate, the running max (new value on >=), mmr and the local argmax
        best = 0;
        for (uint32_t j = warp; j < sn; j += MMR_WARPS) {
            if (where_s[j] == MMR_GONE) continue;
            const float m = warp_score(p.rdims + r0[j], p.rw + r0[j], rn[j], pd, pw, pn, lane);
            if (lane == 0) {
                const float prev = msim[j];
                const float ms = (k == 0 || ord_key(m) >= ord_key(prev)) ? m : prev;
                msim[j] = ms;
                cpu += min(rn[j], pn);
                const float mmr = __fsub_rn(__fmul_rn(lam, rel[j]), __fmul_rn(one_minus, ms));
                const unsigned long long key = pos_key(mmr, where_s[j]);
                best = key > best ? key : best;
            }
        }
    }
    if (lane == 0 && cpu) atomicAdd(&p.cpu[q], cpu);
    if (rank == 0 && tid == 0) p.out_counts[q] = L;
    cluster.sync();   // no CTA leaves while a peer may still read its slot
}

}  // namespace

// ------------------------------------------------------------------------------------------------ the entry
extern "C" qb_status qb_mmr_sparse_batch(qb_sparse_storage* s, const uint64_t* q_indptr, const uint32_t* q_dims, const float* q_weights, uint32_t n_queries,
                                         const float* lambdas, const qb_scored_point* candidates, const uint32_t* candidate_counts, uint32_t max_candidates,
                                         uint32_t limit, qb_scored_point* out, uint32_t* out_counts, qb_hw_counters* counters) {
    const char* who = "mmr_sparse_batch";
    QB_CHECK(s && out_counts && (out || n_queries == 0), QB_ERR_INVALID, "%s: null argument", who);
    QB_CHECK(n_queries == 0 || (q_indptr && lambdas && candidate_counts && (candidates || max_candidates == 0)), QB_ERR_INVALID, "%s: null argument", who);
    QB_CHECK(max_candidates <= QB_MMR_MAX_CANDIDATES, QB_ERR_UNSUPPORTED, "%s: max_candidates %u > %u", who, max_candidates, QB_MMR_MAX_CANDIDATES);
    QB_CHECK(limit >= 1, QB_ERR_INVALID, "%s: limit must be >= 1", who);
    if (n_queries == 0) return QB_OK;
    QB_CHECK(q_indptr[0] == 0, QB_ERR_INVALID, "%s: q_indptr[0] must be 0", who);
    for (uint32_t q = 0; q < n_queries; ++q) QB_CHECK(q_indptr[q + 1] >= q_indptr[q], QB_ERR_INVALID, "%s: q_indptr descends at query %u", who, q);
    const uint64_t q_nnz = q_indptr[n_queries];
    QB_CHECK(q_nnz == 0 || (q_dims && q_weights), QB_ERR_INVALID, "%s: null argument", who);
    // every query sorted by dim (VectorInternal::preprocess); a repeated dim fails SparseVector validation
    std::vector<uint32_t> qd(q_nnz);
    std::vector<float> qw(q_nnz);
    std::vector<std::pair<uint32_t, float>> v;
    uint64_t max_len = 1;
    for (uint32_t q = 0; q < n_queries; ++q) {
        v.clear();
        for (uint64_t e = q_indptr[q]; e < q_indptr[q + 1]; ++e) v.emplace_back(q_dims[e], q_weights[e]);
        std::sort(v.begin(), v.end(), [](const std::pair<uint32_t, float>& a, const std::pair<uint32_t, float>& b) { return a.first < b.first; });
        for (size_t i = 1; i < v.size(); ++i) QB_CHECK(v[i].first != v[i - 1].first, QB_ERR_INVALID, "%s: dim %u repeated in query %u", who, v[i].first, q);
        for (size_t i = 0; i < v.size(); ++i) {
            qd[q_indptr[q] + i] = v[i].first;
            qw[q_indptr[q] + i] = v[i].second;
        }
        max_len = std::max<uint64_t>(max_len, v.size());
    }
    uint32_t n_max = 0;
    for (uint32_t q = 0; q < n_queries; ++q) {
        const float l = lambdas[q];
        QB_CHECK(l >= 0.0f && l <= 1.0f, QB_ERR_INVALID, "%s: lambda %g of query %u outside [0, 1]", who, (double)l, q);
        QB_CHECK(candidate_counts[q] <= max_candidates, QB_ERR_INVALID, "%s: %u candidates for query %u > max_candidates %u", who, candidate_counts[q], q,
                 max_candidates);
        n_max = std::max(n_max, candidate_counts[q]);
        for (uint32_t i = 0; i < candidate_counts[q]; ++i) {
            const uint32_t id = candidates[(size_t)q * max_candidates + i].idx;
            QB_CHECK(id < s->n_points, QB_ERR_INVALID, "%s: id %u >= n_points %u", who, id, s->n_points);
            max_len = std::max<uint64_t>(max_len, s->h_rptr[id + 1] - s->h_rptr[id]);
        }
    }
    QB_TRY(qb_use_device(s->device));
    std::lock_guard<std::mutex> lk(s->mu);
    const uint32_t C = mmr_ctas(n_max), out_stride = std::max<uint32_t>(1, std::min(limit, max_candidates));
    // scratch = [cpu nq (u64) | query offsets nq + 1 | lambdas nq | counts nq | candidates nq x max | query dims | query weights |
    //            selections nq x out_stride | out counts nq]; everything before the selections goes up, the cpu counts start at 0
    const size_t qp_at = (size_t)n_queries * 8, lam_at = qp_at + ((size_t)n_queries + 1) * 8, cnt_at = lam_at + (size_t)n_queries * 4;
    const size_t cand_at = round_up_u64(cnt_at + (size_t)n_queries * 4, 16), qd_at = cand_at + (size_t)n_queries * max_candidates * sizeof(qb_scored_point);
    const size_t qw_at = qd_at + q_nnz * 4, out_at = round_up_u64(qw_at + q_nnz * 4, 16), oc_at = out_at + (size_t)n_queries * out_stride * sizeof(qb_scored_point);
    const size_t bytes = oc_at + (size_t)n_queries * 4;
    QB_TRY(qb_ensure_device(&s->d_scratch, &s->scratch_bytes, bytes));
    std::vector<uint8_t> h(out_at, 0);
    memcpy(h.data() + qp_at, q_indptr, ((size_t)n_queries + 1) * 8);
    memcpy(h.data() + lam_at, lambdas, (size_t)n_queries * 4);
    memcpy(h.data() + cnt_at, candidate_counts, (size_t)n_queries * 4);
    if (max_candidates) memcpy(h.data() + cand_at, candidates, (size_t)n_queries * max_candidates * sizeof(qb_scored_point));
    if (q_nnz) {
        memcpy(h.data() + qd_at, qd.data(), q_nnz * 4);
        memcpy(h.data() + qw_at, qw.data(), q_nnz * 4);
    }
    uint8_t* d = reinterpret_cast<uint8_t*>(s->d_scratch);
    QB_CUDA(cudaMemcpyAsync(d, h.data(), out_at, cudaMemcpyHostToDevice, s->stream));
    MspParams p{};
    p.rptr = s->d_rptr; p.rdims = s->d_rdims; p.rw = s->d_rw; p.n_points = s->n_points;
    p.q_ptr = reinterpret_cast<const uint64_t*>(d + qp_at); p.q_dims = reinterpret_cast<const uint32_t*>(d + qd_at); p.q_w = reinterpret_cast<const float*>(d + qw_at);
    p.lambdas = reinterpret_cast<const float*>(d + lam_at);
    p.cand = reinterpret_cast<const qb_scored_point*>(d + cand_at); p.cand_counts = reinterpret_cast<const uint32_t*>(d + cnt_at);
    p.max_cand = max_candidates; p.limit = limit;
    p.out = reinterpret_cast<qb_scored_point*>(d + out_at); p.out_stride = out_stride; p.out_counts = reinterpret_cast<uint32_t*>(d + oc_at);
    p.cpu = reinterpret_cast<unsigned long long*>(d);
    p.sm.stage_e = (uint32_t)round_up_u64(std::min<uint64_t>(MSP_STAGE_MAX, max_len), 2);
    p.sm.slice = std::max<uint32_t>(1, (uint32_t)ceil_div_u64(n_max, C));
    p.sm.n_cap = (uint32_t)round_up_u64(std::max<uint32_t>(n_max, 1), 8);
    const size_t smem = p.sm.bytes();
    QB_CUDA(cudaFuncSetAttribute(mmr_sparse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(n_queries * C);
    cfg.blockDim = dim3(MMR_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    QB_CUDA(cudaLaunchKernelEx(&cfg, mmr_sparse_kernel, p));
    QB_LAUNCHED();
    std::vector<uint8_t> r(bytes - out_at);
    std::vector<unsigned long long> cpu(n_queries);
    QB_CUDA(cudaMemcpyAsync(r.data(), d + out_at, r.size(), cudaMemcpyDeviceToHost, s->stream));
    QB_CUDA(cudaMemcpyAsync(cpu.data(), d, (size_t)n_queries * 8, cudaMemcpyDeviceToHost, s->stream));
    QB_CUDA(cudaStreamSynchronize(s->stream));
    const qb_scored_point* h_res = reinterpret_cast<const qb_scored_point*>(r.data());
    const uint32_t* h_cnt = reinterpret_cast<const uint32_t*>(r.data() + (oc_at - out_at));
    for (uint32_t q = 0; q < n_queries; ++q) {
        out_counts[q] = h_cnt[q];
        memcpy(out + (size_t)q * limit, h_res + (size_t)q * out_stride, (size_t)h_cnt[q] * sizeof(qb_scored_point));
        // SparseMetricQueryScorer: cpu multiplier 1, min(|a|, |b|) per scored pair; vector_io_read: the volatile storage is in memory,
        // whether or not this storage is on disk
        if (counters) counters->cpu += cpu[q];
    }
    return QB_OK;
}
