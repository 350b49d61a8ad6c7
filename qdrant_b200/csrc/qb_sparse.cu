// qb_sparse.cu — sparse vectors: an inverted index in HBM, its batched search (SearchContext::search,
// lib/sparse/src/index/search_context.rs:263-414) and plain search over caller-filtered ids (plain_search, :92-143).
//
// Index (qb_sparse_index_create): the points' CSR rows are sorted by (row, dim) and kept for plain search; the posting lists are the
// same elements sorted by (dim, id), laid out as ids / weights / max_next_weight arrays with one offset per dim
// (PostingBuilder::build, posting_list.rs:140-170).  Both sorts are CUB radix sorts.
//
// Search: one CTA per query, queries drawn from a work counter.  The kernel replays the reference's state machine exactly:
//   - a batch [min_id, min(min_id + 10 000, max_record_id)] zeroes a shared f32 score array, then every list in its current order
//     adds weight * query_weight for its elements in the batch (ids are distinct within a list, so the CTA adds one list's elements
//     in parallel; a barrier between lists keeps the reference's summation order 0 + p1 + p2 + ...);
//   - the batch's scores that are non-zero, pass the filter and beat the running threshold are pushed, in id order, into an exact
//     emulation of TopK (common/src/top_k.rs:22-64): a buffer of 2k keys; when it fills, the k-th largest becomes the threshold and
//     the k best stay.  Keys order by (score desc, id asc), so the kept tie members are the smaller ids;
//   - one thread then retains the live lists, pushes the last list's remaining elements (no non-zero test), or promotes the longest
//     list (the last of equal lengths) and prunes it against the threshold, as the reference does.
// Plain search: one warp per id merge-joins the point's row with the query in ascending dim order, and the existing top-k selection
// (qb_topk.cu) keeps the best.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cfloat>

#include "qb_internal.h"

namespace {

constexpr uint32_t SP_THREADS = 256;
constexpr uint32_t SP_WARPS = SP_THREADS / 32;
constexpr uint32_t SP_BATCH = 10000;              // ADVANCE_BATCH_SIZE (search_context.rs:25): a batch spans up to 10 001 ids
constexpr uint32_t SP_SCORES = SP_BATCH + 1;
constexpr uint32_t SP_SCORES_BYTES = (SP_SCORES * 4 + 15) / 16 * 16;
constexpr uint32_t SP_PLAIN_IDS_PER_BLOCK = 64;

struct SpList { uint32_t pos, end, bend; float qw; };   // a posting list's cursor, its end, its end in the current batch, the query weight

__device__ __forceinline__ bool sp_deleted(const uint32_t* del, uint32_t id) { return del && ((del[id >> 5] >> (id & 31)) & 1u); }

__device__ __forceinline__ void sp_bitonic_desc(unsigned long long* buf, uint32_t n_pow2) {
    for (uint32_t k = 2; k <= n_pow2; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < n_pow2; i += blockDim.x) {
                const uint32_t ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = buf[i], b = buf[ixj];
                    const bool desc = (i & k) == 0;
                    if (desc ? (a < b) : (a > b)) { buf[i] = b; buf[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
}

// rank of a true flag among the CTA's flags in thread order, and their total; every thread calls it
__device__ __forceinline__ uint32_t sp_block_rank(bool f, uint32_t* s_w, uint32_t* total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned b = __ballot_sync(0xFFFFFFFFu, f);
    if (lane == 0) s_w[warp] = __popc(b);
    __syncthreads();
    uint32_t off = 0, tot = 0;
#pragma unroll
    for (uint32_t w = 0; w < SP_WARPS; ++w) { const uint32_t v = s_w[w]; off += w < warp ? v : 0u; tot += v; }
    __syncthreads();
    *total = tot;
    return off + __popc(b & ((1u << lane) - 1u));
}

struct SpTopK {
    unsigned long long* buf;   // p2 >= 2k keys, zero beyond len
    uint32_t k, p2;
    uint32_t* len; float* thr; uint32_t* s_w;
};

// TopK::push of this thread's candidate, the CTA's candidates taken in thread order: a push needs score > threshold; when the buffer
// reaches 2k the k-th largest key's score becomes the threshold and the k largest keys stay.  `want` holds the pushes' other
// conditions; the threshold test is applied here, again after every compaction.
__device__ void sp_push(const SpTopK& t, bool want, float score, uint32_t id) {
    want = want && score > *t.thr;
    for (;;) {
        uint32_t tot;
        const uint32_t r = sp_block_rank(want, t.s_w, &tot);
        if (tot == 0) return;
        const uint32_t len = *t.len, room = 2 * t.k - len;
        if (want && r < room) t.buf[len + r] = qb_pack_key(score, id);
        __syncthreads();
        if (tot < room) {
            if (threadIdx.x == 0) *t.len = len + tot;
            __syncthreads();
            return;
        }
        sp_bitonic_desc(t.buf, t.p2);
        for (uint32_t i = t.k + threadIdx.x; i < 2 * t.k; i += blockDim.x) t.buf[i] = 0ull;
        if (threadIdx.x == 0) { *t.thr = qb_key_score(t.buf[t.k - 1]); *t.len = t.k; }
        __syncthreads();
        want = want && r >= room && score > *t.thr;
    }
}

struct SparseSearchParams {
    const uint32_t* ids; const float* w; const float* mnw; const uint64_t* dptr; uint32_t n_dims;
    const uint64_t* q_ptr; const uint32_t* q_dims; const float* q_w; uint32_t nq, max_nnz;
    const uint32_t* deleted;   // 32-bit words, bit = 1 deleted; or null
    uint32_t top, p2; int allow_pruning;
    qb_scored_point* out; uint32_t* out_counts;
    unsigned int* work;
};

// the first index in [lo, hi) whose id is >= x (binary_search_by's Ok / Err position for distinct ids, posting_list.rs:268-290)
__device__ __forceinline__ uint32_t sp_lower_bound(const uint32_t* ids, uint32_t lo, uint32_t hi, uint32_t x) {
    while (lo < hi) { const uint32_t m = lo + (hi - lo) / 2; if (ids[m] < x) lo = m + 1; else hi = m; }
    return lo;
}

__global__ void __launch_bounds__(SP_THREADS) sparse_search_kernel(const SparseSearchParams p) {
    extern __shared__ __align__(16) unsigned char sp_smem[];
    float* scores = reinterpret_cast<float*>(sp_smem);
    SpList* lists = reinterpret_cast<SpList*>(sp_smem + SP_SCORES_BYTES);
    unsigned long long* buf = reinterpret_cast<unsigned long long*>(sp_smem + SP_SCORES_BYTES + (size_t)p.max_nnz * sizeof(SpList));
    __shared__ uint32_t s_w[SP_WARPS];
    __shared__ uint32_t s_q, s_len, s_nl, s_nkept, s_state, s_start, s_last;
    __shared__ float s_thr;
    const SpTopK t{buf, p.top, p.p2, &s_len, &s_thr, s_w};
    for (;;) {
        if (threadIdx.x == 0) s_q = atomicAdd(p.work, 1u);
        __syncthreads();
        const uint32_t q = s_q;
        if (q >= p.nq) return;
        // the query, sorted by (dim, position) with the dims >= n_dims dropped (remap_vector, indices_tracker.rs:53-72), staged in lists[]
        const uint64_t qb = p.q_ptr[q];
        const uint32_t n_raw = (uint32_t)min((unsigned long long)(p.q_ptr[q + 1] - qb), (unsigned long long)p.max_nnz);
        uint2* raw = reinterpret_cast<uint2*>(scores);
        for (uint32_t i = threadIdx.x; i < n_raw; i += blockDim.x) raw[i] = make_uint2(p.q_dims[qb + i], __float_as_uint(p.q_w[qb + i]));
        for (uint32_t i = threadIdx.x; i < p.p2; i += blockDim.x) buf[i] = 0ull;
        if (threadIdx.x == 0) { s_len = 0; s_thr = -FLT_MAX; s_nkept = 0; }
        __syncthreads();
        bool nonneg = true;
        uint32_t kept = 0;
        for (uint32_t i = threadIdx.x; i < n_raw; i += blockDim.x) {
            const uint2 e = raw[i];
            if (e.x >= p.n_dims) continue;
            uint32_t r = 0;
            for (uint32_t j = 0; j < n_raw; ++j) { const uint32_t d = raw[j].x; r += d < p.n_dims && (d < e.x || (d == e.x && j < i)); }
            lists[r] = SpList{e.x, 0u, 0u, __uint_as_float(e.y)};
            nonneg = nonneg && __uint_as_float(e.y) >= 0.0f;
            ++kept;
        }
        // pruning needs reliable max_next_weight (the RAM lists) and no negative query weight (search_context.rs:67-72)
        const int use_pruning = __syncthreads_and(nonneg) && p.allow_pruning;
        if (kept) atomicAdd(&s_nkept, kept);
        __syncthreads();
        uint32_t min_id = 0, max_id = 0;
        if (threadIdx.x == 0) {
            // the lists that exist and are non-empty, in query order (:42-87)
            uint32_t nl = 0;
            min_id = 0xFFFFFFFFu;
            for (uint32_t j = 0; j < s_nkept; ++j) {
                const SpList e = lists[j];
                const uint32_t b = (uint32_t)p.dptr[e.pos], en = (uint32_t)p.dptr[e.pos + 1];
                if (b == en) continue;
                lists[nl++] = SpList{b, en, b, e.qw};
                min_id = min(min_id, p.ids[b]);
                max_id = max(max_id, p.ids[en - 1]);
            }
            s_nl = nl;
            s_state = nl ? 0u : 1u;   // 0 = next batch, 1 = done, 2 = the last list
            s_start = min_id;
        }
        __syncthreads();
        float best_min = -FLT_MAX;   // thread 0's copy
        while (s_state == 0) {
            const uint32_t start = s_start;
            if (threadIdx.x == 0) s_last = (uint32_t)min((unsigned long long)start + SP_BATCH, (unsigned long long)max_id);
            const uint32_t nl = s_nl;
            // every list's end in this batch (for_each_till_id, posting_list.rs:211-226)
            __syncthreads();
            const uint32_t last = s_last, blen = last - start + 1;
            for (uint32_t j = threadIdx.x; j < nl; j += blockDim.x) lists[j].bend = sp_lower_bound(p.ids, lists[j].pos, lists[j].end, last + 1);
            for (uint32_t i = threadIdx.x; i < blen; i += blockDim.x) scores[i] = 0.0f;
            __syncthreads();
            // advance_batch (:146-187): the lists in their current order, one barrier apart
            for (uint32_t j = 0; j < nl; ++j) {
                const SpList L = lists[j];
                if (L.pos == L.bend) continue;
                for (uint32_t i = L.pos + threadIdx.x; i < L.bend; i += blockDim.x) {
                    const uint32_t li = p.ids[i] - start;
                    scores[li] = __fadd_rn(scores[li], __fmul_rn(p.w[i], L.qw));
                }
                __syncthreads();
            }
            for (uint32_t base = 0; base < blen; base += blockDim.x) {
                const uint32_t i = base + threadIdx.x;
                const float sc = i < blen ? scores[i] : 0.0f;
                sp_push(t, i < blen && sc != 0.0f && !sp_deleted(p.deleted, start + i), sc, start + i);
            }
            if (threadIdx.x == 0) {
                // retain the lists with elements left, in order; the next min id
                uint32_t n = 0;
                for (uint32_t j = 0; j < nl; ++j) { SpList L = lists[j]; L.pos = L.bend; if (L.pos != L.end) lists[n++] = L; }
                uint32_t nmin = 0xFFFFFFFFu;
                for (uint32_t j = 0; j < n; ++j) nmin = min(nmin, p.ids[lists[j].pos]);
                s_nl = n;
                if (n == 0) s_state = 1;
                else if (n == 1) s_state = 2;
                else if (use_pruning && s_len >= p.top && s_thr != best_min) {
                    const float min_score = s_thr;
                    best_min = min_score;
                    // promote_longest_posting_lists_to_the_front (:232-252): max_by keeps the last of equal lengths
                    uint32_t li = 0;
                    for (uint32_t j = 1; j < n; ++j) if (lists[j].end - lists[j].pos >= lists[li].end - lists[li].pos) li = j;
                    if (li != 0) { const SpList tmp = lists[0]; lists[0] = lists[li]; lists[li] = tmp; }
                    // prune_longest_posting_list (:350-414); with n >= 2 the other lists are never all exhausted here
                    const SpList L = lists[0];
                    uint32_t nm = 0xFFFFFFFFu;
                    for (uint32_t j = 1; j < n; ++j) nm = min(nm, p.ids[lists[j].pos]);
                    const uint32_t eid = p.ids[L.pos];
                    if (nm > eid && __fmul_rn(fmaxf(p.w[L.pos], p.mnw[L.pos]), L.qw) <= min_score) {
                        lists[0].pos = sp_lower_bound(p.ids, L.pos, L.end, nm);
                        if (lists[0].pos != L.pos) {
                            nmin = 0xFFFFFFFFu;
                            for (uint32_t j = 0; j < n; ++j) if (lists[j].pos != lists[j].end) nmin = min(nmin, p.ids[lists[j].pos]);
                        }
                    }
                }
                s_start = nmin;
            }
            __syncthreads();
        }
        if (s_state == 2) {
            // process_last_posting_list (:189-205): every remaining element that passes the filter, no non-zero test
            const SpList L = lists[0];
            for (uint32_t base = L.pos; base < L.end; base += blockDim.x) {
                const uint32_t i = base + threadIdx.x;
                const bool in = i < L.end;
                const uint32_t id = in ? p.ids[i] : 0u;
                const float sc = in ? __fmul_rn(p.w[i], L.qw) : 0.0f;
                sp_push(t, in && !sp_deleted(p.deleted, id), sc, id);
            }
        }
        // into_vec: sorted, at most k
        sp_bitonic_desc(buf, p.p2);
        const uint32_t n_out = min(s_len, p.top);
        for (uint32_t i = threadIdx.x; i < n_out; i += blockDim.x) {
            const unsigned long long k = buf[i];
            p.out[(size_t)q * p.top + i] = qb_scored_point{qb_key_id(k), qb_key_score(k)};
        }
        if (threadIdx.x == 0) p.out_counts[q] = n_out;
        __syncthreads();
    }
}

// plain_search (:92-143) of query blockIdx.y over ids [blockIdx.x * 64, +64) of its list: one warp per id merge-joins the point's row
// (ascending dims) with the query (ascending kept dims) and sums stored * query from +0.0 in that order (score_vectors,
// sparse_vector.rs:66-90).  An id with no common dim is not pushed, nor is a score <= f32::MIN (TopK's initial threshold) or NaN.
__global__ void __launch_bounds__(SP_THREADS) sparse_plain_kernel(const uint64_t* rptr, const uint32_t* rdims, const float* rw, const uint64_t* q_ptr,
                                                                  const uint32_t* q_dims, const float* q_w, const uint64_t* id_ptr, const uint32_t* ids,
                                                                  uint32_t q0, unsigned long long* cand, uint64_t cap, unsigned long long* cpu) {
    extern __shared__ __align__(16) unsigned char sp_smem[];
    const uint32_t q = q0 + blockIdx.y;
    const uint64_t qb = q_ptr[q];
    const uint32_t nk = (uint32_t)(q_ptr[q + 1] - qb);
    uint32_t* sd = reinterpret_cast<uint32_t*>(sp_smem);
    float* sw = reinterpret_cast<float*>(sp_smem + (size_t)nk * 4);
    for (uint32_t i = threadIdx.x; i < nk; i += blockDim.x) { sd[i] = q_dims[qb + i]; sw[i] = q_w[qb + i]; }
    __syncthreads();
    const uint64_t ib = id_ptr[q], n_ids = id_ptr[q + 1] - ib;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long units = 0;
    for (uint64_t k = (uint64_t)blockIdx.x * SP_PLAIN_IDS_PER_BLOCK + warp; k < min((unsigned long long)n_ids, (unsigned long long)(blockIdx.x + 1) * SP_PLAIN_IDS_PER_BLOCK); k += SP_WARPS) {
        const uint32_t id = ids[ib + k];
        const uint64_t r0 = rptr[id], r1 = rptr[id + 1];
        float s = 0.0f;
        uint32_t matched = 0;
        for (uint64_t c = r0; c < r1; c += 32) {
            const uint64_t e = c + lane;
            float prod = 0.0f;
            bool hit = false;
            if (e < r1) {
                const uint32_t d = rdims[e];
                uint32_t lo = 0, hi = nk;
                while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (sd[m] < d) lo = m + 1; else hi = m; }
                if (lo < nk && sd[lo] == d) { hit = true; prod = __fmul_rn(rw[e], sw[lo]); }
            }
            unsigned mask = __ballot_sync(0xFFFFFFFFu, hit);
            matched += __popc(mask);
            while (mask) {
                const int b = __ffs(mask) - 1;
                s = __fadd_rn(s, __shfl_sync(0xFFFFFFFFu, prod, b));
                mask &= mask - 1;
            }
        }
        if (lane == 0) {
            cand[(uint64_t)blockIdx.y * cap + k] = (matched && s > -FLT_MAX) ? qb_pack_key(s, id) : 0ull;
            if (matched) units += nk + (unsigned long long)matched * 4;   // query.len + matched * size_of::<DimWeight>()
        }
    }
    if (lane == 0 && units) atomicAdd(cpu + q, units);
}

// the rows' (row, dim) keys and the checks of every element: bit 0 a dim >= n_dims, bit 1 a non-finite weight
__global__ void sparse_row_keys_kernel(const uint64_t* indptr, uint32_t n_points, const uint32_t* dims, const float* w, uint32_t n_dims,
                                       unsigned long long* keys, unsigned int* flags) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_points) return;
    unsigned int f = 0;
    for (uint64_t e = indptr[r]; e < indptr[r + 1]; ++e) {
        const uint32_t d = dims[e];
        f |= (d >= n_dims ? 1u : 0u) | (isfinite(w[e]) ? 0u : 2u);
        keys[e] = ((unsigned long long)r << 32) | d;
    }
    if (f) atomicOr(flags, f);
}

// bit 2: a dim repeated within a row; and the posting keys (dim, id) of the sorted rows
__global__ void sparse_posting_keys_kernel(const unsigned long long* row_keys, uint64_t n, uint32_t* rdims, unsigned long long* post_keys, unsigned int* flags) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long k = row_keys[i];
    if (i > 0 && row_keys[i - 1] == k) atomicOr(flags, 4u);
    rdims[i] = (uint32_t)k;
    post_keys[i] = (k << 32) | (k >> 32);
}

// ids of the posting elements, and dptr[d] = the first element of dim d (dptr[n_dims] = n)
__global__ void sparse_split_kernel(const unsigned long long* post_keys, uint64_t n, uint32_t n_dims, uint32_t* ids, uint64_t* dptr) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long k = post_keys[i];
    ids[i] = (uint32_t)k;
    const uint32_t d = (uint32_t)(k >> 32);
    const uint32_t prev = i == 0 ? 0u : (uint32_t)(post_keys[i - 1] >> 32) + 1u;
    if (i == 0 || prev <= d)
        for (uint32_t x = i == 0 ? 0u : prev; x <= d; ++x) dptr[x] = i;
    if (i == n - 1)
        for (uint32_t x = d + 1; x <= n_dims; ++x) dptr[x] = n;
}

// max_next_weight: a segmented reverse max-scan, one warp per posting list from its end (-inf for the last element)
__global__ void sparse_max_next_kernel(const uint64_t* dptr, uint32_t n_dims, const float* w, float* mnw) {
    const uint32_t d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (d >= n_dims) return;
    const uint64_t b = dptr[d], e = dptr[d + 1];
    float carry = -INFINITY;
    for (uint64_t c = e; c > b;) {
        const uint64_t lo = c >= b + 32 ? c - 32 : b;
        const uint64_t i = c - 1 - lane;          // lane 0 takes the chunk's last element
        const bool in = i >= lo && i < c;
        float v = in ? w[i] : -INFINITY;
        // inclusive max over this lane and the lanes before it (the later elements)
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const float t = __shfl_up_sync(0xFFFFFFFFu, v, o); if (lane >= (uint32_t)o) v = fmaxf(v, t); }
        const float before = __shfl_up_sync(0xFFFFFFFFu, v, 1);
        if (in) mnw[i] = fmaxf(carry, lane == 0 ? -INFINITY : before);
        carry = fmaxf(carry, __shfl_sync(0xFFFFFFFFu, v, 31));
        c = lo;
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------ the handle
struct qb_sparse_index {
    int device = 0;
    qb_sparse_kind kind = QB_SPARSE_RAM;
    uint32_t n_points = 0, n_dims = 0;
    uint64_t nnz = 0, hbm_bytes = 0;
    cudaStream_t stream = nullptr;
    uint32_t* d_ids = nullptr; float* d_w = nullptr; float* d_mnw = nullptr; uint64_t* d_dptr = nullptr;   // posting lists
    uint64_t* d_rptr = nullptr; uint32_t* d_rdims = nullptr; float* d_rw = nullptr;                       // rows, sorted by dim
    std::vector<uint64_t> h_dptr;
    unsigned int* d_work = nullptr;
    std::mutex mu;
    void* d_scratch = nullptr; size_t scratch_bytes = 0;
    void* h_stage = nullptr; size_t stage_bytes = 0;
    int sm_count = 132;
};

static void sparse_free(qb_sparse_index* x) {
    if (!x) return;
    cudaSetDevice(x->device);
    if (x->stream) cudaStreamSynchronize(x->stream);
    cudaFree(x->d_ids); cudaFree(x->d_w); cudaFree(x->d_mnw); cudaFree(x->d_dptr);
    cudaFree(x->d_rptr); cudaFree(x->d_rdims); cudaFree(x->d_rw); cudaFree(x->d_work); cudaFree(x->d_scratch);
    if (x->h_stage) cudaFreeHost(x->h_stage);
    if (x->stream) cudaStreamDestroy(x->stream);
    delete x;
}

template <typename T>
static qb_status sp_alloc(qb_sparse_index* x, T** p, size_t elems) {
    const size_t b = std::max<size_t>(elems * sizeof(T), 16);
    QB_CUDA(cudaMalloc(reinterpret_cast<void**>(p), b));
    x->hbm_bytes += b;
    return QB_OK;
}

// The CSR rows (offsets already in d_rptr) sorted by (row, dim) into d_rdims / d_rw, with the checks of every element: bit 0 of
// *h_flags a dim >= dim_bound (any_dim: no bound, every u32 is a dim), bit 1 a non-finite weight, bit 2 a dim repeated within a row.
// d_post_keys (n entries) receives the (dim, id) keys of the sorted elements.  The index and the sparse vector storage (qb_sparse_custom.cu)
// both build their rows here.  Synchronous.
qb_status qb_sparse_sort_rows(cudaStream_t st, uint32_t n_points, uint64_t n, const uint64_t* d_rptr, const uint32_t* dims, const float* weights,
                              uint32_t dim_bound, bool any_dim, uint32_t* d_rdims, float* d_rw, unsigned long long* d_post_keys, unsigned int* h_flags) {
    unsigned long long *k0 = nullptr, *k1 = nullptr;
    uint32_t* in_dims = nullptr; float* in_w = nullptr; unsigned int* flags = nullptr; void* tmp = nullptr;
    size_t tmp_bytes = 0;
    const int row_bits = 32 + std::max(1, 32 - __builtin_clz(std::max(n_points, 1u)));
    // any_dim: the bound 0xFFFFFFFF flags only dim 0xFFFFFFFF, a valid dim; bit 0 is dropped
    const unsigned int keep = any_dim ? ~1u : ~0u;
    if (any_dim) dim_bound = 0xFFFFFFFFu;
    if (n) QB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, k0, k1, in_w, d_rw, (int64_t)n, 0, row_bits, st));
    *h_flags = 0;
    auto run = [&]() -> qb_status {
        QB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&flags), 16, st));
        QB_CUDA(cudaMemsetAsync(flags, 0, 4, st));
        if (n) {
            QB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&k0), n * 8, st));
            QB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&k1), n * 8, st));
            QB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&in_dims), n * 4, st));
            QB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&in_w), n * 4, st));
            QB_CUDA(cudaMallocAsync(&tmp, std::max<size_t>(tmp_bytes, 16), st));
            QB_CUDA(cudaMemcpyAsync(in_dims, dims, n * 4, cudaMemcpyHostToDevice, st));
            QB_CUDA(cudaMemcpyAsync(in_w, weights, n * 4, cudaMemcpyHostToDevice, st));
            if (n_points) {
                sparse_row_keys_kernel<<<(n_points + 255) / 256, 256, 0, st>>>(d_rptr, n_points, in_dims, in_w, dim_bound, k0, flags);
                QB_LAUNCHED();
            }
            // the index lays its lists out by dim: stop here when a dim is out of range
            QB_CUDA(cudaMemcpyAsync(h_flags, flags, 4, cudaMemcpyDeviceToHost, st));
            QB_CUDA(cudaStreamSynchronize(st));
            if (*h_flags & keep) return QB_OK;
            size_t b = tmp_bytes;
            QB_CUDA(cub::DeviceRadixSort::SortPairs(tmp, b, k0, k1, in_w, d_rw, (int64_t)n, 0, row_bits, st));
            sparse_posting_keys_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(k1, n, d_rdims, d_post_keys, flags);
            QB_LAUNCHED();
            QB_CUDA(cudaGetLastError());
        }
        QB_CUDA(cudaMemcpyAsync(h_flags, flags, 4, cudaMemcpyDeviceToHost, st));
        return QB_OK;
    };
    const qb_status rc = run();
    cudaFreeAsync(k0, st); cudaFreeAsync(k1, st); cudaFreeAsync(in_dims, st); cudaFreeAsync(in_w, st); cudaFreeAsync(tmp, st); cudaFreeAsync(flags, st);
    const cudaError_t e = cudaStreamSynchronize(st);
    QB_TRY(rc);
    QB_CHECK(e == cudaSuccess, QB_ERR_CUDA, "sparse rows: %s", cudaGetErrorString(e));
    *h_flags &= keep;
    return QB_OK;
}

static qb_status sparse_build(qb_sparse_index* x, const uint64_t* indptr, const uint32_t* dims, const float* weights) {
    const uint64_t n = x->nnz;
    cudaStream_t st = x->stream;
    QB_TRY(sp_alloc(x, &x->d_rptr, (size_t)x->n_points + 1));
    QB_TRY(sp_alloc(x, &x->d_rdims, n));
    QB_TRY(sp_alloc(x, &x->d_rw, n));
    QB_TRY(sp_alloc(x, &x->d_ids, n));
    QB_TRY(sp_alloc(x, &x->d_w, n));
    QB_TRY(sp_alloc(x, &x->d_mnw, n));
    QB_TRY(sp_alloc(x, &x->d_dptr, (size_t)x->n_dims + 1));
    QB_CUDA(cudaMemcpyAsync(x->d_rptr, indptr, ((size_t)x->n_points + 1) * 8, cudaMemcpyHostToDevice, st));
    QB_CUDA(cudaMemsetAsync(x->d_dptr, 0, ((size_t)x->n_dims + 1) * 8, st));
    // the rows, then the posting lists: the (dim, id) keys sorted with the weights, split into ids and dim offsets
    unsigned long long *k0 = nullptr, *k1 = nullptr;
    void* tmp = nullptr;
    size_t tmp_bytes = 0;
    const int dim_bits = 32 + std::max(1, 32 - __builtin_clz(std::max(x->n_dims, 1u)));
    if (n) QB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, k0, k1, x->d_rw, x->d_w, (int64_t)n, 0, dim_bits, st));
    unsigned int h_flags = 0;
    auto run = [&]() -> qb_status {
        if (n) QB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&k0), n * 8, st));
        QB_TRY(qb_sparse_sort_rows(st, x->n_points, n, x->d_rptr, dims, weights, x->n_dims, false, x->d_rdims, x->d_rw, k0, &h_flags));
        if (!n || h_flags) return QB_OK;
        QB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&k1), n * 8, st));
        QB_CUDA(cudaMallocAsync(&tmp, std::max<size_t>(tmp_bytes, 16), st));
        size_t b = tmp_bytes;
        QB_CUDA(cub::DeviceRadixSort::SortPairs(tmp, b, k0, k1, x->d_rw, x->d_w, (int64_t)n, 0, dim_bits, st));
        sparse_split_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(k1, n, x->n_dims, x->d_ids, x->d_dptr);
        QB_LAUNCHED();
        if (x->n_dims) {
            sparse_max_next_kernel<<<(unsigned)(((uint64_t)x->n_dims * 32 + 255) / 256), 256, 0, st>>>(x->d_dptr, x->n_dims, x->d_w, x->d_mnw);
            QB_LAUNCHED();
        }
        QB_CUDA(cudaGetLastError());
        return QB_OK;
    };
    const qb_status rc = run();
    cudaFreeAsync(k0, st); cudaFreeAsync(k1, st); cudaFreeAsync(tmp, st);
    const cudaError_t e = cudaStreamSynchronize(st);
    QB_TRY(rc);
    QB_CHECK(e == cudaSuccess, QB_ERR_CUDA, "sparse_index_create: %s", cudaGetErrorString(e));
    QB_CHECK(!(h_flags & 1u), QB_ERR_INVALID, "sparse_index_create: a dim >= n_dims %u", x->n_dims);
    QB_CHECK(!(h_flags & 2u), QB_ERR_INVALID, "sparse_index_create: a weight is not finite");
    QB_CHECK(!(h_flags & 4u), QB_ERR_INVALID, "sparse_index_create: a dim is repeated within a row");
    x->h_dptr.resize((size_t)x->n_dims + 1);
    QB_CUDA(cudaMemcpy(x->h_dptr.data(), x->d_dptr, x->h_dptr.size() * 8, cudaMemcpyDeviceToHost));
    return QB_OK;
}

extern "C" qb_status qb_sparse_index_create(int32_t device, qb_sparse_kind kind, uint32_t n_points, uint32_t n_dims, const uint64_t* indptr,
                                            const uint32_t* dims, const float* weights, qb_sparse_index** out) {
    QB_CHECK(out && indptr, QB_ERR_INVALID, "sparse_index_create: null argument");
    *out = nullptr;
    QB_CHECK(kind == QB_SPARSE_RAM || kind == QB_SPARSE_COMPRESSED || kind == QB_SPARSE_COMPRESSED_F16 || kind == QB_SPARSE_COMPRESSED_U8,
             QB_ERR_INVALID, "sparse_index_create: unknown kind %d", (int)kind);
    QB_CHECK(kind != QB_SPARSE_COMPRESSED_F16 && kind != QB_SPARSE_COMPRESSED_U8, QB_ERR_UNSUPPORTED,
             "sparse_index_create: compressed posting lists with f16 / u8 weights are not supported");
    QB_CHECK(indptr[0] == 0, QB_ERR_INVALID, "sparse_index_create: indptr[0] must be 0");
    for (uint32_t r = 0; r < n_points; ++r)
        QB_CHECK(indptr[r + 1] >= indptr[r], QB_ERR_INVALID, "sparse_index_create: indptr descends at row %u", r);
    const uint64_t nnz = indptr[n_points];
    QB_CHECK(nnz == 0 || (dims && weights), QB_ERR_INVALID, "sparse_index_create: null argument");
    QB_CHECK(nnz < 0xFFFFFFFFull, QB_ERR_UNSUPPORTED, "sparse_index_create: %llu elements (the lists use 32-bit positions)", (unsigned long long)nnz);
    QB_CHECK(n_points < 0xFFFFFFFFu - SP_BATCH, QB_ERR_UNSUPPORTED, "sparse_index_create: %u points", n_points);
    QB_TRY(qb_use_device(device));
    qb_sparse_index* x = new qb_sparse_index();
    x->device = device; x->kind = kind; x->n_points = n_points; x->n_dims = n_dims; x->nnz = nnz;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) x->sm_count = prop.multiProcessorCount;
    qb_status rc = cudaStreamCreateWithFlags(&x->stream, cudaStreamNonBlocking) == cudaSuccess ? QB_OK : QB_ERR_CUDA;
    if (rc != QB_OK) qb_set_error("sparse_index_create: cudaStreamCreate failed");
    if (rc == QB_OK) rc = sp_alloc(x, &x->d_work, 4);
    if (rc == QB_OK) rc = sparse_build(x, indptr, dims, weights);
    if (rc != QB_OK) { sparse_free(x); return rc; }
    *out = x;
    return QB_OK;
}

extern "C" void qb_sparse_index_destroy(qb_sparse_index* idx) { sparse_free(idx); }

extern "C" qb_status qb_sparse_index_info(const qb_sparse_index* idx, uint32_t* n_points, uint32_t* n_dims, uint64_t* n_elements, uint64_t* hbm_bytes) {
    QB_CHECK(idx, QB_ERR_INVALID, "sparse_index_info: null index");
    if (n_points) *n_points = idx->n_points;
    if (n_dims) *n_dims = idx->n_dims;
    if (n_elements) *n_elements = idx->nnz;
    if (hbm_bytes) *hbm_bytes = idx->hbm_bytes;
    return QB_OK;
}

extern "C" void* qb_sparse_index_stream(qb_sparse_index* idx) { return idx ? idx->stream : nullptr; }

// ------------------------------------------------------------------------------------------------ searches
constexpr uint32_t QB_SPARSE_MAX_TOP = 4096;
constexpr uint32_t QB_SPARSE_MAX_QUERY_DIMS = 4096;

static uint32_t sp_p2(uint32_t top) { uint32_t p2 = 32; while (p2 < 2 * top) p2 <<= 1; return p2; }

static qb_status sparse_launch(qb_sparse_index* x, const uint64_t* d_qptr, const uint32_t* d_qdims, const float* d_qw, uint32_t nq, uint32_t max_nnz,
                               uint32_t top, const uint32_t* d_deleted, qb_scored_point* d_out, uint32_t* d_counts) {
    SparseSearchParams p{x->d_ids, x->d_w, x->d_mnw, x->d_dptr, x->n_dims, d_qptr, d_qdims, d_qw, nq, std::max(max_nnz, 1u), d_deleted, top, sp_p2(top),
                         x->kind == QB_SPARSE_RAM, d_out, d_counts, x->d_work};
    const size_t smem = SP_SCORES_BYTES + (size_t)p.max_nnz * sizeof(SpList) + (size_t)p.p2 * 8;
    QB_CUDA(cudaFuncSetAttribute(sparse_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 1;
    QB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sparse_search_kernel, SP_THREADS, smem));
    const unsigned grid = (unsigned)std::min<uint64_t>(nq, (uint64_t)x->sm_count * std::max(per_sm, 1));
    QB_CUDA(cudaMemsetAsync(x->d_work, 0, 4, x->stream));
    sparse_search_kernel<<<grid, SP_THREADS, smem, x->stream>>>(p);
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return QB_OK;
}

// a query as the reference takes it: duplicate dims rejected (the user's SparseVector is validated before remapping), the dims >= n_dims
// dropped (the tracker does not know them), the rest sorted by dim
static qb_status sparse_prepare_queries(const qb_sparse_index* x, const uint64_t* q_indptr, const uint32_t* q_dims, const float* q_weights, uint32_t nq,
                                        std::vector<uint64_t>& ptr, std::vector<uint32_t>& kd, std::vector<float>& kw, uint32_t* max_nnz, const char* who) {
    ptr.assign(1, 0);
    *max_nnz = 0;
    std::vector<std::pair<uint32_t, float>> v;
    for (uint32_t q = 0; q < nq; ++q) {
        QB_CHECK(q_indptr[q + 1] >= q_indptr[q], QB_ERR_INVALID, "%s: q_indptr descends at query %u", who, q);
        v.clear();
        for (uint64_t e = q_indptr[q]; e < q_indptr[q + 1]; ++e) v.emplace_back(q_dims[e], q_weights[e]);
        std::sort(v.begin(), v.end(), [](const std::pair<uint32_t, float>& a, const std::pair<uint32_t, float>& b) { return a.first < b.first; });
        for (size_t i = 1; i < v.size(); ++i) QB_CHECK(v[i].first != v[i - 1].first, QB_ERR_INVALID, "%s: dim %u repeated in query %u", who, v[i].first, q);
        uint32_t n = 0;
        for (const auto& e : v) if (e.first < x->n_dims) { kd.push_back(e.first); kw.push_back(e.second); ++n; }
        QB_CHECK(n <= QB_SPARSE_MAX_QUERY_DIMS, QB_ERR_UNSUPPORTED, "%s: query %u has %u known dims > %u", who, q, n, QB_SPARSE_MAX_QUERY_DIMS);
        *max_nnz = std::max(*max_nnz, n);
        ptr.push_back(kd.size());
    }
    return QB_OK;
}

static qb_status sparse_common_check(const qb_sparse_index* x, const uint64_t* q_indptr, const uint32_t* q_dims, const float* q_weights, uint32_t nq,
                                     uint32_t top, const void* out, const uint32_t* out_counts, const char* who) {
    QB_CHECK(x && out_counts && (out || nq == 0), QB_ERR_INVALID, "%s: null argument", who);
    QB_CHECK(nq == 0 || q_indptr, QB_ERR_INVALID, "%s: null argument", who);
    QB_CHECK(nq == 0 || q_indptr[nq] == q_indptr[0] || (q_dims && q_weights), QB_ERR_INVALID, "%s: null argument", who);
    QB_CHECK(top >= 1, QB_ERR_INVALID, "%s: top must be >= 1", who);
    QB_CHECK(top <= QB_SPARSE_MAX_TOP, QB_ERR_UNSUPPORTED, "%s: top %u > %u", who, top, QB_SPARSE_MAX_TOP);
    return QB_OK;
}

static qb_status sp_ensure_pinned(qb_sparse_index* x, size_t need) { return qb_ensure_pinned(&x->h_stage, &x->stage_bytes, need); }

extern "C" qb_status qb_sparse_search_batch(qb_sparse_index* idx, const uint64_t* q_indptr, const uint32_t* q_dims, const float* q_weights, uint32_t n_queries,
                                            uint32_t top, const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped, qb_scored_point* out,
                                            uint32_t* out_counts, qb_hw_counters* counters) {
    const char* who = "sparse_search_batch";
    QB_TRY(sparse_common_check(idx, q_indptr, q_dims, q_weights, n_queries, top, out, out_counts, who));
    std::vector<uint64_t> ptr; std::vector<uint32_t> kd; std::vector<float> kw;
    uint32_t max_nnz = 0;
    QB_TRY(sparse_prepare_queries(idx, q_indptr, q_dims, q_weights, n_queries, ptr, kd, kw, &max_nnz, who));
    if (n_queries == 0) return QB_OK;
    QB_CHECK(!(is_stopped && *is_stopped), QB_ERR_CANCELLED, "%s: cancelled", who);
    QB_TRY(qb_use_device(idx->device));
    std::lock_guard<std::mutex> lk(idx->mu);
    const size_t nk = kd.size(), words = ((size_t)idx->n_points + 63) / 64;
    // scratch = [q ptr | dims | weights | deleted words | out | counts]
    const size_t dims_at = round_up_u64(ptr.size() * 8, 16), w_at = round_up_u64(dims_at + nk * 4, 16), del_at = round_up_u64(w_at + nk * 4, 16);
    const size_t out_at = round_up_u64(del_at + (deleted_bitmap ? words * 8 : 0), 16), cnt_at = out_at + (size_t)n_queries * top * 8;
    const size_t bytes = cnt_at + (size_t)n_queries * 4;
    QB_TRY(qb_ensure_device(&idx->d_scratch, &idx->scratch_bytes, bytes));
    QB_TRY(sp_ensure_pinned(idx, bytes));
    uint8_t* h = reinterpret_cast<uint8_t*>(idx->h_stage);
    uint8_t* d = reinterpret_cast<uint8_t*>(idx->d_scratch);
    memcpy(h, ptr.data(), ptr.size() * 8);
    if (nk) { memcpy(h + dims_at, kd.data(), nk * 4); memcpy(h + w_at, kw.data(), nk * 4); }
    if (deleted_bitmap) memcpy(h + del_at, deleted_bitmap, words * 8);
    QB_CUDA(cudaMemcpyAsync(d, h, out_at, cudaMemcpyHostToDevice, idx->stream));
    QB_TRY(sparse_launch(idx, reinterpret_cast<const uint64_t*>(d), reinterpret_cast<const uint32_t*>(d + dims_at), reinterpret_cast<const float*>(d + w_at),
                         n_queries, max_nnz, top, deleted_bitmap ? reinterpret_cast<const uint32_t*>(d + del_at) : nullptr,
                         reinterpret_cast<qb_scored_point*>(d + out_at), reinterpret_cast<uint32_t*>(d + cnt_at)));
    QB_CUDA(cudaMemcpyAsync(h + out_at, d + out_at, bytes - out_at, cudaMemcpyDeviceToHost, idx->stream));
    QB_CUDA(cudaStreamSynchronize(idx->stream));
    memcpy(out, h + out_at, (size_t)n_queries * top * 8);
    memcpy(out_counts, h + cnt_at, (size_t)n_queries * 4);
    if (counters) {
        // SearchContext::search: cpu += len_to_end * size_of::<DimWeight>() over the lists at the start (:272-283)
        for (size_t i = 0; i < nk; ++i) counters->cpu += (idx->h_dptr[kd[i] + 1] - idx->h_dptr[kd[i]]) * 4;
    }
    return QB_OK;
}

extern "C" qb_status qb_sparse_search_batch_device(qb_sparse_index* idx, const uint64_t* dev_q_indptr, const uint32_t* dev_q_dims, const float* dev_q_weights,
                                                   uint32_t n_queries, uint32_t max_query_nnz, uint32_t top, const uint64_t* dev_deleted_bitmap,
                                                   qb_scored_point* dev_out, uint32_t* dev_out_counts) {
    const char* who = "sparse_search_batch_device";
    QB_CHECK(idx, QB_ERR_INVALID, "%s: null argument", who);
    QB_CHECK(n_queries == 0 || (dev_q_indptr && dev_q_dims && dev_q_weights && dev_out && dev_out_counts), QB_ERR_INVALID, "%s: null argument", who);
    QB_CHECK(top >= 1, QB_ERR_INVALID, "%s: top must be >= 1", who);
    QB_CHECK(top <= QB_SPARSE_MAX_TOP, QB_ERR_UNSUPPORTED, "%s: top %u > %u", who, top, QB_SPARSE_MAX_TOP);
    QB_CHECK(max_query_nnz <= QB_SPARSE_MAX_QUERY_DIMS, QB_ERR_UNSUPPORTED, "%s: max_query_nnz %u > %u", who, max_query_nnz, QB_SPARSE_MAX_QUERY_DIMS);
    if (n_queries == 0) return QB_OK;
    QB_TRY(qb_use_device(idx->device));
    std::lock_guard<std::mutex> lk(idx->mu);
    return sparse_launch(idx, dev_q_indptr, dev_q_dims, dev_q_weights, n_queries, max_query_nnz, top, reinterpret_cast<const uint32_t*>(dev_deleted_bitmap),
                         dev_out, dev_out_counts);
}

extern "C" qb_status qb_sparse_search_plain_batch(qb_sparse_index* idx, const uint64_t* q_indptr, const uint32_t* q_dims, const float* q_weights, uint32_t n_queries,
                                                  const uint64_t* id_indptr, const uint32_t* ids, uint32_t top, const volatile int32_t* is_stopped,
                                                  qb_scored_point* out, uint32_t* out_counts, qb_hw_counters* counters) {
    const char* who = "sparse_search_plain_batch";
    QB_TRY(sparse_common_check(idx, q_indptr, q_dims, q_weights, n_queries, top, out, out_counts, who));
    QB_CHECK(n_queries == 0 || id_indptr, QB_ERR_INVALID, "%s: null argument", who);
    std::vector<uint64_t> ptr; std::vector<uint32_t> kd; std::vector<float> kw;
    uint32_t max_nnz = 0;
    QB_TRY(sparse_prepare_queries(idx, q_indptr, q_dims, q_weights, n_queries, ptr, kd, kw, &max_nnz, who));
    // each query's ids: in range and distinct; sorted as plain_search sorts them
    std::vector<uint64_t> iptr(1, 0);
    std::vector<uint32_t> sid;
    uint64_t max_ids = 0;
    for (uint32_t q = 0; q < n_queries; ++q) {
        QB_CHECK(id_indptr[q + 1] >= id_indptr[q], QB_ERR_INVALID, "%s: id_indptr descends at query %u", who, q);
        QB_CHECK(id_indptr[q + 1] == id_indptr[q] || ids, QB_ERR_INVALID, "%s: null argument", who);
        const size_t b = sid.size();
        for (uint64_t e = id_indptr[q]; e < id_indptr[q + 1]; ++e) {
            QB_CHECK(ids[e] < idx->n_points, QB_ERR_INVALID, "%s: id %u of query %u >= n_points %u", who, ids[e], q, idx->n_points);
            sid.push_back(ids[e]);
        }
        std::sort(sid.begin() + b, sid.end());
        for (size_t i = b + 1; i < sid.size(); ++i) QB_CHECK(sid[i] != sid[i - 1], QB_ERR_INVALID, "%s: id %u repeated in query %u", who, sid[i], q);
        max_ids = std::max<uint64_t>(max_ids, sid.size() - b);
        iptr.push_back(sid.size());
    }
    if (n_queries == 0) return QB_OK;
    QB_CHECK(!(is_stopped && *is_stopped), QB_ERR_CANCELLED, "%s: cancelled", who);
    QB_TRY(qb_use_device(idx->device));
    std::lock_guard<std::mutex> lk(idx->mu);
    const size_t nk = kd.size(), ni = sid.size(), cap = std::max<uint64_t>(max_ids, 1);
    // scratch = [q ptr | id ptr | dims | weights | ids | cnt | cpu | out | counts | candidates]
    const size_t iptr_at = ptr.size() * 8, dims_at = round_up_u64(iptr_at + iptr.size() * 8, 16), w_at = round_up_u64(dims_at + nk * 4, 16);
    const size_t ids_at = round_up_u64(w_at + nk * 4, 16), cnt_at = round_up_u64(ids_at + ni * 4, 16), cpu_at = round_up_u64(cnt_at + (size_t)n_queries * 4, 16);
    const size_t out_at = cpu_at + (size_t)n_queries * 8, ocnt_at = out_at + (size_t)n_queries * top * 8, cand_at = round_up_u64(ocnt_at + (size_t)n_queries * 4, 16);
    const size_t bytes = cand_at + (size_t)n_queries * cap * 8;
    QB_TRY(qb_ensure_device(&idx->d_scratch, &idx->scratch_bytes, bytes));
    QB_TRY(sp_ensure_pinned(idx, cand_at));
    uint8_t* h = reinterpret_cast<uint8_t*>(idx->h_stage);
    uint8_t* d = reinterpret_cast<uint8_t*>(idx->d_scratch);
    memcpy(h, ptr.data(), ptr.size() * 8);
    memcpy(h + iptr_at, iptr.data(), iptr.size() * 8);
    if (nk) { memcpy(h + dims_at, kd.data(), nk * 4); memcpy(h + w_at, kw.data(), nk * 4); }
    if (ni) memcpy(h + ids_at, sid.data(), ni * 4);
    for (uint32_t q = 0; q < n_queries; ++q) reinterpret_cast<uint32_t*>(h + cnt_at)[q] = (uint32_t)(iptr[q + 1] - iptr[q]);
    memset(h + cpu_at, 0, (size_t)n_queries * 8);
    QB_CUDA(cudaMemcpyAsync(d, h, out_at, cudaMemcpyHostToDevice, idx->stream));
    const size_t smem = (size_t)std::max(max_nnz, 1u) * 8;
    const unsigned gx = (unsigned)((cap + SP_PLAIN_IDS_PER_BLOCK - 1) / SP_PLAIN_IDS_PER_BLOCK);
    QB_CHECK(gx <= 0x7FFFFFFFu, QB_ERR_UNSUPPORTED, "%s: %llu ids in one query", who, (unsigned long long)cap);
    for (uint32_t q0 = 0; q0 < n_queries; q0 += 65535) {
        const uint32_t nqc = std::min<uint32_t>(65535, n_queries - q0);
        sparse_plain_kernel<<<dim3(gx, nqc), SP_THREADS, smem, idx->stream>>>(
            idx->d_rptr, idx->d_rdims, idx->d_rw, reinterpret_cast<const uint64_t*>(d), reinterpret_cast<const uint32_t*>(d + dims_at),
            reinterpret_cast<const float*>(d + w_at), reinterpret_cast<const uint64_t*>(d + iptr_at), reinterpret_cast<const uint32_t*>(d + ids_at), q0,
            reinterpret_cast<unsigned long long*>(d + cand_at) + (size_t)q0 * cap, cap, reinterpret_cast<unsigned long long*>(d + cpu_at));
        QB_LAUNCHED();
        QB_CUDA(cudaGetLastError());
    }
    QB_TRY(qb_launch_select(reinterpret_cast<const unsigned long long*>(d + cand_at), reinterpret_cast<const unsigned int*>(d + cnt_at), cap, 0, n_queries, top, 0,
                            reinterpret_cast<qb_scored_point*>(d + out_at), reinterpret_cast<uint32_t*>(d + ocnt_at), nullptr, nullptr, idx->stream));
    QB_CUDA(cudaMemcpyAsync(h + cpu_at, d + cpu_at, cand_at - cpu_at, cudaMemcpyDeviceToHost, idx->stream));
    QB_CUDA(cudaStreamSynchronize(idx->stream));
    memcpy(out, h + out_at, (size_t)n_queries * top * 8);
    memcpy(out_counts, h + ocnt_at, (size_t)n_queries * 4);
    if (counters)
        for (uint32_t q = 0; q < n_queries; ++q) counters->cpu += reinterpret_cast<const uint64_t*>(h + cpu_at)[q];
    return QB_OK;
}
