// qb_api.cu — the C ABI (include/qb200.h): storages in HBM, RawScorer handles, fused brute-force search.
//
// Host-side orchestration only; every arithmetic step runs in the CUDA kernels of qb_dense.cu / qb_quant.cu /
// qb_topk.cu.  There is no CPU scoring path anywhere in this library.
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>

#include <algorithm>
#include <cmath>

#include "qb_internal.h"

// kernels' host entry points (qb_dense.cu / qb_quant.cu / qb_dtype.cu)
qb_status qb_dense_f32_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream);
qb_status qb_dense_f32_score_points(const qb_storage* s, const void* d_q_enc, const uint32_t* d_ids, uint64_t n, float* d_scores, cudaStream_t stream);
qb_status qb_dense_f32_scan_localk(const qb_storage* s, const QbScanArgs& a, uint32_t top, uint64_t* n_slots, cudaStream_t stream, uint64_t min_rows = 65536);
qb_status qb_dense_f32_scan_fold(const qb_storage* s, const QbScanArgs& a, int kind, uint32_t n_a, uint32_t n_b, const float* d_coef, bool* done, cudaStream_t stream);
qb_status qb_dense_x_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream);
qb_status qb_dense_x_score_points(const qb_storage* s, const void* d_q_enc, const uint32_t* d_ids, uint64_t n, float* d_scores, cudaStream_t stream);
qb_status qb_dense_x_convert_queries(const qb_storage* s, const float* d_q_pre, uint32_t q_stride_f, uint32_t nq, void* d_out, cudaStream_t stream);
qb_status qb_sq8_repack(const qb_storage* s, const uint8_t* d_rows_in, uint32_t row_bytes, uint64_t first, uint64_t n, cudaStream_t stream);
qb_status qb_sq8_encode_queries(const qb_storage* s, const float* d_q_pre, uint32_t q_stride_f, uint32_t nq, uint8_t* d_codes, float* d_q_off, cudaStream_t stream);
qb_status qb_sq8_internal_query(const qb_storage* s, uint32_t id, uint8_t* d_code, float* d_q_off, cudaStream_t stream);
qb_status qb_sq8_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream);
qb_status qb_sq8_score_points(const qb_storage* s, const void* d_q_enc, const float* d_q_off, const uint32_t* d_ids, uint64_t n, float* d_scores, cudaStream_t stream);
qb_status qb_pq_build_luts(const qb_storage* s, const float* d_q_pre, uint32_t q_stride_f, uint32_t nq, float* d_luts, cudaStream_t stream);
qb_status qb_pq_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream);
qb_status qb_pq_score_points(const qb_storage* s, const void* d_q_enc, const uint32_t* d_ids, uint64_t n, float* d_scores, cudaStream_t stream);
qb_status qb_pq_score_internal(const qb_storage* s, uint32_t a, uint32_t b, float* d_out, cudaStream_t stream);
uint32_t qb_sq8_mma_block(const qb_storage* s, uint32_t nq);
size_t qb_sq8_mma_scratch_bytes(const qb_storage* s, uint32_t nq_pad);
qb_status qb_sq8_mma_scan(const qb_storage* s, const uint8_t* d_q_codes, uint32_t nq_pad, const float* d_q_off, uint32_t nq, uint32_t n_blk,
                          uint64_t row_begin, uint64_t row_end, const QbEmit& emit, unsigned int* d_flags, unsigned long long* seg_len,
                          void* d_scratch, size_t scratch_bytes, cudaStream_t stream);
uint32_t qb_f32_mma_block(qb_storage* s, uint32_t nq, cudaStream_t stream);
size_t qb_f32_mma_scratch_bytes(const qb_storage* s, uint32_t nq_pad);
qb_status qb_f32_mma_scan(qb_storage* s, const float* d_q_pre, uint32_t q_stride_f, uint32_t nq, uint32_t nq_pad, uint32_t n_blk, uint64_t row_end, const QbEmit& emit,
                          unsigned int* d_flags, void* d_scratch, size_t scratch_bytes, cudaStream_t stream);
qb_status qb_bq_encode_queries(const qb_storage* s, const float* d_q_pre, uint32_t q_stride_f, uint32_t nq, int force_binary, void* d_out, cudaStream_t stream);
qb_status qb_bq_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream);
qb_status qb_bq_score_points(const qb_storage* s, const void* d_q_enc, int bits, const uint32_t* d_ids, uint64_t n, float* d_scores, cudaStream_t stream);

uint32_t qb_custom_examples(int kind, uint32_t n_a, uint32_t n_b);
qb_status qb_launch_custom_combine(int kind, uint32_t n_a, uint32_t n_b, const float* d_coef, const float* d_sims, uint64_t stride, uint64_t n, float* d_scores,
                                   const uint32_t* d_ids, const QbEmit* emit, cudaStream_t stream);
qb_status qb_launch_iota(uint32_t* d, uint64_t n, cudaStream_t stream);
qb_status qb_launch_maxsim_fold(const float* d_sims, uint64_t stride, uint32_t n_query_tokens, const uint32_t* d_row_offsets, const uint32_t* d_point_ids,
                                uint64_t n_points, float* d_scores, const QbEmit* emit, cudaStream_t stream);

// ------------------------------------------------------------------------------------------------ errors
static thread_local char g_err[1024] = "";
std::atomic<uint64_t> g_qb_launches{0};

// Process-wide switches (debugging / experiments).  The environment is read ONCE, at first use; qb_set_option changes a
// switch at run time.  Nothing on a search path calls getenv.
QbOptions& qb_opt() {
    static QbOptions o = [] {
        QbOptions v;
        auto num = [](const char* name, long long dflt) { const char* e = getenv(name); return e ? strtoll(e, nullptr, 10) : dflt; };
        v.disable_localk = getenv("QB_DISABLE_LOCALK") != nullptr;
        v.disable_prefilter = getenv("QB_DISABLE_PREFILTER") != nullptr;
        v.prefilter_plane = (int)num("QB_PREFILTER_PLANE", 0);
        v.prefilter_stage1 = (int)num("QB_PREFILTER_STAGE1", 0);
        v.prefilter_slot_bytes = (uint32_t)num("QB_PREFILTER_SLOT_BYTES", 0);
        v.disable_mma = getenv("QB_DISABLE_MMA") != nullptr;
        v.mma_no_segments = getenv("QB_MMA_NO_SEGMENTS") != nullptr;
        v.mma_debug = (int)num("QB_MMA_DEBUG", 0);
        v.sample_rows = (uint64_t)num("QB_SAMPLE_ROWS", 0);
        v.verbose = getenv("QB_VERBOSE") != nullptr;
        v.pq_queries_per_pass = (int)num("QB_PQ_QUERIES", 0);
        v.mma_seg_cap = (uint32_t)num("QB_MMA_SEG_CAP", 0);
        v.hnsw_threads = (int)num("QB_HNSW_THREADS", 0);
        return v;
    }();
    return o;
}

extern "C" qb_status qb_set_option(const char* name, int64_t value) {
    QB_CHECK(name, QB_ERR_INVALID, "set_option: null name");
    QbOptions& o = qb_opt();
    const std::string n(name);
    if (n == "disable_localk") o.disable_localk = value != 0;
    else if (n == "disable_prefilter") o.disable_prefilter = value != 0;
    else if (n == "prefilter_plane") o.prefilter_plane = (int)value;
    else if (n == "prefilter_stage1") o.prefilter_stage1 = (int)value;
    else if (n == "prefilter_slot_bytes") o.prefilter_slot_bytes = (uint32_t)value;
    else if (n == "prefilter_producers") o.prefilter_producers = (int)value;
    else if (n == "disable_mma") o.disable_mma = value != 0;
    else if (n == "mma_no_segments") o.mma_no_segments = value != 0;
    else if (n == "mma_debug") o.mma_debug = (int)value;
    else if (n == "sample_rows") o.sample_rows = (uint64_t)value;
    else if (n == "verbose") o.verbose = value != 0;
    else if (n == "pq_queries_per_pass") o.pq_queries_per_pass = (int)value;
    else if (n == "hnsw_threads") o.hnsw_threads = (int)value;
    else if (n == "mma_seg_cap") o.mma_seg_cap = (uint32_t)value;
    else if (n == "hnsw_no_prefetch") o.hnsw_no_prefetch = value != 0;
    else { qb_set_error("set_option: unknown option '%s'", name); return QB_ERR_INVALID; }
    return QB_OK;
}

void qb_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char* qb_last_error(void) { return g_err; }
extern "C" int32_t qb_abi_version(void) { return QB200_ABI_VERSION; }
extern "C" uint64_t qb_kernel_launch_count(void) { return g_qb_launches.load(); }

extern "C" qb_status qb_device_count(int32_t* out) {
    QB_CHECK(out, QB_ERR_INVALID, "qb_device_count: null out");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        *out = 0;
        qb_set_error("no CUDA device: %s (this library has no CPU fallback)", cudaGetErrorString(e));
        cudaGetLastError();
        return QB_ERR_NO_DEVICE;
    }
    *out = n;
    return QB_OK;
}

static qb_status use_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        qb_set_error("no CUDA device: %s (this library has no CPU fallback)", cudaGetErrorString(e));
        cudaGetLastError();
        return QB_ERR_NO_DEVICE;
    }
    QB_CHECK(device >= 0 && device < n, QB_ERR_INVALID, "device %d out of range (have %d)", device, n);
    QB_CUDA(cudaSetDevice(device));
    return QB_OK;
}

// Point ids crossing the C ABI are the ids searches on this storage report: local row + id_base (qb_storage_set_id_base).
// Every id-taking entry point validates the range and works on local rows.
static qb_status localize_ids(const qb_storage* s, const uint32_t* ids, uint64_t n, uint32_t* dst, const char* who) {
    const uint32_t base = s->id_base;
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t l = ids[i] - base;
        QB_CHECK(ids[i] >= base && l < s->count, QB_ERR_INVALID, "%s: id %u out of range [%u, %llu)", who, ids[i], base, (unsigned long long)base + s->count);
        dst[i] = l;
    }
    return QB_OK;
}

// ------------------------------------------------------------------------------------------------ buffers
qb_status qb_ensure_device(void** p, size_t* have, size_t need_bytes) {
    if (*have >= need_bytes && *p) return QB_OK;
    if (*p) { QB_CUDA(cudaFree(*p)); *p = nullptr; *have = 0; }
    size_t sz = std::max<size_t>(need_bytes, 256);
    QB_CUDA(cudaMalloc(p, sz));
    *have = sz;
    return QB_OK;
}
qb_status qb_ensure_pinned(void** p, size_t* have, size_t need_bytes) {
    if (*have >= need_bytes && *p) return QB_OK;
    if (*p) { QB_CUDA(cudaFreeHost(*p)); *p = nullptr; *have = 0; }
    size_t sz = std::max<size_t>(need_bytes, 4096);
    QB_CUDA(cudaMallocHost(p, sz));
    *have = sz;
    return QB_OK;
}
template <typename T>
static qb_status ensure_dev_elems(T** p, size_t* have_elems, size_t need_elems) {
    size_t have_b = *have_elems * sizeof(T);
    void* vp = *p;
    QB_TRY(qb_ensure_device(&vp, &have_b, need_elems * sizeof(T)));
    *p = reinterpret_cast<T*>(vp);
    *have_elems = have_b / sizeof(T);
    return QB_OK;
}

static qb_status ctx_new(QbSearchCtx** out) {
    QbSearchCtx* c = new QbSearchCtx();
    cudaError_t e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { delete c; qb_set_error("cudaStreamCreate: %s", cudaGetErrorString(e)); return QB_ERR_CUDA; }
    cudaEventCreate(&c->ev0);
    cudaEventCreate(&c->ev1);
    c->in_use = true;
    *out = c;
    return QB_OK;
}
qb_status qb_ctx_acquire(qb_storage* s, QbSearchCtx** out) {
    std::lock_guard<std::mutex> lk(s->mu);
    for (QbSearchCtx* c : s->ctxs)
        if (!c->in_use) { c->in_use = true; *out = c; return QB_OK; }
    QbSearchCtx* c = nullptr;
    QB_TRY(ctx_new(&c));
    s->ctxs.push_back(c);
    *out = c;
    return QB_OK;
}
// the context of the device-resident entry points (qb_search_batch_device, qb_hnsw_search_batch_device) and of qb_storage_stream:
// its stream is the one the caller times and orders against, so it is never shared with the pooled host-facing searches
qb_status qb_ctx_device(qb_storage* s, QbSearchCtx** out) {
    std::lock_guard<std::mutex> lk(s->mu);
    if (!s->dev_ctx) QB_TRY(ctx_new(&s->dev_ctx));
    *out = s->dev_ctx;
    return QB_OK;
}
void qb_ctx_release(qb_storage* s, QbSearchCtx* c) {
    std::lock_guard<std::mutex> lk(s->mu);
    c->in_use = false;
}
static void ctx_destroy(QbSearchCtx* c) {
    if (!c) return;
    if (c->stream) cudaStreamSynchronize(c->stream);
    cudaFree(c->d_queries_raw); cudaFree(c->d_queries_enc); cudaFree(c->d_q_off); cudaFree(c->d_thr); cudaFree(c->d_cnt); cudaFree(c->d_done);
    cudaFree(c->d_cand); cudaFree(c->d_out); cudaFree(c->d_out_counts); cudaFree(c->d_deleted2); cudaFree(c->d_ids); cudaFree(c->d_mma); cudaFree(c->d_pf); cudaFree(c->d_pf_up5);
    if (c->h_stage) cudaFreeHost(c->h_stage);
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

// ------------------------------------------------------------------------------------------------ storages
static qb_storage* new_storage(int device, QbKind kind, uint32_t dim, uint64_t count) {
    qb_storage* s = new qb_storage();
    s->device = device; s->kind = kind; s->dim = dim; s->count = count;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) s->sm_count = prop.multiProcessorCount;
    return s;
}

static uint32_t elem_size_of(qb_dtype dt) { return dt == QB_DT_F32 ? 4 : (dt == QB_DT_F16 ? 2 : 1); }

extern "C" qb_status qb_storage_create_dense(int32_t device, qb_dtype dt, qb_distance distance, uint32_t dim, uint64_t count,
                                             const void* host_rows, uint64_t row_stride_bytes, qb_storage** out) {
    QB_CHECK(out, QB_ERR_INVALID, "create_dense: null out");
    *out = nullptr;
    QB_CHECK(dim >= 1 && dim <= 65536, QB_ERR_INVALID, "create_dense: dim %u outside [1,65536]", dim);
    QB_CHECK((int)dt >= 0 && (int)dt <= 2, QB_ERR_INVALID, "create_dense: bad dtype %d", (int)dt);
    QB_CHECK((int)distance >= 0 && (int)distance <= 3, QB_ERR_INVALID, "create_dense: bad distance %d", (int)distance);
    QB_CHECK(count <= 0xFFFFFFFFull, QB_ERR_INVALID, "create_dense: count exceeds PointOffsetType (u32)");
    QB_TRY(use_device(device));
    qb_storage* s = new_storage(device, QB_KIND_DENSE, dim, count);
    s->dtype = dt; s->distance = distance; s->elem_size = elem_size_of(dt);
    s->row_stride = (uint32_t)round_up_u64((uint64_t)dim * s->elem_size, 16);
    const size_t bytes = std::max<size_t>((size_t)count * s->row_stride, 256);
    cudaError_t e = cudaMalloc(&s->d_rows, bytes);
    if (e != cudaSuccess) { delete s; qb_set_error("cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e)); return QB_ERR_OOM; }
    s->hbm_bytes = bytes;
    if (s->row_stride != dim * s->elem_size) cudaMemset(s->d_rows, 0, bytes);
    *out = s;
    if (host_rows && count) {
        qb_status st = qb_storage_write_rows(s, 0, count, host_rows, row_stride_bytes);
        if (st != QB_OK) { qb_storage_destroy(s); *out = nullptr; return st; }
    }
    return QB_OK;
}

extern "C" qb_status qb_storage_write_rows(qb_storage* s, uint64_t first_row, uint64_t n_rows, const void* host_rows, uint64_t row_stride_bytes) {
    QB_CHECK(s && host_rows, QB_ERR_INVALID, "write_rows: null argument");
    QB_CHECK(s->kind == QB_KIND_DENSE, QB_ERR_UNSUPPORTED, "write_rows: dense storages only");
    QB_CHECK(first_row + n_rows <= s->count, QB_ERR_INVALID, "write_rows: range beyond count");
    const size_t rb = (size_t)s->dim * s->elem_size;
    if (row_stride_bytes == 0) row_stride_bytes = rb;
    QB_CHECK(row_stride_bytes >= rb, QB_ERR_INVALID, "write_rows: stride smaller than a row");
    QB_TRY(use_device(s->device));
    QB_CUDA(cudaMemcpy2D(reinterpret_cast<uint8_t*>(s->d_rows) + first_row * s->row_stride, s->row_stride, host_rows, row_stride_bytes, rb, n_rows,
                         cudaMemcpyHostToDevice));
    s->bf16_ready = false;   // the bf16 shadow (if any) no longer mirrors the rows
    s->q8_ready = false;
    s->q6_ready = false;
    s->q4b_ready = false;
    return QB_OK;
}

extern "C" qb_status qb_storage_write_rows_device(qb_storage* s, uint64_t first_row, uint64_t n_rows, const void* dev_rows, uint64_t row_stride_bytes) {
    QB_CHECK(s && dev_rows, QB_ERR_INVALID, "write_rows_device: null argument");
    QB_CHECK(s->kind == QB_KIND_DENSE, QB_ERR_UNSUPPORTED, "write_rows_device: dense storages only");
    QB_CHECK(first_row + n_rows <= s->count, QB_ERR_INVALID, "write_rows_device: range beyond count");
    const size_t rb = (size_t)s->dim * s->elem_size;
    if (row_stride_bytes == 0) row_stride_bytes = rb;
    QB_TRY(use_device(s->device));
    QB_CUDA(cudaMemcpy2D(reinterpret_cast<uint8_t*>(s->d_rows) + first_row * s->row_stride, s->row_stride, dev_rows, row_stride_bytes, rb, n_rows,
                         cudaMemcpyDeviceToDevice));
    s->bf16_ready = false;
    s->q8_ready = false;
    s->q6_ready = false;
    s->q4b_ready = false;
    return QB_OK;
}

__global__ void gather_rows_kernel(const uint8_t* __restrict__ rows, uint32_t stride, uint32_t row_bytes, const uint32_t* __restrict__ ids, uint64_t n,
                                   uint8_t* __restrict__ out) {
    for (uint64_t r = blockIdx.x; r < n; r += gridDim.x) {
        const uint8_t* src = rows + (size_t)ids[r] * stride;
        uint8_t* dst = out + r * row_bytes;
        for (uint32_t i = threadIdx.x; i < row_bytes; i += blockDim.x) dst[i] = src[i];
    }
}

extern "C" qb_status qb_storage_read_rows(const qb_storage* s, const uint32_t* ids, uint64_t n, void* host_out) {
    QB_CHECK(s && ids && host_out, QB_ERR_INVALID, "read_rows: null argument");
    QB_CHECK(s->kind == QB_KIND_DENSE, QB_ERR_UNSUPPORTED, "read_rows: dense storages only");
    if (n == 0) return QB_OK;
    std::vector<uint32_t> local(n);
    QB_TRY(localize_ids(s, ids, n, local.data(), "read_rows"));
    ids = local.data();
    QB_TRY(use_device(s->device));
    const uint32_t rb = s->dim * s->elem_size;
    uint32_t* d_ids = nullptr; uint8_t* d_out = nullptr;
    QB_CUDA(cudaMalloc(&d_ids, n * 4));
    cudaError_t e = cudaMalloc(&d_out, n * rb);
    if (e != cudaSuccess) { cudaFree(d_ids); qb_set_error("read_rows: cudaMalloc: %s", cudaGetErrorString(e)); return QB_ERR_OOM; }
    cudaMemcpy(d_ids, ids, n * 4, cudaMemcpyHostToDevice);
    gather_rows_kernel<<<(unsigned)std::min<uint64_t>(n, 4096), 128>>>(reinterpret_cast<const uint8_t*>(s->d_rows), s->row_stride, rb, d_ids, n, d_out);
    QB_LAUNCHED();
    e = cudaMemcpy(host_out, d_out, n * rb, cudaMemcpyDeviceToHost);
    cudaFree(d_ids); cudaFree(d_out);
    if (e != cudaSuccess) { qb_set_error("read_rows: %s", cudaGetErrorString(e)); return QB_ERR_CUDA; }
    return QB_OK;
}

extern "C" qb_status qb_storage_create_sq8(int32_t device, uint32_t dim, uint64_t count, const uint8_t* rows, uint32_t row_bytes, float alpha,
                                           float offset, float multiplier, qb_qdistance dt, int32_t invert, qb_distance metric, qb_storage** out) {
    QB_CHECK(out, QB_ERR_INVALID, "create_sq8: null out");
    *out = nullptr;
    QB_CHECK(dim >= 1 && dim <= 65536, QB_ERR_INVALID, "create_sq8: dim %u outside [1,65536]", dim);
    const uint32_t ad = dim + (16 - dim % 16) % 16;  // get_actual_dim, encoded_vectors_u8.rs:622-624
    QB_CHECK(row_bytes == ad + 4, QB_ERR_INVALID, "create_sq8: row_bytes %u != 4 + actual_dim %u (load validation, encoded_vectors_u8.rs:328)", row_bytes, ad);
    QB_CHECK(count == 0 || rows, QB_ERR_INVALID, "create_sq8: null rows");
    QB_CHECK(count <= 0xFFFFFFFFull, QB_ERR_INVALID, "create_sq8: count exceeds u32");
    QB_TRY(use_device(device));
    qb_storage* s = new_storage(device, QB_KIND_SQ8, dim, count);
    s->actual_dim = ad; s->alpha = alpha; s->offset = offset; s->multiplier = multiplier; s->qdist = dt; s->invert = invert ? 1 : 0;
    s->distance = metric;
    const size_t cb = std::max<size_t>((size_t)count * ad, 256), ob = std::max<size_t>((size_t)count * 4, 256);
    if (cudaMalloc(&s->d_codes, cb) != cudaSuccess || cudaMalloc(&s->d_voff, ob) != cudaSuccess) {
        qb_set_error("create_sq8: cudaMalloc failed: %s", cudaGetErrorString(cudaGetLastError()));
        qb_storage_destroy(s);
        return QB_ERR_OOM;
    }
    s->hbm_bytes = cb + ob;
    // upload in chunks through a device staging buffer, repacking 772-B rows into a 768-B code plane + f32 plane
    const uint64_t chunk_rows = std::max<uint64_t>(1, (64ull << 20) / row_bytes);
    uint8_t* d_stage = nullptr;
    if (count) {
        if (cudaMalloc(&d_stage, std::min<uint64_t>(chunk_rows, count) * row_bytes) != cudaSuccess) {
            qb_set_error("create_sq8: staging cudaMalloc failed"); qb_storage_destroy(s); return QB_ERR_OOM;
        }
        std::vector<float> h_voff;
        for (uint64_t r = 0; r < count; r += chunk_rows) {
            const uint64_t n = std::min<uint64_t>(chunk_rows, count - r);
            cudaError_t e = cudaMemcpy(d_stage, rows + r * row_bytes, n * row_bytes, cudaMemcpyDefault);  // host or device source
            qb_status st = (e == cudaSuccess) ? qb_sq8_repack(s, d_stage, row_bytes, r, n, 0) : QB_ERR_CUDA;
            if (st == QB_OK && cudaDeviceSynchronize() != cudaSuccess) st = QB_ERR_CUDA;
            // the largest |v_off| (inf once one is not finite) bounds the scores the tensor-core path can produce (qb_sq8_mma_block)
            h_voff.resize(n);
            if (st == QB_OK && cudaMemcpy(h_voff.data(), s->d_voff + r, n * 4, cudaMemcpyDeviceToHost) != cudaSuccess) st = QB_ERR_CUDA;
            if (st == QB_OK)
                for (const float v : h_voff) s->voff_absmax = std::isfinite(v) ? std::max(s->voff_absmax, std::fabs(v)) : INFINITY;
            if (st != QB_OK) { qb_set_error("create_sq8: upload failed: %s", cudaGetErrorString(cudaGetLastError())); cudaFree(d_stage); qb_storage_destroy(s); return st; }
        }
        cudaFree(d_stage);
    }
    *out = s;
    return QB_OK;
}

extern "C" qb_status qb_storage_create_pq(int32_t device, uint32_t dim, uint32_t m, const uint32_t* div_start_end, const float* centroids,
                                          uint32_t n_centroids, const uint8_t* codes, uint64_t count, qb_qdistance dt, int32_t invert,
                                          qb_distance metric, qb_storage** out) {
    QB_CHECK(out, QB_ERR_INVALID, "create_pq: null out");
    *out = nullptr;
    QB_CHECK(dim >= 1 && m >= 1 && div_start_end && centroids, QB_ERR_INVALID, "create_pq: bad arguments");
    QB_CHECK(n_centroids >= 1 && n_centroids <= 256, QB_ERR_INVALID, "create_pq: n_centroids %u outside [1,256]", n_centroids);
    QB_CHECK(count == 0 || codes, QB_ERR_INVALID, "create_pq: null codes");
    QB_CHECK(count <= 0xFFFFFFFFull, QB_ERR_INVALID, "create_pq: count exceeds u32");
    for (uint32_t j = 0; j < m; ++j)
        QB_CHECK(div_start_end[2 * j] < div_start_end[2 * j + 1] && div_start_end[2 * j + 1] <= dim, QB_ERR_INVALID, "create_pq: bad division %u", j);
    QB_TRY(use_device(device));
    qb_storage* s = new_storage(device, QB_KIND_PQ, dim, count);
    s->pq_m = m; s->pq_stride = (uint32_t)round_up_u64(m, 16); s->n_centroids = n_centroids; s->qdist = dt; s->invert = invert ? 1 : 0;
    s->distance = metric;
    s->pq_div.assign(div_start_end, div_start_end + 2 * m);
    const size_t cb = std::max<size_t>((size_t)count * s->pq_stride, 256);
    bool ok = cudaMalloc(&s->d_pq_codes, cb) == cudaSuccess && cudaMalloc(&s->d_centroids, (size_t)n_centroids * dim * 4) == cudaSuccess &&
              cudaMalloc(&s->d_pq_div, (size_t)2 * m * 4) == cudaSuccess;
    if (!ok) { qb_set_error("create_pq: cudaMalloc failed: %s", cudaGetErrorString(cudaGetLastError())); qb_storage_destroy(s); return QB_ERR_OOM; }
    s->hbm_bytes = cb + (size_t)n_centroids * dim * 4;
    cudaMemset(s->d_pq_codes, 0, cb);
    cudaError_t e = cudaMemcpy(s->d_centroids, centroids, (size_t)n_centroids * dim * 4, cudaMemcpyDefault);
    if (e == cudaSuccess) e = cudaMemcpy(s->d_pq_div, div_start_end, (size_t)2 * m * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && count) e = cudaMemcpy2D(s->d_pq_codes, s->pq_stride, codes, m, m, count, cudaMemcpyDefault);
    if (e != cudaSuccess) { qb_set_error("create_pq: upload: %s", cudaGetErrorString(e)); qb_storage_destroy(s); return QB_ERR_CUDA; }
    *out = s;
    return QB_OK;
}

static uint32_t bq_row_bytes_for(uint32_t dim, qb_bq_encoding enc) {  // get_quantized_vector_size_from_params :829-839
    uint64_t ext = dim;
    if (enc == QB_BQ_TWO_BITS) ext = (uint64_t)dim * 2;
    else if (enc == QB_BQ_ONE_AND_HALF_BITS) ext = ((uint64_t)dim * 3 + 1) / 2;
    if (ext < 1) ext = 1;
    return (uint32_t)(((ext + 127) / 128) * 16);
}

extern "C" qb_status qb_storage_create_bq(int32_t device, uint32_t dim, qb_bq_encoding enc, qb_bq_query_encoding qenc, const uint8_t* rows,
                                          uint32_t row_bytes, uint64_t count, qb_qdistance dt, int32_t invert, const float* mean_std,
                                          qb_distance metric, qb_storage** out) {
    QB_CHECK(out, QB_ERR_INVALID, "create_bq: null out");
    *out = nullptr;
    QB_CHECK(dim >= 1 && dim <= 65536, QB_ERR_INVALID, "create_bq: dim %u outside [1,65536]", dim);
    // EncodedVectorsBin<u128, _> rows (single vectors) are whole u128 words; multivector storages use EncodedVectorsBin<u8, _> whose rows
    // are ceil(bits / 8) bytes (quantized_vectors.rs:270-282).  Bit i sits in byte i / 8, bit i % 8 for both word types (little-endian
    // words), so a u8 row is the prefix of the u128 row: it is zero-padded to whole u128 words at upload and scored by the same kernels
    // (padding bits are zero in rows and queries alike and add nothing to any popcount).
    const uint32_t rb128 = bq_row_bytes_for(dim, enc);
    uint64_t ext_bits = dim;
    if (enc == QB_BQ_TWO_BITS) ext_bits = (uint64_t)dim * 2;
    else if (enc == QB_BQ_ONE_AND_HALF_BITS) ext_bits = ((uint64_t)dim * 3 + 1) / 2;
    const uint32_t rb_u8 = (uint32_t)((std::max<uint64_t>(ext_bits, 1) + 7) / 8);
    QB_CHECK(row_bytes == rb128 || row_bytes == rb_u8, QB_ERR_INVALID, "create_bq: row_bytes %u is neither the u128 row size %u nor the u8 row size %u", row_bytes, rb128, rb_u8);
    const uint32_t src_row_bytes = row_bytes;
    row_bytes = rb128;
    QB_CHECK(count == 0 || rows, QB_ERR_INVALID, "create_bq: null rows");
    QB_CHECK(count <= 0xFFFFFFFFull, QB_ERR_INVALID, "create_bq: count exceeds u32");
    QB_TRY(use_device(device));
    qb_storage* s = new_storage(device, QB_KIND_BQ, dim, count);
    s->bq_enc = enc; s->bq_qenc = qenc; s->bq_row_bytes = row_bytes; s->qdist = dt; s->invert = invert ? 1 : 0; s->distance = metric;
    const size_t rb = std::max<size_t>((size_t)count * row_bytes, 256);
    bool ok = cudaMalloc(&s->d_bq_rows, rb) == cudaSuccess;
    if (ok && mean_std) ok = cudaMalloc(&s->d_mean_std, (size_t)dim * 8) == cudaSuccess;
    if (!ok) { qb_set_error("create_bq: cudaMalloc failed: %s", cudaGetErrorString(cudaGetLastError())); qb_storage_destroy(s); return QB_ERR_OOM; }
    s->hbm_bytes = rb;
    cudaError_t e = cudaSuccess;
    if (count && src_row_bytes == row_bytes) e = cudaMemcpy(s->d_bq_rows, rows, (size_t)count * row_bytes, cudaMemcpyDefault);
    else if (count) {
        e = cudaMemset(s->d_bq_rows, 0, rb);
        if (e == cudaSuccess) e = cudaMemcpy2D(s->d_bq_rows, row_bytes, rows, src_row_bytes, src_row_bytes, count, cudaMemcpyDefault);
    }
    if (e == cudaSuccess && mean_std) e = cudaMemcpy(s->d_mean_std, mean_std, (size_t)dim * 8, cudaMemcpyDefault);
    if (e != cudaSuccess) { qb_set_error("create_bq: upload: %s", cudaGetErrorString(e)); qb_storage_destroy(s); return QB_ERR_CUDA; }
    *out = s;
    return QB_OK;
}

extern "C" void qb_storage_destroy(qb_storage* s) {
    if (!s) return;
    cudaSetDevice(s->device);
    for (QbSearchCtx* c : s->ctxs) ctx_destroy(c);
    ctx_destroy(s->dev_ctx);
    for (auto& pr : s->prof_pending) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
    for (auto& pr : s->prof_free) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
    cudaFree(s->d_rows); cudaFree(s->d_bf16); cudaFree(s->d_bf16_meta); cudaFree(s->d_q8); cudaFree(s->d_q8_meta); cudaFree(s->d_q6); cudaFree(s->d_q6_lo); cudaFree(s->d_q6_meta); cudaFree(s->d_q4b); cudaFree(s->d_codes); cudaFree(s->d_voff); cudaFree(s->d_pq_div); cudaFree(s->d_centroids); cudaFree(s->d_pq_codes);
    cudaFree(s->d_bq_rows); cudaFree(s->d_mean_std); cudaFree(s->d_deleted); cudaFree(s->d_pf_fallbacks);
    cudaGetLastError();
    delete s;
}

extern "C" qb_status qb_storage_info(const qb_storage* s, uint32_t* dim, uint64_t* count, uint64_t* hbm_bytes) {
    QB_CHECK(s, QB_ERR_INVALID, "storage_info: null storage");
    if (dim) *dim = s->dim;
    if (count) *count = s->count;
    if (hbm_bytes) *hbm_bytes = s->hbm_bytes;
    return QB_OK;
}

extern "C" qb_status qb_storage_set_deleted(qb_storage* s, const uint64_t* bitmap_words, uint64_t n_words) {
    QB_CHECK(s, QB_ERR_INVALID, "set_deleted: null storage");
    QB_TRY(use_device(s->device));
    std::lock_guard<std::mutex> lk(s->mu);
    if (!bitmap_words) { if (s->d_deleted) { cudaDeviceSynchronize(); cudaFree(s->d_deleted); s->d_deleted = nullptr; } return QB_OK; }
    const uint64_t need = ceil_div_u64(s->count, 64);
    QB_CHECK(n_words >= need, QB_ERR_INVALID, "set_deleted: bitmap has %llu words, need %llu", (unsigned long long)n_words, (unsigned long long)need);
    if (!s->d_deleted) QB_CUDA(cudaMalloc(&s->d_deleted, std::max<uint64_t>(need, 1) * 8));
    // searches in flight on this storage's (non-blocking) streams may be reading the flags: a rare control call, so simply wait for them
    QB_CUDA(cudaDeviceSynchronize());
    QB_CUDA(cudaMemcpy(s->d_deleted, bitmap_words, need * 8, cudaMemcpyHostToDevice));
    return QB_OK;
}

extern "C" void* qb_storage_stream(qb_storage* s) {
    if (!s) return nullptr;
    if (cudaSetDevice(s->device) != cudaSuccess) return nullptr;
    QbSearchCtx* c = nullptr;
    if (qb_ctx_device(s, &c) != QB_OK) return nullptr;
    return c->stream;
}

// ------------------------------------------------------------------------------------------------ Metric::preprocess
extern "C" qb_status qb_metric_preprocess(int32_t device, qb_distance distance, uint32_t dim, uint64_t n, const float* in, float* out) {
    QB_CHECK(in && out && dim >= 1, QB_ERR_INVALID, "metric_preprocess: bad arguments");
    QB_TRY(use_device(device));
    if (n == 0) return QB_OK;
    float* d = nullptr;
    QB_CUDA(cudaMalloc(&d, n * dim * 4));
    cudaError_t e = cudaMemcpy(d, in, n * dim * 4, cudaMemcpyHostToDevice);
    qb_status st = (e == cudaSuccess) ? qb_launch_preprocess_rows(distance, dim, n, d, dim, d, dim, 0) : QB_ERR_CUDA;
    if (st == QB_OK) e = cudaMemcpy(out, d, n * dim * 4, cudaMemcpyDeviceToHost);
    cudaFree(d);
    if (st != QB_OK || e != cudaSuccess) { qb_set_error("metric_preprocess: %s", cudaGetErrorString(e)); return st != QB_OK ? st : QB_ERR_CUDA; }
    return QB_OK;
}

extern "C" qb_status qb_metric_preprocess_device(int32_t device, qb_distance distance, uint32_t dim, uint64_t n, float* dev_rows, uint64_t row_stride_bytes) {
    QB_CHECK(dev_rows && dim >= 1, QB_ERR_INVALID, "metric_preprocess_device: bad arguments");
    QB_TRY(use_device(device));
    if (row_stride_bytes == 0) row_stride_bytes = (uint64_t)dim * 4;
    QB_CHECK(row_stride_bytes % 4 == 0, QB_ERR_INVALID, "metric_preprocess_device: stride must be a multiple of 4");
    QB_TRY(qb_launch_preprocess_rows(distance, dim, n, dev_rows, row_stride_bytes / 4, dev_rows, row_stride_bytes / 4, 0));
    QB_CUDA(cudaStreamSynchronize(0));
    return QB_OK;
}

extern "C" float qb_metric_postprocess(qb_distance distance, float score) {
    // MetricPostProcessing::postprocess, spaces/simple.rs:74-78,118-122 (host arithmetic on one scalar per result)
    if (distance == QB_DIST_EUCLID) return sqrtf(fabsf(score));
    if (distance == QB_DIST_MANHATTAN) return fabsf(score);
    return score;
}

// ------------------------------------------------------------------------------------------------ queries
size_t qb_encoded_query_bytes(const qb_storage* s) {
    switch (s->kind) {
        case QB_KIND_DENSE: return s->row_stride;
        case QB_KIND_SQ8: return s->actual_dim;
        case QB_KIND_PQ: return (size_t)s->pq_m * s->n_centroids * 4;
        default: return (size_t)s->bq_row_bytes * (s->bq_qenc == QB_BQQ_SCALAR4 ? 4 : (s->bq_qenc == QB_BQQ_SCALAR8 ? 8 : 1));
    }
}

// f32 stride (floats) of the preprocessed-query staging rows
static uint32_t pre_stride_f(const qb_storage* s) { return (uint32_t)round_up_u64(s->dim, 4); }

// Metric::preprocess then (for quantized storages) EncodedVectors::encode_query, all on the device.
// d_pre: scratch of nq * pre_stride_f floats (ignored for dense f32 where the output IS the preprocessed query)
static qb_status prepare_queries(const qb_storage* s, const float* d_q_raw, uint32_t nq, float* d_pre, void* d_q_enc, float* d_q_off, cudaStream_t stream) {
    if (nq == 0) return QB_OK;
    if (s->kind == QB_KIND_DENSE && s->dtype == QB_DT_F32) {
        return qb_launch_preprocess_rows(s->distance, s->dim, nq, d_q_raw, s->dim, reinterpret_cast<float*>(d_q_enc), s->row_stride / 4, stream);
    }
    const uint32_t ps = pre_stride_f(s);
    // u8 / f16 storages: only CosineMetric<f32>-style preprocess applies to f32/f16 (metric_f16/simple_cosine.rs); u8 cosine has none
    qb_distance pre_dist = s->distance;
    if (s->kind == QB_KIND_DENSE && s->dtype == QB_DT_U8) pre_dist = QB_DIST_DOT;
    QB_TRY(qb_launch_preprocess_rows(pre_dist, s->dim, nq, d_q_raw, s->dim, d_pre, ps, stream));
    switch (s->kind) {
        case QB_KIND_DENSE: return qb_dense_x_convert_queries(s, d_pre, ps, nq, d_q_enc, stream);
        case QB_KIND_SQ8: return qb_sq8_encode_queries(s, d_pre, ps, nq, reinterpret_cast<uint8_t*>(d_q_enc), d_q_off, stream);
        case QB_KIND_PQ: return qb_pq_build_luts(s, d_pre, ps, nq, reinterpret_cast<float*>(d_q_enc), stream);
        default: return qb_bq_encode_queries(s, d_pre, ps, nq, 0, d_q_enc, stream);
    }
}

qb_status qb_launch_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream) {
    switch (s->kind) {
        case QB_KIND_DENSE: return s->dtype == QB_DT_F32 ? qb_dense_f32_scan(s, a, stream) : qb_dense_x_scan(s, a, stream);
        case QB_KIND_SQ8: return qb_sq8_scan(s, a, stream);
        case QB_KIND_PQ: return qb_pq_scan(s, a, stream);
        default: return qb_bq_scan(s, a, stream);
    }
}

qb_status qb_launch_score_points(const qb_storage* s, const void* d_q_enc, const float* d_q_off, const uint32_t* d_ids, uint64_t n, float* d_scores,
                                 cudaStream_t stream) {
    switch (s->kind) {
        case QB_KIND_DENSE:
            return s->dtype == QB_DT_F32 ? qb_dense_f32_score_points(s, d_q_enc, d_ids, n, d_scores, stream)
                                         : qb_dense_x_score_points(s, d_q_enc, d_ids, n, d_scores, stream);
        case QB_KIND_SQ8: return qb_sq8_score_points(s, d_q_enc, d_q_off, d_ids, n, d_scores, stream);
        case QB_KIND_PQ: return qb_pq_score_points(s, d_q_enc, d_ids, n, d_scores, stream);
        default: return QB_ERR_INVALID;  // BQ goes through the scorer (needs bits)
    }
}

// ------------------------------------------------------------------------------------------------ search
struct SearchPlan {
    uint64_t n_cand;       // candidates per query (rows or listed ids)
    bool direct;           // one dense pass + select
    uint64_t sample;       // sample prefix length (dense pass -> per-query threshold)
    uint64_t sample2;      // 0, or a longer prefix scanned with that threshold to refine it before the full pass (three levels)
    uint64_t cap;          // per-query candidate capacity of the filter pass
    uint32_t q_chunk;      // queries per pass
};

static SearchPlan make_plan(uint64_t n_cand, uint32_t nq, uint32_t top, bool force_direct, bool refine) {
    SearchPlan p{};
    p.n_cand = n_cand;
    const uint64_t kDirectRows = 65536;
    const uint64_t kCandBudgetBytes = 2ull << 30;  // candidate buffer budget per pass
    if (force_direct || n_cand <= kDirectRows) {
        p.direct = true;
        p.cap = std::max<uint64_t>(n_cand, 1);
    } else if (refine && n_cand >= (1ull << 20)) {
        // Batched tensor-core scan: a dense sample costs 8 B per (row, query) to write and ~4x that to select from, and every survivor
        // of the filter pass costs a trip through the epilogue's slow path.  Three levels keep both small:
        //   S1 rows dense -> thr1;  S2 = 1.5 sqrt(N S1) rows filtered by thr1 -> thr2 (k-th best of S2);  all rows filtered by thr2.
        p.direct = false;
        p.sample = round_up_u64(std::max<uint64_t>(4096, 16ull * top), 256);
        p.sample2 = std::min<uint64_t>(round_up_u64((uint64_t)(1.5 * sqrt((double)n_cand * (double)p.sample)), 1024), n_cand / 4);
        const uint64_t expect = std::max<uint64_t>(p.sample2 * top / p.sample, n_cand * top / p.sample2);
        p.cap = std::max<uint64_t>(p.sample, 8 * expect + 4096);
    } else {
        p.direct = false;
        // minimise sample + expected survivors (N*k/S): S ~ sqrt(N*k); x2 keeps the survivor list short
        // batches pay for every survivor in the epilogue of the tensor-core scan (a global atomic each): a 4x larger sample
        // costs < 1 % more scan work and cuts survivors 4x
        uint64_t sgoal = (uint64_t)((nq >= 32 ? 8.0 : 2.0) * sqrt((double)n_cand * (double)top));
        sgoal = round_up_u64(std::max<uint64_t>(sgoal, 8192), 1024);
        if (qb_opt().sample_rows) sgoal = std::max<uint64_t>(256, qb_opt().sample_rows);  // tuning experiments
        p.sample = std::min<uint64_t>(sgoal, n_cand / 2);
        const uint64_t expect = (uint64_t)((double)n_cand * (double)top / (double)p.sample);
        p.cap = std::max<uint64_t>(p.sample, 8 * expect + 4096);
        p.cap = std::min<uint64_t>(p.cap, n_cand);
    }
    uint64_t qc = kCandBudgetBytes / (p.cap * 8);
    if (qc < 1) qc = 1;
    p.q_chunk = (uint32_t)std::min<uint64_t>(qc, nq);
    return p;
}

static void profile_begin(qb_storage* s, QbSearchCtx* c, cudaStream_t stream, cudaEvent_t* e0, cudaEvent_t* e1) {
    *e0 = *e1 = nullptr;
    if (!s->profile) return;
    {
        std::lock_guard<std::mutex> lk(s->mu);
        if (!s->prof_free.empty()) { *e0 = s->prof_free.back().first; *e1 = s->prof_free.back().second; s->prof_free.pop_back(); }
    }
    if (!*e0) { cudaEventCreate(e0); cudaEventCreate(e1); }
    cudaEventRecord(*e0, stream);
}
// the same pair without recording: the callee brackets its dominant kernel itself
static void profile_acquire(qb_storage* s, cudaEvent_t* e0, cudaEvent_t* e1) {
    *e0 = *e1 = nullptr;
    if (!s->profile) return;
    {
        std::lock_guard<std::mutex> lk(s->mu);
        if (!s->prof_free.empty()) { *e0 = s->prof_free.back().first; *e1 = s->prof_free.back().second; s->prof_free.pop_back(); }
    }
    if (!*e0) { cudaEventCreate(e0); cudaEventCreate(e1); }
}
static void profile_commit(qb_storage* s, cudaEvent_t e0, cudaEvent_t e1) {
    if (!e0) return;
    std::lock_guard<std::mutex> lk(s->mu);
    s->prof_pending.emplace_back(e0, e1);
}
static void profile_end(qb_storage* s, cudaStream_t stream, cudaEvent_t e0, cudaEvent_t e1) {
    if (!e0) return;
    cudaEventRecord(e1, stream);
    std::lock_guard<std::mutex> lk(s->mu);
    s->prof_pending.emplace_back(e0, e1);
}

// Core of the fused scan: queries already encoded in c->d_queries_enc (+ c->d_q_off).  Results to d_out/d_counts
// (device).  Sets *overflow_possible when the filter pass is used (caller checks c->d_cnt overflow flag at [nq]).
enum { RS_FORCE_DIRECT = 1, RS_NO_MMA = 2, RS_NO_SEGMENTS = 4, RS_NO_REFINE = 8 };
static qb_status run_search(qb_storage* s, QbSearchCtx* c, uint32_t nq, uint32_t top, const uint32_t* d_ids, uint64_t n_ids, const uint32_t* d_deleted2,
                            const volatile int32_t* is_stopped, uint32_t rs_flags, qb_scored_point* d_out, uint32_t* d_counts, unsigned int* d_overflow,
                            bool* can_flag = nullptr) {
    const bool force_direct = (rs_flags & RS_FORCE_DIRECT) != 0;
    if (can_flag) *can_flag = true;  // cleared on the paths that have no heuristic to fall back from
    const uint64_t n_cand = d_ids ? n_ids : s->count;
    cudaStream_t stream = c->stream;
    if (n_cand == 0) { QB_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)nq * 4, stream)); return QB_OK; }
    // single query, small top, dense f32: one streaming scan with per-CTA top-k lists + one small select (qb_dense.cu, LOCALK)
    if (nq == 1 && top <= 16 && !d_ids && !force_direct && s->kind == QB_KIND_DENSE && s->dtype == QB_DT_F32 && n_cand > 65536 && !qb_opt().disable_localk) {
        QB_TRY(ensure_dev_elems(&c->d_cand, &c->cand_elems, (size_t)4096));
        QbScanArgs a{};
        a.d_q_enc = c->d_queries_enc; a.nq = 1; a.row_begin = 0; a.row_end = n_cand;
        a.emit.deleted = s->d_deleted; a.emit.deleted2 = d_deleted2; a.emit.id_base = s->id_base; a.emit.cand = c->d_cand; a.emit.cap = 4096;
        // the last CTA of the scan merges the per-CTA lists into d_out itself (d_done = its arrival counter: zeroed once, reset by the kernel)
        if (!c->d_done) { QB_CUDA(cudaMalloc(&c->d_done, 256)); QB_CUDA(cudaMemsetAsync(c->d_done, 0, 256, stream)); }
        a.emit.final_out = d_out; a.emit.final_count = d_counts; a.emit.done_counter = c->d_done;
        uint64_t n_slots = 0;
        cudaEvent_t e0, e1;
        // dot / cosine on a large storage: the scan reads the bf16 shadow plane (half the bytes), survivors are re-scored exactly and a
        // device-side flag falls back to the exact scan below when the prefilter's candidate list overflowed (qb_prefilter.cu)
        if (qb_f32_prefilter_usable(s, n_cand, top, stream)) {
            if (!c->d_pf) { QB_CUDA(cudaMalloc(&c->d_pf, qb_f32_prefilter_scratch_bytes())); QB_CUDA(cudaMemsetAsync(c->d_pf, 0, 256, stream)); }
            QB_TRY(ensure_dev_elems(&c->d_pf_up5, &c->pf_up5_elems, (size_t)round_up_u64(n_cand, 4)));
            {
                std::lock_guard<std::mutex> lk(s->mu);
                if (!s->d_pf_fallbacks) { QB_CUDA(cudaMalloc(&s->d_pf_fallbacks, 256)); QB_CUDA(cudaMemsetAsync(s->d_pf_fallbacks, 0, 256, stream)); }
            }
            profile_acquire(s, &e0, &e1);
            QB_TRY(qb_f32_prefilter_search(s, a, top, c->d_pf, c->d_pf_up5, s->d_pf_fallbacks, d_out, d_counts, e0, e1, stream));
            profile_commit(s, e0, e1);
            if (can_flag) *can_flag = false;
            return QB_OK;
        }
        profile_begin(s, c, stream, &e0, &e1);
        QB_TRY(qb_dense_f32_scan_localk(s, a, top, &n_slots, stream));
        if (n_slots != 0 && n_slots <= 4096) {
            profile_end(s, stream, e0, e1);
            if (can_flag) *can_flag = false;
            return QB_OK;
        }
        if (e0) { cudaEventDestroy(e0); cudaEventDestroy(e1); }
        QB_CHECK(n_slots == 0, QB_ERR_CUDA, "local top-k scan wrote %llu slots", (unsigned long long)n_slots);
    }
    const bool mma_ok = !d_ids && !(rs_flags & RS_NO_MMA) && !qb_opt().disable_mma;
    // dense f32 (dot / cosine) batches: bf16 tensor-core prefilter + exact rescoring of the survivors (qb_sq8_mma.cu, F16)
    const bool f32_mma = mma_ok && s->kind == QB_KIND_DENSE && n_cand >= (1ull << 17) && qb_f32_mma_block(s, nq, stream) != 0;
    const SearchPlan plan = make_plan(n_cand, nq, top, force_direct, mma_ok && (f32_mma || qb_sq8_mma_block(s, nq) != 0) && !(rs_flags & RS_NO_REFINE));
    if (can_flag && plan.direct) *can_flag = false;  // full materialisation: no threshold, no counters, nothing to overflow
    QB_TRY(ensure_dev_elems(&c->d_cand, &c->cand_elems, (size_t)plan.q_chunk * plan.cap));
    QB_TRY(ensure_dev_elems(&c->d_thr, &c->thr_elems, (size_t)2 * nq));   // [nq] thresholds + [nq] scratch (adjusted thresholds of the PQ prefilter)
    QB_TRY(ensure_dev_elems(&c->d_cnt, &c->cnt_elems, (size_t)nq + 1));
    const size_t enc_bytes = qb_encoded_query_bytes(s);

    for (uint32_t q0 = 0; q0 < nq; q0 += plan.q_chunk) {
        if (is_stopped && *is_stopped) { qb_set_error("search cancelled"); return QB_ERR_CANCELLED; }
        const uint32_t qn = std::min<uint32_t>(plan.q_chunk, nq - q0);
        QbScanArgs a{};
        a.d_q_enc = reinterpret_cast<const uint8_t*>(c->d_queries_enc) + (size_t)q0 * enc_bytes;
        a.d_q_off = c->d_q_off ? c->d_q_off + q0 : nullptr;
        a.nq = qn;
        a.d_ids = d_ids;
        a.emit.deleted = s->d_deleted;
        a.emit.deleted2 = d_deleted2;
        a.emit.id_base = s->id_base;
        a.emit.cand = c->d_cand;
        a.emit.cap = plan.cap;
        a.d_thr_scratch = c->d_thr + nq + q0;
        if (s->kind == QB_KIND_PQ && !d_ids && !plan.direct) {
            const size_t need = qb_pq_scratch_bytes(s, qn);
            if (need) { QB_TRY(qb_ensure_device(&c->d_mma, &c->mma_bytes, need)); a.d_scratch = c->d_mma; a.scratch_bytes = c->mma_bytes; }
        }
        cudaEvent_t e0, e1;
        if (plan.direct) {
            a.row_begin = 0; a.row_end = n_cand;
            a.emit.dense = 1; a.emit.dense_base = 0;
            profile_begin(s, c, stream, &e0, &e1);
            QB_TRY(qb_launch_scan(s, a, stream));
            profile_end(s, stream, e0, e1);
            QB_TRY(qb_launch_select(c->d_cand, nullptr, plan.cap, n_cand, qn, top, 0, d_out + (size_t)q0 * top, d_counts + q0, nullptr, nullptr, stream));
        } else {
            // pass 1: sample prefix, materialised densely -> per-query threshold = k-th best of the sample
            a.row_begin = 0; a.row_end = plan.sample;
            a.emit.dense = 1; a.emit.dense_base = 0;
            const bool f32b = f32_mma && qb_f32_mma_block(s, qn, stream) != 0;   // this chunk of the batch is wide enough for the tensor-core prefilter
            const uint32_t mma_blk = mma_ok ? (f32b ? qb_f32_mma_block(s, qn, stream) : qb_sq8_mma_block(s, qn)) : 0;
            const uint32_t nq_pad = mma_blk ? (uint32_t)round_up_u64(qn, mma_blk) : 0;
            const uint32_t q_stride_f = s->row_stride / 4;              // dense f32: encoded queries = preprocessed f32 rows
            if (mma_blk && !f32b) {
                QB_TRY(qb_sq8_mma_scan(s, reinterpret_cast<const uint8_t*>(a.d_q_enc), nq_pad, a.d_q_off, qn, mma_blk, 0, plan.sample, a.emit, d_overflow, nullptr,
                                       nullptr, 0, stream));
            } else {
                QB_TRY(qb_launch_scan(s, a, stream));                   // the sample is always scored exactly for f32 storages
            }
            QB_TRY(qb_launch_select(c->d_cand, nullptr, plan.cap, plan.sample, qn, top, 1, nullptr, nullptr, c->d_thr + q0, nullptr, stream));
            if (mma_blk) QB_TRY(qb_ensure_device(&c->d_mma, &c->mma_bytes, f32b ? qb_f32_mma_scratch_bytes(s, nq_pad) : qb_sq8_mma_scratch_bytes(s, nq_pad)));
            if (plan.sample2) {
                // level 2: a longer prefix filtered by the level-1 threshold; its k-th best survivor is the threshold of the full pass
                QB_CUDA(cudaMemsetAsync(c->d_cnt + q0, 0, (size_t)qn * 4, stream));
                a.row_end = plan.sample2;
                a.emit.dense = 0; a.emit.thr = c->d_thr + q0; a.emit.cnt = c->d_cnt + q0;
                unsigned long long seg2 = 0;
                if (f32b) {
                    QB_TRY(qb_f32_mma_scan(s, reinterpret_cast<const float*>(a.d_q_enc), q_stride_f, qn, nq_pad, mma_blk, plan.sample2, a.emit, d_overflow, c->d_mma,
                                           c->mma_bytes, stream));
                } else if (mma_blk) {
                    QB_TRY(qb_sq8_mma_scan(s, reinterpret_cast<const uint8_t*>(a.d_q_enc), nq_pad, a.d_q_off, qn, mma_blk, 0, plan.sample2, a.emit, d_overflow,
                                           (rs_flags & RS_NO_SEGMENTS) ? nullptr : &seg2, c->d_mma, c->mma_bytes, stream));
                } else {
                    QB_TRY(qb_launch_scan(s, a, stream));  // a chunk too small for the tensor-core kernel
                }
                QB_TRY(qb_launch_select(c->d_cand, c->d_cnt + q0, plan.cap, seg2, qn, top, 1, nullptr, nullptr, c->d_thr + q0, d_overflow, stream));
            }
            // pass 2: everything, keeping only score >= threshold
            QB_CUDA(cudaMemsetAsync(c->d_cnt + q0, 0, (size_t)qn * 4, stream));
            a.row_begin = 0; a.row_end = n_cand;
            a.emit.dense = 0; a.emit.thr = c->d_thr + q0; a.emit.cnt = c->d_cnt + q0;
            if (is_stopped && *is_stopped) { qb_set_error("search cancelled"); return QB_ERR_CANCELLED; }
            profile_begin(s, c, stream, &e0, &e1);
            unsigned long long seg_len = 0;
            if (f32b) {
                // batched dense f32: bf16 tensor-core prefilter, survivors re-scored exactly (qb_sq8_mma.cu, F16)
                QB_TRY(qb_f32_mma_scan(s, reinterpret_cast<const float*>(a.d_q_enc), q_stride_f, qn, nq_pad, mma_blk, n_cand, a.emit, d_overflow, c->d_mma, c->mma_bytes,
                                       stream));
            } else if (mma_blk) {
                // batched SQ8: tensor-core GEMM with the fused epilogue/filter (qb_sq8_mma.cu)
                QB_TRY(qb_sq8_mma_scan(s, reinterpret_cast<const uint8_t*>(a.d_q_enc), nq_pad, a.d_q_off, qn, mma_blk, 0, n_cand, a.emit, d_overflow,
                                       (rs_flags & RS_NO_SEGMENTS) ? nullptr : &seg_len, c->d_mma, c->mma_bytes, stream));
            } else {
                QB_TRY(qb_launch_scan(s, a, stream));
            }
            profile_end(s, stream, e0, e1);
            // seg_len != 0: per-(query, CTA) segments with empty (zero) slots -> fixed-length selection
            QB_TRY(qb_launch_select(c->d_cand, c->d_cnt + q0, plan.cap, seg_len, qn, top, 0, d_out + (size_t)q0 * top, d_counts + q0, nullptr, d_overflow, stream));
        }
    }
    return QB_OK;
}

static uint64_t cpu_units_per_point(const qb_storage* s) {
    switch (s->kind) {
        case QB_KIND_DENSE: return (uint64_t)s->dim * s->elem_size;  // set_cpu_multiplier(dim * size_of::<TElement>()), metric_query_scorer.rs:43
        case QB_KIND_SQ8: return s->dim;                             // encoded_vectors_u8.rs:785-787
        case QB_KIND_PQ: return s->pq_m;                             // encoded_vectors_pq.rs:693-695
        default: return s->bq_row_bytes;                             // encoded_vectors_binary.rs:999
    }
}

// vector_io_read per scored point: dim * size_of::<TElement>() for on-disk dense storages (metric_query_scorer.rs:44-48), the
// quantized row size for on-disk quantized data (quantized_query_scorer.rs:48,84-86), 0 for RAM-resident storages
static uint64_t io_units_per_point(const qb_storage* s) {
    if (!s->on_disk) return 0;
    switch (s->kind) {
        case QB_KIND_DENSE: return (uint64_t)s->dim * s->elem_size;
        case QB_KIND_SQ8: return (uint64_t)s->actual_dim + 4;
        case QB_KIND_PQ: return s->pq_m;
        default: return s->bq_row_bytes;
    }
}

extern "C" qb_status qb_search_batch(qb_storage* s, const float* queries, uint32_t n_queries, uint32_t top, const uint64_t* deleted_bitmap,
                                     const uint32_t* id_list, uint64_t n_ids, const volatile int32_t* is_stopped, qb_scored_point* out,
                                     uint32_t* out_counts, qb_hw_counters* counters) {
    QB_CHECK(s && out && out_counts, QB_ERR_INVALID, "search_batch: null argument");
    QB_CHECK(n_queries == 0 || queries, QB_ERR_INVALID, "search_batch: null queries");
    QB_CHECK(top >= 1, QB_ERR_INVALID, "search_batch: top must be >= 1 (FixedLengthPriorityQueue::new panics on 0)");
    QB_CHECK(top <= QB_MAX_TOP, QB_ERR_UNSUPPORTED, "search_batch: top %u > %u not supported by the fused selection", top, QB_MAX_TOP);
    if (n_queries == 0) return QB_OK;
    if (is_stopped && *is_stopped) { qb_set_error("search cancelled"); return QB_ERR_CANCELLED; }
    QB_TRY(use_device(s->device));
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_acquire(s, &c));
    struct Rel { qb_storage* s; QbSearchCtx* c; ~Rel() { qb_ctx_release(s, c); } } rel{s, c};
    cudaStream_t stream = c->stream;

    const size_t raw_bytes = (size_t)n_queries * s->dim * 4;
    const size_t res_bytes = (size_t)n_queries * top * sizeof(qb_scored_point);
    const size_t cnt_bytes = (size_t)n_queries * 4;
    // pinned staging: [queries | results | counts | overflow flag | candidate ids]
    const size_t ids_off = round_up_u64(raw_bytes + res_bytes + cnt_bytes + 16, 16);
    QB_TRY(qb_ensure_pinned(&c->h_stage, &c->h_stage_bytes, ids_off + (id_list ? n_ids * 4 : 0)));
    uint8_t* hs = reinterpret_cast<uint8_t*>(c->h_stage);
    memcpy(hs, queries, raw_bytes);
    if (id_list) QB_TRY(localize_ids(s, id_list, n_ids, reinterpret_cast<uint32_t*>(hs + ids_off), "search_batch"));
    QB_TRY(qb_ensure_device(&c->d_queries_raw, &c->queries_raw_bytes, raw_bytes + (size_t)n_queries * pre_stride_f(s) * 4));
    // +256 rows: the tensor-core SQ8 path reads whole query blocks (rows past n_queries are masked, never scored)
    QB_TRY(qb_ensure_device(&c->d_queries_enc, &c->queries_enc_bytes, ((size_t)n_queries + 256) * qb_encoded_query_bytes(s)));
    QB_TRY(ensure_dev_elems(&c->d_q_off, &c->q_off_elems, (size_t)n_queries));
    QB_TRY(ensure_dev_elems(&c->d_out, &c->out_elems, (size_t)n_queries * top));
    QB_TRY(ensure_dev_elems(&c->d_out_counts, &c->out_counts_elems, (size_t)n_queries + 4));
    QB_CUDA(cudaMemcpyAsync(c->d_queries_raw, hs, raw_bytes, cudaMemcpyHostToDevice, stream));
    float* d_pre = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(c->d_queries_raw) + raw_bytes);
    QB_TRY(prepare_queries(s, reinterpret_cast<const float*>(c->d_queries_raw), n_queries, d_pre, c->d_queries_enc, c->d_q_off, stream));

    const uint32_t* d_del2 = nullptr;
    if (deleted_bitmap) {
        const uint64_t words64 = ceil_div_u64(s->count, 64);
        QB_TRY(ensure_dev_elems(&c->d_deleted2, &c->deleted2_words, (size_t)words64 * 2));
        QB_CUDA(cudaMemcpyAsync(c->d_deleted2, deleted_bitmap, words64 * 8, cudaMemcpyHostToDevice, stream));
        d_del2 = c->d_deleted2;
    }
    const uint32_t* d_ids = nullptr;
    if (id_list) {
        QB_TRY(ensure_dev_elems(&c->d_ids, &c->ids_elems, (size_t)std::max<uint64_t>(n_ids, 1)));
        QB_CUDA(cudaMemcpyAsync(c->d_ids, hs + ids_off, n_ids * 4, cudaMemcpyHostToDevice, stream));
        d_ids = c->d_ids;
    }
    unsigned int* d_overflow = reinterpret_cast<unsigned int*>(c->d_out_counts + n_queries);
    uint8_t* h_res = hs + raw_bytes;
    uint8_t* h_cnt = h_res + res_bytes;
    // Fast path first; the device reports (flags word) when one of its assumptions did not hold and the host reruns without it:
    //   1 candidate buffer overflow (threshold admitted too much: mass ties, mostly-deleted sample) -> full materialisation
    //   2 a tensor-core dot product left the f32-exact window (>= 2^24)                           -> lane-exact CUDA-core kernel
    //   8 a per-(query, CTA) survivor segment filled up                                            -> global counters
    uint32_t rs_flags = 0;
    for (int attempt = 0; attempt < 4; ++attempt) {
        QB_CUDA(cudaMemsetAsync(d_overflow, 0, 4, stream));
        QB_TRY(run_search(s, c, n_queries, top, d_ids, n_ids, d_del2, is_stopped, rs_flags, c->d_out, c->d_out_counts, d_overflow));
        QB_CUDA(cudaMemcpyAsync(h_res, c->d_out, res_bytes, cudaMemcpyDeviceToHost, stream));
        QB_CUDA(cudaMemcpyAsync(h_cnt, c->d_out_counts, cnt_bytes + 4, cudaMemcpyDeviceToHost, stream));
        QB_CUDA(cudaStreamSynchronize(stream));
        unsigned int flags = 0;
        memcpy(&flags, h_cnt + cnt_bytes, 4);
        uint32_t next = rs_flags;
        if (flags & 8u) next |= RS_NO_SEGMENTS;
        if (flags & 2u) next |= RS_NO_MMA;
        if (flags & 1u) next |= RS_FORCE_DIRECT | RS_NO_MMA;
        if (next == rs_flags) break;
        s->n_reruns.fetch_add(1, std::memory_order_relaxed);
        if (qb_opt().verbose) fprintf(stderr, "[qb200] search rerun: device flags=0x%x, mode 0x%x -> 0x%x\n", flags, rs_flags, next);
        rs_flags = next;
    }
    s->n_searches.fetch_add(1, std::memory_order_relaxed);
    memcpy(out, h_res, res_bytes);
    memcpy(out_counts, h_cnt, cnt_bytes);
    if (counters) {
        const uint64_t n_cand = id_list ? n_ids : s->count;
        counters->cpu += n_cand * (uint64_t)n_queries * cpu_units_per_point(s);
        counters->vector_io_read += n_cand * (uint64_t)n_queries * io_units_per_point(s);
    }
    return QB_OK;
}

extern "C" qb_status qb_search_batch_device(qb_storage* s, const float* dev_queries, uint32_t n_queries, uint32_t top, qb_scored_point* dev_out,
                                            uint32_t* dev_counts) {
    QB_CHECK(s && dev_queries && dev_out && dev_counts, QB_ERR_INVALID, "search_batch_device: null argument");
    QB_CHECK(top >= 1 && top <= QB_MAX_TOP, QB_ERR_INVALID, "search_batch_device: top %u outside [1,%u]", top, QB_MAX_TOP);
    if (n_queries == 0) return QB_OK;
    QB_TRY(use_device(s->device));
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_device(s, &c));
    QB_TRY(qb_ensure_device(&c->d_queries_raw, &c->queries_raw_bytes, (size_t)n_queries * pre_stride_f(s) * 4 + 256));
    QB_TRY(qb_ensure_device(&c->d_queries_enc, &c->queries_enc_bytes, ((size_t)n_queries + 256) * qb_encoded_query_bytes(s)));
    QB_TRY(ensure_dev_elems(&c->d_q_off, &c->q_off_elems, (size_t)n_queries));
    QB_TRY(ensure_dev_elems(&c->d_out_counts, &c->out_counts_elems, (size_t)n_queries + 4));
    QB_TRY(prepare_queries(s, dev_queries, n_queries, reinterpret_cast<float*>(c->d_queries_raw), c->d_queries_enc, c->d_q_off, c->stream));
    unsigned int* d_overflow = reinterpret_cast<unsigned int*>(c->d_out_counts + n_queries);
    // same contract as qb_search_batch: the device reports a broken fast-path assumption in a flags word and the host reruns
    // without it; reading that word is the one synchronisation of this call
    QB_TRY(qb_ensure_pinned(&c->h_stage, &c->h_stage_bytes, 64));
    uint32_t rs_flags = 0;
    for (int attempt = 0; attempt < 4; ++attempt) {
        QB_CUDA(cudaMemsetAsync(d_overflow, 0, 4, c->stream));
        bool can_flag = true;
        QB_TRY(run_search(s, c, n_queries, top, nullptr, 0, nullptr, nullptr, rs_flags, dev_out, dev_counts, d_overflow, &can_flag));
        if (!can_flag) break;  // exact single-pass path: nothing to check, the call stays asynchronous
        QB_CUDA(cudaMemcpyAsync(c->h_stage, d_overflow, 4, cudaMemcpyDeviceToHost, c->stream));
        QB_CUDA(cudaStreamSynchronize(c->stream));
        unsigned int flags = 0;
        memcpy(&flags, c->h_stage, 4);
        uint32_t next = rs_flags;
        if (flags & 8u) next |= RS_NO_SEGMENTS;
        if (flags & 2u) next |= RS_NO_MMA;
        if (flags & 1u) next |= RS_FORCE_DIRECT | RS_NO_MMA;
        if (next == rs_flags) break;
        s->n_reruns.fetch_add(1, std::memory_order_relaxed);
        if (qb_opt().verbose) fprintf(stderr, "[qb200] search rerun: device flags=0x%x, mode 0x%x -> 0x%x\n", flags, rs_flags, next);
        rs_flags = next;
    }
    s->n_searches.fetch_add(1, std::memory_order_relaxed);
    return QB_OK;
}

// ------------------------------------------------------------------------------------------------ RawScorer
static qb_status scorer_alloc(qb_storage* s, qb_scorer** out) {
    qb_scorer* sc = new qb_scorer();
    sc->st = s;
    if (cudaStreamCreateWithFlags(&sc->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete sc; qb_set_error("scorer: cudaStreamCreate failed"); return QB_ERR_CUDA;
    }
    sc->query_bytes = std::max<size_t>(qb_encoded_query_bytes(s), s->bq_row_bytes);
    if (cudaMalloc(&sc->d_query, std::max<size_t>(sc->query_bytes, 256)) != cudaSuccess || cudaMalloc(&sc->d_q_off, 256) != cudaSuccess) {
        qb_set_error("scorer: cudaMalloc failed"); qb_scorer_destroy(sc); return QB_ERR_OOM;
    }
    *out = sc;
    return QB_OK;
}

extern "C" qb_status qb_scorer_create(qb_storage* s, const float* query, qb_scorer** out) {
    QB_CHECK(s && query && out, QB_ERR_INVALID, "scorer_create: null argument");
    *out = nullptr;
    QB_TRY(use_device(s->device));
    qb_scorer* sc = nullptr;
    QB_TRY(scorer_alloc(s, &sc));
    float* d_raw = nullptr;
    const size_t raw = (size_t)s->dim * 4, pre = (size_t)pre_stride_f(s) * 4;
    if (cudaMalloc(&d_raw, raw + pre + 256) != cudaSuccess) { qb_scorer_destroy(sc); qb_set_error("scorer_create: cudaMalloc failed"); return QB_ERR_OOM; }
    cudaError_t e = cudaMemcpyAsync(d_raw, query, raw, cudaMemcpyHostToDevice, sc->stream);
    qb_status st = e == cudaSuccess ? prepare_queries(s, d_raw, 1, reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(d_raw) + round_up_u64(raw, 16)),
                                                      sc->d_query, sc->d_q_off, sc->stream)
                                    : QB_ERR_CUDA;
    if (st == QB_OK && cudaStreamSynchronize(sc->stream) != cudaSuccess) st = QB_ERR_CUDA;
    cudaFree(d_raw);
    if (st != QB_OK) { qb_set_error("scorer_create: %s", cudaGetErrorString(cudaGetLastError())); qb_scorer_destroy(sc); return st; }
    *out = sc;
    return QB_OK;
}

extern "C" qb_status qb_scorer_create_internal(qb_storage* s, uint32_t point_id, qb_scorer** out) {
    QB_CHECK(s && out, QB_ERR_INVALID, "scorer_create_internal: null argument");
    *out = nullptr;
    QB_TRY(localize_ids(s, &point_id, 1, &point_id, "scorer_create_internal"));
    QB_CHECK(s->kind != QB_KIND_PQ, QB_ERR_UNSUPPORTED, "PQ has no internal query encoding (encode_internal_vector = None, encoded_vectors_pq.rs:624-627)");
    QB_TRY(use_device(s->device));
    qb_scorer* sc = nullptr;
    QB_TRY(scorer_alloc(s, &sc));
    sc->internal = true; sc->internal_id = point_id;
    qb_status st = QB_OK;
    cudaError_t e = cudaSuccess;
    switch (s->kind) {
        case QB_KIND_DENSE:
            e = cudaMemcpyAsync(sc->d_query, reinterpret_cast<const uint8_t*>(s->d_rows) + (size_t)point_id * s->row_stride, s->row_stride,
                                cudaMemcpyDeviceToDevice, sc->stream);
            break;
        case QB_KIND_SQ8: st = qb_sq8_internal_query(s, point_id, reinterpret_cast<uint8_t*>(sc->d_query), sc->d_q_off, sc->stream); break;
        default:
            e = cudaMemcpyAsync(sc->d_query, s->d_bq_rows + (size_t)point_id * s->bq_row_bytes, s->bq_row_bytes, cudaMemcpyDeviceToDevice, sc->stream);
            break;
    }
    if (e != cudaSuccess) st = QB_ERR_CUDA;
    if (st == QB_OK && cudaStreamSynchronize(sc->stream) != cudaSuccess) st = QB_ERR_CUDA;
    if (st != QB_OK) { qb_set_error("scorer_create_internal: %s", cudaGetErrorString(cudaGetLastError())); qb_scorer_destroy(sc); return st; }
    *out = sc;
    return QB_OK;
}

static qb_status launch_example(const qb_storage* s, const void* d_enc, const float* d_q_off, uint32_t e, bool internal, const uint32_t* d_ids, uint64_t n,
                                float* d_scores, cudaStream_t stream);

static qb_status check_custom(qb_query_kind kind, uint32_t n_a, uint32_t n_b, uint32_t* n_examples) {
    QB_CHECK(kind >= QB_QUERY_RECO_BEST_SCORE && kind <= QB_QUERY_FEEDBACK_NAIVE, QB_ERR_INVALID, "custom query: unknown kind %d", (int)kind);
    QB_CHECK((kind != QB_QUERY_DISCOVER && kind != QB_QUERY_CONTEXT && kind != QB_QUERY_FEEDBACK_NAIVE) || n_b == 0, QB_ERR_INVALID, "custom query: n_b must be 0 for discover / context (n_a = pairs)");
    const uint32_t e = qb_custom_examples((int)kind, n_a, n_b);
    QB_CHECK(e >= 1 && e <= 4096, QB_ERR_INVALID, "custom query: %u example vectors (need 1..4096)", e);
    *n_examples = e;
    return QB_OK;
}

static qb_status scorer_create_custom_impl(qb_storage* s, qb_query_kind kind, const float* vectors, uint32_t n_a, uint32_t n_b, const float* coef, uint32_t n_coef,
                                           qb_scorer** out) {
    QB_CHECK(s && vectors && out, QB_ERR_INVALID, "scorer_create_custom: null argument");
    *out = nullptr;
    uint32_t ne = 0;
    QB_TRY(check_custom(kind, n_a, n_b, &ne));
    QB_TRY(use_device(s->device));
    qb_scorer* sc = new qb_scorer();
    sc->st = s;
    sc->custom_kind = (int)kind; sc->n_a = n_a; sc->n_b = n_b; sc->n_examples = ne;
    sc->query_bytes = (size_t)ne * qb_encoded_query_bytes(s);
    float* d_raw = nullptr;
    const size_t raw = round_up_u64((size_t)ne * s->dim * 4, 16), pre = (size_t)ne * pre_stride_f(s) * 4;
    qb_status st = QB_OK;
    if (cudaStreamCreateWithFlags(&sc->stream, cudaStreamNonBlocking) != cudaSuccess || cudaMalloc(&sc->d_query, sc->query_bytes + 256) != cudaSuccess ||
        cudaMalloc(&sc->d_q_off, (size_t)ne * 4 + 256) != cudaSuccess || cudaMalloc(&d_raw, raw + pre + 256) != cudaSuccess) {
        st = QB_ERR_OOM;
    } else if (cudaMemcpyAsync(d_raw, vectors, (size_t)ne * s->dim * 4, cudaMemcpyHostToDevice, sc->stream) != cudaSuccess) {
        st = QB_ERR_CUDA;
    } else {
        st = prepare_queries(s, d_raw, ne, reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(d_raw) + raw), sc->d_query, sc->d_q_off, sc->stream);
        if (st == QB_OK && n_coef) {
            if (cudaMalloc(&sc->d_coef, (size_t)n_coef * 4 + 256) != cudaSuccess) st = QB_ERR_OOM;
            else if (cudaMemcpyAsync(sc->d_coef, coef, (size_t)n_coef * 4, cudaMemcpyHostToDevice, sc->stream) != cudaSuccess) st = QB_ERR_CUDA;
        }
        if (st == QB_OK && cudaStreamSynchronize(sc->stream) != cudaSuccess) st = QB_ERR_CUDA;
    }
    cudaFree(d_raw);
    if (st != QB_OK) { qb_set_error("scorer_create_custom: %s", cudaGetErrorString(cudaGetLastError())); qb_scorer_destroy(sc); return st; }
    *out = sc;
    return QB_OK;
}

extern "C" qb_status qb_scorer_create_custom(qb_storage* s, qb_query_kind kind, const float* vectors, uint32_t n_a, uint32_t n_b, qb_scorer** out) {
    QB_CHECK(kind != QB_QUERY_FEEDBACK_NAIVE, QB_ERR_INVALID, "scorer_create_custom: feedback queries carry coefficients, use qb_scorer_create_feedback");
    return scorer_create_custom_impl(s, kind, vectors, n_a, n_b, nullptr, 0, out);
}

// [a, partial_computation...] as one host array
static std::vector<float> feedback_coef(float a, const float* partial, uint32_t n_pairs) {
    std::vector<float> c(1 + n_pairs);
    c[0] = a;
    for (uint32_t i = 0; i < n_pairs; ++i) c[1 + i] = partial[i];
    return c;
}

extern "C" qb_status qb_scorer_create_feedback(qb_storage* s, const float* vectors, uint32_t n_pairs, float a, const float* partial, qb_scorer** out) {
    QB_CHECK(n_pairs == 0 || partial, QB_ERR_INVALID, "scorer_create_feedback: null partial computations");
    const std::vector<float> c = feedback_coef(a, partial, n_pairs);
    return scorer_create_custom_impl(s, QB_QUERY_FEEDBACK_NAIVE, vectors, n_pairs, 0, c.data(), (uint32_t)c.size(), out);
}

static qb_status search_custom_impl(qb_storage* s, qb_query_kind kind, const float* vectors, uint32_t n_a, uint32_t n_b, const float* coef, uint32_t n_coef, uint32_t top,
                                    const uint64_t* deleted_bitmap, const uint32_t* id_list, uint64_t n_ids, const volatile int32_t* is_stopped,
                                    qb_scored_point* out, uint32_t* out_count, qb_hw_counters* counters) {
    QB_CHECK(s && vectors && out && out_count, QB_ERR_INVALID, "search_custom: null argument");
    QB_CHECK(top >= 1 && top <= QB_MAX_TOP, QB_ERR_INVALID, "search_custom: top %u outside [1,%u]", top, QB_MAX_TOP);
    uint32_t ne = 0;
    QB_TRY(check_custom(kind, n_a, n_b, &ne));
    const uint64_t n = id_list ? n_ids : s->count;
    *out_count = 0;
    if (n == 0) return QB_OK;
    // dense f32 scans with up to 16 example vectors fold inside the streaming kernel (rows read once, no similarity matrix);
    // otherwise every candidate needs its similarity to every example before the fold: E x n floats + n keys of scratch
    const bool try_fold = !id_list && s->kind == QB_KIND_DENSE && s->dtype == QB_DT_F32 && s->dim >= 32 && ne <= 16 && n >= 1024;
    QB_CHECK(try_fold || n * (12ull + 4ull * ne) <= (16ull << 30), QB_ERR_UNSUPPORTED, "search_custom: %llu candidates x %u examples exceed the 16 GB scratch budget",
             (unsigned long long)n, ne);
    if (is_stopped && *is_stopped) { qb_set_error("search cancelled"); return QB_ERR_CANCELLED; }
    QB_TRY(use_device(s->device));
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_acquire(s, &c));
    struct Rel { qb_storage* s; QbSearchCtx* c; ~Rel() { qb_ctx_release(s, c); } } rel{s, c};
    cudaStream_t stream = c->stream;
    const size_t raw_bytes = (size_t)ne * s->dim * 4, res_bytes = (size_t)top * sizeof(qb_scored_point);
    const size_t ids_off = round_up_u64(raw_bytes + res_bytes + 16, 16);
    QB_TRY(qb_ensure_pinned(&c->h_stage, &c->h_stage_bytes, ids_off + (id_list ? n_ids * 4 : 0)));
    uint8_t* hs = reinterpret_cast<uint8_t*>(c->h_stage);
    memcpy(hs, vectors, raw_bytes);
    if (id_list) QB_TRY(localize_ids(s, id_list, n_ids, reinterpret_cast<uint32_t*>(hs + ids_off), "search_custom"));
    QB_TRY(qb_ensure_device(&c->d_queries_raw, &c->queries_raw_bytes, round_up_u64(raw_bytes, 16) + (size_t)ne * pre_stride_f(s) * 4));
    QB_TRY(qb_ensure_device(&c->d_queries_enc, &c->queries_enc_bytes, ((size_t)ne + 256) * qb_encoded_query_bytes(s)));
    QB_TRY(ensure_dev_elems(&c->d_q_off, &c->q_off_elems, (size_t)ne));
    QB_TRY(ensure_dev_elems(&c->d_out, &c->out_elems, (size_t)top));
    QB_TRY(ensure_dev_elems(&c->d_out_counts, &c->out_counts_elems, (size_t)8));
    QB_TRY(ensure_dev_elems(&c->d_cand, &c->cand_elems, (size_t)n));
    QB_TRY(ensure_dev_elems(&c->d_thr, &c->thr_elems, (size_t)n_coef + 64));
    QB_CUDA(cudaMemcpyAsync(c->d_queries_raw, hs, raw_bytes, cudaMemcpyHostToDevice, stream));
    QB_TRY(prepare_queries(s, reinterpret_cast<const float*>(c->d_queries_raw), ne,
                           reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(c->d_queries_raw) + round_up_u64(raw_bytes, 16)), c->d_queries_enc, c->d_q_off, stream));
    const uint32_t* d_del2 = nullptr;
    if (deleted_bitmap) {
        const size_t words64 = (size_t)ceil_div_u64(s->count, 64);
        QB_TRY(ensure_dev_elems(&c->d_deleted2, &c->deleted2_words, words64 * 2));
        QB_CUDA(cudaMemcpyAsync(c->d_deleted2, deleted_bitmap, words64 * 8, cudaMemcpyHostToDevice, stream));
        d_del2 = c->d_deleted2;
    }
    QbEmit emit{};
    emit.cand = c->d_cand; emit.cap = n; emit.dense = 1; emit.dense_base = 0; emit.deleted = s->d_deleted; emit.deleted2 = d_del2; emit.id_base = s->id_base;
    const float* d_coef = nullptr;
    if (n_coef) {
        QB_CUDA(cudaMemcpyAsync(c->d_thr, coef, (size_t)n_coef * 4, cudaMemcpyHostToDevice, stream));
        d_coef = c->d_thr;
    }
    bool folded = false;
    if (try_fold) {
        QbScanArgs a{};
        a.d_q_enc = c->d_queries_enc; a.nq = ne; a.row_begin = 0; a.row_end = n; a.emit = emit;
        QB_TRY(qb_dense_f32_scan_fold(s, a, (int)kind, n_a, n_b, d_coef, &folded, stream));
    }
    if (!folded) {
        QB_CHECK(n * (12ull + 4ull * ne) <= (16ull << 30), QB_ERR_UNSUPPORTED, "search_custom: %llu candidates x %u examples exceed the 16 GB scratch budget",
                 (unsigned long long)n, ne);
        QB_TRY(ensure_dev_elems(&c->d_ids, &c->ids_elems, (size_t)n));
        QB_TRY(qb_ensure_device(&c->d_mma, &c->mma_bytes, (size_t)ne * n * 4 + 256));
        if (id_list) QB_CUDA(cudaMemcpyAsync(c->d_ids, hs + ids_off, n * 4, cudaMemcpyHostToDevice, stream));
        else QB_TRY(qb_launch_iota(c->d_ids, n, stream));
        float* d_sims = reinterpret_cast<float*>(c->d_mma);
        for (uint32_t e = 0; e < ne; ++e) {
            if (is_stopped && *is_stopped) { qb_set_error("search cancelled"); return QB_ERR_CANCELLED; }
            QB_TRY(launch_example(s, c->d_queries_enc, c->d_q_off, e, false, c->d_ids, n, d_sims + (size_t)e * n, stream));
        }
        QB_TRY(qb_launch_custom_combine((int)kind, n_a, n_b, d_coef, d_sims, n, n, nullptr, c->d_ids, &emit, stream));
    }
    QB_TRY(qb_launch_select(c->d_cand, nullptr, n, n, 1, top, 0, c->d_out, c->d_out_counts, nullptr, nullptr, stream));
    QB_CUDA(cudaMemcpyAsync(hs + raw_bytes, c->d_out, res_bytes, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaMemcpyAsync(hs + raw_bytes + res_bytes, c->d_out_counts, 4, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaStreamSynchronize(stream));
    memcpy(out, hs + raw_bytes, res_bytes);
    memcpy(out_count, hs + raw_bytes + res_bytes, 4);
    if (counters) { counters->cpu += n * (uint64_t)ne * cpu_units_per_point(s); counters->vector_io_read += n * (uint64_t)ne * io_units_per_point(s); }
    return QB_OK;
}

extern "C" qb_status qb_search_custom(qb_storage* s, qb_query_kind kind, const float* vectors, uint32_t n_a, uint32_t n_b, uint32_t top,
                                      const uint64_t* deleted_bitmap, const uint32_t* id_list, uint64_t n_ids, const volatile int32_t* is_stopped,
                                      qb_scored_point* out, uint32_t* out_count, qb_hw_counters* counters) {
    QB_CHECK(kind != QB_QUERY_FEEDBACK_NAIVE, QB_ERR_INVALID, "search_custom: feedback queries carry coefficients, use qb_search_feedback");
    return search_custom_impl(s, kind, vectors, n_a, n_b, nullptr, 0, top, deleted_bitmap, id_list, n_ids, is_stopped, out, out_count, counters);
}

extern "C" qb_status qb_search_feedback(qb_storage* s, const float* vectors, uint32_t n_pairs, float a, const float* partial, uint32_t top,
                                        const uint64_t* deleted_bitmap, const uint32_t* id_list, uint64_t n_ids, const volatile int32_t* is_stopped,
                                        qb_scored_point* out, uint32_t* out_count, qb_hw_counters* counters) {
    QB_CHECK(n_pairs == 0 || partial, QB_ERR_INVALID, "search_feedback: null partial computations");
    const std::vector<float> c = feedback_coef(a, partial, n_pairs);
    return search_custom_impl(s, QB_QUERY_FEEDBACK_NAIVE, vectors, n_pairs, 0, c.data(), (uint32_t)c.size(), top, deleted_bitmap, id_list, n_ids, is_stopped, out,
                              out_count, counters);
}

// ------------------------------------------------------------------------------------------------ multivector MaxSim
// Shared body of qb_search_maxsim / qb_score_maxsim.  point_ids = null: every point (search); else the listed points (scores).
static qb_status maxsim_run(qb_storage* s, const uint32_t* point_offsets, uint32_t n_points, const float* query_tokens, uint32_t nqt, const uint32_t* point_ids,
                            uint64_t n_sel, const uint64_t* deleted_points, uint32_t top, qb_scored_point* out, uint32_t* out_count, float* scores,
                            qb_hw_counters* counters) {
    QB_CHECK(s && point_offsets && query_tokens, QB_ERR_INVALID, "maxsim: null argument");
    QB_CHECK(nqt >= 1 && nqt <= 4096, QB_ERR_INVALID, "maxsim: %u query vectors (need 1..4096)", nqt);
    for (uint32_t p = 0; p < n_points; ++p) QB_CHECK(point_offsets[p] <= point_offsets[p + 1], QB_ERR_INVALID, "maxsim: point_offsets not ascending at %u", p);
    QB_CHECK(n_points == 0 || point_offsets[n_points] <= s->count, QB_ERR_INVALID, "maxsim: point_offsets end %u beyond the %llu stored vectors",
             n_points ? point_offsets[n_points] : 0u, (unsigned long long)s->count);
    const uint64_t n_pts = point_ids ? n_sel : n_points;
    if (n_pts == 0) return QB_OK;
    // rows to score and, per selected point, its column range in the similarity matrix
    std::vector<uint32_t> h_off(n_pts + 1), h_rows;
    uint64_t n_rows;
    if (point_ids) {
        uint64_t acc = 0;
        for (uint64_t i = 0; i < n_pts; ++i) {
            QB_CHECK(point_ids[i] < n_points, QB_ERR_INVALID, "maxsim: point id %u out of range", point_ids[i]);
            h_off[i] = (uint32_t)acc;
            for (uint32_t r = point_offsets[point_ids[i]]; r < point_offsets[point_ids[i] + 1]; ++r) h_rows.push_back(r);
            acc = h_rows.size();
        }
        h_off[n_pts] = (uint32_t)acc;
        n_rows = acc;
    } else {
        for (uint64_t i = 0; i <= n_pts; ++i) h_off[i] = point_offsets[i];
        n_rows = point_offsets[n_points];
    }
    QB_CHECK(n_rows * (4ull * nqt + 4) + n_pts * 20 <= (16ull << 30), QB_ERR_UNSUPPORTED, "maxsim: %llu vectors x %u query vectors exceed the 16 GB scratch budget",
             (unsigned long long)n_rows, nqt);
    QB_TRY(use_device(s->device));
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_acquire(s, &c));
    struct Rel { qb_storage* s; QbSearchCtx* c; ~Rel() { qb_ctx_release(s, c); } } rel{s, c};
    cudaStream_t stream = c->stream;
    const size_t raw_bytes = (size_t)nqt * s->dim * 4;
    const size_t res_bytes = scores ? (size_t)n_pts * 4 : (size_t)top * sizeof(qb_scored_point);
    QB_TRY(qb_ensure_pinned(&c->h_stage, &c->h_stage_bytes, raw_bytes + res_bytes + 16));
    uint8_t* hs = reinterpret_cast<uint8_t*>(c->h_stage);
    memcpy(hs, query_tokens, raw_bytes);
    QB_TRY(qb_ensure_device(&c->d_queries_raw, &c->queries_raw_bytes, round_up_u64(raw_bytes, 16) + (size_t)nqt * pre_stride_f(s) * 4));
    QB_TRY(qb_ensure_device(&c->d_queries_enc, &c->queries_enc_bytes, ((size_t)nqt + 256) * qb_encoded_query_bytes(s)));
    QB_TRY(ensure_dev_elems(&c->d_q_off, &c->q_off_elems, (size_t)nqt));
    QB_TRY(ensure_dev_elems(&c->d_ids, &c->ids_elems, (size_t)std::max<uint64_t>(n_rows, 1)));
    // scratch: [similarities nqt x n_rows][column offsets n_pts + 1][point ids n_pts][scores n_pts]
    const size_t sims_bytes = round_up_u64((size_t)nqt * n_rows * 4, 256), off_bytes = round_up_u64((n_pts + 1) * 4, 256), pid_bytes = round_up_u64(n_pts * 4, 256);
    QB_TRY(qb_ensure_device(&c->d_mma, &c->mma_bytes, sims_bytes + off_bytes + pid_bytes + n_pts * 4 + 256));
    uint8_t* sc = reinterpret_cast<uint8_t*>(c->d_mma);
    float* d_sims = reinterpret_cast<float*>(sc);
    uint32_t* d_off = reinterpret_cast<uint32_t*>(sc + sims_bytes);
    uint32_t* d_pid = reinterpret_cast<uint32_t*>(sc + sims_bytes + off_bytes);
    float* d_scores = reinterpret_cast<float*>(sc + sims_bytes + off_bytes + pid_bytes);
    QB_CUDA(cudaMemcpyAsync(c->d_queries_raw, hs, raw_bytes, cudaMemcpyHostToDevice, stream));
    QB_TRY(prepare_queries(s, reinterpret_cast<const float*>(c->d_queries_raw), nqt,
                           reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(c->d_queries_raw) + round_up_u64(raw_bytes, 16)), c->d_queries_enc, c->d_q_off, stream));
    QB_CUDA(cudaMemcpyAsync(d_off, h_off.data(), (n_pts + 1) * 4, cudaMemcpyHostToDevice, stream));
    if (point_ids) {
        QB_CUDA(cudaMemcpyAsync(d_pid, point_ids, n_pts * 4, cudaMemcpyHostToDevice, stream));
        if (n_rows) QB_CUDA(cudaMemcpyAsync(c->d_ids, h_rows.data(), n_rows * 4, cudaMemcpyHostToDevice, stream));
    } else {
        QB_TRY(qb_launch_iota(c->d_ids, n_rows, stream));
    }
    for (uint32_t e = 0; e < nqt && n_rows; ++e) QB_TRY(launch_example(s, c->d_queries_enc, c->d_q_off, e, false, c->d_ids, n_rows, d_sims + (size_t)e * n_rows, stream));
    if (scores) {
        QB_TRY(qb_launch_maxsim_fold(d_sims, n_rows, nqt, d_off, nullptr, n_pts, d_scores, nullptr, stream));
        QB_CUDA(cudaMemcpyAsync(hs + raw_bytes, d_scores, n_pts * 4, cudaMemcpyDeviceToHost, stream));
        QB_CUDA(cudaStreamSynchronize(stream));  // also orders the reads of h_off / h_rows / point_ids before they go out of scope
        memcpy(scores, hs + raw_bytes, n_pts * 4);
    } else {
        const uint32_t* d_del2 = nullptr;
        if (deleted_points) {
            const size_t words64 = (size_t)ceil_div_u64(n_points, 64);
            QB_TRY(ensure_dev_elems(&c->d_deleted2, &c->deleted2_words, words64 * 2));
            QB_CUDA(cudaMemcpyAsync(c->d_deleted2, deleted_points, words64 * 8, cudaMemcpyHostToDevice, stream));
            d_del2 = c->d_deleted2;
        }
        QB_TRY(ensure_dev_elems(&c->d_cand, &c->cand_elems, (size_t)n_pts));
        QB_TRY(ensure_dev_elems(&c->d_out, &c->out_elems, (size_t)top));
        QB_TRY(ensure_dev_elems(&c->d_out_counts, &c->out_counts_elems, (size_t)8));
        QbEmit emit{};
        emit.cand = c->d_cand; emit.cap = n_pts; emit.dense = 1; emit.dense_base = 0; emit.deleted = nullptr; emit.deleted2 = d_del2; emit.id_base = 0;
        QB_TRY(qb_launch_maxsim_fold(d_sims, n_rows, nqt, d_off, nullptr, n_pts, nullptr, &emit, stream));
        QB_TRY(qb_launch_select(c->d_cand, nullptr, n_pts, n_pts, 1, top, 0, c->d_out, c->d_out_counts, nullptr, nullptr, stream));
        QB_CUDA(cudaMemcpyAsync(hs + raw_bytes, c->d_out, res_bytes, cudaMemcpyDeviceToHost, stream));
        QB_CUDA(cudaMemcpyAsync(hs + raw_bytes + res_bytes, c->d_out_counts, 4, cudaMemcpyDeviceToHost, stream));
        QB_CUDA(cudaStreamSynchronize(stream));
        memcpy(out, hs + raw_bytes, res_bytes);
        memcpy(out_count, hs + raw_bytes + res_bytes, 4);
    }
    if (counters) counters->cpu += n_rows * (uint64_t)nqt * cpu_units_per_point(s);
    return QB_OK;
}

extern "C" qb_status qb_search_maxsim(qb_storage* s, const uint32_t* point_offsets, uint32_t n_points, const float* query_vectors, uint32_t n_query_vectors,
                                      uint32_t top, const uint64_t* deleted_points, qb_scored_point* out, uint32_t* out_count, qb_hw_counters* counters) {
    QB_CHECK(out && out_count, QB_ERR_INVALID, "search_maxsim: null output");
    QB_CHECK(top >= 1 && top <= QB_MAX_TOP, QB_ERR_INVALID, "search_maxsim: top %u outside [1,%u]", top, QB_MAX_TOP);
    *out_count = 0;
    return maxsim_run(s, point_offsets, n_points, query_vectors, n_query_vectors, nullptr, 0, deleted_points, top, out, out_count, nullptr, counters);
}

extern "C" qb_status qb_score_maxsim(qb_storage* s, const uint32_t* point_offsets, uint32_t n_points, const float* query_vectors, uint32_t n_query_vectors,
                                     const uint32_t* point_ids, size_t n, float* scores) {
    QB_CHECK(n == 0 || (point_ids && scores), QB_ERR_INVALID, "score_maxsim: null argument");
    if (n == 0) return QB_OK;
    return maxsim_run(s, point_offsets, n_points, query_vectors, n_query_vectors, point_ids, n, nullptr, 0, nullptr, nullptr, scores, nullptr);
}

// MultiCustomQueryScorer (query_scorer/multi_custom_query_scorer.rs:88-104) / QuantizedMultiCustomQueryScorer: a custom query whose
// examples are MULTIVECTORS; a point's similarity to an example is MaxSim (score_multi -> score_max_similarity), the per-example
// similarities are folded by Query::score_by exactly like the single-vector custom queries.
static qb_status maxsim_custom_run(qb_storage* s, const uint32_t* point_offsets, uint32_t n_points, qb_query_kind kind, const float* example_vectors,
                                   const uint32_t* example_offsets, uint32_t n_a, uint32_t n_b, const float* coef, const uint32_t* point_ids, uint64_t n_sel,
                                   const uint64_t* deleted_points, uint32_t top, qb_scored_point* out, uint32_t* out_count, float* scores, qb_hw_counters* counters) {
    QB_CHECK(s && point_offsets && example_vectors && example_offsets, QB_ERR_INVALID, "maxsim_custom: null argument");
    uint32_t ne = 0;
    QB_TRY(check_custom(kind, n_a, n_b, &ne));
    QB_CHECK(kind != QB_QUERY_FEEDBACK_NAIVE || coef, QB_ERR_INVALID, "maxsim_custom: feedback queries need [a, partial computations]");
    for (uint32_t e = 0; e < ne; ++e) QB_CHECK(example_offsets[e] < example_offsets[e + 1], QB_ERR_INVALID, "maxsim_custom: example %u has no vectors", e);
    for (uint32_t p = 0; p < n_points; ++p) QB_CHECK(point_offsets[p] <= point_offsets[p + 1], QB_ERR_INVALID, "maxsim_custom: point_offsets not ascending at %u", p);
    QB_CHECK(n_points == 0 || point_offsets[n_points] <= s->count, QB_ERR_INVALID, "maxsim_custom: point_offsets end beyond the stored vectors");
    const uint64_t n_pts = point_ids ? n_sel : n_points;
    if (n_pts == 0) return QB_OK;
    std::vector<uint32_t> h_off(n_pts + 1), h_rows;
    uint64_t n_rows;
    if (point_ids) {
        uint64_t acc = 0;
        for (uint64_t i = 0; i < n_pts; ++i) {
            QB_CHECK(point_ids[i] < n_points, QB_ERR_INVALID, "maxsim_custom: point id %u out of range", point_ids[i]);
            h_off[i] = (uint32_t)acc;
            for (uint32_t r = point_offsets[point_ids[i]]; r < point_offsets[point_ids[i] + 1]; ++r) h_rows.push_back(r);
            acc = h_rows.size();
        }
        h_off[n_pts] = (uint32_t)acc;
        n_rows = acc;
    } else {
        for (uint64_t i = 0; i <= n_pts; ++i) h_off[i] = point_offsets[i];
        n_rows = point_offsets[n_points];
    }
    uint32_t max_tok = 0;
    const uint32_t total_tok = example_offsets[ne];
    for (uint32_t e = 0; e < ne; ++e) max_tok = std::max(max_tok, example_offsets[e + 1] - example_offsets[e]);
    QB_CHECK(max_tok <= 4096, QB_ERR_INVALID, "maxsim_custom: %u vectors in one example (max 4096)", max_tok);
    QB_CHECK(n_rows * (4ull * max_tok + 4) + n_pts * (4ull * ne + 20) <= (16ull << 30), QB_ERR_UNSUPPORTED, "maxsim_custom: scratch budget exceeded");
    QB_TRY(use_device(s->device));
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_acquire(s, &c));
    struct Rel { qb_storage* s; QbSearchCtx* c; ~Rel() { qb_ctx_release(s, c); } } rel{s, c};
    cudaStream_t stream = c->stream;
    const uint32_t n_coef = (kind == QB_QUERY_FEEDBACK_NAIVE) ? 1 + n_a : 0;
    const size_t raw_bytes = (size_t)total_tok * s->dim * 4;
    const size_t res_bytes = scores ? (size_t)n_pts * 4 : (size_t)top * sizeof(qb_scored_point);
    QB_TRY(qb_ensure_pinned(&c->h_stage, &c->h_stage_bytes, raw_bytes + res_bytes + (size_t)n_coef * 4 + 16));
    uint8_t* hs = reinterpret_cast<uint8_t*>(c->h_stage);
    memcpy(hs, example_vectors, raw_bytes);
    if (n_coef) memcpy(hs + raw_bytes + res_bytes, coef, (size_t)n_coef * 4);
    QB_TRY(qb_ensure_device(&c->d_queries_raw, &c->queries_raw_bytes, round_up_u64(raw_bytes, 16) + (size_t)total_tok * pre_stride_f(s) * 4));
    QB_TRY(qb_ensure_device(&c->d_queries_enc, &c->queries_enc_bytes, ((size_t)total_tok + 256) * qb_encoded_query_bytes(s)));
    QB_TRY(ensure_dev_elems(&c->d_q_off, &c->q_off_elems, (size_t)total_tok));
    QB_TRY(ensure_dev_elems(&c->d_ids, &c->ids_elems, (size_t)std::max<uint64_t>(n_rows, 1)));
    QB_TRY(ensure_dev_elems(&c->d_thr, &c->thr_elems, (size_t)n_coef + 64));
    // scratch: [token similarities max_tok x n_rows][per-example MaxSim ne x n_pts][column offsets n_pts + 1][final scores n_pts]
    const size_t sims_bytes = round_up_u64((size_t)max_tok * n_rows * 4, 256), ex_bytes = round_up_u64((size_t)ne * n_pts * 4, 256), off_bytes = round_up_u64((n_pts + 1) * 4, 256);
    QB_TRY(qb_ensure_device(&c->d_mma, &c->mma_bytes, sims_bytes + ex_bytes + off_bytes + n_pts * 4 + 256));
    uint8_t* sc = reinterpret_cast<uint8_t*>(c->d_mma);
    float* d_sims = reinterpret_cast<float*>(sc);
    float* d_ex = reinterpret_cast<float*>(sc + sims_bytes);
    uint32_t* d_off = reinterpret_cast<uint32_t*>(sc + sims_bytes + ex_bytes);
    float* d_scores = reinterpret_cast<float*>(sc + sims_bytes + ex_bytes + off_bytes);
    QB_CUDA(cudaMemcpyAsync(c->d_queries_raw, hs, raw_bytes, cudaMemcpyHostToDevice, stream));
    QB_TRY(prepare_queries(s, reinterpret_cast<const float*>(c->d_queries_raw), total_tok,
                           reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(c->d_queries_raw) + round_up_u64(raw_bytes, 16)), c->d_queries_enc, c->d_q_off, stream));
    QB_CUDA(cudaMemcpyAsync(d_off, h_off.data(), (n_pts + 1) * 4, cudaMemcpyHostToDevice, stream));
    if (point_ids) { if (n_rows) QB_CUDA(cudaMemcpyAsync(c->d_ids, h_rows.data(), n_rows * 4, cudaMemcpyHostToDevice, stream)); }
    else QB_TRY(qb_launch_iota(c->d_ids, n_rows, stream));
    const float* d_coef = nullptr;
    if (n_coef) { QB_CUDA(cudaMemcpyAsync(c->d_thr, hs + raw_bytes + res_bytes, (size_t)n_coef * 4, cudaMemcpyHostToDevice, stream)); d_coef = c->d_thr; }
    for (uint32_t e = 0; e < ne; ++e) {
        const uint32_t t0 = example_offsets[e], nt = example_offsets[e + 1] - t0;
        for (uint32_t t = 0; t < nt && n_rows; ++t) QB_TRY(launch_example(s, c->d_queries_enc, c->d_q_off, t0 + t, false, c->d_ids, n_rows, d_sims + (size_t)t * n_rows, stream));
        QB_TRY(qb_launch_maxsim_fold(d_sims, n_rows, nt, d_off, nullptr, n_pts, d_ex + (size_t)e * n_pts, nullptr, stream));
    }
    if (scores) {
        QB_TRY(qb_launch_custom_combine((int)kind, n_a, n_b, d_coef, d_ex, n_pts, n_pts, d_scores, nullptr, nullptr, stream));
        QB_CUDA(cudaMemcpyAsync(hs + raw_bytes, d_scores, n_pts * 4, cudaMemcpyDeviceToHost, stream));
        QB_CUDA(cudaStreamSynchronize(stream));
        memcpy(scores, hs + raw_bytes, n_pts * 4);
    } else {
        const uint32_t* d_del2 = nullptr;
        if (deleted_points) {
            const size_t words64 = (size_t)ceil_div_u64(n_points, 64);
            QB_TRY(ensure_dev_elems(&c->d_deleted2, &c->deleted2_words, words64 * 2));
            QB_CUDA(cudaMemcpyAsync(c->d_deleted2, deleted_points, words64 * 8, cudaMemcpyHostToDevice, stream));
            d_del2 = c->d_deleted2;
        }
        QB_TRY(ensure_dev_elems(&c->d_cand, &c->cand_elems, (size_t)n_pts));
        QB_TRY(ensure_dev_elems(&c->d_out, &c->out_elems, (size_t)top));
        QB_TRY(ensure_dev_elems(&c->d_out_counts, &c->out_counts_elems, (size_t)8));
        QbEmit emit{};
        emit.cand = c->d_cand; emit.cap = n_pts; emit.dense = 1; emit.dense_base = 0; emit.deleted = nullptr; emit.deleted2 = d_del2; emit.id_base = 0;
        QB_TRY(qb_launch_custom_combine((int)kind, n_a, n_b, d_coef, d_ex, n_pts, n_pts, nullptr, nullptr, &emit, stream));
        QB_TRY(qb_launch_select(c->d_cand, nullptr, n_pts, n_pts, 1, top, 0, c->d_out, c->d_out_counts, nullptr, nullptr, stream));
        QB_CUDA(cudaMemcpyAsync(hs + raw_bytes, c->d_out, res_bytes, cudaMemcpyDeviceToHost, stream));
        QB_CUDA(cudaMemcpyAsync(hs + raw_bytes + res_bytes + (size_t)n_coef * 4, c->d_out_counts, 4, cudaMemcpyDeviceToHost, stream));
        QB_CUDA(cudaStreamSynchronize(stream));
        memcpy(out, hs + raw_bytes, res_bytes);
        memcpy(out_count, hs + raw_bytes + res_bytes + (size_t)n_coef * 4, 4);
    }
    if (counters) { counters->cpu += n_rows * (uint64_t)total_tok * cpu_units_per_point(s); counters->vector_io_read += n_rows * (uint64_t)ne * (s->on_disk ? 1 : 0); }
    return QB_OK;
}

extern "C" qb_status qb_search_maxsim_custom(qb_storage* s, const uint32_t* point_offsets, uint32_t n_points, qb_query_kind kind, const float* example_vectors,
                                             const uint32_t* example_offsets, uint32_t n_a, uint32_t n_b, const float* coef, uint32_t top, const uint64_t* deleted_points,
                                             qb_scored_point* out, uint32_t* out_count, qb_hw_counters* counters) {
    QB_CHECK(out && out_count, QB_ERR_INVALID, "search_maxsim_custom: null output");
    QB_CHECK(top >= 1 && top <= QB_MAX_TOP, QB_ERR_INVALID, "search_maxsim_custom: top %u outside [1,%u]", top, QB_MAX_TOP);
    *out_count = 0;
    return maxsim_custom_run(s, point_offsets, n_points, kind, example_vectors, example_offsets, n_a, n_b, coef, nullptr, 0, deleted_points, top, out, out_count, nullptr, counters);
}

extern "C" qb_status qb_score_maxsim_custom(qb_storage* s, const uint32_t* point_offsets, uint32_t n_points, qb_query_kind kind, const float* example_vectors,
                                            const uint32_t* example_offsets, uint32_t n_a, uint32_t n_b, const float* coef, const uint32_t* point_ids, size_t n, float* scores) {
    QB_CHECK(n == 0 || (point_ids && scores), QB_ERR_INVALID, "score_maxsim_custom: null argument");
    if (n == 0) return QB_OK;
    return maxsim_custom_run(s, point_offsets, n_points, kind, example_vectors, example_offsets, n_a, n_b, coef, point_ids, n, nullptr, 0, nullptr, nullptr, scores, nullptr);
}

extern "C" void qb_scorer_destroy(qb_scorer* sc) {
    if (!sc) return;
    cudaSetDevice(sc->st->device);
    if (sc->stream) cudaStreamSynchronize(sc->stream);
    cudaFree(sc->d_query); cudaFree(sc->d_q_off); cudaFree(sc->d_ids); cudaFree(sc->d_scores); cudaFree(sc->d_sims); cudaFree(sc->d_coef);
    if (sc->h_ids) cudaFreeHost(sc->h_ids);
    if (sc->h_scores) cudaFreeHost(sc->h_scores);
    if (sc->stream) cudaStreamDestroy(sc->stream);
    cudaGetLastError();
    delete sc;
}

static qb_status scorer_reserve(qb_scorer* sc, size_t n) {
    if (n <= sc->cap) return QB_OK;
    size_t cap = std::max<size_t>(n, 256);
    cap = round_up_u64(cap, 256);
    cudaFree(sc->d_ids); cudaFree(sc->d_scores);
    if (sc->h_ids) cudaFreeHost(sc->h_ids);
    if (sc->h_scores) cudaFreeHost(sc->h_scores);
    sc->d_ids = nullptr; sc->d_scores = nullptr; sc->h_ids = nullptr; sc->h_scores = nullptr; sc->cap = 0;
    QB_CUDA(cudaMalloc(&sc->d_ids, cap * 4));
    QB_CUDA(cudaMalloc(&sc->d_scores, cap * 4));
    // pinned AND mapped: small batches (an HNSW hop is <= 32 ids) are read / written by the kernel straight through PCIe, which
    // leaves one launch and one synchronisation per call instead of two copies around them
    QB_CUDA(cudaHostAlloc(&sc->h_ids, cap * 4, cudaHostAllocMapped));
    QB_CUDA(cudaHostAlloc(&sc->h_scores, cap * 4, cudaHostAllocMapped));
    QB_CUDA(cudaHostGetDevicePointer(&sc->m_ids, sc->h_ids, 0));
    QB_CUDA(cudaHostGetDevicePointer(&sc->m_scores, sc->h_scores, 0));
    sc->cap = cap;
    return QB_OK;
}

// similarities of `n` ids to encoded query `e` of a buffer of encoded queries
static qb_status launch_example(const qb_storage* s, const void* d_enc, const float* d_q_off, uint32_t e, bool internal, const uint32_t* d_ids, uint64_t n,
                                float* d_scores, cudaStream_t stream) {
    const void* q = reinterpret_cast<const uint8_t*>(d_enc) + (size_t)e * qb_encoded_query_bytes(s);
    if (s->kind == QB_KIND_BQ) {
        const int bits = internal ? 1 : (s->bq_qenc == QB_BQQ_SCALAR4 ? 4 : (s->bq_qenc == QB_BQQ_SCALAR8 ? 8 : 1));
        return qb_bq_score_points(s, q, bits, d_ids, n, d_scores, stream);
    }
    return qb_launch_score_points(s, q, d_q_off ? d_q_off + e : nullptr, d_ids, n, d_scores, stream);
}

static qb_status scorer_launch(qb_scorer* sc, const uint32_t* d_ids, uint64_t n, float* d_scores) {
    qb_storage* s = sc->st;
    if (!sc->custom_kind) return launch_example(s, sc->d_query, sc->d_q_off, 0, sc->internal, d_ids, n, d_scores, sc->stream);
    // custom query: one launch per example vector, then Query::score_by per candidate
    if (n > sc->sims_cap) {
        cudaFree(sc->d_sims); sc->d_sims = nullptr; sc->sims_cap = 0;
        const size_t cap = round_up_u64(std::max<uint64_t>(n, 256), 256);
        QB_CUDA(cudaMalloc(&sc->d_sims, (size_t)sc->n_examples * cap * 4));
        sc->sims_cap = cap;
    }
    for (uint32_t e = 0; e < sc->n_examples; ++e)
        QB_TRY(launch_example(s, sc->d_query, sc->d_q_off, e, false, d_ids, n, sc->d_sims + (size_t)e * sc->sims_cap, sc->stream));
    return qb_launch_custom_combine(sc->custom_kind, sc->n_a, sc->n_b, sc->d_coef, sc->d_sims, sc->sims_cap, n, d_scores, nullptr, nullptr, sc->stream);
}

extern "C" qb_status qb_score_points(qb_scorer* sc, const uint32_t* ids, size_t n, float* scores) {
    QB_CHECK(sc && (n == 0 || (ids && scores)), QB_ERR_INVALID, "score_points: null argument");
    if (n == 0) return QB_OK;
    qb_storage* s = sc->st;
    QB_TRY(use_device(s->device));
    QB_TRY(scorer_reserve(sc, n));
    QB_TRY(localize_ids(s, ids, n, sc->h_ids, "score_points"));
    if (n <= 2048) {
        QB_TRY(scorer_launch(sc, reinterpret_cast<const uint32_t*>(sc->m_ids), n, reinterpret_cast<float*>(sc->m_scores)));
    } else {
        QB_CUDA(cudaMemcpyAsync(sc->d_ids, sc->h_ids, n * 4, cudaMemcpyHostToDevice, sc->stream));
        QB_TRY(scorer_launch(sc, sc->d_ids, n, sc->d_scores));
        QB_CUDA(cudaMemcpyAsync(sc->h_scores, sc->d_scores, n * 4, cudaMemcpyDeviceToHost, sc->stream));
    }
    QB_CUDA(cudaStreamSynchronize(sc->stream));
    memcpy(scores, sc->h_scores, n * 4);
    sc->hw.cpu += (uint64_t)n * cpu_units_per_point(s) * (sc->custom_kind ? sc->n_examples : 1);
    sc->hw.vector_io_read += (uint64_t)n * io_units_per_point(s);
    return QB_OK;
}

extern "C" qb_status qb_score_point(qb_scorer* sc, uint32_t id, float* score) { return qb_score_points(sc, &id, 1, score); }

extern "C" qb_status qb_score_internal(qb_scorer* sc, uint32_t a, uint32_t b, float* score) {
    QB_CHECK(sc && score, QB_ERR_INVALID, "score_internal: null argument");
    QB_CHECK(!sc->custom_kind, QB_ERR_UNSUPPORTED, "score_internal: custom scorers compare against several vectors (custom_query_scorer.rs:111-113: unimplemented!)");
    qb_storage* s = sc->st;
    {
        uint32_t ab[2] = {a, b};
        QB_TRY(localize_ids(s, ab, 2, ab, "score_internal (the reference panics)"));
        a = ab[0]; b = ab[1];
    }
    QB_TRY(use_device(s->device));
    QB_TRY(scorer_reserve(sc, 1));
    if (s->kind == QB_KIND_PQ) {
        QB_TRY(qb_pq_score_internal(s, a, b, sc->d_scores, sc->stream));
    } else {
        // point `a` becomes the query (MetricQueryScorer::score_internal; SQ8 encode_internal_vector; BQ binary)
        qb_scorer* tmp = nullptr;
        const uint32_t ga = a + s->id_base, gb = b + s->id_base;   // the public entry points take reported (global) ids
        QB_TRY(qb_scorer_create_internal(s, ga, &tmp));
        qb_status st = qb_score_points(tmp, &gb, 1, score);
        qb_scorer_destroy(tmp);
        sc->hw.cpu += cpu_units_per_point(s);
        return st;
    }
    QB_CUDA(cudaMemcpyAsync(sc->h_scores, sc->d_scores, 4, cudaMemcpyDeviceToHost, sc->stream));
    QB_CUDA(cudaStreamSynchronize(sc->stream));
    *score = sc->h_scores[0];
    sc->hw.cpu += (uint64_t)s->pq_m * (s->pq_div[1] - s->pq_div[0]);
    return QB_OK;
}

extern "C" qb_status qb_scorer_take_counters(qb_scorer* sc, qb_hw_counters* out) {
    QB_CHECK(sc && out, QB_ERR_INVALID, "take_counters: null argument");
    *out = sc->hw;
    sc->hw.cpu = 0; sc->hw.vector_io_read = 0;
    return QB_OK;
}

extern "C" qb_status qb_rescore(qb_scorer* orig, const uint32_t* ids, size_t n, uint32_t top, qb_scored_point* out, uint32_t* out_count) {
    QB_CHECK(orig && out && out_count && (n == 0 || ids), QB_ERR_INVALID, "rescore: null argument");
    QB_CHECK(top >= 1 && top <= QB_MAX_TOP, QB_ERR_INVALID, "rescore: top %u outside [1,%u]", top, QB_MAX_TOP);
    *out_count = 0;
    if (n == 0) return QB_OK;
    qb_storage* s = orig->st;
    QB_TRY(use_device(s->device));
    QB_TRY(scorer_reserve(orig, std::max<size_t>(n, (size_t)top * 2 + 8)));
    QB_TRY(localize_ids(s, ids, n, orig->h_ids, "rescore"));
    QB_CUDA(cudaMemcpyAsync(orig->d_ids, orig->h_ids, n * 4, cudaMemcpyHostToDevice, orig->stream));
    // score into candidate keys, select top on the device (postprocess_search_result: sort_unstable desc + truncate)
    unsigned long long* d_cand = nullptr;
    QB_CUDA(cudaMalloc(&d_cand, n * 8 + top * sizeof(qb_scored_point) + 64));
    QbScanArgs a{};
    a.d_q_enc = orig->d_query; a.d_q_off = orig->d_q_off; a.nq = 1; a.row_begin = 0; a.row_end = n; a.d_ids = orig->d_ids;
    a.emit.cand = d_cand; a.emit.cap = n; a.emit.dense = 1; a.emit.dense_base = 0; a.emit.id_base = s->id_base;
    qb_status st = QB_OK;
    if (s->kind == QB_KIND_BQ) st = QB_ERR_UNSUPPORTED;  // rescoring always uses the original (dense) vectors
    else st = qb_launch_scan(s, a, orig->stream);
    qb_scored_point* d_res = reinterpret_cast<qb_scored_point*>(d_cand + n);
    uint32_t* d_cnt = reinterpret_cast<uint32_t*>(d_res + top);
    if (st == QB_OK) st = qb_launch_select(d_cand, nullptr, n, n, 1, top, 0, d_res, d_cnt, nullptr, nullptr, orig->stream);
    cudaError_t e = cudaSuccess;
    if (st == QB_OK) {
        e = cudaMemcpyAsync(out, d_res, (size_t)top * sizeof(qb_scored_point), cudaMemcpyDeviceToHost, orig->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out_count, d_cnt, 4, cudaMemcpyDeviceToHost, orig->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(orig->stream);
    }
    cudaFree(d_cand);
    if (e != cudaSuccess) { qb_set_error("rescore: %s", cudaGetErrorString(e)); return QB_ERR_CUDA; }
    orig->hw.cpu += (uint64_t)n * cpu_units_per_point(s);
    orig->hw.vector_io_read += (uint64_t)n * io_units_per_point(s);
    return st;
}

// ------------------------------------------------------------------------------------------------ sharding
extern "C" qb_status qb_storage_set_id_base(qb_storage* s, uint32_t id_base) {
    QB_CHECK(s, QB_ERR_INVALID, "set_id_base: null storage");
    s->id_base = id_base;
    return QB_OK;
}

__global__ void lists_to_keys_kernel(const qb_scored_point* __restrict__ lists, const uint32_t* __restrict__ counts, uint32_t n_lists, uint32_t nq,
                                     uint32_t top, unsigned long long* __restrict__ keys) {
    // lists: [n_lists][nq][top], counts: [n_lists][nq]  ->  keys: [nq][n_lists*top] (0 = empty)
    const uint64_t total = (uint64_t)n_lists * nq * top;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t k = (uint32_t)(i % top);
        const uint32_t q = (uint32_t)((i / top) % nq);
        const uint32_t l = (uint32_t)(i / ((uint64_t)top * nq));
        const qb_scored_point sp = lists[i];
        keys[(uint64_t)q * n_lists * top + (uint64_t)l * top + k] = (k < counts[(uint64_t)l * nq + q]) ? qb_pack_key(sp.score, sp.idx) : 0ull;
    }
}

// BatchResultAggregator (lib/shard/src/search_result_aggregator.rs:50-117) for per-GPU shards: merge n_lists sorted
// top-k lists per query (as gathered over NVLink) into one.  All pointers are device memory; enqueued on `stream`.
extern "C" qb_status qb_topk_merge_device(int32_t device, const qb_scored_point* dev_lists, const uint32_t* dev_counts, uint32_t n_lists,
                                          uint32_t n_queries, uint32_t top, qb_scored_point* dev_out, uint32_t* dev_out_counts,
                                          void* dev_scratch, uint64_t scratch_bytes, void* stream) {
    QB_CHECK(dev_lists && dev_counts && dev_out && dev_out_counts && dev_scratch, QB_ERR_INVALID, "topk_merge: null argument");
    QB_CHECK(top >= 1 && top <= QB_MAX_TOP, QB_ERR_INVALID, "topk_merge: top %u outside [1,%u]", top, QB_MAX_TOP);
    const uint64_t need = (uint64_t)n_queries * n_lists * top * 8;
    QB_CHECK(scratch_bytes >= need, QB_ERR_INVALID, "topk_merge: scratch %llu < %llu bytes", (unsigned long long)scratch_bytes, (unsigned long long)need);
    if (n_queries == 0 || n_lists == 0) return QB_OK;
    QB_TRY(use_device(device));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const uint64_t total = (uint64_t)n_lists * n_queries * top;
    lists_to_keys_kernel<<<(unsigned)std::min<uint64_t>(ceil_div_u64(total, 256), 4096), 256, 0, st>>>(
        dev_lists, dev_counts, n_lists, n_queries, top, reinterpret_cast<unsigned long long*>(dev_scratch));
    QB_LAUNCHED();
    QB_CUDA(cudaGetLastError());
    return qb_launch_select(reinterpret_cast<unsigned long long*>(dev_scratch), nullptr, (unsigned long long)n_lists * top,
                            (unsigned long long)n_lists * top, n_queries, top, 0, dev_out, dev_out_counts, nullptr, nullptr, st);
}

// ------------------------------------------------------------------------------------------------ profiling
extern "C" qb_status qb_profile_enable(qb_storage* s, int32_t on) {
    QB_CHECK(s, QB_ERR_INVALID, "profile_enable: null storage");
    std::lock_guard<std::mutex> lk(s->mu);
    s->profile = on != 0;
    return QB_OK;
}

extern "C" qb_status qb_profile_read(qb_storage* s, uint64_t* launches, double* total_ms, int32_t reset) {
    QB_CHECK(s, QB_ERR_INVALID, "profile_read: null storage");
    QB_TRY(use_device(s->device));
    std::lock_guard<std::mutex> lk(s->mu);
    for (auto& pr : s->prof_pending) {
        float ms = 0.f;
        if (cudaEventSynchronize(pr.second) == cudaSuccess && cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) {
            s->prof_ms += ms;
            s->prof_launches += 1;
        }
        s->prof_free.push_back(pr);
    }
    s->prof_pending.clear();
    if (launches) *launches = s->prof_launches;
    if (total_ms) *total_ms = s->prof_ms;
    if (reset) { s->prof_launches = 0; s->prof_ms = 0.0; }
    return QB_OK;
}

extern "C" qb_status qb_search_stats(qb_storage* s, uint64_t* searches, uint64_t* reruns, int32_t reset) {
    QB_CHECK(s, QB_ERR_INVALID, "search_stats: null storage");
    // single-query prefilter searches fall back on the device (no host round trip): their count lives in device memory
    unsigned int dev_fallbacks = 0;
    if (s->d_pf_fallbacks) {
        QB_TRY(use_device(s->device));
        QB_CUDA(cudaDeviceSynchronize());
        QB_CUDA(cudaMemcpy(&dev_fallbacks, s->d_pf_fallbacks, 4, cudaMemcpyDeviceToHost));
        if (reset) QB_CUDA(cudaMemset(s->d_pf_fallbacks, 0, 4));
    }
    if (searches) *searches = s->n_searches.load();
    if (reruns) *reruns = s->n_reruns.load() + dev_fallbacks;
    if (reset) { s->n_searches = 0; s->n_reruns = 0; }
    return QB_OK;
}

extern "C" qb_status qb_storage_set_on_disk(qb_storage* s, int32_t on_disk) {
    QB_CHECK(s, QB_ERR_INVALID, "set_on_disk: null storage");
    s->on_disk = on_disk != 0;
    return QB_OK;
}

// ------------------------------------------------------------------------------------------------ HNSW on the device
extern "C" qb_status qb_hnsw_search_batch_algo(qb_hnsw* g, const float* queries, uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point,
                                               uint32_t entry_level, const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped, qb_scored_point* out,
                                               uint32_t* out_counts, qb_hw_counters* counters, qb_hnsw_algorithm algorithm) {
    QB_CHECK(g && out && out_counts, QB_ERR_INVALID, "hnsw_search_batch: null argument");
    QB_CHECK(n_queries == 0 || queries, QB_ERR_INVALID, "hnsw_search_batch: null queries");
    QB_CHECK(top >= 1 && top <= 4096, QB_ERR_INVALID, "hnsw_search_batch: top %u outside [1,4096]", top);
    if (n_queries == 0) return QB_OK;
    if (is_stopped && *is_stopped) { qb_set_error("search cancelled"); return QB_ERR_CANCELLED; }
    qb_storage* s = g->st;
    QB_TRY(use_device(s->device));
    std::lock_guard<std::mutex> glk(g->mu);
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_acquire(s, &c));
    struct Rel { qb_storage* s; QbSearchCtx* c; ~Rel() { qb_ctx_release(s, c); } } rel{s, c};
    cudaStream_t stream = c->stream;
    const size_t raw_bytes = (size_t)n_queries * s->dim * 4, res_bytes = (size_t)n_queries * top * sizeof(qb_scored_point), cnt_bytes = (size_t)n_queries * 4;
    QB_TRY(qb_ensure_pinned(&c->h_stage, &c->h_stage_bytes, raw_bytes + res_bytes + cnt_bytes + 16));
    uint8_t* hs = reinterpret_cast<uint8_t*>(c->h_stage);
    memcpy(hs, queries, raw_bytes);
    QB_TRY(qb_ensure_device(&c->d_queries_raw, &c->queries_raw_bytes, raw_bytes + (size_t)n_queries * pre_stride_f(s) * 4));
    QB_TRY(qb_ensure_device(&c->d_queries_enc, &c->queries_enc_bytes, ((size_t)n_queries + 256) * qb_encoded_query_bytes(s)));
    QB_TRY(ensure_dev_elems(&c->d_q_off, &c->q_off_elems, (size_t)n_queries));
    QB_TRY(ensure_dev_elems(&c->d_out, &c->out_elems, (size_t)n_queries * top));
    QB_TRY(ensure_dev_elems(&c->d_out_counts, &c->out_counts_elems, (size_t)n_queries + 4));
    QB_CUDA(cudaMemcpyAsync(c->d_queries_raw, hs, raw_bytes, cudaMemcpyHostToDevice, stream));
    float* d_pre = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(c->d_queries_raw) + raw_bytes);
    QB_TRY(prepare_queries(s, reinterpret_cast<const float*>(c->d_queries_raw), n_queries, d_pre, c->d_queries_enc, c->d_q_off, stream));
    const uint32_t* d_del2 = nullptr;
    if (deleted_bitmap) {
        const uint64_t words64 = ceil_div_u64(s->count, 64);
        QB_TRY(ensure_dev_elems(&c->d_deleted2, &c->deleted2_words, (size_t)words64 * 2));
        QB_CUDA(cudaMemcpyAsync(c->d_deleted2, deleted_bitmap, words64 * 8, cudaMemcpyHostToDevice, stream));
        d_del2 = c->d_deleted2;
    }
    QB_TRY(qb_hnsw_launch(g, c->d_queries_enc, c->d_q_off, n_queries, top, ef, entry_point, entry_level, d_del2, c->d_out, c->d_out_counts, stream,
                          (int)algorithm));
    QB_CUDA(cudaMemcpyAsync(hs + raw_bytes, c->d_out, res_bytes, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaMemcpyAsync(hs + raw_bytes + res_bytes, c->d_out_counts, cnt_bytes, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaStreamSynchronize(stream));
    memcpy(out, hs + raw_bytes, res_bytes);
    memcpy(out_counts, hs + raw_bytes + res_bytes, cnt_bytes);
    if (counters) {
        const uint64_t before = g->evals;
        QB_TRY(qb_hnsw_read_stats(g, stream));
        counters->cpu += (g->evals - before) * cpu_units_per_point(s);
        counters->vector_io_read += (g->evals - before) * io_units_per_point(s);
    }
    if (is_stopped && *is_stopped) { qb_set_error("search cancelled"); return QB_ERR_CANCELLED; }
    return QB_OK;
}

extern "C" qb_status qb_hnsw_search_batch(qb_hnsw* g, const float* queries, uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point,
                                          uint32_t entry_level, const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped, qb_scored_point* out,
                                          uint32_t* out_counts, qb_hw_counters* counters) {
    return qb_hnsw_search_batch_algo(g, queries, n_queries, top, ef, entry_point, entry_level, deleted_bitmap, is_stopped, out, out_counts, counters,
                                     QB_HNSW_ALGO_HNSW);
}

extern "C" qb_status qb_hnsw_search_batch_device_algo(qb_hnsw* g, const float* dev_queries, uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point,
                                                      uint32_t entry_level, qb_scored_point* dev_out, uint32_t* dev_counts, qb_hnsw_algorithm algorithm) {
    QB_CHECK(g && dev_queries && dev_out && dev_counts, QB_ERR_INVALID, "hnsw_search_batch_device: null argument");
    QB_CHECK(top >= 1 && top <= 4096, QB_ERR_INVALID, "hnsw_search_batch_device: top %u outside [1,4096]", top);
    if (n_queries == 0) return QB_OK;
    qb_storage* s = g->st;
    QB_TRY(use_device(s->device));
    std::lock_guard<std::mutex> glk(g->mu);
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_device(s, &c));
    QB_TRY(qb_ensure_device(&c->d_queries_raw, &c->queries_raw_bytes, (size_t)n_queries * pre_stride_f(s) * 4 + 256));
    QB_TRY(qb_ensure_device(&c->d_queries_enc, &c->queries_enc_bytes, ((size_t)n_queries + 256) * qb_encoded_query_bytes(s)));
    QB_TRY(ensure_dev_elems(&c->d_q_off, &c->q_off_elems, (size_t)n_queries));
    QB_TRY(prepare_queries(s, dev_queries, n_queries, reinterpret_cast<float*>(c->d_queries_raw), c->d_queries_enc, c->d_q_off, c->stream));
    cudaEvent_t e0, e1;
    profile_begin(s, c, c->stream, &e0, &e1);
    QB_TRY(qb_hnsw_launch(g, c->d_queries_enc, c->d_q_off, n_queries, top, ef, entry_point, entry_level, nullptr, dev_out, dev_counts, c->stream,
                          (int)algorithm));
    profile_end(s, c->stream, e0, e1);
    return QB_OK;
}

extern "C" qb_status qb_hnsw_search_batch_device(qb_hnsw* g, const float* dev_queries, uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point,
                                                 uint32_t entry_level, qb_scored_point* dev_out, uint32_t* dev_counts) {
    return qb_hnsw_search_batch_device_algo(g, dev_queries, n_queries, top, ef, entry_point, entry_level, dev_out, dev_counts, QB_HNSW_ALGO_HNSW);
}

// GraphLayers::search_with_vectors on a graph with inline vectors (qb_hnsw_inline.cu).  Counters as the reference meters its three scorers:
// the entry point's score_point through the quantized storage (cpu and, on disk, vector_io_read, quantized_query_scorer.rs:95-101),
// each link score through EncodedVectorsU8::score_bytes (cpu only), each base score through MetricQueryScorer::score_bytes (cpu,
// dim * 4 per point, metric_query_scorer.rs:43-64,101-104); inline bytes never count vector_io_read.
static qb_status hnsw_with_vectors_counters(qb_hnsw* g, uint32_t n_queries, cudaStream_t stream, qb_hw_counters* counters) {
    const uint64_t ev0 = g->evals, bev0 = g->base_evals;
    QB_TRY(qb_hnsw_read_stats(g, stream));
    if (counters) {
        qb_storage* s = g->st;
        counters->cpu += (g->evals - ev0) * cpu_units_per_point(s) + (g->base_evals - bev0) * (uint64_t)s->dim * 4;
        counters->vector_io_read += (uint64_t)n_queries * io_units_per_point(s);
    }
    return QB_OK;
}

extern "C" qb_status qb_hnsw_search_with_vectors_batch(qb_hnsw* g, const float* queries, uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point,
                                                       uint32_t entry_level, const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped,
                                                       qb_scored_point* out, uint32_t* out_counts, qb_hw_counters* counters) {
    QB_CHECK(g && out && out_counts, QB_ERR_INVALID, "hnsw_search_with_vectors_batch: null argument");
    QB_CHECK(n_queries == 0 || queries, QB_ERR_INVALID, "hnsw_search_with_vectors_batch: null queries");
    QB_CHECK(top >= 1 && top <= 4096, QB_ERR_INVALID, "hnsw_search_with_vectors_batch: top %u outside [1,4096]", top);
    QB_CHECK(g->d_blob, QB_ERR_UNSUPPORTED, "hnsw_search_with_vectors_batch: the graph has no inline vectors (load it with qb_hnsw_create_with_vectors)");
    if (n_queries == 0) return QB_OK;
    if (is_stopped && *is_stopped) { qb_set_error("search cancelled"); return QB_ERR_CANCELLED; }
    qb_storage* s = g->st;
    QB_TRY(use_device(s->device));
    std::lock_guard<std::mutex> glk(g->mu);
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_acquire(s, &c));
    struct Rel { qb_storage* s; QbSearchCtx* c; ~Rel() { qb_ctx_release(s, c); } } rel{s, c};
    cudaStream_t stream = c->stream;
    const size_t raw_bytes = (size_t)n_queries * s->dim * 4, res_bytes = (size_t)n_queries * top * sizeof(qb_scored_point), cnt_bytes = (size_t)n_queries * 4;
    QB_TRY(qb_ensure_pinned(&c->h_stage, &c->h_stage_bytes, raw_bytes + res_bytes + cnt_bytes + 16));
    uint8_t* hs = reinterpret_cast<uint8_t*>(c->h_stage);
    memcpy(hs, queries, raw_bytes);
    const size_t pre_off = round_up_u64(raw_bytes, 16);
    QB_TRY(qb_ensure_device(&c->d_queries_raw, &c->queries_raw_bytes, pre_off + (size_t)n_queries * pre_stride_f(s) * 4));
    QB_TRY(qb_ensure_device(&c->d_queries_enc, &c->queries_enc_bytes, ((size_t)n_queries + 256) * qb_encoded_query_bytes(s)));
    QB_TRY(ensure_dev_elems(&c->d_q_off, &c->q_off_elems, (size_t)n_queries));
    QB_TRY(ensure_dev_elems(&c->d_out, &c->out_elems, (size_t)n_queries * top));
    QB_TRY(ensure_dev_elems(&c->d_out_counts, &c->out_counts_elems, (size_t)n_queries + 4));
    QB_CUDA(cudaMemcpyAsync(c->d_queries_raw, hs, raw_bytes, cudaMemcpyHostToDevice, stream));
    float* d_pre = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(c->d_queries_raw) + pre_off);
    QB_TRY(prepare_queries(s, reinterpret_cast<const float*>(c->d_queries_raw), n_queries, d_pre, c->d_queries_enc, c->d_q_off, stream));
    const uint32_t* d_del2 = nullptr;
    if (deleted_bitmap) {
        const uint64_t words64 = ceil_div_u64(s->count, 64);
        QB_TRY(ensure_dev_elems(&c->d_deleted2, &c->deleted2_words, (size_t)words64 * 2));
        QB_CUDA(cudaMemcpyAsync(c->d_deleted2, deleted_bitmap, words64 * 8, cudaMemcpyHostToDevice, stream));
        d_del2 = c->d_deleted2;
    }
    QB_TRY(qb_hnsw_inline_launch(g, d_pre, pre_stride_f(s), c->d_queries_enc, c->d_q_off, n_queries, top, ef, entry_point, entry_level, d_del2, c->d_out,
                                 c->d_out_counts, stream));
    QB_CUDA(cudaMemcpyAsync(hs + raw_bytes, c->d_out, res_bytes, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaMemcpyAsync(hs + raw_bytes + res_bytes, c->d_out_counts, cnt_bytes, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaStreamSynchronize(stream));
    memcpy(out, hs + raw_bytes, res_bytes);
    memcpy(out_counts, hs + raw_bytes + res_bytes, cnt_bytes);
    QB_TRY(hnsw_with_vectors_counters(g, n_queries, stream, counters));
    if (is_stopped && *is_stopped) { qb_set_error("search cancelled"); return QB_ERR_CANCELLED; }
    return QB_OK;
}

extern "C" qb_status qb_hnsw_search_with_vectors_batch_device(qb_hnsw* g, const float* dev_queries, uint32_t n_queries, uint32_t top, uint32_t ef,
                                                              uint32_t entry_point, uint32_t entry_level, qb_scored_point* dev_out, uint32_t* dev_counts) {
    QB_CHECK(g && dev_queries && dev_out && dev_counts, QB_ERR_INVALID, "hnsw_search_with_vectors_batch_device: null argument");
    QB_CHECK(top >= 1 && top <= 4096, QB_ERR_INVALID, "hnsw_search_with_vectors_batch_device: top %u outside [1,4096]", top);
    QB_CHECK(g->d_blob, QB_ERR_UNSUPPORTED, "hnsw_search_with_vectors_batch_device: the graph has no inline vectors (load it with qb_hnsw_create_with_vectors)");
    if (n_queries == 0) return QB_OK;
    qb_storage* s = g->st;
    QB_TRY(use_device(s->device));
    std::lock_guard<std::mutex> glk(g->mu);
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_device(s, &c));
    QB_TRY(qb_ensure_device(&c->d_queries_raw, &c->queries_raw_bytes, (size_t)n_queries * pre_stride_f(s) * 4 + 256));
    QB_TRY(qb_ensure_device(&c->d_queries_enc, &c->queries_enc_bytes, ((size_t)n_queries + 256) * qb_encoded_query_bytes(s)));
    QB_TRY(ensure_dev_elems(&c->d_q_off, &c->q_off_elems, (size_t)n_queries));
    float* d_pre = reinterpret_cast<float*>(c->d_queries_raw);
    QB_TRY(prepare_queries(s, dev_queries, n_queries, d_pre, c->d_queries_enc, c->d_q_off, c->stream));
    cudaEvent_t e0, e1;
    profile_begin(s, c, c->stream, &e0, &e1);
    QB_TRY(qb_hnsw_inline_launch(g, d_pre, pre_stride_f(s), c->d_queries_enc, c->d_q_off, n_queries, top, ef, entry_point, entry_level, nullptr, dev_out,
                                 dev_counts, c->stream));
    profile_end(s, c->stream, e0, e1);
    return QB_OK;
}

// custom queries through the device traversal; discover_pairs > 0: the two-stage discover of that many pairs (kind = DISCOVER)
static qb_status hnsw_custom_run(qb_hnsw* g, qb_query_kind kind, const float* vectors, uint32_t n_a, uint32_t n_b, const float* coef, uint32_t n_queries,
                                 uint32_t top, uint32_t ef, uint32_t entry_point, uint32_t entry_level, const uint32_t* cep, const uint32_t* cep_counts,
                                 uint32_t n_custom, const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped, qb_scored_point* out,
                                 uint32_t* out_counts, qb_hw_counters* counters, qb_hnsw_algorithm algorithm, bool discover, const char* what) {
    QB_CHECK(g && out && out_counts, QB_ERR_INVALID, "%s: null argument", what);
    QB_CHECK(n_queries == 0 || vectors, QB_ERR_INVALID, "%s: null vectors", what);
    QB_CHECK(top >= 1 && top <= 4096, QB_ERR_INVALID, "%s: top %u outside [1,4096]", what, top);
    uint32_t ne = 0;
    QB_TRY(check_custom(kind, n_a, n_b, &ne));
    QB_CHECK(!discover || n_a >= 1, QB_ERR_INVALID, "%s: discover needs at least one (positive, negative) pair for its context stage", what);
    const bool fb = kind == QB_QUERY_FEEDBACK_NAIVE;
    QB_CHECK(fb == (coef != nullptr), QB_ERR_INVALID, "%s: coef is required for feedback queries and must be NULL otherwise", what);
    QB_CHECK(!cep || (cep_counts && n_custom >= 1), QB_ERR_INVALID, "%s: custom_entry_points need custom_counts and n_custom >= 1", what);
    qb_storage* s = g->st;
    QB_CHECK((s->kind == QB_KIND_DENSE && s->dtype == QB_DT_F32) || s->kind == QB_KIND_SQ8, QB_ERR_UNSUPPORTED,
             "%s: device traversal supports dense f32 and SQ8 storages (others go through qb_score_points per hop)", what);
    if (cep) {
        for (uint32_t q = 0; q < n_queries; ++q) {
            QB_CHECK(cep_counts[q] <= n_custom, QB_ERR_INVALID, "%s: custom_counts[%u] = %u > n_custom %u", what, q, cep_counts[q], n_custom);
            for (uint32_t i = 0; i < cep_counts[q]; ++i)
                QB_CHECK(cep[(size_t)q * n_custom + i] < g->n_points, QB_ERR_INVALID, "%s: custom entry point %u out of range", what, cep[(size_t)q * n_custom + i]);
        }
    }
    if (n_queries == 0) return QB_OK;
    if (is_stopped && *is_stopped) { qb_set_error("search cancelled"); return QB_ERR_CANCELLED; }
    QB_TRY(use_device(s->device));
    std::lock_guard<std::mutex> glk(g->mu);
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_acquire(s, &c));
    struct Rel { qb_storage* s; QbSearchCtx* c; ~Rel() { qb_ctx_release(s, c); } } rel{s, c};
    cudaStream_t stream = c->stream;
    const size_t nv = (size_t)n_queries * ne;   // example vectors, encoded back to back: query q's are [q * ne, (q + 1) * ne)
    const size_t raw_bytes = nv * s->dim * 4, res_bytes = (size_t)n_queries * top * sizeof(qb_scored_point), cnt_bytes = (size_t)n_queries * 4;
    QB_TRY(qb_ensure_pinned(&c->h_stage, &c->h_stage_bytes, raw_bytes + res_bytes + cnt_bytes + 16));
    uint8_t* hs = reinterpret_cast<uint8_t*>(c->h_stage);
    memcpy(hs, vectors, raw_bytes);
    QB_TRY(qb_ensure_device(&c->d_queries_raw, &c->queries_raw_bytes, raw_bytes + nv * pre_stride_f(s) * 4));
    QB_TRY(qb_ensure_device(&c->d_queries_enc, &c->queries_enc_bytes, (nv + 256) * qb_encoded_query_bytes(s)));
    QB_TRY(ensure_dev_elems(&c->d_q_off, &c->q_off_elems, nv));
    QB_TRY(ensure_dev_elems(&c->d_out, &c->out_elems, (size_t)n_queries * top));
    QB_TRY(ensure_dev_elems(&c->d_out_counts, &c->out_counts_elems, (size_t)n_queries + 4));
    QB_CUDA(cudaMemcpyAsync(c->d_queries_raw, hs, raw_bytes, cudaMemcpyHostToDevice, stream));
    float* d_pre = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(c->d_queries_raw) + raw_bytes);
    QB_TRY(prepare_queries(s, reinterpret_cast<const float*>(c->d_queries_raw), (uint32_t)nv, d_pre, c->d_queries_enc, c->d_q_off, stream));
    const uint32_t* d_del2 = nullptr;
    if (deleted_bitmap) {
        const uint64_t words64 = ceil_div_u64(s->count, 64);
        QB_TRY(ensure_dev_elems(&c->d_deleted2, &c->deleted2_words, (size_t)words64 * 2));
        QB_CUDA(cudaMemcpyAsync(c->d_deleted2, deleted_bitmap, words64 * 8, cudaMemcpyHostToDevice, stream));
        d_del2 = c->d_deleted2;
    }
    // per-call buffers: coefficients, custom entry points (as scored points: the stage-1 lists of discover have that layout), counts
    constexpr uint32_t DISCOVERY_ENTRY_POINT_COUNT = 10;   // search.rs:325
    const uint32_t n_coef = fb ? 1 + n_a : 0;
    const uint32_t n_cep = discover ? DISCOVERY_ENTRY_POINT_COUNT : (cep ? n_custom : 0);
    const size_t coef_bytes = round_up_u64((size_t)n_queries * n_coef * 4, 256), cep_bytes = round_up_u64((size_t)n_queries * n_cep * sizeof(qb_scored_point), 256);
    std::vector<uint8_t> h_extra(coef_bytes + cep_bytes + (size_t)n_queries * 4, 0);
    if (fb) memcpy(h_extra.data(), coef, (size_t)n_queries * n_coef * 4);
    if (cep && !discover) {
        qb_scored_point* hp = reinterpret_cast<qb_scored_point*>(h_extra.data() + coef_bytes);
        for (size_t i = 0; i < (size_t)n_queries * n_cep; ++i) hp[i].idx = cep[i];
        memcpy(h_extra.data() + coef_bytes + cep_bytes, cep_counts, (size_t)n_queries * 4);
    }
    struct Scratch { void* p = nullptr; ~Scratch() { cudaFree(p); } } extra;
    QB_CUDA(cudaMalloc(&extra.p, h_extra.size() + 256));
    uint8_t* d_extra = reinterpret_cast<uint8_t*>(extra.p);
    if (fb || (cep && !discover)) QB_CUDA(cudaMemcpyAsync(d_extra, h_extra.data(), h_extra.size(), cudaMemcpyHostToDevice, stream));
    QbHnswCustom cq{};
    cq.kind = (int)kind; cq.n_a = n_a; cq.n_b = n_b; cq.n_ex = ne; cq.ex_first = 0; cq.ex_stride = ne;
    cq.d_coef = fb ? reinterpret_cast<const float*>(d_extra) : nullptr; cq.n_coef = n_coef;
    qb_scored_point* d_cep = reinterpret_cast<qb_scored_point*>(d_extra + coef_bytes);
    uint32_t* d_cep_counts = reinterpret_cast<uint32_t*>(d_extra + coef_bytes + cep_bytes);
    if (n_cep) { cq.d_cep = d_cep; cq.d_cep_counts = d_cep_counts; cq.n_cep = n_cep; }
    cudaEvent_t e0, e1;
    profile_begin(s, c, stream, &e0, &e1);   // qb_profile_*: the traversal kernels (both stages of discover)
    if (discover) {
        // stage 1: the context search over the pairs (encoded examples 1 .. 2 n_pairs of each query), top 10, its lists left on the device
        QbHnswCustom ctx{};
        ctx.kind = QB_QUERY_CONTEXT; ctx.n_a = n_a; ctx.n_b = 0; ctx.n_ex = 2 * n_a; ctx.ex_first = 1; ctx.ex_stride = ne;
        ctx.stats_slot = 1; ctx.internal_out = true;
        QB_TRY(qb_hnsw_launch(g, c->d_queries_enc, c->d_q_off, n_queries, DISCOVERY_ENTRY_POINT_COUNT, ef, entry_point, entry_level, d_del2, d_cep,
                              d_cep_counts, stream, (int)algorithm, &ctx));
    }
    QB_TRY(qb_hnsw_launch(g, c->d_queries_enc, c->d_q_off, n_queries, top, ef, entry_point, entry_level, d_del2, c->d_out, c->d_out_counts, stream,
                          (int)algorithm, &cq));
    profile_end(s, stream, e0, e1);
    QB_CUDA(cudaMemcpyAsync(hs + raw_bytes, c->d_out, res_bytes, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaMemcpyAsync(hs + raw_bytes + res_bytes, c->d_out_counts, cnt_bytes, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaStreamSynchronize(stream));
    memcpy(out, hs + raw_bytes, res_bytes);
    memcpy(out_counts, hs + raw_bytes + res_bytes, cnt_bytes);
    if (counters) {
        // per scored point: E similarities of cpu units, one read of the vector (custom_query_scorer.rs:78-111, qb_score_points)
        uint64_t ev[2] = {0, 0};
        QB_TRY(qb_hnsw_read_stats(g, stream, ev));
        counters->cpu += (ev[0] * ne + ev[1] * (2ull * n_a)) * cpu_units_per_point(s);
        counters->vector_io_read += (ev[0] + ev[1]) * io_units_per_point(s);
    }
    if (is_stopped && *is_stopped) { qb_set_error("search cancelled"); return QB_ERR_CANCELLED; }
    return QB_OK;
}

extern "C" qb_status qb_hnsw_search_custom_batch(qb_hnsw* g, qb_query_kind kind, const float* vectors, uint32_t n_a, uint32_t n_b, const float* coef,
                                                 uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point, uint32_t entry_level,
                                                 const uint32_t* custom_entry_points, const uint32_t* custom_counts, uint32_t n_custom,
                                                 const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped, qb_scored_point* out,
                                                 uint32_t* out_counts, qb_hw_counters* counters, qb_hnsw_algorithm algorithm) {
    return hnsw_custom_run(g, kind, vectors, n_a, n_b, coef, n_queries, top, ef, entry_point, entry_level, custom_entry_points, custom_counts, n_custom,
                           deleted_bitmap, is_stopped, out, out_counts, counters, algorithm, false, "hnsw_search_custom_batch");
}

extern "C" qb_status qb_hnsw_search_discover_batch(qb_hnsw* g, const float* vectors, uint32_t n_pairs, uint32_t n_queries, uint32_t top, uint32_t ef,
                                                   uint32_t entry_point, uint32_t entry_level, const uint64_t* deleted_bitmap,
                                                   const volatile int32_t* is_stopped, qb_scored_point* out, uint32_t* out_counts,
                                                   qb_hw_counters* counters, qb_hnsw_algorithm algorithm) {
    return hnsw_custom_run(g, QB_QUERY_DISCOVER, vectors, n_pairs, 0, nullptr, n_queries, top, ef, entry_point, entry_level, nullptr, nullptr, 0,
                           deleted_bitmap, is_stopped, out, out_counts, counters, algorithm, true, "hnsw_search_discover_batch");
}

extern "C" qb_status qb_hnsw_stats(qb_hnsw* g, uint64_t* hops, uint64_t* scored_points, int32_t reset) {
    QB_CHECK(g, QB_ERR_INVALID, "hnsw_stats: null graph");
    QB_TRY(use_device(g->st->device));
    std::lock_guard<std::mutex> glk(g->mu);
    QB_CUDA(cudaDeviceSynchronize());
    QB_TRY(qb_hnsw_read_stats(g, 0));
    if (hops) *hops = g->hops;
    if (scored_points) *scored_points = g->evals;
    if (reset) { g->hops = 0; g->evals = 0; }
    return QB_OK;
}

// ------------------------------------------------------------------------------------------------ sharded search: one collective call per shard
// The reference runs one blocking task per segment and aggregates their lists (segments_searcher.rs:255, search_result_aggregator.rs:50-117);
// here every shard's task calls qb_multi_search_batch with the same queries, and the aggregation happens on the GPUs (qb_comm.cu).
extern "C" qb_status qb_multi_search_batch(qb_comm* cm, qb_storage* s, const float* queries, uint32_t n_queries, uint32_t top, const uint64_t* deleted_bitmap,
                                           const volatile int32_t* is_stopped, qb_scored_point* out, uint32_t* out_counts, qb_hw_counters* counters) {
    QB_CHECK(cm && s && out && out_counts, QB_ERR_INVALID, "multi_search_batch: null argument");
    QB_CHECK(n_queries == 0 || queries, QB_ERR_INVALID, "multi_search_batch: null queries");
    QB_CHECK(top >= 1, QB_ERR_INVALID, "multi_search_batch: top must be >= 1");
    QB_CHECK(cm->device == s->device, QB_ERR_INVALID, "multi_search_batch: communicator on device %d, shard on device %d", cm->device, s->device);
    if (n_queries == 0) return QB_OK;
    QB_TRY(use_device(s->device));
    std::lock_guard<std::mutex> clk(cm->mu);
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_acquire(s, &c));
    struct Rel { qb_storage* s; QbSearchCtx* c; ~Rel() { qb_ctx_release(s, c); } } rel{s, c};
    cudaStream_t stream = c->stream;
    const size_t raw_bytes = (size_t)n_queries * s->dim * 4, res_bytes = (size_t)n_queries * top * sizeof(qb_scored_point), cnt_bytes = (size_t)n_queries * 4;
    QB_TRY(qb_ensure_pinned(&c->h_stage, &c->h_stage_bytes, raw_bytes + res_bytes + cnt_bytes + 32));
    uint8_t* hs = reinterpret_cast<uint8_t*>(c->h_stage);
    memcpy(hs, queries, raw_bytes);
    QB_TRY(qb_ensure_device(&c->d_queries_raw, &c->queries_raw_bytes, raw_bytes + (size_t)n_queries * pre_stride_f(s) * 4));
    QB_TRY(qb_ensure_device(&c->d_queries_enc, &c->queries_enc_bytes, ((size_t)n_queries + 256) * qb_encoded_query_bytes(s)));
    QB_TRY(ensure_dev_elems(&c->d_q_off, &c->q_off_elems, (size_t)n_queries));
    QB_TRY(ensure_dev_elems(&c->d_out, &c->out_elems, (size_t)n_queries * top));
    QB_TRY(ensure_dev_elems(&c->d_out_counts, &c->out_counts_elems, (size_t)n_queries + 4));
    if (cm->local_cap < (size_t)n_queries * top) {
        cudaFree(cm->d_local); cudaFree(cm->d_local_cnt); cm->d_local = nullptr; cm->d_local_cnt = nullptr; cm->local_cap = 0;
        QB_CUDA(cudaMalloc(&cm->d_local, (size_t)n_queries * top * sizeof(qb_scored_point)));
        QB_CUDA(cudaMalloc(&cm->d_local_cnt, ((size_t)n_queries * top + 4) * 4));
        cm->local_cap = (size_t)n_queries * top;
    }
    QB_CUDA(cudaMemcpyAsync(c->d_queries_raw, hs, raw_bytes, cudaMemcpyHostToDevice, stream));
    float* d_pre = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(c->d_queries_raw) + raw_bytes);
    QB_TRY(prepare_queries(s, reinterpret_cast<const float*>(c->d_queries_raw), n_queries, d_pre, c->d_queries_enc, c->d_q_off, stream));
    const uint32_t* d_del2 = nullptr;
    if (deleted_bitmap) {
        const uint64_t words64 = ceil_div_u64(s->count, 64);
        QB_TRY(ensure_dev_elems(&c->d_deleted2, &c->deleted2_words, (size_t)words64 * 2));
        QB_CUDA(cudaMemcpyAsync(c->d_deleted2, deleted_bitmap, words64 * 8, cudaMemcpyHostToDevice, stream));
        d_del2 = c->d_deleted2;
    }
    unsigned int* d_overflow = reinterpret_cast<unsigned int*>(cm->d_local_cnt + (size_t)n_queries * top);
    uint8_t* h_res = hs + raw_bytes;
    uint8_t* h_cnt = h_res + res_bytes;
    uint32_t rs_flags = 0;
    qb_status st_local = QB_OK;
    for (int attempt = 0; attempt < 4; ++attempt) {
        QB_CUDA(cudaMemsetAsync(d_overflow, 0, 4, stream));
        bool can_flag = true;
        st_local = run_search(s, c, n_queries, top, nullptr, 0, d_del2, is_stopped, rs_flags, cm->d_local, cm->d_local_cnt, d_overflow, &can_flag);
        if (st_local != QB_OK || !can_flag) break;
        QB_CUDA(cudaMemcpyAsync(h_cnt + cnt_bytes, d_overflow, 4, cudaMemcpyDeviceToHost, stream));
        QB_CUDA(cudaStreamSynchronize(stream));
        unsigned int flags = 0;
        memcpy(&flags, h_cnt + cnt_bytes, 4);
        uint32_t next = rs_flags;
        if (flags & 8u) next |= RS_NO_SEGMENTS;
        if (flags & 2u) next |= RS_NO_MMA;
        if (flags & 1u) next |= RS_FORCE_DIRECT | RS_NO_MMA;
        if (next == rs_flags) break;
        s->n_reruns.fetch_add(1, std::memory_order_relaxed);
        rs_flags = next;
    }
    s->n_searches.fetch_add(1, std::memory_order_relaxed);
    // a rank that failed locally still joins the exchange (with empty lists) so that its peers do not wait for it
    if (st_local != QB_OK) QB_CUDA(cudaMemsetAsync(cm->d_local_cnt, 0, (size_t)n_queries * 4, stream));
    QB_TRY(qb_comm_exchange_merge(cm, cm->d_local, cm->d_local_cnt, n_queries, top, c->d_out, c->d_out_counts, stream));
    QB_CUDA(cudaMemcpyAsync(h_res, c->d_out, res_bytes, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaMemcpyAsync(h_cnt, c->d_out_counts, cnt_bytes, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaMemcpyAsync(h_cnt + cnt_bytes + 8, cm->d_error, 4, cudaMemcpyDeviceToHost, stream));
    QB_CUDA(cudaStreamSynchronize(stream));
    unsigned int xerr = 0;
    memcpy(&xerr, h_cnt + cnt_bytes + 8, 4);
    QB_CHECK(xerr == 0, QB_ERR_CUDA, "multi_search_batch: a peer rank never joined the exchange (timeout)");
    if (st_local != QB_OK) return st_local;
    memcpy(out, h_res, res_bytes);
    memcpy(out_counts, h_cnt, cnt_bytes);
    if (counters) {
        counters->cpu += s->count * (uint64_t)n_queries * cpu_units_per_point(s);
        counters->vector_io_read += s->count * (uint64_t)n_queries * io_units_per_point(s);
    }
    return QB_OK;
}

// device-resident form: queries / outputs in HBM, enqueued on qb_storage_stream(s).  dev_local / dev_local_counts receive this shard's own
// lists (n_queries x top) and must stay valid until the stream has run the exchange.
extern "C" qb_status qb_multi_search_batch_device(qb_comm* cm, qb_storage* s, const float* dev_queries, uint32_t n_queries, uint32_t top, qb_scored_point* dev_local,
                                                  uint32_t* dev_local_counts, qb_scored_point* dev_out, uint32_t* dev_counts) {
    QB_CHECK(cm && s && dev_queries && dev_out && dev_counts && (!dev_local == !dev_local_counts), QB_ERR_INVALID, "multi_search_batch_device: null argument");
    QB_CHECK(cm->device == s->device, QB_ERR_INVALID, "multi_search_batch_device: communicator and shard on different devices");
    if (n_queries == 0) return QB_OK;
    QbSearchCtx* c = nullptr;
    QB_TRY(qb_ctx_device(s, &c));
    std::lock_guard<std::mutex> clk(cm->mu);
    if (!dev_local) {
        // pipelined: this step's exchange + merge runs on the communicator's stream while the next step's scan already streams rows
        return qb_comm_pipelined_step(cm, c->stream, n_queries, top, dev_out, dev_counts,
                                      [&](qb_scored_point* d_loc, uint32_t* d_loc_cnt) { return qb_search_batch_device(s, dev_queries, n_queries, top, d_loc, d_loc_cnt); });
    }
    QB_TRY(qb_search_batch_device(s, dev_queries, n_queries, top, dev_local, dev_local_counts));
    return qb_comm_exchange_merge(cm, dev_local, dev_local_counts, n_queries, top, dev_out, dev_counts, c->stream);
}
