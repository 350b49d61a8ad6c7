// qb_internal.h — host-side objects behind the opaque C-ABI handles.
#pragma once
#include <functional>

#include "qb_common.cuh"

enum QbKind { QB_KIND_DENSE = 0, QB_KIND_SQ8 = 1, QB_KIND_PQ = 2, QB_KIND_BQ = 3 };

constexpr uint32_t QB_MAX_TOP = 1u << 20;      // fused top-k limit; <= 4096 sorts in shared memory, larger tops sort in a global scratch (qb_topk.cu)
constexpr uint32_t QB_SELECT_THREADS = 1024;

// A search context: one CUDA stream + the scratch a brute-force scan needs.  Contexts are pooled per
// storage so that concurrent qb_search_batch calls (one blocking task per segment in the reference,
// segments_searcher.rs:255) never share buffers.
struct QbSearchCtx {
    cudaStream_t stream = nullptr;
    // device scratch
    void* d_queries_raw = nullptr;   size_t queries_raw_bytes = 0;   // uploaded raw f32 queries
    void* d_queries_enc = nullptr;   size_t queries_enc_bytes = 0;   // preprocessed / encoded queries
    float* d_q_off = nullptr;        size_t q_off_elems = 0;         // SQ8 query offsets
    float* d_thr = nullptr;          size_t thr_elems = 0;
    unsigned int* d_cnt = nullptr;   size_t cnt_elems = 0;
    unsigned long long* d_cand = nullptr; size_t cand_elems = 0;
    qb_scored_point* d_out = nullptr; size_t out_elems = 0;
    uint32_t* d_out_counts = nullptr; size_t out_counts_elems = 0;
    uint32_t* d_deleted2 = nullptr;  size_t deleted2_words = 0;
    uint32_t* d_ids = nullptr;       size_t ids_elems = 0;
    void* d_pf = nullptr;            // single-query bf16 prefilter: counters, sample top-k, candidate rows (qb_prefilter.cu)
    float* d_pf_up5 = nullptr;       size_t pf_up5_elems = 0;        // single-query prefilter on the 6-bit plane: every row's first-stage bound
    void* d_mma = nullptr;           size_t mma_bytes = 0;           // batched SQ8: sorted query codes / permutation / chunk thresholds
    // pinned host staging
    void* h_stage = nullptr;         size_t h_stage_bytes = 0;
    // profiling
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    bool in_use = false;
    unsigned int* d_done = nullptr;      // arrival counter of the single-query in-kernel top-k (zeroed once, the kernel resets it)
};

struct qb_storage {
    int device = 0;
    QbKind kind = QB_KIND_DENSE;
    uint32_t dim = 0;
    uint64_t count = 0;
    uint64_t hbm_bytes = 0;

    // ---- dense
    qb_dtype dtype = QB_DT_F32;
    qb_distance distance = QB_DIST_DOT;
    void* d_rows = nullptr;          // row-major, stride padded to 16 B
    // bf16 shadow of the f32 rows for the tensor-core prefilter of batched searches (qb_sq8_mma.cu, F16): built on first use
    uint16_t* d_bf16 = nullptr;  uint32_t bf16_row_h = 0;  unsigned int* d_bf16_meta = nullptr;   // meta: [0] max |row| (float bits), [1] non-finite flag
    bool bf16_ready = false, bf16_usable = false;
    // int8 shadow (per-row scale) for single-query searches (qb_prefilter.cu): a quarter of the f32 bytes per scan; built on first use
    int8_t* d_q8 = nullptr;  uint32_t q8_row_b = 0;  unsigned int* d_q8_meta = nullptr;   // meta as above
    bool q8_ready = false, q8_usable = false;
    // 6-bit shadow for single-query searches (qb_prefilter.cu): main records of 5-bit codes, the row's scale and residual-norm bounds (0.16 of the
    // f32 bytes, streamed by every scan) and a side plane of the codes' low bits (read for the rows the 5-bit codes let through)
    uint8_t* d_q6 = nullptr;  uint32_t q6_row_b = 0;  unsigned int* d_q6_meta = nullptr;   // meta as above
    uint8_t* d_q6_lo = nullptr;
    bool q6_ready = false, q6_usable = false;
    // block-scaled 4-bit records (codes, a u8 scale per 16 dims, the row's scale and residual-norm bound: 0.14 of the f32 bytes), streamed
    // by the first stage of the 6-bit plane's scan in place of its 5-bit codes
    uint8_t* d_q4b = nullptr;  uint32_t q4b_row_b = 0;
    bool q4b_ready = false;
    uint32_t row_stride = 0;         // bytes
    uint32_t elem_size = 4;

    // ---- quantized common
    qb_qdistance qdist = QB_QD_DOT;
    int invert = 0;

    // ---- SQ8 (rows repacked: code plane + offset plane; the HBM copy is a cache, SURVEY §7 hard parts)
    uint32_t actual_dim = 0;
    uint8_t* d_codes = nullptr;      // [count][actual_dim], actual_dim % 16 == 0
    float* d_voff = nullptr;         // [count]
    float alpha = 0, offset = 0, multiplier = 0;
    float voff_absmax = 0;           // max |v_off| over the rows; inf when one is not finite (qb_sq8_mma_block)

    // ---- PQ
    uint32_t pq_m = 0, pq_stride = 0, n_centroids = 0;
    std::vector<uint32_t> pq_div;    // 2*m {start,end}
    uint32_t* d_pq_div = nullptr;
    float* d_centroids = nullptr;    // [n_centroids][dim]
    uint8_t* d_pq_codes = nullptr;   // [count][pq_stride], stride = round_up(m,16)

    // ---- BQ
    qb_bq_encoding bq_enc = QB_BQ_ONE_BIT;
    qb_bq_query_encoding bq_qenc = QB_BQQ_SAME_AS_STORAGE;
    uint32_t bq_row_bytes = 0;
    uint8_t* d_bq_rows = nullptr;
    float* d_mean_std = nullptr;

    // ---- sharding: ids reported by searches are local row + id_base
    uint32_t id_base = 0;

    // ---- soft deletes
    uint32_t* d_deleted = nullptr;   // resident bits (32-bit words), or null

    // ---- hardware counters: the reference meters vector_io_read only for on-disk storages (metric_query_scorer.rs:44-48)
    bool on_disk = false;

    // ---- contexts / profiling
    std::mutex mu;
    std::vector<QbSearchCtx*> ctxs;       // pool for the host-facing searches (one per concurrent call)
    unsigned int* d_pf_fallbacks = nullptr;   // device-side count of prefilter searches answered by the exact fallback scan
    QbSearchCtx* dev_ctx = nullptr;       // reserved for qb_storage_stream / the *_device entry points; never handed out by the pool
    std::atomic<uint64_t> n_searches{0}, n_reruns{0};
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_free;
    bool profile = false;
    uint64_t prof_launches = 0;
    double prof_ms = 0.0;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_pending;
    int sm_count = 132;
};

struct qb_scorer {
    qb_storage* st = nullptr;
    cudaStream_t stream = nullptr;
    void* d_query = nullptr;         // preprocessed f32 / u8 / f16 query, SQ8 code, PQ LUT, BQ encoded query
    size_t query_bytes = 0;
    float* d_q_off = nullptr;        // SQ8 query offset (device scalar)
    bool internal = false;
    uint32_t internal_id = 0;
    // staging (grown on demand)
    uint32_t* d_ids = nullptr;  float* d_scores = nullptr;  size_t cap = 0;
    uint32_t* h_ids = nullptr;  float* h_scores = nullptr;  size_t h_cap = 0;
    void* m_ids = nullptr;      void* m_scores = nullptr;   // device-side addresses of the mapped host buffers
    // custom queries (recommend / discover / context): d_query holds n_examples encoded queries, d_q_off their SQ8 offsets
    int custom_kind = 0;  uint32_t n_a = 0, n_b = 0, n_examples = 1;
    float* d_sims = nullptr;  size_t sims_cap = 0;          // [n_examples][cap] per-example similarities
    float* d_coef = nullptr;                                // feedback query: [a, partial_computation per pair]
    qb_hw_counters hw = {0, 0};
};

// A device-resident HNSW graph bound to a storage (qb_hnsw.cu)
struct qb_hnsw {
    qb_storage* st = nullptr;
    uint32_t n_points = 0, m = 0, m0 = 0, levels = 0;
    uint32_t* d_links0 = nullptr;
    uint64_t* d_level_offsets = nullptr;
    uint32_t* d_reindex = nullptr;
    uint32_t* d_neighbors = nullptr;
    uint64_t* d_offsets = nullptr;
    uint64_t hbm_bytes = 0;
    // host copy of the level offsets with the extra last element (offset count - 1, view.rs:381-393); offsets / neighbours
    // counts as the file describes them (qb_hnsw_links bounds its reads by these)
    std::vector<uint64_t> level_offsets_ext;
    uint64_t n_offsets = 0, n_neighbors = 0;
    // search scratch (one batch at a time per graph handle; mu serialises)
    std::mutex mu;
    uint32_t* d_visited = nullptr; uint64_t visited_words = 0; unsigned visited_slots = 0;
    uint32_t* d_vlog = nullptr; uint32_t vlog_cap = 0;
    unsigned int* d_work = nullptr;
    unsigned long long* d_stats = nullptr;   // [0..3] the regular searches (two slots), [4..6] the inline-vector search
    uint64_t hops = 0, evals = 0, base_evals = 0;
    // inline vectors (qb_hnsw_create_with_vectors): the records, each entry's first link vector and each point's base vector (byte
    // offsets into d_blob); null for the other loaders
    uint8_t* d_blob = nullptr; uint64_t* d_lvoff = nullptr; uint64_t* d_boff = nullptr; uint32_t link_size = 0;
};

// A batch of custom queries for qb_hnsw_launch: query q's examples are the encoded queries ex_first .. ex_first + n_ex of the
// ex_stride that d_q_enc / d_q_off hold per query.  d_cep: custom entry points [nq][n_cep] (.idx read), d_cep_counts[q] of them valid.
struct QbHnswCustom {
    int kind; uint32_t n_a, n_b;                 // qb_query_kind and its shape
    uint32_t n_ex, ex_first, ex_stride;
    const float* d_coef; uint32_t n_coef;        // feedback: [a, partial...] per query, else null / 0
    const qb_scored_point* d_cep; const uint32_t* d_cep_counts; uint32_t n_cep;
    uint32_t stats_slot;                         // hops / scored points go to stats slot 0 or 1 (qb_hnsw_read_stats)
    bool internal_out;                           // results as point offsets, without the storage's id_base (discover's context stage)
};

qb_status qb_hnsw_launch(qb_hnsw* g, const void* d_q_enc, const float* d_q_off, uint32_t nq, uint32_t top, uint32_t ef, uint32_t entry, uint32_t entry_level,
                         const uint32_t* d_deleted2, qb_scored_point* d_out, uint32_t* d_counts, cudaStream_t stream, int algo /* qb_hnsw_algorithm */,
                         const QbHnswCustom* custom = nullptr);
// completes a handle whose plain arrays (d_level_offsets, d_reindex, d_neighbors, d_offsets and the host-side counts) are on the device:
// the level-0 table and the search scratch (qb_hnsw.cu).  On failure the caller destroys g.  who = the error messages' prefix.
qb_status qb_hnsw_finish_plain(qb_hnsw* g, const char* who);
// the inline-vector search (qb_hnsw_inline.cu): queries preprocessed (d_q_pre, pre_stride floats apart) and SQ8-encoded; enqueued on stream
qb_status qb_hnsw_inline_launch(qb_hnsw* g, const float* d_q_pre, uint32_t pre_stride, const void* d_q_enc, const float* d_q_off, uint32_t nq, uint32_t top,
                                uint32_t ef, uint32_t entry, uint32_t entry_level, const uint32_t* d_deleted2, qb_scored_point* d_out, uint32_t* d_counts,
                                cudaStream_t stream);
// adds the device counters to g->hops / g->evals / g->base_evals and clears them; evals_by_slot (optional, [2]) receives each regular slot's scored points
qb_status qb_hnsw_read_stats(qb_hnsw* g, cudaStream_t stream, uint64_t* evals_by_slot = nullptr);

// One rank of a sharded search (qb_comm.cu): an exchange buffer every peer maps + the peers' buffers
constexpr uint32_t QB_MAX_WORLD = 16;
constexpr uint32_t QB_XCHG_SLOTS = 4;     // ring of exchange slots (window of 2 pipelined steps, see qb_comm.cu)
struct qb_comm {
    int device = 0, rank = 0, world = 1, sm_count = 132;
    uint32_t max_q = 0, max_top = 0;
    void* d_buf = nullptr; uint64_t bytes = 0;
    uint8_t* peers[QB_MAX_WORLD] = {};
    bool ipc_opened[QB_MAX_WORLD] = {};
    bool connected = false;
    uint32_t seq = 0;
    unsigned int* d_error = nullptr;
    qb_scored_point* d_local = nullptr; uint32_t* d_local_cnt = nullptr; size_t local_cap = 0;   // this shard's lists (host-facing entry)
    // pipelined device-resident steps: exchange + merge on its own high-priority stream, this shard's lists in a ring
    cudaStream_t xstream = nullptr;
    cudaEvent_t ev_scan[QB_XCHG_SLOTS] = {}, ev_merge[QB_XCHG_SLOTS] = {};
    qb_scored_point* d_ring[QB_XCHG_SLOTS] = {}; uint32_t* d_ring_cnt[QB_XCHG_SLOTS] = {};
    std::mutex mu;
};
qb_status qb_comm_pipelined_step(qb_comm* c, cudaStream_t scan_stream, uint32_t nq, uint32_t top, qb_scored_point* d_out, uint32_t* d_out_cnt,
                                 const std::function<qb_status(qb_scored_point*, uint32_t*)>& launch_scan);
qb_status qb_comm_exchange_merge(qb_comm* c, const qb_scored_point* d_local, const uint32_t* d_local_cnt, uint32_t nq, uint32_t top, qb_scored_point* d_out,
                                 uint32_t* d_out_cnt, cudaStream_t stream);

// ---------------------------------------------------------------- helpers (qb_api.cu)
qb_status qb_ensure_device(void** p, size_t* have, size_t need_bytes);
qb_status qb_ensure_pinned(void** p, size_t* have, size_t need_bytes);
qb_status qb_ctx_acquire(qb_storage* s, QbSearchCtx** out);
void qb_ctx_release(qb_storage* s, QbSearchCtx* c);
qb_status qb_ctx_device(qb_storage* s, QbSearchCtx** out);

// ---------------------------------------------------------------- kernels' host launchers
// All launchers enqueue on `stream` and never synchronise.

// queries: Metric::preprocess / encode_query on device.  q_raw [nq][dim] f32 -> ctx->d_queries_enc (+ d_q_off)
qb_status qb_launch_prepare_queries(const qb_storage* s, const float* d_q_raw, uint32_t nq, void* d_q_enc, float* d_q_off,
                                    cudaStream_t stream);
// size in bytes of one encoded query for this storage
size_t qb_encoded_query_bytes(const qb_storage* s);

// scan rows [row_begin,row_end) (id_list == null) or the listed ids [0,n_ids) against nq encoded queries
struct QbScanArgs {
    const void* d_q_enc;
    const float* d_q_off;
    uint32_t nq;
    uint64_t row_begin, row_end;
    const uint32_t* d_ids;  // optional gather list; then row_begin/row_end index into it
    QbEmit emit;
    float* d_thr_scratch;   // optional: nq floats a scan may use for adjusted thresholds (PQ prefilter); null = exact kernels only
    void* d_scratch; size_t scratch_bytes;   // optional per-call scratch (PQ: interleaved u8 tables of the sixteen-query prefilter)
};
size_t qb_pq_scratch_bytes(const qb_storage* s, uint32_t nq);
// single-query dense f32 searches through the bf16 shadow plane (qb_prefilter.cu)
qb_status qb_f32_shadow_ensure(qb_storage* s, cudaStream_t stream);
bool qb_f32_prefilter_usable(qb_storage* s, uint64_t n_rows, uint32_t top, cudaStream_t stream);
size_t qb_f32_prefilter_scratch_bytes();
qb_status qb_f32_prefilter_search(qb_storage* s, const QbScanArgs& a, uint32_t top, void* d_scratch, float* d_up5, unsigned int* d_n_fallbacks, qb_scored_point* d_out,
                                  uint32_t* d_out_cnt, cudaEvent_t prof0, cudaEvent_t prof1, cudaStream_t stream);
qb_status qb_launch_scan(const qb_storage* s, const QbScanArgs& a, cudaStream_t stream);

// score listed ids for ONE encoded query into d_scores (RawScorer::score_points)
qb_status qb_launch_score_points(const qb_storage* s, const void* d_q_enc, const float* d_q_off, const uint32_t* d_ids,
                                 uint64_t n, float* d_scores, cudaStream_t stream);
// encoded query taken from a stored point (internal scorer)
qb_status qb_launch_encode_internal(const qb_storage* s, uint32_t point_id, void* d_q_enc, float* d_q_off, cudaStream_t stream);

// selection (qb_topk.cu)
//  mode 0: write top-k (desc) of each query's candidate list to out/out_counts
//  mode 1: write the score of the k-th best candidate of each query to thr (or -inf when fewer than k)
qb_status qb_launch_select(const unsigned long long* d_cand, const unsigned int* d_cnt, unsigned long long cap,
                           unsigned long long fixed_n /* !=0: dense lists of this length */, uint32_t nq, uint32_t top, int mode,
                           qb_scored_point* d_out, uint32_t* d_out_counts, float* d_thr, unsigned int* d_overflow,
                           cudaStream_t stream);
qb_status qb_launch_fill_u32(unsigned int* p, unsigned int v, size_t n, cudaStream_t stream);

// dense preprocess of rows in place (qb_dense.cu)
qb_status qb_launch_preprocess_rows(qb_distance distance, uint32_t dim, uint64_t n, const float* in, uint64_t in_stride_f,
                                    float* out, uint64_t out_stride_f, cudaStream_t stream);
