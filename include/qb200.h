/*
 * qb200.h — C ABI of libqdrant_b200.so: Qdrant's vector-scoring hot path on NVIDIA H100 (sm_90a).
 *
 * This is the drop-in boundary.  The reference has no FFI seam for scorers; its seam is the Rust trait
 * object `RawScorer` (lib/segment/src/vector_storage/raw_scorer.rs:39-54) built by `RawScorerBuilder`
 * (:122-128) / `QuantizedVectorsRead::raw_scorer` (quantized_vectors/read_access.rs:26-34) and driven by
 * `BatchFilteredSearcher::peek_top_iter` (lib/segment/src/index/hnsw_index/point_scorer.rs:423-472) and
 * `FilteredScorer::score_points` (:265-295).  Each entry point below names the reference interface it
 * replaces.  INTEGRATION.md shows the Rust `extern "C"` block + `impl RawScorer` adapter a maintainer adds.
 *
 * Conventions
 *   - every function returns qb_status (0 = ok, < 0 = error); qb_last_error() gives the thread-local text.
 *     No exception crosses the ABI.  Scoring calls on valid handles fail only on CUDA errors, which the Rust
 *     adapter `expect`s exactly like the reference's `.expect("read vectors")` (metric_query_scorer.rs:91).
 *   - handles are opaque and owned by the library; host buffers are borrowed for the duration of a call;
 *     outputs are caller-allocated.
 *   - any thread may call any function.  One qb_scorer must not be used from two threads at once (the Rust
 *     `&mut FilteredScorer`), but many scorers / searches over one qb_storage may run concurrently
 *     (segments_searcher.rs:255): each scorer and each search context owns a CUDA stream.
 *   - there is NO CPU fallback: without a CUDA device every create call returns QB_ERR_NO_DEVICE.
 *   - "greater score = closer" everywhere, exactly as Metric::similarity (spaces/metric.rs:8-17).
 */
#ifndef QB200_H
#define QB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QB200_ABI_VERSION 2
#if defined(__GNUC__)
#define QB_API __attribute__((visibility("default")))
#else
#define QB_API
#endif

typedef int32_t qb_status;
enum {
    QB_OK = 0,
    QB_ERR_INVALID = -1,      /* bad argument (null, dim mismatch, id out of range, top == 0 ...) */
    QB_ERR_CUDA = -2,         /* CUDA runtime / driver error, text in qb_last_error() */
    QB_ERR_UNSUPPORTED = -3,  /* e.g. internal scorer on PQ (encode_internal_vector = None, encoded_vectors_pq.rs:624) */
    QB_ERR_OOM = -4,
    QB_ERR_CANCELLED = -5,    /* *is_stopped became non-zero (check_process_stopped, point_scorer.rs:433) */
    QB_ERR_NO_DEVICE = -6
};

/* Distance — same order as lib/segment/src/types.rs:313-322 */
typedef enum { QB_DIST_COSINE = 0, QB_DIST_EUCLID = 1, QB_DIST_DOT = 2, QB_DIST_MANHATTAN = 3 } qb_distance;
/* VectorStorageDatatype (types.rs) of a dense storage */
typedef enum { QB_DT_F32 = 0, QB_DT_F16 = 1, QB_DT_U8 = 2 } qb_dtype;
/* quantization::DistanceType — lib/quantization/src/encoded_vectors.rs:13 */
typedef enum { QB_QD_COSINE = 0, QB_QD_DOT = 1, QB_QD_L1 = 2, QB_QD_L2 = 3 } qb_qdistance;
/* BQ Encoding / QueryEncoding — lib/quantization/src/encoded_vectors_binary.rs:34-54 */
typedef enum { QB_BQ_ONE_BIT = 0, QB_BQ_TWO_BITS = 1, QB_BQ_ONE_AND_HALF_BITS = 2 } qb_bq_encoding;
typedef enum { QB_BQQ_SAME_AS_STORAGE = 0, QB_BQQ_SCALAR4 = 1, QB_BQQ_SCALAR8 = 2 } qb_bq_query_encoding;
/* QueryVector variants beyond Nearest (lib/segment/src/data_types/vectors.rs QueryVector; vector_storage/query/*.rs) */
typedef enum { QB_QUERY_RECO_BEST_SCORE = 1, QB_QUERY_RECO_SUM_SCORES = 2, QB_QUERY_DISCOVER = 3, QB_QUERY_CONTEXT = 4, QB_QUERY_FEEDBACK_NAIVE = 5 } qb_query_kind;

/* #[repr(C)] ScoredPointOffset — lib/common/common/src/types.rs:12-17 */
typedef struct { uint32_t idx; float score; } qb_scored_point;

/* HardwareCounterCell deltas a drop-in scorer must keep reporting (metric_query_scorer.rs:43-49,84-85;
 * encoded_vectors_u8.rs:785-787).  Values are already multiplied by the reference's multipliers. */
typedef struct { uint64_t cpu; uint64_t vector_io_read; } qb_hw_counters;

typedef struct qb_storage qb_storage;  /* one segment's vectors (dense or quantized) resident in HBM */
typedef struct qb_scorer qb_scorer;    /* Box<dyn RawScorer>: a preprocessed/encoded query bound to a storage */
typedef struct qb_sparse_storage qb_sparse_storage;   /* a sparse vector storage in user dims (qb_sparse_storage_create) */

/* ---------------------------------------------------------------- library / device ------------------ */
QB_API const char* qb_last_error(void);
QB_API int32_t qb_abi_version(void);
QB_API qb_status qb_device_count(int32_t* out);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
QB_API uint64_t qb_kernel_launch_count(void);
/* Debugging / experiment switches (README.md lists them); the QB_* environment variables of the same names are read once,
 * at first use, as defaults.  Not needed for normal operation. */
QB_API qb_status qb_set_option(const char* name, int64_t value);

/* ---------------------------------------------------------------- storages -------------------------- */
/* Dense vectors as the reference stores them: row-major, `dim` elements of `dt`, rows `row_stride_bytes`
 * apart (dense/immutable_dense_vectors.rs:100-113).  Cosine rows must already be normalised the way
 * Distance::preprocess_vector does at insert time (types.rs:334-347) — see qb_metric_preprocess.
 * host_rows may be NULL to allocate an empty storage filled later with qb_storage_write_rows*. */
QB_API qb_status qb_storage_create_dense(int32_t device, qb_dtype dt, qb_distance distance, uint32_t dim, uint64_t count,
                                  const void* host_rows, uint64_t row_stride_bytes, qb_storage** out);
/* chunked upload (the reference uploads in chunks too, UPLOAD_CHUNK_SIZE, gpu_vector_storage/mod.rs) */
QB_API qb_status qb_storage_write_rows(qb_storage* s, uint64_t first_row, uint64_t n_rows, const void* host_rows, uint64_t row_stride_bytes);
QB_API qb_status qb_storage_write_rows_device(qb_storage* s, uint64_t first_row, uint64_t n_rows, const void* dev_rows, uint64_t row_stride_bytes);
/* read back stored rows (dense storages; used by rescoring and by the full-size parity tests) */
QB_API qb_status qb_storage_read_rows(const qb_storage* s, const uint32_t* ids, uint64_t n, void* host_out);

/* Quantized storages.  `dt` + `invert` are the quantizer's VectorParameters (construct_vector_parameters,
 * quantized_vectors.rs:205-234: Cosine is stored as Dot, invert = Euclid || Manhattan); `metric` is the segment's
 * Distance and only decides Metric::preprocess of incoming queries (QuantizedQueryScorer::new,
 * quantized_query_scorer.rs:29-55).
 *
 * SQ8: rows exactly as `quantized.data` holds them — [f32 v_off][actual_dim u8], stride row_bytes =
 * 4 + ceil(dim/16)*16 (encoded_vectors_u8.rs:22,240-283,622-629) — plus MetadataInt8 (:84-91). */
QB_API qb_status qb_storage_create_sq8(int32_t device, uint32_t dim, uint64_t count, const uint8_t* rows, uint32_t row_bytes,
                                float alpha, float offset, float multiplier, qb_qdistance dt, int32_t invert,
                                qb_distance metric, qb_storage** out);
/* PQ: codes [count x m] u8, centroids as 256 (n_centroids) full-dim vectors and the chunk division
 * (Metadata, encoded_vectors_pq.rs:46-51); division = 2*m uint32 {start,end}. */
QB_API qb_status qb_storage_create_pq(int32_t device, uint32_t dim, uint32_t m, const uint32_t* div_start_end,
                               const float* centroids, uint32_t n_centroids, const uint8_t* codes, uint64_t count,
                               qb_qdistance dt, int32_t invert, qb_distance metric, qb_storage** out);
/* BQ: rows of row_bytes = ceil(bits/128)*16 (EncodedVectorsBin<u128>, single vectors, encoded_vectors_binary.rs:829-839) or
 * ceil(bits/8) (EncodedVectorsBin<u8>, the token rows of multivector storages, quantized_vectors.rs:270-282; zero-padded to u128 words
 * at upload); mean_std = dim x {mean, stddev} for the 2-bit / 1.5-bit encodings (VectorStats), or NULL. */
QB_API qb_status qb_storage_create_bq(int32_t device, uint32_t dim, qb_bq_encoding enc, qb_bq_query_encoding qenc,
                               const uint8_t* rows, uint32_t row_bytes, uint64_t count, qb_qdistance dt, int32_t invert,
                               const float* mean_std, qb_distance metric, qb_storage** out);
/* The same storages from a segment directory's files AS THEY LIE ON DISK (SURVEY Appendix C): the caller hands over the (mmapped) bytes.
 *   matrix.dat           b"data" + count x dim x size_of::<T>() row-major (dense/dense_vector_storage.rs:31, immutable_dense_vectors.rs:100-113);
 *                        every complete row after the header is loaded
 *   quantized.meta.json  serde_json of MetadataInt8 / PQ Metadata / BQ Metadata (encoded_vectors_u8.rs:84-91, encoded_vectors_pq.rs:46-51,
 *                        encoded_vectors_binary.rs:112-125) — the kind is recognised from its fields
 *   quantized.data       headerless rows of quantized_vector_size bytes (quantized/quantized_storage.rs:63-69); count = 0 means
 *                        "as many rows as the bytes hold" (mmap files are page-padded: pass the real count when known)
 * `metric` is the segment's Distance (decides Metric::preprocess of incoming queries), as in qb_storage_create_*. */
QB_API qb_status qb_storage_load_dense_file(int32_t device, qb_dtype dt, qb_distance distance, uint32_t dim, const uint8_t* file_bytes, uint64_t n_bytes,
                                            qb_storage** out);
QB_API qb_status qb_storage_load_quantized(int32_t device, qb_distance metric, const char* meta_json, uint64_t json_len, const uint8_t* data, uint64_t n_bytes,
                                           uint64_t count, qb_storage** out);
QB_API void qb_storage_destroy(qb_storage* s);

QB_API qb_status qb_storage_info(const qb_storage* s, uint32_t* dim, uint64_t* count, uint64_t* hbm_bytes);
/* Resident soft-delete flags (bit i = 1 => point i deleted): the storage-level `deleted` BitSlice that
 * ScorerFilters / not_deleted_checker consult (point_scorer.rs:351-352).  NULL clears. */
QB_API qb_status qb_storage_set_deleted(qb_storage* s, const uint64_t* bitmap_words, uint64_t n_words);
/* VectorStorage::is_on_disk of the segment storage this HBM copy caches: decides whether scoring calls meter
 * hardware_counter.vector_io_read (dim * size_of::<TElement>() per scored point for on-disk dense storages,
 * metric_query_scorer.rs:44-48; the quantized row size for on-disk quantized data, quantized_query_scorer.rs:48,84-86).
 * Default 0 (RAM storage: multiplier 0). */
QB_API qb_status qb_storage_set_on_disk(qb_storage* s, int32_t on_disk);
/* CUDA stream (cudaStream_t) of the storage's device-resident entry points (qb_search_batch_device,
 * qb_hnsw_search_batch_device) — for event timing and stream ordering; host-facing searches use pooled streams of their own */
QB_API void* qb_storage_stream(qb_storage* s);

/* Metric::preprocess for `n` vectors (spaces/metric.rs:14; cosine = cosine_preprocess_avx arithmetic,
 * simple_avx.rs:127-165).  in/out are host buffers of n*dim f32 (may alias). */
QB_API qb_status qb_metric_preprocess(int32_t device, qb_distance distance, uint32_t dim, uint64_t n, const float* in, float* out);
/* same, in place on device memory (synthetic data generated on the GPU) */
QB_API qb_status qb_metric_preprocess_device(int32_t device, qb_distance distance, uint32_t dim, uint64_t n, float* dev_rows, uint64_t row_stride_bytes);
/* MetricPostProcessing::postprocess applied by the caller at shard level (local_shard/search.rs:150-170) */
QB_API float qb_metric_postprocess(qb_distance distance, float score);

/* ---------------------------------------------------------------- RawScorer ------------------------- */
/* RawScorerBuilder::build_raw_scorer / QuantizedVectorsRead::raw_scorer for QueryVector::Nearest:
 * runs Metric::preprocess + (quantized) EncodedVectors::encode_query on the device. query = dim raw f32. */
QB_API qb_status qb_scorer_create(qb_storage* s, const float* query, qb_scorer** out);
/* QuantizedVectorsRead::raw_internal_scorer / FilteredScorer::new_internal: the stored point is the query.
 * QB_ERR_UNSUPPORTED for PQ (encoded_vectors_pq.rs:624-627), as in the reference. */
QB_API qb_status qb_scorer_create_internal(qb_storage* s, uint32_t point_id, qb_scorer** out);
QB_API void qb_scorer_destroy(qb_scorer* sc);
/* RawScorer::score_points(&[PointOffsetType], &mut [ScoreType]) — raw_scorer.rs:40 */
QB_API qb_status qb_score_points(qb_scorer* sc, const uint32_t* ids, size_t n, float* scores);
/* RawScorer::score_point — raw_scorer.rs:43 */
QB_API qb_status qb_score_point(qb_scorer* sc, uint32_t id, float* score);
/* RawScorer::score_internal — raw_scorer.rs:50 (QB_ERR_INVALID when an id is out of range; Rust adapter panics) */
QB_API qb_status qb_score_internal(qb_scorer* sc, uint32_t a, uint32_t b, float* score);
/* read and reset the hardware-counter deltas accumulated by this scorer */
QB_API qb_status qb_scorer_take_counters(qb_scorer* sc, qb_hw_counters* out);

/* ---------------------------------------------------------------- brute-force scan ------------------ */
/* BatchFilteredSearcher::{new, peek_top_iter} fused: scores every candidate point against every query and
 * keeps the `top` best per query, sorted by descending score (FixedLengthPriorityQueue::into_sorted_vec).
 *   queries        n_queries x dim raw f32 (preprocessed + encoded on the device)
 *   deleted_bitmap optional per-call soft-delete bits (bit=1 deleted), OR-ed with the resident flags; the caller
 *                  provides ceil(count / 64) 64-bit words (the library reads exactly that many)
 *   id_list/n_ids  optional explicit candidate ids (a payload filter's result); NULL = all rows
 *   is_stopped     optional cancellation flag, polled between kernel launches
 *   out            n_queries x top; out_counts[q] = number of valid entries (< top when fewer candidates)
 * Ties: ScoredPointOffset orders by score only, so which of several equal-score points survives at the
 * k-th boundary is unspecified in the reference; this library orders by (score desc, id asc).
 * How the scan is carried out never changes the result: large dense f32 storages keep compact shadow planes of their rows
 * (built on the first search that uses them, rebuilt after qb_storage_write_rows*: single-query searches on >= 2^19 rows take + 19 % HBM
 * for the 6-bit plane and + 14 % for its block-scaled 4-bit first stage at dim 768 (5.9 + 4.4 GB at 10M x 768; option prefilter_stage1 = 5
 * drops the latter), or + 26 % for the int8 plane, + 50 % for the bf16 plane of batches of >= 32 queries; dot / cosine only), batched SQ8 / PQ scans run
 * prefilter kernels — in every case the rows that can reach the top-k are re-scored with the reference's exact arithmetic before
 * selection, and a case the prefilter cannot decide falls back to the exact scan (qb_search_stats counts those).
 * qb_set_option("disable_prefilter" / "disable_mma", 1) keeps a process on the exact kernels and allocates no plane. */
QB_API qb_status qb_search_batch(qb_storage* s, const float* queries, uint32_t n_queries, uint32_t top,
                          const uint64_t* deleted_bitmap, const uint32_t* id_list, uint64_t n_ids,
                          const volatile int32_t* is_stopped, qb_scored_point* out, uint32_t* out_counts,
                          qb_hw_counters* counters /* optional */);
/* Same scan with queries and outputs already resident in HBM, enqueued on qb_storage_stream(s) (bench.py's
 * kernel-only `value`).  Paths with a fallback (threshold filter, tensor-core batch) wait for that stream once to
 * read the device's "fast-path assumption broken" flags word (reruns happen inside, as in qb_search_batch); the
 * single-pass paths (single-query dense f32 with top <= 16, small scans) return without synchronising.  It uses the storage's first search context:
 * do not run it concurrently with other searches on the same storage. */
QB_API qb_status qb_search_batch_device(qb_storage* s, const float* dev_queries, uint32_t n_queries, uint32_t top,
                                 qb_scored_point* dev_out, uint32_t* dev_counts);

/* ---------------------------------------------------------------- custom queries (SURVEY §8f rank 1) -- */
/* RawScorer for a recommend / discover / context query: CustomQueryScorer (query_scorer/custom_query_scorer.rs:16-122)
 * and QuantizedCustomQueryScorer.  Every example vector goes through Metric::preprocess (+ encode_query on quantized
 * storages) exactly like a plain query; a candidate's score is Query::score_by over its similarities to the examples:
 *   QB_QUERY_RECO_BEST_SCORE  vectors = n_a positives, then n_b negatives      (query/reco_query.rs:64-90)
 *   QB_QUERY_RECO_SUM_SCORES  same layout                                       (query/reco_query.rs:116-133)
 *   QB_QUERY_DISCOVER         vectors = target, then n_a (positive, negative) pairs; n_b = 0   (query/discover_query.rs:66-76)
 *   QB_QUERY_CONTEXT          vectors = n_a (positive, negative) pairs; n_b = 0  (query/context_query.rs:111-119)
 * The scorer works with qb_score_points / qb_score_point; qb_score_internal returns QB_ERR_UNSUPPORTED (the reference's
 * score_internal is unimplemented!() for custom scorers). */
QB_API qb_status qb_scorer_create_custom(qb_storage* s, qb_query_kind kind, const float* vectors, uint32_t n_a, uint32_t n_b, qb_scorer** out);
/* Brute-force scan with a custom query: BatchFilteredSearcher::peek_top_iter driven by a custom RawScorer.  Same
 * deleted_bitmap / id_list / is_stopped / out conventions as qb_search_batch, one query per call. */
QB_API qb_status qb_search_custom(qb_storage* s, qb_query_kind kind, const float* vectors, uint32_t n_a, uint32_t n_b, uint32_t top,
                                  const uint64_t* deleted_bitmap, const uint32_t* id_list, uint64_t n_ids, const volatile int32_t* is_stopped,
                                  qb_scored_point* out, uint32_t* out_count, qb_hw_counters* counters /* optional */);

/* QueryVector::FeedbackNaive — FeedbackQuery (vector_storage/query/feedback_query.rs:150-226, dispatched at raw_scorer.rs:322-323,
 * 376-377): score = a * sim(target) + sum over context pairs of partial_computation * (sim(positive) - sim(negative)), f32, the
 * product rounded before the add.  vectors = target, then n_pairs (positive, negative) pairs; `partial` = the pairs'
 * partial_computation values exactly as FeedbackQuery::new derived them (confidence^b * c, feedback_query.rs:121-146 — host
 * arithmetic on the feedback scores, done once per query by the caller). */
QB_API qb_status qb_scorer_create_feedback(qb_storage* s, const float* vectors, uint32_t n_pairs, float a, const float* partial, qb_scorer** out);
QB_API qb_status qb_search_feedback(qb_storage* s, const float* vectors, uint32_t n_pairs, float a, const float* partial, uint32_t top,
                                    const uint64_t* deleted_bitmap, const uint32_t* id_list, uint64_t n_ids, const volatile int32_t* is_stopped,
                                    qb_scored_point* out, uint32_t* out_count, qb_hw_counters* counters /* optional */);

/* ---------------------------------------------------------------- multivector MaxSim (SURVEY §8f rank 3) -- */
/* ColBERT MaxSim, score_max_similarity (vector_storage/query_scorer/mod.rs:77-98) as used by MultiMetricQueryScorer
 * (multi_metric_query_scorer.rs) and the quantized multivector storage: a point is a run of consecutive vectors of `s`
 * (point p = rows [point_offsets[p], point_offsets[p+1]), the layout of the reference's flattened multivector storage,
 * vector_storage/multi_dense/*.rs); score = sum over the query's vectors (sequential f32 from 0.0) of the best similarity
 * (`sim > max`, from -inf) to any vector of the point.  Similarities are the storage's ordinary bit-exact ones, so `s`
 * may be dense or quantized.  deleted_points: optional bitmap over POINTS (1 = skip). */
QB_API qb_status qb_search_maxsim(qb_storage* s, const uint32_t* point_offsets, uint32_t n_points, const float* query_vectors,
                                  uint32_t n_query_vectors, uint32_t top, const uint64_t* deleted_points, qb_scored_point* out, uint32_t* out_count,
                                  qb_hw_counters* counters /* optional */);
QB_API qb_status qb_score_maxsim(qb_storage* s, const uint32_t* point_offsets, uint32_t n_points, const float* query_vectors,
                                 uint32_t n_query_vectors, const uint32_t* point_ids, size_t n, float* scores);

/* MultiCustomQueryScorer / QuantizedMultiCustomQueryScorer (query_scorer/multi_custom_query_scorer.rs:88-104, quantized/
 * quantized_multi_custom_query_scorer.rs): a recommend / discover / context / feedback query whose EXAMPLES are multivectors.  A
 * point's similarity to an example is MaxSim (score_multi), the per-example similarities are folded by Query::score_by like the
 * single-vector custom queries.  example e = example_vectors rows [example_offsets[e], example_offsets[e + 1]) (raw f32 x dim), the
 * examples ordered as qb_scorer_create_custom / qb_scorer_create_feedback order their vectors; coef = [a, partial computations...] for
 * QB_QUERY_FEEDBACK_NAIVE, else NULL. */
QB_API qb_status qb_search_maxsim_custom(qb_storage* s, const uint32_t* point_offsets, uint32_t n_points, qb_query_kind kind, const float* example_vectors,
                                         const uint32_t* example_offsets, uint32_t n_a, uint32_t n_b, const float* coef, uint32_t top, const uint64_t* deleted_points,
                                         qb_scored_point* out, uint32_t* out_count, qb_hw_counters* counters /* optional */);
QB_API qb_status qb_score_maxsim_custom(qb_storage* s, const uint32_t* point_offsets, uint32_t n_points, qb_query_kind kind, const float* example_vectors,
                                        const uint32_t* example_offsets, uint32_t n_a, uint32_t n_b, const float* coef, const uint32_t* point_ids, size_t n, float* scores);

/* ---------------------------------------------------------------- quantizer encode on the device (SURVEY §8f rank 2) -- */
/* The ENCODE half of the quantizers, on f32 rows already resident in HBM; outputs are the reference's row formats bit
 * for bit and can be passed straight to qb_storage_create_{sq8,pq,bq} (device pointers are accepted there) or copied
 * into a segment's quantized.data.  Training (SQ quantiles, PQ k-means, BQ mean/std) stays with the caller.
 * row_stride_bytes = 0 means dim * 4.  `stream` is a cudaStream_t (NULL = default stream). */
/* alpha = (max - min) / 127, offset = min over all values: EncodedVectorsU8 with quantile = None (encoded_vectors_u8.rs:194-225,523-527) */
QB_API qb_status qb_sq8_find_alpha_offset_device(int32_t device, uint32_t dim, uint64_t count, const float* dev_rows, uint64_t row_stride_bytes,
                                                 float* alpha, float* offset);
/* EncodedVectorsU8::encode (encoded_vectors_u8.rs:240-283): dev_out = count x [f32 v_off][actual_dim u8], actual_dim = dim rounded up to 16 */
QB_API qb_status qb_sq8_encode_rows_device(int32_t device, uint32_t dim, uint64_t count, const float* dev_rows, uint64_t row_stride_bytes, float alpha,
                                           float offset, qb_qdistance dt, int invert, uint8_t* dev_out, void* stream);
/* get_quantized_vector_size_from_params for u128 words (encoded_vectors_binary.rs:829-839) */
QB_API uint32_t qb_bq_row_bytes(uint32_t dim, qb_bq_encoding encoding);
/* EncodedVectorsBin::encode_vector (encoded_vectors_binary.rs:531-671); mean_std = dim x (mean, stddev) on the HOST, NULL for one-bit */
QB_API qb_status qb_bq_encode_rows_device(int32_t device, uint32_t dim, uint64_t count, const float* dev_rows, uint64_t row_stride_bytes,
                                          qb_bq_encoding encoding, const float* mean_std, uint8_t* dev_out, void* stream);
/* EncodedVectorsPQ::encode_vector (encoded_vectors_pq.rs:301-329); centroids = n_centroids x dim on the HOST; dev_codes = count x ceil(dim / chunk) */
QB_API qb_status qb_pq_encode_rows_device(int32_t device, uint32_t dim, uint32_t chunk, uint32_t n_centroids, const float* centroids, uint64_t count,
                                          const float* dev_rows, uint64_t row_stride_bytes, uint8_t* dev_codes, void* stream);

/* ---------------------------------------------------------------- quantizer TRAINING on the device (SURVEY §8f rank 2) -- */
/* The steps before encode.  What the reference computes deterministically is reproduced operation for operation; what it draws from an
 * unseeded RNG is an input: the caller passes the sampled vectors (the reference samples rows with a randomly keyed Permutor,
 * quantile.rs:286-314, encoded_vectors_pq.rs:365-372) and a seed for re-seeding empty k-means clusters (kmeans.rs:113-121).
 * row_stride_bytes = 0 means dim * 4; all row pointers are DEVICE memory, outputs are host memory. */
/* VectorStats::build (vector_stats.rs:48-117): per-coordinate f64 Welford over ALL `count` rows in order -> mean_std_out = dim x
 * {mean, stddev} (what qb_storage_create_bq / qb_bq_encode_rows_device take), min_max_out = dim x {min, max} or NULL */
QB_API qb_status qb_bq_vector_stats_device(int32_t device, uint32_t dim, uint64_t count, const float* dev_rows, uint64_t row_stride_bytes, float* mean_std_out,
                                           float* min_max_out);
/* find_quantile_interval (quantile.rs:35-88) on the n_sample sampled vectors + alpha_offset_from_min_max (encoded_vectors_u8.rs:523-527).
 * *found = 0 when the reference would return None (keep the min/max alpha / offset of qb_sq8_find_alpha_offset_device). */
QB_API qb_status qb_sq8_quantile_interval_device(int32_t device, uint32_t dim, uint64_t n_sample, const float* dev_sample_rows, uint64_t row_stride_bytes,
                                                 float quantile, float* alpha, float* offset, int32_t* found);
/* EncodedVectorsPQ::find_centroids -> kmeans (encoded_vectors_pq.rs:342-407, kmeans.rs:9-167) on the sampled vectors, all chunks at once:
 * first-minimum assignment on sequential f32 squared distances, means as f64 partial sums over `max_threads` contiguous sample ranges
 * merged in range order (update_centroids' per-thread counters), stop when the L1 shift of a chunk's centroids < accuracy or after
 * max_iterations (reference: 100, 1e-5, KMEANS_SAMPLE_SIZE = 10 000 vectors).  centroids_out = n_centroids x dim (Metadata.centroids).
 * iterations_out (optional) = Lloyd iterations launched (a multiple-of-4 upper bound of the slowest chunk's count). */
QB_API qb_status qb_pq_train_device(int32_t device, uint32_t dim, uint32_t chunk, uint32_t n_centroids, uint64_t n_sample, const float* dev_sample_rows,
                                    uint64_t row_stride_bytes, uint32_t max_iterations, float accuracy, uint32_t max_threads, uint64_t seed, float* centroids_out,
                                    uint32_t* iterations_out);

/* Oversampling + rescoring contract (index/vector_index_search_common.rs:27-91): rescore `n` candidate ids of
 * one query with the ORIGINAL-vector scorer `orig`, sort descending, truncate to `top`. */
QB_API qb_status qb_rescore(qb_scorer* orig, const uint32_t* ids, size_t n, uint32_t top, qb_scored_point* out, uint32_t* out_count);

/* ---------------------------------------------------------------- sharded segments (multi-GPU) ------- */
/* Rows of a sharded data set live on several GPUs (one process per GPU); ids reported by searches on this shard
 * are `local row + id_base`, and every id-taking entry point (qb_score_points, qb_score_internal, qb_scorer_create_internal,
 * qb_rescore, qb_storage_read_rows, the id_list of qb_search_batch / qb_search_custom) takes ids in that same numbering,
 * i.e. id_base <= id < id_base + count.  Bitmaps (deleted flags) stay indexed by local row. */
QB_API qb_status qb_storage_set_id_base(qb_storage* s, uint32_t id_base);
/* BatchResultAggregator (lib/shard/src/search_result_aggregator.rs:50-117) on the device: merge `n_lists` per-shard
 * top-k lists per query — as all-gathered over NVLink by the caller: dev_lists[n_lists][n_queries][top],
 * dev_counts[n_lists][n_queries] — into dev_out[n_queries][top].  dev_scratch >= n_queries*n_lists*top*8 bytes.
 * Enqueued on `stream` (cudaStream_t), no host synchronisation. */
QB_API qb_status qb_topk_merge_device(int32_t device, const qb_scored_point* dev_lists, const uint32_t* dev_counts, uint32_t n_lists,
                                      uint32_t n_queries, uint32_t top, qb_scored_point* dev_out, uint32_t* dev_out_counts,
                                      void* dev_scratch, uint64_t scratch_bytes, void* stream);

/* A sharded search as ONE collective per shard (SURVEY §8e).  The reference runs one blocking task per segment and merges the
 * tasks' lists on the host (segments_searcher.rs:255 -> BatchResultAggregator, search_result_aggregator.rs:50-117); here the
 * task of every shard calls qb_multi_search_batch with the same queries, the `n_queries x top x 8 B` lists cross GPUs through
 * peer-mapped exchange buffers over NVLink (no NCCL call, no host hop) and every caller receives the merged top-k.
 *   - one qb_comm per shard / GPU: qb_comm_create(device, rank, world, ...).
 *   - shards in ONE process (threads): qb_comm_connect_local(all comms) enables peer access and wires them up.
 *   - shards in separate processes (one per GPU): each publishes qb_comm_local_handle (64 bytes, a CUDA IPC handle), the host
 *     gathers the `world` handles by whatever transport it has, and every rank calls qb_comm_connect(handles).
 *   - every rank must issue the same sequence of qb_multi_search_batch* calls (same n_queries / top), like any collective.
 *   world x max_top <= 4096. */
typedef struct qb_comm qb_comm;
QB_API qb_status qb_comm_create(int32_t device, int32_t rank, int32_t world, uint32_t max_queries, uint32_t max_top, qb_comm** out);
QB_API qb_status qb_comm_local_handle(qb_comm* c, uint8_t* handle_out /* 64 bytes */);
QB_API qb_status qb_comm_connect(qb_comm* c, const uint8_t* handles /* world x 64 bytes, indexed by rank */);
QB_API qb_status qb_comm_connect_local(qb_comm* const* comms, int32_t n);
QB_API void qb_comm_destroy(qb_comm* c);
/* qb_search_batch over this rank's shard (ids = local row + id_base) + exchange + merge: out = the global top-k, on every rank */
QB_API qb_status qb_multi_search_batch(qb_comm* c, qb_storage* shard, const float* queries, uint32_t n_queries, uint32_t top,
                                       const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped, qb_scored_point* out,
                                       uint32_t* out_counts, qb_hw_counters* counters /* optional */);
/* same with queries / outputs resident in HBM, no host synchronisation on the exact single-pass paths.
 *   dev_local / dev_local_counts != NULL: they receive the shard's own lists (n_queries x top, n_queries); scan, exchange and merge are all
 *     enqueued on qb_storage_stream(shard).
 *   dev_local == NULL (both): PIPELINED — the scan runs on qb_storage_stream(shard), the exchange + merge on qb_comm_stream(c), and the next
 *     call's scan does not wait for this call's merge (a window of two steps over rings of four list buffers / exchange slots): consecutive independent query
 *     batches overlap across GPUs instead of meeting at a barrier per batch.  dev_out / dev_counts of a call are complete once
 *     qb_comm_stream(c) has drained; successive calls write them in order. */
QB_API qb_status qb_multi_search_batch_device(qb_comm* c, qb_storage* shard, const float* dev_queries, uint32_t n_queries, uint32_t top,
                                              qb_scored_point* dev_local, uint32_t* dev_local_counts, qb_scored_point* dev_out, uint32_t* dev_counts);
/* cudaStream_t the pipelined exchange + merge kernels run on */
QB_API void* qb_comm_stream(qb_comm* c);
/* synchronise qb_comm_stream(c) and report a failed exchange of the device-resident calls made so far (a peer that never made the matching
 * call: the waiting rank gives up after ~10 s, leaves that step's results empty and this returns QB_ERR_CUDA) */
QB_API qb_status qb_comm_check(qb_comm* c);

/* ---------------------------------------------------------------- HNSW graph search on the device ---- */
/* GraphLayers::search (lib/segment/src/index/hnsw_index/graph_layers.rs:530-561) for a BATCH of queries with the
 * traversal itself on the GPU: search_entry (greedy descent through the upper levels, :247-316) and search_on_level
 * (beam search on level 0 with SearchContext, :108-148, search_context.rs:8-41), every hop scored with the storage's
 * bit-exact per-pair arithmetic.  This is the throughput form of `RawScorer` under HNSW: the per-hop qb_score_points
 * boundary stays available (qb_scorer_*), this entry removes it.
 *
 * links_bin = the bytes of the segment's `links.bin` in GraphLinksFormat::Plain (graph_links/header.rs:9-20,
 * graph_links/view.rs:121-135): HeaderPlain, level offsets, reindex, neighbors, padding, offsets.  m / m0 = HnswM
 * (hnsw_index/mod.rs:34-40), both <= 64.  The graph is bound to `s` (dense f32, dense Uint8 or SQ8; the quantized storage when
 * the segment searches quantized) and must outlive neither it nor its searches.  Float16 storages load but are not searched on the
 * device (QB_ERR_UNSUPPORTED). */
typedef struct qb_hnsw qb_hnsw;
QB_API qb_status qb_hnsw_create_plain(qb_storage* s, const uint8_t* links_bin, uint64_t n_bytes, uint32_t m, uint32_t m0, qb_hnsw** out);
/* The same graph from `links.bin` in GraphLinksFormat::Compressed, the format the reference writes for every HNSW index it
 * builds (graph_links/header.rs:22-34, view.rs:137-163; hnsw/build.rs:548-562).  m / m0 come from the header.  The file is
 * copied to the device once and decoded there into the arrays qb_hnsw_create_plain uploads; the search is the same.
 * Every value taken from the file is checked before it is followed: a malformed file returns QB_ERR_INVALID and leaves the
 * device usable.  CompressedWithVectors (version word ...FF02, inline storage) and m0 > 64 return QB_ERR_UNSUPPORTED: those
 * graphs load through qb_hnsw_create_with_vectors below. */
QB_API qb_status qb_hnsw_create_compressed(qb_storage* s, const uint8_t* bytes, uint64_t n_bytes, qb_hnsw** out);
/* A graph from `links.bin` in GraphLinksFormat::CompressedWithVectors, which the reference writes for an index with
 * HnswConfig.inline_storage and quantization (graph_links/header.rs:37-70, serializer.rs:91-171, view.rs:165-207,276-352): each
 * level-0 record holds the point's original vector (base), and every link is followed by that neighbour's quantized vector.
 *   s   the segment's SQ8 storage: link vectors are its rows ([f32 offset][actual_dim codes], layout alignment 1), and the link
 *       layout size must be 4 + actual_dim (QB_ERR_INVALID otherwise).  BQ / PQ / dense storages: QB_ERR_UNSUPPORTED.
 *   base vectors must be f32 (layout size dim * 4); f16 / u8 base layouts return QB_ERR_UNSUPPORTED, any other size QB_ERR_INVALID.
 *       They live in the file, so the original f32 storage need not be resident.
 * Every value is checked as qb_hnsw_create_compressed checks it, and every record's count (varint), packed links, padding,
 * link vectors and (level 0) base vector must end inside the record: a malformed file returns QB_ERR_INVALID and leaves the
 * device usable; a list of more than 128 links returns QB_ERR_UNSUPPORTED.  The links are decoded into the arrays the other
 * loaders fill, so qb_hnsw_links, qb_hnsw_export_plain and the regular searches (HNSW, ACORN, custom) work on this handle; the
 * records stay resident for qb_hnsw_search_with_vectors_batch.  HBM: the records (about dim * 4 + m0 * (actual_dim + 4) bytes per
 * point: ~28 KB at 768-d and m0 = 32, so ~28 GB per million points), the plain arrays and 8 bytes per entry and per point of
 * offsets; qb_hnsw_info reports the total.  Synchronous. */
QB_API qb_status qb_hnsw_create_with_vectors(qb_storage* quantized, const uint8_t* bytes, uint64_t n_bytes, qb_hnsw** out);
/* GraphLinks::links (view.rs:238-263) for n_ids points on one level, from the device-resident graph of either loader:
 * out[i * cap .. i * cap + min(counts[i], cap)) = point ids[i]'s links in the graph's stored order, counts[i] = their full
 * number.  QB_ERR_INVALID when a point is out of range or its top level is below `level` (view.rs:354-369).  Synchronous. */
QB_API qb_status qb_hnsw_links(const qb_hnsw* g, uint32_t level, const uint32_t* ids, uint32_t n_ids, uint32_t cap, uint32_t* out /* n_ids x cap */,
                               uint32_t* counts);
QB_API void qb_hnsw_destroy(qb_hnsw* g);
QB_API qb_status qb_hnsw_info(const qb_hnsw* g, uint32_t* n_points, uint32_t* levels, uint64_t* hbm_bytes);
/* Builds the HNSW graph of a dense f32 or Uint8 storage on the device, with the schedule of the reference's GPU builder
 * (gpu/gpu_graph_builder.rs:19-101, gpu_level_builder.rs:12-96, batched_points.rs:36-163) and the CPU builder's per-point
 * arithmetic (search_on_level with ef = max(ef_construct, m0), fill_from_sorted_with_heuristic, connect_with_heuristic):
 *   - points sorted by level descending, then id; the first is the entry point (returned in entry_point / entry_level);
 *   - the first serial_points points of that order are inserted one at a time (0 = 256, SINGLE_THREADED_HNSW_BUILD_THRESHOLD);
 *   - the rest in batches of at most `batch` points on one level (0 = 512, GPU_GROUPS_COUNT_DEFAULT), level by level from the top.
 * A batch's points search the level as it was before the batch; their backlinks are then applied target by target in batch order
 * (the reference races them under per-point locks).  So the graph is a pure function of (rows, levels, m, m0, ef_construct, batch,
 * serial_points): two builds give the same graph, and batch = 1 gives the serial CPU build in the sorted order.
 *   levels    one per point, <= 30: the reference draws them from an unseeded RNG (get_random_layer), the caller draws them here
 * Points with the storage's resident deleted flag (qb_storage_set_deleted) are not inserted (iter_internal_excluding(deleted)): they keep
 * their level and have no links.  m, m0 <= 64 and ef <= 4096 (else QB_ERR_UNSUPPORTED); a level > 30, an empty storage or no point left
 * to insert: QB_ERR_INVALID.  Other storages (Float16 included): QB_ERR_UNSUPPORTED (build over the original vectors, then bind the
 * exported graph to the quantized storage).  The result is the handle qb_hnsw_create_plain would make from the graph's plain links.bin.
 * Uint8: an insert's query is the point's stored row, and every score is Metric<u8>::similarity of two stored rows (score_internal),
 * as both reference builders score u8 (FilteredScorer::new_internal, run_insert_vector.comp:41).  Its Dot / Euclid / Manhattan scores
 * are integers, so ties are common: the graph equals the reference's build with every level-0 comparison of the inserts' searches on
 * (score desc, id asc) keys; the greedy descent through the upper levels moves only to a strictly greater score.  Synchronous. */
QB_API qb_status qb_hnsw_build(qb_storage* s, uint32_t m, uint32_t m0, uint32_t ef_construct, const uint8_t* levels /* n */, uint32_t batch,
                               uint32_t serial_points, qb_hnsw** out, uint32_t* entry_point, uint32_t* entry_level);
/* Builds a segment's graph incrementally on the device: the old segment's graph is healed where its points have gone, renumbered into
 * this storage's ids and extended with the points it did not have (hnsw/build.rs:225-357 with an old index; the reference's own GPU
 * builder drops the old graph instead, build.rs:259-274).  In the reference's order:
 *   1. to-heal items: every (point, level) of `old` whose first level_m links (in the handle's stored order) include an unmapped point,
 *      point ascending, then level ascending (GraphLayersHealer::new over to_edges_impl, graph_layers_healer.rs:33-47,
 *      graph_links/links.rs:174-186), unmapped points included, as the reference does;
 *   2. each item is healed as heal_point_on_level does it (graph_layers_healer.rs:82-207): a stack-based search through the unmapped
 *      points collects the ef_construct best border points, fill_from_sorted_with_heuristic keeps up to level_m - |valid links| of
 *      them, the valid links follow, and every kept link gets a backlink (connect_with_heuristic) unless it holds the item already.
 *      The query is the item's stored row in old's storage;
 *   3. the reference heals in parallel under per-list locks; here each level heals in two phases: every item searches the lists as
 *      loaded and writes its own list, then the backlinks are applied target by target in item order, the "already linked" test
 *      made as each is applied.  The graph is a pure function of the inputs;
 *   4. each mapped point's lists move to its new id without the unmapped links (save_into_builder, :236-256); the entry is the first
 *      mapped point, in old-offset order, with the strictly highest level (EntryPoints::new_point, entry_points.rs:46-86);
 *   5. the points of s that are neither mapped nor resident-deleted are inserted with qb_hnsw_build's schedule and arithmetic (ef =
 *      max(ef_construct, m0)), the first serial_points of them one at a time.  A new point above the top links up to the top from
 *      the entry and becomes the entry (link_new_point, graph_layers_builder.rs:417-475); batch = 1 equals serial insertion.
 *   old_to_new  one per old point: its id in s, or 0xFFFFFFFF (not carried over)
 *   levels      one per point of s, <= 30; a mapped point's must equal its old level (build.rs:235-239)
 * m / m0 are old's (the reference reuses no graph of another configuration, old_index.rs:67-71); batch / serial_points as for
 * qb_hnsw_build (0 = 512 / 256).  The decision to reuse a graph (OldIndexCandidate::evaluate, healing_threshold) stays with the
 * caller.  Errors, checked before any device work: s not dense f32 or Uint8, old's storage not of s's datatype (f32 and Uint8 do not
 * mix), another dim / distance / device, a multivector
 * or inline-vector (CompressedWithVectors, old_index.rs:72-76) handle, ef > 4096: QB_ERR_UNSUPPORTED; a null argument, ef_construct
 * = 0, a target >= s's count, two old points on one target, a target with the resident deleted flag, no mapped point (build from
 * scratch with qb_hnsw_build), a level > 30 or a mapped level that differs: QB_ERR_INVALID.  Healing and inserting read the stored
 * f32 or Uint8 rows (quantized vectors are out of scope, as for qb_hnsw_build).  Uint8: the keyed tie contract of qb_hnsw_build, in
 * the inserts and in the heal's `nearest` (the heal's stack test stays score-only, as in the reference).  The result is the handle
 * qb_hnsw_create_plain would make from the new graph's plain links.bin, bound to s.  Synchronous. */
QB_API qb_status qb_hnsw_build_incremental(qb_storage* s, const qb_hnsw* old, const uint32_t* old_to_new /* old n_points */, uint32_t ef_construct,
                                           const uint8_t* levels /* s->count */, uint32_t batch, uint32_t serial_points, qb_hnsw** out,
                                           uint32_t* entry_point, uint32_t* entry_level);
/* The graph of any handle as a plain links.bin (graph_links/header.rs:9-20, serializer.rs:53-200).  *n_bytes = its size; out = NULL
 * asks for the size only, else cap must hold it (QB_ERR_INVALID).  Synchronous. */
QB_API qb_status qb_hnsw_export_plain(const qb_hnsw* g, uint8_t* out, uint64_t cap, uint64_t* n_bytes);
/*   queries         n_queries x dim raw f32 (Metric::preprocess + encode_query on the device)
 *   ef              beam width; max(ef, top) is used (graph_layers.rs:551)
 *   entry_point / entry_level   GraphLayers::get_entry_point's answer (entry_points.rs; it depends on the filter, so the
 *                   host passes it per call)
 *   deleted_bitmap  optional filter (bit = 1: point fails ScorerFilters::check_vector), OR-ed with the resident flags;
 *                   filtered-out links are neither scored nor traversed (point_scorer.rs:270-277)
 *   out             n_queries x top, descending; out_counts[q] valid entries
 * Result lists equal the reference traversal's whenever scores are distinct (ties are ordered by id).  Storages: dense f32, dense
 * Uint8 (queries `x as u8` after Metric<u8>::preprocess, the identity even for Cosine; counters cpu += dim per scored point,
 * vector_io_read += dim on disk) and SQ8; Float16: QB_ERR_UNSUPPORTED (qb_score_points per hop).  Uint8 Dot / Euclid / Manhattan
 * scores are integers, so ties are common there: lists equal the reference traversal with every level-0 comparison on (score desc,
 * id asc) keys; the greedy upper-level descent moves only to a strictly greater score. */
QB_API qb_status qb_hnsw_search_batch(qb_hnsw* g, const float* queries, uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point,
                                      uint32_t entry_level, const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped,
                                      qb_scored_point* out, uint32_t* out_counts, qb_hw_counters* counters /* optional */);
/* same with queries / outputs resident in HBM, enqueued on qb_storage_stream(s); no host synchronisation */
QB_API qb_status qb_hnsw_search_batch_device(qb_hnsw* g, const float* dev_queries, uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point,
                                             uint32_t entry_level, qb_scored_point* dev_out, uint32_t* dev_counts);
/* The level-0 algorithm of GraphLayers::search (SearchAlgorithm, graph_layers.rs:80-84); search_entry through the upper
 * levels is the same for both.
 *   QB_HNSW_ALGO_HNSW   search_on_level (:108-148): links that fail the filter are neither scored nor traversed.
 *   QB_HNSW_ALGO_ACORN  search_on_level_acorn (:154-243), ACORN-1: a filtered-out link is explored instead, and those of its own
 *                       links that pass the filter are scored (up to m0 per explored list).  Hops and scored points are counted
 *                       per scorer call, as for HNSW.  Unfiltered, it visits and scores exactly what HNSW does.
 * The choice stays with the caller, as in hnsw/read_view/search.rs:59-86: ACORN when the request sets
 * SearchParams.acorn.enable, the graph has m0 != 0, there is a filter, and the filter's estimated cardinality over the
 * segment's available points is at most acorn.max_selectivity (default 0.4, types.rs:622); HNSW otherwise.  Searches over a
 * CompressedWithVectors graph never use ACORN (search.rs:91-92); qb_hnsw_search_with_vectors_batch serves them.  ACORN uses the
 * same visited state as HNSW; its per-hop buffers take up to 16 * m0 * m0 bytes of shared memory per query in flight. */
typedef enum { QB_HNSW_ALGO_HNSW = 0, QB_HNSW_ALGO_ACORN = 1 } qb_hnsw_algorithm;
/* qb_hnsw_search_batch / qb_hnsw_search_batch_device with the level-0 algorithm chosen; the two calls above are these with
 * QB_HNSW_ALGO_HNSW */
QB_API qb_status qb_hnsw_search_batch_algo(qb_hnsw* g, const float* queries, uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point,
                                           uint32_t entry_level, const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped,
                                           qb_scored_point* out, uint32_t* out_counts, qb_hw_counters* counters /* optional */,
                                           qb_hnsw_algorithm algorithm);
QB_API qb_status qb_hnsw_search_batch_device_algo(qb_hnsw* g, const float* dev_queries, uint32_t n_queries, uint32_t top, uint32_t ef,
                                                  uint32_t entry_point, uint32_t entry_level, qb_scored_point* dev_out, uint32_t* dev_counts,
                                                  qb_hnsw_algorithm algorithm);
/* scorer calls (hops) and scored points since the last reset, summed over all searches on this graph (waits for them).  For
 * qb_hnsw_search_with_vectors_batch: hops and link-scored points (the entry point's score included); base scores are not
 * counted here (one per popped candidate; they show in the cpu counter). */
QB_API qb_status qb_hnsw_stats(qb_hnsw* g, uint64_t* hops, uint64_t* scored_points, int32_t reset);
/* GraphLayers::search_with_vectors (graph_layers.rs:336-452,564-596) on a qb_hnsw_create_with_vectors handle; the same arguments as
 * qb_hnsw_search_batch, and QB_ERR_UNSUPPORTED on a handle without inline vectors.  The caller passes ef = max(ef, oversampled top)
 * as search.rs:128 does; max(top, ef) is used.  Which search a request takes stays with the caller (hnsw/read_view/search.rs:88-178):
 * this one when the graph has inline vectors, the search is quantized and the algorithm is HNSW; otherwise the regular search on
 * the same handle.
 *   - the query is Metric::preprocess-ed for the storage's distance, then SQ8-encoded for the link scores;
 *   - the entry point is scored from the storage's SQ8 row; upper levels move greedily on the inline link vectors;
 *   - level 0 runs the beam on link scores (filter, then truncate to m0, then score) and scores every candidate it pops exactly
 *     from its base vector (the f32 chain of qb_score_points on a dense storage), including the candidate whose pop ends the
 *     search below the beam's lower bound;
 *   - the result is the best `top` exact scores, with no rescoring step.
 * Ties: every level-0 comparison, in both lists, orders by (score desc, id asc).  Duplicate ids within one list are outside the
 * contract (the first copy is scored).  Counters: cpu = link-scored points (the entry included) * dim + base-scored points * dim * 4;
 * vector_io_read = the entry's quantized row per query for on-disk storages; inline bytes never count.
 * Not covered: BQ / PQ link vectors, f16 / u8 base vectors, custom queries (the reference scores recommend / context / discover /
 * feedback through the inline vectors as well; here they run as the regular device search on this handle, which differs from the
 * reference on inline segments), ACORN (the reference has none with vectors), writing such files. */
QB_API qb_status qb_hnsw_search_with_vectors_batch(qb_hnsw* g, const float* queries, uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point,
                                                   uint32_t entry_level, const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped,
                                                   qb_scored_point* out, uint32_t* out_counts, qb_hw_counters* counters /* optional */);
/* same with queries / outputs resident in HBM, enqueued on qb_storage_stream(s); no host synchronisation */
QB_API qb_status qb_hnsw_search_with_vectors_batch_device(qb_hnsw* g, const float* dev_queries, uint32_t n_queries, uint32_t top, uint32_t ef,
                                                          uint32_t entry_point, uint32_t entry_level, qb_scored_point* dev_out, uint32_t* dev_counts);

/* A graph over the POINTS of a multivector collection whose token rows live in `tokens` (dense f32 or SQ8; others:
 * QB_ERR_UNSUPPORTED).  point p = token rows [point_offsets[p], point_offsets[p+1]) — the layout of qb_search_maxsim; the offsets
 * must ascend and end at or before the storage's count (QB_ERR_INVALID).  The graph's point count must equal n_points
 * (QB_ERR_INVALID otherwise).  The offsets are copied to the device (4 * (n_points + 1) bytes, in qb_hnsw_info's total).  The files
 * are read and checked as qb_hnsw_create_plain / qb_hnsw_create_compressed read them; CompressedWithVectors: QB_ERR_UNSUPPORTED.
 * This is the graph the reference builds for a multivector named vector with an HNSW index (a links.bin like any other), searched
 * through GraphLayers::search with MultiMetricQueryScorer (query_scorer/multi_metric_query_scorer.rs) for dense tokens and
 * QuantizedMultivectorStorage::score_point_max_similarity (quantized/quantized_multivector_storage/mod.rs:328-352) for SQ8 tokens.
 * qb_hnsw_links, qb_hnsw_export_plain, qb_hnsw_info, qb_hnsw_stats and qb_hnsw_destroy work on the handle; the single-vector searches
 * (qb_hnsw_search_batch*, _custom_, _discover_, _with_vectors_) return QB_ERR_UNSUPPORTED.  Search it with qb_hnsw_search_maxsim_batch
 * (nearest queries) and qb_hnsw_search_maxsim_custom_batch / qb_hnsw_search_maxsim_discover_batch (custom queries with multivector
 * examples).  Synchronous. */
QB_API qb_status qb_hnsw_create_plain_multivector(qb_storage* tokens, const uint32_t* point_offsets, uint32_t n_points, const uint8_t* links_bin,
                                                  uint64_t n_bytes, uint32_t m, uint32_t m0, qb_hnsw** out);
QB_API qb_status qb_hnsw_create_compressed_multivector(qb_storage* tokens, const uint32_t* point_offsets, uint32_t n_points, const uint8_t* bytes,
                                                       uint64_t n_bytes, qb_hnsw** out);
/* Builds the graph over the POINTS of a multivector collection on the device: qb_hnsw_build's schedule and arithmetic (levels
 * descending then id, serial_points batches of one, batches of at most `batch` cut where the level changes, two-phase backlinks), so the
 * graph is a pure function of its inputs, with every score the MaxSim S(a, b) of two stored points: point a's token rows are the
 * query, scored against point b's rows with the arithmetic of qb_hnsw_search_maxsim_batch (per query row the sequential `sim > max`
 * fold from -inf, the maxima summed in row order from +0.0).  An insert's search scores S(inserted, p); the heuristic keeps a
 * candidate c unless S(c, kept) > S(inserted, c) for a kept link; connect_with_heuristic scores S(target, link)
 * (MultiMetricQueryScorer::score_internal behind FilteredScorer::new_internal, multi_metric_query_scorer.rs:64-121).
 *   tokens, point_offsets, n_points   the layout qb_hnsw_create_plain_multivector takes, checked the same way (QB_ERR_INVALID)
 *   deleted_points  optional bitmap over POINTS, ceil(n_points / 64) words: such a point is not inserted, keeps its level and has
 *                   no links.  The token storage's resident flags are per row and do not apply.
 * The query is the stored token rows as they are, as qb_scorer_create_internal and qb_hnsw_build use them; the reference passes
 * them through Metric::preprocess again, which leaves a cosine row unchanged when its squared length is within 1e-6 of 1
 * (spaces/tools.rs:14-16), so the two agree on rows the storage normalised.  A point with no token rows scores +0.0 against every
 * point as the query and -inf as the scored point.  Errors: f16 / u8 / SQ8 / PQ / BQ tokens, m or m0 > 64 or ef > 4096:
 * QB_ERR_UNSUPPORTED (build over the f32 tokens, then bind the exported graph to the quantized storage); bad offsets, a level > 30,
 * n_points = 0 or every point deleted: QB_ERR_INVALID.  The result is the handle qb_hnsw_create_plain_multivector would make from the
 * graph's plain links.bin with the same offsets: search it with qb_hnsw_search_maxsim_batch.  Synchronous. */
QB_API qb_status qb_hnsw_build_multivector(qb_storage* tokens, const uint32_t* point_offsets, uint32_t n_points, uint32_t m, uint32_t m0,
                                           uint32_t ef_construct, const uint8_t* levels /* n_points */, const uint64_t* deleted_points,
                                           uint32_t batch, uint32_t serial_points, qb_hnsw** out, uint32_t* entry_point, uint32_t* entry_level);
/* GraphLayers::search (graph_layers.rs:530-561) with a MaxSim FilteredScorer, for a batch of multivector queries, on a
 * qb_hnsw_create_*_multivector handle (QB_ERR_UNSUPPORTED on any other).  Replaces the per-hop qb_score_maxsim boundary.
 *   query i         rows [query_offsets[i], query_offsets[i+1]) of query_vectors (raw f32 x dim), 1..4096 vectors each
 *   deleted_points  optional bitmap over POINTS, ceil(n_points / 64) words, as qb_search_maxsim takes it; a point that fails it is
 *                   neither scored nor traversed.  The token storage's resident deleted flags are per token row and do not apply.
 *   out             point offsets 0 .. n_points - 1 (the numbering of qb_search_maxsim), descending
 * The other arguments and the traversal are qb_hnsw_search_batch_algo's (max(ef, top), ef <= 4096, keyed ties, is_stopped).
 * A point's score equals qb_score_maxsim on that point bit for bit: each query vector prepared as a plain query, every (vector,
 * token) similarity by the storage's chain, per vector the sequential `sim > max` fold over the point's tokens from -inf (NaN
 * never wins, the earlier of -0.0 / +0.0 keeps its bits, an empty run stays -inf), the maxima summed in vector order from +0.0.
 * (For SQ8 tokens the reference sums with Iterator::sum, which starts from -0.0: the two differ only when every maximum is -0.0.)
 * Counters: cpu += query vectors x token rows x the storage's per-vector units per scored point (dim * 4 for f32, dim for SQ8),
 * vector_io_read += token rows x the row size on disk.  qb_hnsw_stats counts hops and scored points (points, not token rows). */
QB_API qb_status qb_hnsw_search_maxsim_batch(qb_hnsw* g, const float* query_vectors, const uint32_t* query_offsets, uint32_t n_queries, uint32_t top,
                                             uint32_t ef, uint32_t entry_point, uint32_t entry_level, const uint64_t* deleted_points,
                                             const volatile int32_t* is_stopped, qb_scored_point* out, uint32_t* out_counts,
                                             qb_hw_counters* counters /* optional */, qb_hnsw_algorithm algorithm);
/* same with query vectors (n_query_vectors x dim), offsets (n_queries + 1) and outputs resident in HBM, enqueued on
 * qb_storage_stream(tokens), no host synchronisation and no filter.  max_query_vectors (1..4096) bounds the largest query's vector
 * count; it sizes the shared-memory staging of the query vectors only (a larger query is read from HBM, with the same results).
 * Offsets beyond n_query_vectors are clamped to it. */
QB_API qb_status qb_hnsw_search_maxsim_batch_device(qb_hnsw* g, const float* dev_query_vectors, uint32_t n_query_vectors, const uint32_t* dev_query_offsets,
                                                    uint32_t n_queries, uint32_t max_query_vectors, uint32_t top, uint32_t ef, uint32_t entry_point,
                                                    uint32_t entry_level, qb_scored_point* dev_out, uint32_t* dev_counts, qb_hnsw_algorithm algorithm);
/* Custom queries whose examples are multivectors, through the device traversal of a graph over multivector points: GraphLayers::search
 * with a MultiCustomQueryScorer (hnsw/read_view/search.rs:181-208, query_scorer/multi_custom_query_scorer.rs).  Only
 * qb_hnsw_create_*_multivector and qb_hnsw_build_multivector handles (QB_ERR_UNSUPPORTED on any other); dense f32 and SQ8 tokens.
 *   kind, n_a, n_b   one kind and one shape per call, as qb_hnsw_search_custom_batch takes them; query q has E =
 *                    qb_custom_examples(kind, n_a, n_b) examples in the qb_scorer_create_custom order
 *   example_vectors, example_offsets   example j of query q is rows [example_offsets[q*E + j], example_offsets[q*E + j + 1]) of
 *                    example_vectors (raw f32 x dim): n_queries*E + 1 ascending offsets, 1..4096 vectors per example (QB_ERR_INVALID)
 *   coef, custom_entry_points, custom_counts, n_custom   as qb_hnsw_search_custom_batch takes them (get_entry_point included)
 *   deleted_points, out   over POINTS, as qb_hnsw_search_maxsim_batch takes and returns them; the token storage's resident flags do
 *                    not apply
 * The traversal is qb_hnsw_search_batch_algo's (max(ef, top), ef <= 4096 else QB_ERR_UNSUPPORTED, HNSW or ACORN-1, is_stopped) with
 * the keyed tie contract of qb_hnsw_search_custom_batch.  A point's score equals qb_score_maxsim_custom on that point bit for bit: per
 * example the MaxSim of qb_hnsw_search_maxsim_batch (the sequential `sim > max` fold from -inf per example vector, the maxima summed in
 * vector order from +0.0; a point with no token rows scores -inf), then the E values folded by Query::score_by.
 * Counters (multi_custom_query_scorer.rs:90-133): per scored point of T token rows, cpu += (the vectors of all E examples) x T x the
 * storage's per-vector units (as qb_hnsw_search_maxsim_batch), vector_io_read += T x io units.  qb_hnsw_stats counts hops and
 * scored points (points, not token rows). */
QB_API qb_status qb_hnsw_search_maxsim_custom_batch(qb_hnsw* g, qb_query_kind kind, const float* example_vectors, const uint32_t* example_offsets,
                                                    uint32_t n_a, uint32_t n_b, const float* coef, uint32_t n_queries, uint32_t top, uint32_t ef,
                                                    uint32_t entry_point, uint32_t entry_level, const uint32_t* custom_entry_points,
                                                    const uint32_t* custom_counts, uint32_t n_custom, const uint64_t* deleted_points,
                                                    const volatile int32_t* is_stopped, qb_scored_point* out, uint32_t* out_counts,
                                                    qb_hw_counters* counters /* optional */, qb_hnsw_algorithm algorithm);
/* Discover with multivector examples as one call: the two stages of qb_hnsw_search_discover_batch over the examples above (E = 1 +
 * 2 n_pairs: the target, then the pairs; n_pairs >= 1).  Stage 1 is a context search over examples 1 .. 2 n_pairs for the top 10
 * with the same ef, filter, algorithm and entry point; stage 2 the discover search from that list as custom entry points.  Scores,
 * ties and counters as qb_hnsw_search_maxsim_custom_batch; hops, scored points and counters sum both stages. */
QB_API qb_status qb_hnsw_search_maxsim_discover_batch(qb_hnsw* g, const float* example_vectors, const uint32_t* example_offsets, uint32_t n_pairs,
                                                      uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point, uint32_t entry_level,
                                                      const uint64_t* deleted_points, const volatile int32_t* is_stopped, qb_scored_point* out,
                                                      uint32_t* out_counts, qb_hw_counters* counters /* optional */, qb_hnsw_algorithm algorithm);

/* Custom queries (recommend, context, feedback) through the device traversal: GraphLayers::search with a custom FilteredScorer
 * (hnsw/read_view/search.rs:181-208).  A point's score is qb_score_points on a qb_scorer_create_custom / qb_scorer_create_feedback
 * scorer of the same examples, bit for bit.
 *   kind, n_a, n_b  one kind and one shape per call (qb_scorer_create_custom's table); queries of other shapes go in other calls.
 *                   QB_QUERY_DISCOVER here is ONE discover search (the reference's second stage); qb_hnsw_search_discover_batch
 *                   below runs both stages
 *   vectors         n_queries x E x dim raw f32, each query's E examples in the qb_scorer_create_custom layout
 *   coef            QB_QUERY_FEEDBACK_NAIVE: n_queries x (1 + n_a) values [a, partial_computation of pair 0, ...]; NULL otherwise
 *   custom_entry_points  optional, n_queries x n_custom point offsets in entry_point's id space (GraphLayers::search's
 *                   custom_entry_points), custom_counts[q] of
 *                   them valid.  Per query the device restates get_entry_point (graph_layers.rs:506-528): of the candidates that pass
 *                   the filter, the one with the highest point level, the LAST of several equal maxima (Iterator::max_by_key); if
 *                   none passes, entry_point / entry_level
 *   counters        cpu += scored points x E x cpu units, vector_io_read += scored points x io units (custom_query_scorer.rs:78-111)
 * The rest is as for qb_hnsw_search_batch_algo.  Dense f32, dense Uint8 and SQ8 storages only (QB_ERR_UNSUPPORTED otherwise).
 *
 * Ties.  Context scores are sums of fast_sigmoid(min(d, 0)): every point that satisfies all pairs scores exactly 0.0, so custom
 * scores tie often.  The device orders equal scores by id (score desc, id asc) in every comparison of the level-0 search:
 * `nearest` insertion and eviction, the candidate order and the stop test; the greedy descent through the upper levels moves
 * only to a strictly greater score, as the reference does.  The reference leaves ties to heap order, so on a plateau the two
 * traversals may visit different points.  The contract: lists equal the reference traversal whenever scores are distinct, and
 * on ties they equal the reference traversal with every level-0 comparison made on (score desc, id asc) keys. */
QB_API qb_status qb_hnsw_search_custom_batch(qb_hnsw* g, qb_query_kind kind, const float* vectors, uint32_t n_a, uint32_t n_b, const float* coef,
                                             uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point, uint32_t entry_level,
                                             const uint32_t* custom_entry_points, const uint32_t* custom_counts, uint32_t n_custom,
                                             const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped, qb_scored_point* out,
                                             uint32_t* out_counts, qb_hw_counters* counters /* optional */, qb_hnsw_algorithm algorithm);
/* Discover (discover_search_with_graph, search.rs:314-349) as one call with no host round trip between its stages:
 *   1. a context search over the query's pairs: top 10 (DISCOVERY_ENTRY_POINT_COUNT), the same ef, filter, algorithm and entry
 *      point; it scores the encoded pair examples of the discover query (the target is skipped, nothing is encoded twice);
 *   2. the discover search, with the stage-1 list as the query's custom entry points (get_entry_point, as above).
 *   vectors   n_queries x (1 + 2 n_pairs) x dim raw f32: the target, then n_pairs (positive, negative) pairs; n_pairs >= 1
 * Hops, scored points and counters sum both stages (one HardwareCounterCell in the reference); the tie contract is the one above.
 * This is the reference's path when the search is not rescored: dense storages, or quantized searches without oversampling or
 * rescoring.  A rescored quantized discover oversamples and rescores stage 1 against the original vectors
 * (search_with_graph -> postprocess_search_result); compose it from the parts: qb_hnsw_search_custom_batch(QB_QUERY_CONTEXT) with
 * the oversampled top, qb_scorer_create_custom(original storage, QB_QUERY_CONTEXT, ...) + qb_rescore down to 10, then
 * qb_hnsw_search_custom_batch(QB_QUERY_DISCOVER) with those ids as custom_entry_points. */
QB_API qb_status qb_hnsw_search_discover_batch(qb_hnsw* g, const float* vectors, uint32_t n_pairs, uint32_t n_queries, uint32_t top, uint32_t ef,
                                               uint32_t entry_point, uint32_t entry_level, const uint64_t* deleted_bitmap,
                                               const volatile int32_t* is_stopped, qb_scored_point* out, uint32_t* out_counts,
                                               qb_hw_counters* counters /* optional */, qb_hnsw_algorithm algorithm);

/* ---------------------------------------------------------------- MMR reranking ---------------------- */
/* Maximal marginal relevance, the diversity rerank of the universal query API, for dense vectors: mmr_from_points_with_vector +
 * maximal_marginal_relevance (lib/shard/src/query/mmr/mod.rs:42-279) with its LazyMatrix (lazy_matrix.rs:25-68).
 *   s           the storage of the candidates' vectors: dense f32 of the collection's distance, rows as they are (the reference's volatile
 *               storage does not preprocess them, volatile_dense_vector_storage.rs:170-182) — a temporary storage the caller fills with
 *               the candidates' vectors, or the resident segment storage whose rows are the vectors `with_vector` returns.  Others:
 *               QB_ERR_UNSUPPORTED
 *   queries     n_queries x dim raw f32 (Metric::preprocess on the device, as qb_scorer_create)
 *   lambdas     one per query: 1 - diversity, in [0, 1] (NaN or outside: QB_ERR_INVALID)
 *   candidates  n_queries x max_candidates, candidate_counts[q] of them valid: the layout qb_search_batch* / qb_hnsw_search_batch* return
 *               with top = max_candidates.  Ids in the storage's numbering (id_base included); max_candidates <= 16384 (candidates_limit's
 *               cap, api/src/rest/schema.rs:771), else QB_ERR_UNSUPPORTED
 *   out         n_queries x limit: the selected candidates in selection order with their ORIGINAL scores; out_counts[q] of them
 * Per query: unique_by(id) keeps the first occurrence; 0 or 1 candidates left are returned as they are (no scoring, no truncation).
 * Otherwise rel[i] = sim(preprocess(query), v_i) (qb_score_points on qb_scorer_create(s, query)), pair(c, t) = sim(preprocess(v_c), v_t)
 * (candidate c's scorer, lazy_matrix.rs:45-52), the first pick is the argmax of rel, and each later pick the argmax over the remaining
 * candidates of lambda * rel - (1 - lambda) * (max over the picks so far, in pick order, of pair(c, pick)), four f32 operations each
 * rounded; until `limit` picks or none remain.  Every max / argmax is max_by_key(OrderedFloat): the last maximal element wins, NaN is above
 * everything and equal to NaN, -0.0 equals +0.0.  Remaining candidates are in IndexSet order and a pick is swap_remove-d (the last
 * remaining one takes its position), so ties go to the later current position.  Scores are bit-exact with the reference's f32 chains.
 * Counters: cpu += dim * 4 * (n + sum over k = 1 .. L-1 of (n - k)) per query of n >= 2 unique candidates and L picks (the relevance
 * pass, then one pair per remaining candidate and later pick); vector_io_read += 0 (the volatile storage is never on disk).
 * Errors, checked before any device work: a null argument, limit = 0, a lambda outside [0, 1], candidate_counts[q] > max_candidates or
 * an id outside the storage: QB_ERR_INVALID.  Synchronous. */
QB_API qb_status qb_mmr_batch(qb_storage* s, const float* queries, uint32_t n_queries, const float* lambdas, const qb_scored_point* candidates,
                              const uint32_t* candidate_counts, uint32_t max_candidates, uint32_t limit, qb_scored_point* out, uint32_t* out_counts,
                              qb_hw_counters* counters /* optional */);
/* same with every array resident in HBM, enqueued on qb_storage_stream(s) with no host synchronisation, so it chains after
 * qb_search_batch_device / qb_hnsw_search_batch_device on the same storage (top = max_candidates).  The host checks the storage,
 * max_candidates and limit; lambdas and ids stay on the device unchecked: a count above max_candidates is clamped to it and an id outside
 * the storage is dropped from its list.  dev_out is n_queries x limit. */
QB_API qb_status qb_mmr_batch_device(qb_storage* s, const float* dev_queries, uint32_t n_queries, const float* dev_lambdas,
                                     const qb_scored_point* dev_candidates, const uint32_t* dev_candidate_counts, uint32_t max_candidates,
                                     uint32_t limit, qb_scored_point* dev_out, uint32_t* dev_out_counts);

/* The same rerank over a multivector named vector (ColBERT MaxSim): mmr_from_points_with_vector (mod.rs:42-125) puts the candidates'
 * multivectors into a volatile multi-dense f32 storage, which does not preprocess them (volatile_multi_dense_vector_storage.rs:138-148),
 * and its LazyMatrix scores pairs with MultiMetricQueryScorer.
 *   tokens, point_offsets, n_points   dense f32 token rows (others, e.g. f16 / u8 / SQ8: QB_ERR_UNSUPPORTED), point p = rows
 *               [point_offsets[p], point_offsets[p+1]) used as they are — the layout qb_search_maxsim takes; the offsets must ascend and
 *               end within the storage.  Candidate ids are point offsets 0 .. n_points - 1, the numbering the MaxSim searches return
 *   query q     rows [query_offsets[q], query_offsets[q+1]) of query_vectors: 1..4096 raw f32 vectors, each prepared with
 *               Metric::preprocess (MultiMetricQueryScorer::new)
 *   lambdas, candidates, candidate_counts, max_candidates (<= 16384, else QB_ERR_UNSUPPORTED), limit, out, out_counts   as qb_mmr_batch
 * MaxSim(A, B) = for each vector a of A in order, the sequential `sim > max` fold from -inf over B's vectors (NaN never wins, an empty run
 * stays -inf, the earlier of -0.0 / +0.0 keeps its bits), the maxima summed sequentially in f32 from +0.0 — qb_score_maxsim's rule.
 *   rel[i]     = MaxSim(preprocess(Q), P_i), equal to qb_score_maxsim on that point bit for bit
 *   pair(c, s) = MaxSim(preprocess(P_c), P_s): candidate c's tokens are the query side, the pick's the stored side (lazy_matrix.rs:45-52);
 *                MaxSim is not symmetric
 * The selection is qb_mmr_batch's: unique_by(id) keeps the first occurrence, fewer than two are returned as they are, every max / argmax
 * keeps the last maximum under OrderedFloat, mmr = lambda * rel - (1 - lambda) * maxsim in four rounded f32 operations, picks are
 * swap_remove-d, the output keeps the input scores in pick order.
 * Counters (MultiMetricQueryScorer: dim * 4 per vector pair of a MaxSim): per query of n >= 2 unique candidates and L picks,
 * cpu += dim * 4 * (T_q * sum_i T_i + sum over picks k = 1 .. L-1 of T_pick_k * (sum of T_c over the candidates remaining after pick k));
 * vector_io_read += 0.
 * Errors, checked before any device work: a null argument, limit = 0, a lambda NaN or outside [0, 1], a count above max_candidates, an id
 * >= n_points, offsets that do not ascend or end past the storage, a query with 0 or more than 4096 vectors, or a candidate point with no
 * token rows (the reference cannot hold an empty multivector): QB_ERR_INVALID.
 * Device scratch: for Cosine, every candidate's preprocessed token rows, max_candidates x (the longest candidate's row count) x the row
 * size per query, the batch in chunks of at most 512 MB (one query per chunk when a query needs more); nothing for the other distances.
 * Synchronous. */
QB_API qb_status qb_mmr_maxsim_batch(qb_storage* tokens, const uint32_t* point_offsets, uint32_t n_points, const float* query_vectors,
                                     const uint32_t* query_offsets, uint32_t n_queries, const float* lambdas, const qb_scored_point* candidates,
                                     const uint32_t* candidate_counts, uint32_t max_candidates, uint32_t limit, qb_scored_point* out, uint32_t* out_counts,
                                     qb_hw_counters* counters /* optional */);
/* same with the query vectors (n_query_vectors x dim), their offsets (n_queries + 1), lambdas, candidates and outputs resident in HBM,
 * enqueued on qb_storage_stream(tokens) with no host synchronisation, so it chains after qb_hnsw_search_maxsim_batch_device on the same
 * token storage (top = max_candidates).  point_offsets stay in HOST memory: they are the offsets the caller created the graph from, checked
 * here as the host form checks them and copied to the device in stream order (4 * (n_points + 1) bytes per call).  max_query_vectors
 * (1..4096) bounds the largest query's vector count; it sizes the shared-memory staging only.  Query offsets beyond n_query_vectors are
 * clamped to it (a query left with no vectors scores +0.0 relevance).  The host checks the storage, the offsets, max_candidates and
 * limit; lambdas and ids stay on the device unchecked: a count above max_candidates is clamped, and ids outside the points or points
 * without token rows are dropped from their list.  The Cosine scratch bound uses the longest point's row count, never the storage's
 * size.  dev_out is n_queries x limit. */
QB_API qb_status qb_mmr_maxsim_batch_device(qb_storage* tokens, const uint32_t* point_offsets, uint32_t n_points, const float* dev_query_vectors,
                                            uint32_t n_query_vectors, const uint32_t* dev_query_offsets, uint32_t n_queries, uint32_t max_query_vectors,
                                            const float* dev_lambdas, const qb_scored_point* dev_candidates, const uint32_t* dev_candidate_counts,
                                            uint32_t max_candidates, uint32_t limit, qb_scored_point* dev_out, uint32_t* dev_out_counts);

/* The same rerank over a sparse named vector: mmr_from_points_with_vector (mod.rs:42-157) puts the candidates' sparse vectors into a
 * VolatileSparseVectorStorage (mod.rs:130), each sorted by dim on insertion (volatile_sparse_vector_storage.rs:214-226), and its
 * LazyMatrix scores pairs with SparseMetricQueryScorer (query_scorer/sparse_metric_query_scorer.rs).
 *   s           the qb_sparse_storage (below) holding the candidates' vectors; candidate ids are its point ids (< n_points)
 *   query q     CSR entry [q_indptr[q], q_indptr[q+1]) of q_dims / q_weights in user dims, any order (offsets from 0, ascending).  It is
 *               sorted by dim here, as VectorInternal::preprocess sorts it (vectors.rs:68-80) before NearestWithMmr becomes MmrInternal
 *               (collection_query.rs:430, 472-480); its weights are not checked
 *   lambdas, candidates, candidate_counts, max_candidates (<= 16384, else QB_ERR_UNSUPPORTED), limit, out, out_counts   as qb_mmr_batch
 * Per query (mod.rs:42-279):
 *   1. unique_by(id) keeps the first occurrence.  A candidate with an empty row is a vector: it stays and scores +0.0 against everything
 *   2. fewer than two candidates are returned as they are; nothing is scored or counted (mod.rs:77-80)
 *   3. rel[i] = score_vectors(q, v_i) (raw_scorer.rs:142-160, sparse_vector.rs:66-90): both sides sorted by dim, a sum from 0.0 of
 *      q_w * v_w over the shared dims in ascending dim order, every product and sum rounded; no shared dim gives +0.0 (unwrap_or_default)
 *   4. pair(c, s) = score_vectors(v_c, v_s), computed the first time (c, s) is needed (lazy_matrix.rs:45-67); symmetric bit for bit
 *   5. the selection is qb_mmr_batch's: the first pick is the argmax of rel, each later pick the argmax of lambda * rel - (1 - lambda) *
 *      max_sim in four rounded f32 operations, max_sim the max over the picks so far in pick order; every max / argmax keeps the last
 *      maximum under OrderedFloat (NaN above everything, -0.0 == +0.0); the remaining candidates in IndexSet order, a pick swap_remove-d;
 *      the output is the picks in order with their ORIGINAL scores
 *   6. counters (SparseMetricQueryScorer: cpu multiplier 1, min(|a|, |b|) per scored pair): per query of n >= 2 unique candidates and L
 *      picks, cpu += sum_i min(|q|, |v_i|) + sum over picks k = 1 .. L-1 of the sum over the candidates c remaining after pick k of
 *      min(|v_c|, |v_pick_k|); vector_io_read += 0, since the volatile storage is in memory, also when s was created on_disk.
 * Zero scores are common with sparse data (two rows without a shared dim), so plateaus of equal mmr values are frequent and the
 * swap_remove position order decides them.
 * Errors, checked before any device work: a null argument, limit = 0, a lambda NaN or outside [0, 1], query offsets that descend or do not
 * start at 0, a dim repeated within a query, a count above max_candidates or an id >= n_points: QB_ERR_INVALID.  Synchronous. */
QB_API qb_status qb_mmr_sparse_batch(qb_sparse_storage* s, const uint64_t* q_indptr, const uint32_t* q_dims, const float* q_weights,
                                     uint32_t n_queries, const float* lambdas, const qb_scored_point* candidates,
                                     const uint32_t* candidate_counts, uint32_t max_candidates, uint32_t limit,
                                     qb_scored_point* out, uint32_t* out_counts, qb_hw_counters* counters /* optional */);

/* ---------------------------------------------------------------- sparse vectors -------------------- */
/* An inverted index over sparse vectors (SPLADE, BM25 and the like) and the reference's SearchContext over it
 * (lib/sparse/src/index/search_context.rs).  Dims are internal dims: the caller remaps its user dims as the segment's IndicesTracker
 * does (indices_tracker.rs:53-72) and keeps that map on the host.
 *   kind   QB_SPARSE_RAM: the mutable InvertedIndexRam, whose lists report reliable max_next_weight, so search may prune
 *          (posting_list.rs:228).  QB_SPARSE_COMPRESSED: the immutable / mmap compressed indexes with f32 weights, which never prune
 *          (compressed_posting_list.rs:661).  Compressed lists with f16 or u8 weights: QB_ERR_UNSUPPORTED. */
typedef enum { QB_SPARSE_RAM = 0, QB_SPARSE_COMPRESSED = 1, QB_SPARSE_COMPRESSED_F16 = 2, QB_SPARSE_COMPRESSED_U8 = 3 } qb_sparse_kind;
typedef struct qb_sparse_index qb_sparse_index;
/* n_points rows in CSR form: row r = dims / weights [indptr[r], indptr[r + 1]), indptr[0] = 0.  Each row is sorted by dim on creation;
 * one posting list per dim holds (id, weight, max_next_weight) sorted by id, max_next_weight = the largest weight after the element
 * (-inf for the last; PostingBuilder::build, posting_list.rs:140-170).  QB_ERR_INVALID for a null argument, an unknown kind, offsets that
 * descend or do not start at 0, a dim >= n_dims, a dim repeated within a row or a weight that is not finite.  2^32 - 1 or more elements:
 * QB_ERR_UNSUPPORTED.  HBM: 20 bytes per element, 8 per point and 8 per dim.  Synchronous. */
QB_API qb_status qb_sparse_index_create(int32_t device, qb_sparse_kind kind, uint32_t n_points, uint32_t n_dims, const uint64_t* indptr,
                                        const uint32_t* dims, const float* weights, qb_sparse_index** out);
QB_API void qb_sparse_index_destroy(qb_sparse_index* idx);
QB_API qb_status qb_sparse_index_info(const qb_sparse_index* idx, uint32_t* n_points, uint32_t* n_dims, uint64_t* n_elements, uint64_t* hbm_bytes);
/* the cudaStream_t the index's searches run on (qb_sparse_search_batch_device enqueues there) */
QB_API void* qb_sparse_index_stream(qb_sparse_index* idx);
/* SearchContext::new + search (:42-87, :263-414) per query: query q = q_dims / q_weights [q_indptr[q], q_indptr[q + 1]).
 *   The query is sorted by dim and its dims >= n_dims are dropped, as remap_vector drops the dims the tracker does not know; a dim
 *   repeated in a query is QB_ERR_INVALID (SparseVector validation).  An empty query, or one whose lists are all empty, gives an empty list.
 *   Batches of ids [min_id, min(min_id + 10000, max_record_id)]: every list in its current order adds weight * query_weight into a zeroed f32
 *   score (0 + p1 + p2 + ...); a score is pushed when it is non-zero, greater than the running threshold and not deleted.  After each
 *   batch the exhausted lists are removed in order; one list left pushes all its remaining undeleted elements (weight * query_weight, no
 *   non-zero test); otherwise, with pruning on and a full TopK whose threshold changed, the longest list (the last of equal lengths) is
 *   swapped to the front and skipped ahead when max(weight, max_next_weight) * query_weight <= threshold.  Pruning is on for
 *   QB_SPARSE_RAM when every kept query weight is >= 0.
 *   TopK (common/src/top_k.rs:22-64): the threshold starts at f32::MIN, a push needs score > threshold, at 2k entries the threshold
 *   becomes the k-th largest score and k entries stay.  The entries kept order by (score desc, id asc), so among equal scores at the
 *   boundary the smaller ids stay, where the reference keeps an unspecified subset; scores, the threshold history and so pruning are
 *   the reference's bit for bit.
 *   deleted_bitmap  optional, ceil(n_points / 64) words, bit = 1 deleted (the filter)
 *   is_stopped      optional, polled before the launch (QB_ERR_CANCELLED)
 *   out             n_queries x top in (score desc, id asc) order; out_counts[q] valid entries
 * top in 1..4096 (0: QB_ERR_INVALID, above: QB_ERR_UNSUPPORTED); more than 4096 kept dims in a query: QB_ERR_UNSUPPORTED.
 * Counters: cpu += 4 * the total length of the query's posting lists (:272-283); vector_io_read += 0.  Every check runs before any device
 * work.  The choice between this and qb_sparse_search_plain_batch stays with the caller, as in the reference
 * (read_view/search.rs:258-300): plain search when the filter's estimated cardinality is below full_scan_threshold (default 5000).
 * Synchronous. */
QB_API qb_status qb_sparse_search_batch(qb_sparse_index* idx, const uint64_t* q_indptr, const uint32_t* q_dims, const float* q_weights, uint32_t n_queries,
                                        uint32_t top, const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped, qb_scored_point* out,
                                        uint32_t* out_counts, qb_hw_counters* counters /* optional */);
/* same with the queries, the optional bitmap and the outputs resident in HBM, enqueued on qb_sparse_index_stream(idx) with no host
 * synchronisation.  The queries are sorted and their dims >= n_dims dropped on the device; they are not checked: a query's entries past
 * max_query_nnz (<= 4096, else QB_ERR_UNSUPPORTED) are ignored, and a repeated dim counts as two lists.  No counters. */
QB_API qb_status qb_sparse_search_batch_device(qb_sparse_index* idx, const uint64_t* dev_q_indptr, const uint32_t* dev_q_dims, const float* dev_q_weights,
                                               uint32_t n_queries, uint32_t max_query_nnz, uint32_t top, const uint64_t* dev_deleted_bitmap,
                                               qb_scored_point* dev_out, uint32_t* dev_out_counts);
/* SearchContext::plain_search (:92-143) per query over its own ids [id_indptr[q], id_indptr[q + 1]) — already filtered by the caller, as
 * the reference's prefiltered_points are.  For each id, the dims the point shares with the query score 0 + sum of stored * query in
 * ascending dim order (score_vectors, sparse_vector.rs:66-90); an id with no shared dim is skipped; any other score above f32::MIN,
 * zero included, is pushed.  Queries as qb_sparse_search_batch; out in (score desc, id asc) order.  An id >= n_points or repeated within
 * a query: QB_ERR_INVALID.  Counters: cpu += kept query dims + 4 * shared dims per scored id; vector_io_read += 0.  Synchronous. */
QB_API qb_status qb_sparse_search_plain_batch(qb_sparse_index* idx, const uint64_t* q_indptr, const uint32_t* q_dims, const float* q_weights,
                                              uint32_t n_queries, const uint64_t* id_indptr, const uint32_t* ids, uint32_t top,
                                              const volatile int32_t* is_stopped, qb_scored_point* out, uint32_t* out_counts,
                                              qb_hw_counters* counters /* optional */);

/* The segment's sparse vector storage (SparseVectorStorage) and the custom queries over it: every sparse query that is not Nearest
 * (recommend, discover, context, feedback) skips the inverted index and scans the storage (sparse_vector_index/read_view/search.rs:99-151,
 * 302-341) with SparseCustomQueryScorer (query_scorer/sparse_custom_query_scorer.rs).  Dims here are USER dims (any u32): the scorer
 * merges the stored vectors with the examples in user-dim order, which the index's internal dims do not keep. */
/* n_points rows in CSR form as qb_sparse_index_create takes them, in user dims; each row is sorted by dim on creation.  QB_ERR_INVALID for a
 * null argument, offsets that descend or do not start at 0, a dim repeated within a row or a weight that is not finite.  2^32 - 1 or more
 * elements: QB_ERR_UNSUPPORTED.  on_disk != 0: an mmap storage, whose reads count vector_io_read (multiplier 4, size_of::<DimId>()); 0: an
 * in-memory storage (multiplier 0).  HBM: 8 bytes per element and 8 per point.  Synchronous. */
QB_API qb_status qb_sparse_storage_create(int32_t device, uint32_t n_points, const uint64_t* indptr, const uint32_t* dims, const float* weights,
                                          int32_t on_disk, qb_sparse_storage** out);
QB_API void qb_sparse_storage_destroy(qb_sparse_storage* s);
QB_API qb_status qb_sparse_storage_info(const qb_sparse_storage* s, uint32_t* n_points, uint64_t* n_elements, uint64_t* hbm_bytes);
/* search_scored per query: peek_top_iter over the scored points with a SparseCustomQueryScorer.
 *   kind, n_a, n_b  one kind and one shape per call, as qb_hnsw_search_custom_batch takes them; query q has E = qb_custom_examples(kind,
 *                   n_a, n_b) examples in the qb_scorer_create_custom order (feedback: the target, then n_a pairs).  E above 256:
 *                   QB_ERR_UNSUPPORTED
 *   ex_indptr, ex_dims, ex_weights   example j of query q is CSR entry q * E + j (n_queries * E + 1 offsets from 0), user dims, any order;
 *                   more than 4096 non-zeros over one query's examples: QB_ERR_UNSUPPORTED.  Weights are not checked
 *   coef            QB_QUERY_FEEDBACK_NAIVE: n_queries x (1 + n_a) values [a, partial_computation of pair 0, ...]; NULL otherwise
 *   deleted_bitmap  optional, ceil(n_points / 64) words, bit = 1 deleted
 *   id_list         optional, n_ids distinct ids < n_points shared by the whole batch (the reference's prefiltered_points); the scored points
 *                   are the listed ids that are not deleted, or every point that is not deleted when id_list is NULL
 *   is_stopped      optional, polled before the launch (QB_ERR_CANCELLED)
 *   out             n_queries x top in (score desc, id asc) order, out_counts[q] valid entries; NaN ranks above everything (OrderedFloat)
 * A point's similarity to an example is score_vectors (sparse_vector.rs:66-90): both sides sorted by dim, 0 + sum of example weight x stored
 * weight over the shared dims in ascending dim order, every product and sum rounded, +0.0 when no dim is shared; the E similarities are
 * folded by Query::score_by as in qb_scorer_create_custom.  top in 1..4096 (0: QB_ERR_INVALID, above: QB_ERR_UNSUPPORTED).
 * Counters, summed over the batch: per scored point of |v| stored elements, cpu += 4 x the sum over the examples of (|v| + |example|), every
 * given example element counted; vector_io_read += 2 |v| x (4 on disk, else 0).  QB_ERR_INVALID, checked before any device work: a null
 * argument, an unknown kind or a shape qb_scorer_create_custom rejects, example offsets that descend or do not start at 0, a dim repeated
 * within an example, feedback without coef, top 0, an id >= n_points or repeated in id_list.  Synchronous. */
QB_API qb_status qb_sparse_search_custom_batch(qb_sparse_storage* s, qb_query_kind kind, uint32_t n_a, uint32_t n_b, const uint64_t* ex_indptr,
                                               const uint32_t* ex_dims, const float* ex_weights, const float* coef, uint32_t n_queries, uint32_t top,
                                               const uint64_t* deleted_bitmap, const uint32_t* id_list, uint64_t n_ids, const volatile int32_t* is_stopped,
                                               qb_scored_point* out, uint32_t* out_counts, qb_hw_counters* counters /* optional */);
/* score_stored_batch of ONE query (E examples, CSR entries 0 .. E - 1; coef = 1 + n_a values for feedback) over n given ids: scores[k] of
 * ids[k], equal bit for bit to the scores qb_sparse_search_custom_batch ranks.  No filter.  Counters and errors as the batch entry (ids
 * distinct and < n_points).  Synchronous. */
QB_API qb_status qb_sparse_score_custom(qb_sparse_storage* s, qb_query_kind kind, uint32_t n_a, uint32_t n_b, const uint64_t* ex_indptr, const uint32_t* ex_dims,
                                        const float* ex_weights, const float* coef, const uint32_t* ids, uint64_t n, float* scores,
                                        qb_hw_counters* counters /* optional */);

/* ---------------------------------------------------------------- profiling hooks ------------------- */
/* Fused searches run a fast path first and rerun without it when the device reports that one of its assumptions did not
 * hold (candidate buffer overflow, a dot product outside the f32-exact window, a survivor segment full).  searches =
 * fused search calls on this storage, reruns = extra passes they needed: a benchmark or test that claims the fast path
 * asserts reruns == 0. */
QB_API qb_status qb_search_stats(qb_storage* s, uint64_t* searches, uint64_t* reruns, int32_t reset);

/* When enabled, the dominant scan kernel of every search on this storage is bracketed by CUDA events on its
 * launch stream; qb_profile_read returns the number of bracketed launches and their summed duration. */
QB_API qb_status qb_profile_enable(qb_storage* s, int32_t on);
QB_API qb_status qb_profile_read(qb_storage* s, uint64_t* launches, double* total_ms, int32_t reset);

#ifdef __cplusplus
}
#endif
#endif /* QB200_H */
