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
 * (built on the first search that uses them, rebuilt after qb_storage_write_rows*: + 26 % HBM for the int8 plane of single-query
 * searches on >= 2^19 rows, + 50 % for the bf16 plane of batches of >= 32 queries; dot / cosine only), batched SQ8 / PQ scans run
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
 * graph_links/view.rs:121-135): HeaderPlain, level offsets, reindex, neighbors, padding, offsets.  (The compressed
 * formats are decoded by the caller, as GraphLinks::to_edges does.)  m / m0 = HnswM (hnsw_index/mod.rs:34-40), both <= 64.
 * The graph is bound to `s` (dense f32 or SQ8; the quantized storage when the segment searches quantized) and must
 * outlive neither it nor its searches. */
typedef struct qb_hnsw qb_hnsw;
QB_API qb_status qb_hnsw_create_plain(qb_storage* s, const uint8_t* links_bin, uint64_t n_bytes, uint32_t m, uint32_t m0, qb_hnsw** out);
QB_API void qb_hnsw_destroy(qb_hnsw* g);
QB_API qb_status qb_hnsw_info(const qb_hnsw* g, uint32_t* n_points, uint32_t* levels, uint64_t* hbm_bytes);
/*   queries         n_queries x dim raw f32 (Metric::preprocess + encode_query on the device)
 *   ef              beam width; max(ef, top) is used (graph_layers.rs:551)
 *   entry_point / entry_level   GraphLayers::get_entry_point's answer (entry_points.rs; it depends on the filter, so the
 *                   host passes it per call)
 *   deleted_bitmap  optional filter (bit = 1: point fails ScorerFilters::check_vector), OR-ed with the resident flags;
 *                   filtered-out links are neither scored nor traversed (point_scorer.rs:270-277)
 *   out             n_queries x top, descending; out_counts[q] valid entries
 * Result lists equal the reference traversal's whenever scores are distinct (ties are ordered by id). */
QB_API qb_status qb_hnsw_search_batch(qb_hnsw* g, const float* queries, uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point,
                                      uint32_t entry_level, const uint64_t* deleted_bitmap, const volatile int32_t* is_stopped,
                                      qb_scored_point* out, uint32_t* out_counts, qb_hw_counters* counters /* optional */);
/* same with queries / outputs resident in HBM, enqueued on qb_storage_stream(s); no host synchronisation */
QB_API qb_status qb_hnsw_search_batch_device(qb_hnsw* g, const float* dev_queries, uint32_t n_queries, uint32_t top, uint32_t ef, uint32_t entry_point,
                                             uint32_t entry_level, qb_scored_point* dev_out, uint32_t* dev_counts);
/* scorer calls (hops) and scored points since the last reset, summed over all searches on this graph (waits for them) */
QB_API qb_status qb_hnsw_stats(qb_hnsw* g, uint64_t* hops, uint64_t* scored_points, int32_t reset);

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
