//! Raw FFI declarations for libqdrant_b200.so — GENERATED from include/qb200.h by tools/gen_rust_ffi.py; do not edit by hand.
//! SOURCE ONLY: there is no Rust toolchain in the build image, so this file has never been compiled there; it is the binding a
//! Qdrant maintainer would add under `lib/segment/src/vector_storage/b200/ffi.rs`.  One declaration per exported function.
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_void};

pub type qb_status = i32;
pub const QB200_ABI_VERSION: i32 = 2;
pub const QB_OK: qb_status = 0;
pub const QB_ERR_INVALID: qb_status = -1;
pub const QB_ERR_CUDA: qb_status = -2;
pub const QB_ERR_UNSUPPORTED: qb_status = -3;
pub const QB_ERR_OOM: qb_status = -4;
pub const QB_ERR_CANCELLED: qb_status = -5;
pub const QB_ERR_NO_DEVICE: qb_status = -6;

// Distance (types.rs:313-322), VectorStorageDatatype, quantization::DistanceType, BQ encodings, QueryVector kinds — passed as i32
pub const QB_DIST_COSINE: i32 = 0; pub const QB_DIST_EUCLID: i32 = 1; pub const QB_DIST_DOT: i32 = 2; pub const QB_DIST_MANHATTAN: i32 = 3;
pub const QB_DT_F32: i32 = 0; pub const QB_DT_F16: i32 = 1; pub const QB_DT_U8: i32 = 2;
pub const QB_QD_COSINE: i32 = 0; pub const QB_QD_DOT: i32 = 1; pub const QB_QD_L1: i32 = 2; pub const QB_QD_L2: i32 = 3;
// qb_hnsw_algorithm (SearchAlgorithm, graph_layers.rs:80-84)
pub const QB_HNSW_ALGO_HNSW: i32 = 0; pub const QB_HNSW_ALGO_ACORN: i32 = 1;
// qb_sparse_kind: InvertedIndexRam (may prune), the compressed indexes with f32 / f16 / u8 weights
pub const QB_SPARSE_RAM: i32 = 0; pub const QB_SPARSE_COMPRESSED: i32 = 1; pub const QB_SPARSE_COMPRESSED_F16: i32 = 2; pub const QB_SPARSE_COMPRESSED_U8: i32 = 3;

#[repr(C)]
pub struct qb_storage { _private: [u8; 0] }
#[repr(C)]
pub struct qb_scorer { _private: [u8; 0] }
#[repr(C)]
pub struct qb_hnsw { _private: [u8; 0] }
#[repr(C)]
pub struct qb_comm { _private: [u8; 0] }
#[repr(C)]
pub struct qb_sparse_index { _private: [u8; 0] }
#[repr(C)]
pub struct qb_sparse_storage { _private: [u8; 0] }

/// Same layout as `common::types::ScoredPointOffset` (`#[repr(C)] { idx: u32, score: f32 }`).
#[repr(C)]
#[derive(Copy, Clone, Default, Debug, PartialEq)]
pub struct qb_scored_point { pub idx: u32, pub score: f32 }

#[repr(C)]
#[derive(Copy, Clone, Default, Debug)]
pub struct qb_hw_counters { pub cpu: u64, pub vector_io_read: u64 }

#[link(name = "qdrant_b200")]
extern "C" {
    pub fn qb_last_error() -> *const c_char;
    pub fn qb_abi_version() -> i32;
    pub fn qb_device_count(out: *mut i32) -> qb_status;
    pub fn qb_kernel_launch_count() -> u64;
    pub fn qb_set_option(name: *const c_char, value: i64) -> qb_status;
    pub fn qb_storage_create_dense(device: i32, dt: i32, distance: i32, dim: u32, count: u64, host_rows: *const c_void, row_stride_bytes: u64, out: *mut *mut qb_storage) -> qb_status;
    pub fn qb_storage_write_rows(s: *mut qb_storage, first_row: u64, n_rows: u64, host_rows: *const c_void, row_stride_bytes: u64) -> qb_status;
    pub fn qb_storage_write_rows_device(s: *mut qb_storage, first_row: u64, n_rows: u64, dev_rows: *const c_void, row_stride_bytes: u64) -> qb_status;
    pub fn qb_storage_read_rows(s: *const qb_storage, ids: *const u32, n: u64, host_out: *mut c_void) -> qb_status;
    pub fn qb_storage_create_sq8(device: i32, dim: u32, count: u64, rows: *const u8, row_bytes: u32, alpha: f32, offset: f32, multiplier: f32, dt: i32, invert: i32, metric: i32, out: *mut *mut qb_storage) -> qb_status;
    pub fn qb_storage_create_pq(device: i32, dim: u32, m: u32, div_start_end: *const u32, centroids: *const f32, n_centroids: u32, codes: *const u8, count: u64, dt: i32, invert: i32, metric: i32, out: *mut *mut qb_storage) -> qb_status;
    pub fn qb_storage_create_bq(device: i32, dim: u32, enc: i32, qenc: i32, rows: *const u8, row_bytes: u32, count: u64, dt: i32, invert: i32, mean_std: *const f32, metric: i32, out: *mut *mut qb_storage) -> qb_status;
    pub fn qb_storage_load_dense_file(device: i32, dt: i32, distance: i32, dim: u32, file_bytes: *const u8, n_bytes: u64, out: *mut *mut qb_storage) -> qb_status;
    pub fn qb_storage_load_quantized(device: i32, metric: i32, meta_json: *const c_char, json_len: u64, data: *const u8, n_bytes: u64, count: u64, out: *mut *mut qb_storage) -> qb_status;
    pub fn qb_storage_destroy(s: *mut qb_storage);
    pub fn qb_storage_info(s: *const qb_storage, dim: *mut u32, count: *mut u64, hbm_bytes: *mut u64) -> qb_status;
    pub fn qb_storage_set_deleted(s: *mut qb_storage, bitmap_words: *const u64, n_words: u64) -> qb_status;
    pub fn qb_storage_set_on_disk(s: *mut qb_storage, on_disk: i32) -> qb_status;
    pub fn qb_storage_stream(s: *mut qb_storage) -> *mut c_void;
    pub fn qb_metric_preprocess(device: i32, distance: i32, dim: u32, n: u64, r#in: *const f32, out: *mut f32) -> qb_status;
    pub fn qb_metric_preprocess_device(device: i32, distance: i32, dim: u32, n: u64, dev_rows: *mut f32, row_stride_bytes: u64) -> qb_status;
    pub fn qb_metric_postprocess(distance: i32, score: f32) -> f32;
    pub fn qb_scorer_create(s: *mut qb_storage, query: *const f32, out: *mut *mut qb_scorer) -> qb_status;
    pub fn qb_scorer_create_internal(s: *mut qb_storage, point_id: u32, out: *mut *mut qb_scorer) -> qb_status;
    pub fn qb_scorer_destroy(sc: *mut qb_scorer);
    pub fn qb_score_points(sc: *mut qb_scorer, ids: *const u32, n: usize, scores: *mut f32) -> qb_status;
    pub fn qb_score_point(sc: *mut qb_scorer, id: u32, score: *mut f32) -> qb_status;
    pub fn qb_score_internal(sc: *mut qb_scorer, a: u32, b: u32, score: *mut f32) -> qb_status;
    pub fn qb_scorer_take_counters(sc: *mut qb_scorer, out: *mut qb_hw_counters) -> qb_status;
    pub fn qb_search_batch(s: *mut qb_storage, queries: *const f32, n_queries: u32, top: u32, deleted_bitmap: *const u64, id_list: *const u32, n_ids: u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_search_batch_device(s: *mut qb_storage, dev_queries: *const f32, n_queries: u32, top: u32, dev_out: *mut qb_scored_point, dev_counts: *mut u32) -> qb_status;
    pub fn qb_scorer_create_custom(s: *mut qb_storage, kind: i32, vectors: *const f32, n_a: u32, n_b: u32, out: *mut *mut qb_scorer) -> qb_status;
    pub fn qb_search_custom(s: *mut qb_storage, kind: i32, vectors: *const f32, n_a: u32, n_b: u32, top: u32, deleted_bitmap: *const u64, id_list: *const u32, n_ids: u64, is_stopped: *const i32, out: *mut qb_scored_point, out_count: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_scorer_create_feedback(s: *mut qb_storage, vectors: *const f32, n_pairs: u32, a: f32, partial: *const f32, out: *mut *mut qb_scorer) -> qb_status;
    pub fn qb_search_feedback(s: *mut qb_storage, vectors: *const f32, n_pairs: u32, a: f32, partial: *const f32, top: u32, deleted_bitmap: *const u64, id_list: *const u32, n_ids: u64, is_stopped: *const i32, out: *mut qb_scored_point, out_count: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_search_maxsim(s: *mut qb_storage, point_offsets: *const u32, n_points: u32, query_vectors: *const f32, n_query_vectors: u32, top: u32, deleted_points: *const u64, out: *mut qb_scored_point, out_count: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_score_maxsim(s: *mut qb_storage, point_offsets: *const u32, n_points: u32, query_vectors: *const f32, n_query_vectors: u32, point_ids: *const u32, n: usize, scores: *mut f32) -> qb_status;
    pub fn qb_search_maxsim_custom(s: *mut qb_storage, point_offsets: *const u32, n_points: u32, kind: i32, example_vectors: *const f32, example_offsets: *const u32, n_a: u32, n_b: u32, coef: *const f32, top: u32, deleted_points: *const u64, out: *mut qb_scored_point, out_count: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_score_maxsim_custom(s: *mut qb_storage, point_offsets: *const u32, n_points: u32, kind: i32, example_vectors: *const f32, example_offsets: *const u32, n_a: u32, n_b: u32, coef: *const f32, point_ids: *const u32, n: usize, scores: *mut f32) -> qb_status;
    pub fn qb_sq8_find_alpha_offset_device(device: i32, dim: u32, count: u64, dev_rows: *const f32, row_stride_bytes: u64, alpha: *mut f32, offset: *mut f32) -> qb_status;
    pub fn qb_sq8_encode_rows_device(device: i32, dim: u32, count: u64, dev_rows: *const f32, row_stride_bytes: u64, alpha: f32, offset: f32, dt: i32, invert: i32, dev_out: *mut u8, stream: *mut c_void) -> qb_status;
    pub fn qb_bq_row_bytes(dim: u32, encoding: i32) -> u32;
    pub fn qb_bq_encode_rows_device(device: i32, dim: u32, count: u64, dev_rows: *const f32, row_stride_bytes: u64, encoding: i32, mean_std: *const f32, dev_out: *mut u8, stream: *mut c_void) -> qb_status;
    pub fn qb_pq_encode_rows_device(device: i32, dim: u32, chunk: u32, n_centroids: u32, centroids: *const f32, count: u64, dev_rows: *const f32, row_stride_bytes: u64, dev_codes: *mut u8, stream: *mut c_void) -> qb_status;
    pub fn qb_bq_vector_stats_device(device: i32, dim: u32, count: u64, dev_rows: *const f32, row_stride_bytes: u64, mean_std_out: *mut f32, min_max_out: *mut f32) -> qb_status;
    pub fn qb_sq8_quantile_interval_device(device: i32, dim: u32, n_sample: u64, dev_sample_rows: *const f32, row_stride_bytes: u64, quantile: f32, alpha: *mut f32, offset: *mut f32, found: *mut i32) -> qb_status;
    pub fn qb_pq_train_device(device: i32, dim: u32, chunk: u32, n_centroids: u32, n_sample: u64, dev_sample_rows: *const f32, row_stride_bytes: u64, max_iterations: u32, accuracy: f32, max_threads: u32, seed: u64, centroids_out: *mut f32, iterations_out: *mut u32) -> qb_status;
    pub fn qb_rescore(orig: *mut qb_scorer, ids: *const u32, n: usize, top: u32, out: *mut qb_scored_point, out_count: *mut u32) -> qb_status;
    pub fn qb_storage_set_id_base(s: *mut qb_storage, id_base: u32) -> qb_status;
    pub fn qb_topk_merge_device(device: i32, dev_lists: *const qb_scored_point, dev_counts: *const u32, n_lists: u32, n_queries: u32, top: u32, dev_out: *mut qb_scored_point, dev_out_counts: *mut u32, dev_scratch: *mut c_void, scratch_bytes: u64, stream: *mut c_void) -> qb_status;
    pub fn qb_comm_create(device: i32, rank: i32, world: i32, max_queries: u32, max_top: u32, out: *mut *mut qb_comm) -> qb_status;
    pub fn qb_comm_local_handle(c: *mut qb_comm, handle_out: *mut u8) -> qb_status;
    pub fn qb_comm_connect(c: *mut qb_comm, handles: *const u8) -> qb_status;
    pub fn qb_comm_connect_local(comms: *const *mut qb_comm, n: i32) -> qb_status;
    pub fn qb_comm_destroy(c: *mut qb_comm);
    pub fn qb_multi_search_batch(c: *mut qb_comm, shard: *mut qb_storage, queries: *const f32, n_queries: u32, top: u32, deleted_bitmap: *const u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_multi_search_batch_device(c: *mut qb_comm, shard: *mut qb_storage, dev_queries: *const f32, n_queries: u32, top: u32, dev_local: *mut qb_scored_point, dev_local_counts: *mut u32, dev_out: *mut qb_scored_point, dev_counts: *mut u32) -> qb_status;
    pub fn qb_comm_stream(c: *mut qb_comm) -> *mut c_void;
    pub fn qb_comm_check(c: *mut qb_comm) -> qb_status;
    pub fn qb_hnsw_create_plain(s: *mut qb_storage, links_bin: *const u8, n_bytes: u64, m: u32, m0: u32, out: *mut *mut qb_hnsw) -> qb_status;
    pub fn qb_hnsw_create_compressed(s: *mut qb_storage, bytes: *const u8, n_bytes: u64, out: *mut *mut qb_hnsw) -> qb_status;
    pub fn qb_hnsw_create_with_vectors(quantized: *mut qb_storage, bytes: *const u8, n_bytes: u64, out: *mut *mut qb_hnsw) -> qb_status;
    pub fn qb_hnsw_links(g: *const qb_hnsw, level: u32, ids: *const u32, n_ids: u32, cap: u32, out: *mut u32, counts: *mut u32) -> qb_status;
    pub fn qb_hnsw_destroy(g: *mut qb_hnsw);
    pub fn qb_hnsw_info(g: *const qb_hnsw, n_points: *mut u32, levels: *mut u32, hbm_bytes: *mut u64) -> qb_status;
    pub fn qb_hnsw_build(s: *mut qb_storage, m: u32, m0: u32, ef_construct: u32, levels: *const u8, batch: u32, serial_points: u32, out: *mut *mut qb_hnsw, entry_point: *mut u32, entry_level: *mut u32) -> qb_status;
    pub fn qb_hnsw_build_incremental(s: *mut qb_storage, old: *const qb_hnsw, old_to_new: *const u32, ef_construct: u32, levels: *const u8, batch: u32, serial_points: u32, out: *mut *mut qb_hnsw, entry_point: *mut u32, entry_level: *mut u32) -> qb_status;
    pub fn qb_hnsw_export_plain(g: *const qb_hnsw, out: *mut u8, cap: u64, n_bytes: *mut u64) -> qb_status;
    pub fn qb_hnsw_search_batch(g: *mut qb_hnsw, queries: *const f32, n_queries: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, deleted_bitmap: *const u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_hnsw_search_batch_device(g: *mut qb_hnsw, dev_queries: *const f32, n_queries: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, dev_out: *mut qb_scored_point, dev_counts: *mut u32) -> qb_status;
    pub fn qb_hnsw_search_batch_algo(g: *mut qb_hnsw, queries: *const f32, n_queries: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, deleted_bitmap: *const u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters, algorithm: i32) -> qb_status;
    pub fn qb_hnsw_search_batch_device_algo(g: *mut qb_hnsw, dev_queries: *const f32, n_queries: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, dev_out: *mut qb_scored_point, dev_counts: *mut u32, algorithm: i32) -> qb_status;
    pub fn qb_hnsw_stats(g: *mut qb_hnsw, hops: *mut u64, scored_points: *mut u64, reset: i32) -> qb_status;
    pub fn qb_hnsw_search_with_vectors_batch(g: *mut qb_hnsw, queries: *const f32, n_queries: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, deleted_bitmap: *const u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_hnsw_search_with_vectors_batch_device(g: *mut qb_hnsw, dev_queries: *const f32, n_queries: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, dev_out: *mut qb_scored_point, dev_counts: *mut u32) -> qb_status;
    pub fn qb_hnsw_create_plain_multivector(tokens: *mut qb_storage, point_offsets: *const u32, n_points: u32, links_bin: *const u8, n_bytes: u64, m: u32, m0: u32, out: *mut *mut qb_hnsw) -> qb_status;
    pub fn qb_hnsw_create_compressed_multivector(tokens: *mut qb_storage, point_offsets: *const u32, n_points: u32, bytes: *const u8, n_bytes: u64, out: *mut *mut qb_hnsw) -> qb_status;
    pub fn qb_hnsw_build_multivector(tokens: *mut qb_storage, point_offsets: *const u32, n_points: u32, m: u32, m0: u32, ef_construct: u32, levels: *const u8, deleted_points: *const u64, batch: u32, serial_points: u32, out: *mut *mut qb_hnsw, entry_point: *mut u32, entry_level: *mut u32) -> qb_status;
    pub fn qb_hnsw_search_maxsim_batch(g: *mut qb_hnsw, query_vectors: *const f32, query_offsets: *const u32, n_queries: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, deleted_points: *const u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters, algorithm: i32) -> qb_status;
    pub fn qb_hnsw_search_maxsim_batch_device(g: *mut qb_hnsw, dev_query_vectors: *const f32, n_query_vectors: u32, dev_query_offsets: *const u32, n_queries: u32, max_query_vectors: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, dev_out: *mut qb_scored_point, dev_counts: *mut u32, algorithm: i32) -> qb_status;
    pub fn qb_hnsw_search_maxsim_custom_batch(g: *mut qb_hnsw, kind: i32, example_vectors: *const f32, example_offsets: *const u32, n_a: u32, n_b: u32, coef: *const f32, n_queries: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, custom_entry_points: *const u32, custom_counts: *const u32, n_custom: u32, deleted_points: *const u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters, algorithm: i32) -> qb_status;
    pub fn qb_hnsw_search_maxsim_discover_batch(g: *mut qb_hnsw, example_vectors: *const f32, example_offsets: *const u32, n_pairs: u32, n_queries: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, deleted_points: *const u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters, algorithm: i32) -> qb_status;
    pub fn qb_hnsw_search_custom_batch(g: *mut qb_hnsw, kind: i32, vectors: *const f32, n_a: u32, n_b: u32, coef: *const f32, n_queries: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, custom_entry_points: *const u32, custom_counts: *const u32, n_custom: u32, deleted_bitmap: *const u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters, algorithm: i32) -> qb_status;
    pub fn qb_hnsw_search_discover_batch(g: *mut qb_hnsw, vectors: *const f32, n_pairs: u32, n_queries: u32, top: u32, ef: u32, entry_point: u32, entry_level: u32, deleted_bitmap: *const u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters, algorithm: i32) -> qb_status;
    pub fn qb_mmr_batch(s: *mut qb_storage, queries: *const f32, n_queries: u32, lambdas: *const f32, candidates: *const qb_scored_point, candidate_counts: *const u32, max_candidates: u32, limit: u32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_mmr_batch_device(s: *mut qb_storage, dev_queries: *const f32, n_queries: u32, dev_lambdas: *const f32, dev_candidates: *const qb_scored_point, dev_candidate_counts: *const u32, max_candidates: u32, limit: u32, dev_out: *mut qb_scored_point, dev_out_counts: *mut u32) -> qb_status;
    pub fn qb_mmr_maxsim_batch(tokens: *mut qb_storage, point_offsets: *const u32, n_points: u32, query_vectors: *const f32, query_offsets: *const u32, n_queries: u32, lambdas: *const f32, candidates: *const qb_scored_point, candidate_counts: *const u32, max_candidates: u32, limit: u32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_mmr_maxsim_batch_device(tokens: *mut qb_storage, point_offsets: *const u32, n_points: u32, dev_query_vectors: *const f32, n_query_vectors: u32, dev_query_offsets: *const u32, n_queries: u32, max_query_vectors: u32, dev_lambdas: *const f32, dev_candidates: *const qb_scored_point, dev_candidate_counts: *const u32, max_candidates: u32, limit: u32, dev_out: *mut qb_scored_point, dev_out_counts: *mut u32) -> qb_status;
    pub fn qb_mmr_sparse_batch(s: *mut qb_sparse_storage, q_indptr: *const u64, q_dims: *const u32, q_weights: *const f32, n_queries: u32, lambdas: *const f32, candidates: *const qb_scored_point, candidate_counts: *const u32, max_candidates: u32, limit: u32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_sparse_index_create(device: i32, kind: i32, n_points: u32, n_dims: u32, indptr: *const u64, dims: *const u32, weights: *const f32, out: *mut *mut qb_sparse_index) -> qb_status;
    pub fn qb_sparse_index_destroy(idx: *mut qb_sparse_index);
    pub fn qb_sparse_index_info(idx: *const qb_sparse_index, n_points: *mut u32, n_dims: *mut u32, n_elements: *mut u64, hbm_bytes: *mut u64) -> qb_status;
    pub fn qb_sparse_index_stream(idx: *mut qb_sparse_index) -> *mut c_void;
    pub fn qb_sparse_search_batch(idx: *mut qb_sparse_index, q_indptr: *const u64, q_dims: *const u32, q_weights: *const f32, n_queries: u32, top: u32, deleted_bitmap: *const u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_sparse_search_batch_device(idx: *mut qb_sparse_index, dev_q_indptr: *const u64, dev_q_dims: *const u32, dev_q_weights: *const f32, n_queries: u32, max_query_nnz: u32, top: u32, dev_deleted_bitmap: *const u64, dev_out: *mut qb_scored_point, dev_out_counts: *mut u32) -> qb_status;
    pub fn qb_sparse_search_plain_batch(idx: *mut qb_sparse_index, q_indptr: *const u64, q_dims: *const u32, q_weights: *const f32, n_queries: u32, id_indptr: *const u64, ids: *const u32, top: u32, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_sparse_storage_create(device: i32, n_points: u32, indptr: *const u64, dims: *const u32, weights: *const f32, on_disk: i32, out: *mut *mut qb_sparse_storage) -> qb_status;
    pub fn qb_sparse_storage_destroy(s: *mut qb_sparse_storage);
    pub fn qb_sparse_storage_info(s: *const qb_sparse_storage, n_points: *mut u32, n_elements: *mut u64, hbm_bytes: *mut u64) -> qb_status;
    pub fn qb_sparse_search_custom_batch(s: *mut qb_sparse_storage, kind: i32, n_a: u32, n_b: u32, ex_indptr: *const u64, ex_dims: *const u32, ex_weights: *const f32, coef: *const f32, n_queries: u32, top: u32, deleted_bitmap: *const u64, id_list: *const u32, n_ids: u64, is_stopped: *const i32, out: *mut qb_scored_point, out_counts: *mut u32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_sparse_score_custom(s: *mut qb_sparse_storage, kind: i32, n_a: u32, n_b: u32, ex_indptr: *const u64, ex_dims: *const u32, ex_weights: *const f32, coef: *const f32, ids: *const u32, n: u64, scores: *mut f32, counters: *mut qb_hw_counters) -> qb_status;
    pub fn qb_search_stats(s: *mut qb_storage, searches: *mut u64, reruns: *mut u64, reset: i32) -> qb_status;
    pub fn qb_profile_enable(s: *mut qb_storage, on: i32) -> qb_status;
    pub fn qb_profile_read(s: *mut qb_storage, launches: *mut u64, total_ms: *mut f64, reset: i32) -> qb_status;
}
