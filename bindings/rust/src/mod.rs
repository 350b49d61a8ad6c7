//! `lib/segment/src/vector_storage/b200/` — the GPU-resident scorer behind the reference's own seams.  SOURCE ONLY: see ffi.rs.
pub mod ffi;             // generated from include/qb200.h (tools/gen_rust_ffi.py)
pub mod raw_scorer;      // impl RawScorer / RawScorerBuilder
pub mod batch_searcher;  // BatchFilteredSearcher::peek_top_* + oversample / rescore
pub mod hnsw;            // GraphLayers::search, batched, traversal on the device
pub mod sharded;         // per-GPU segments + device-side BatchResultAggregator
pub mod mmr;             // maximal marginal relevance reranking
pub mod sparse;          // sparse vectors: inverted index, SearchContext::search / plain_search; the storage's custom-query scan
