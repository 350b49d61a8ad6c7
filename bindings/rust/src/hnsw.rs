//! `GraphLayers::search` (lib/segment/src/index/hnsw_index/graph_layers.rs:530-561) for a batch of queries with the traversal on the GPU.
//! SOURCE ONLY (see ffi.rs).  The graph is handed over as the bytes of `links.bin`, either in GraphLinksFormat::Compressed (what
//! the reference writes for every index it builds, view.rs:137-163; decoded on the device) or in GraphLinksFormat::Plain (view.rs:121-135).
use common::counter::hardware_counter::HardwareCounterCell;
use common::types::{PointOffsetType, ScoredPointOffset};

use super::ffi::*;
use crate::data_types::vectors::{QueryVector, VectorInternal};
use crate::index::hnsw_index::graph_layers::SearchAlgorithm;
use super::raw_scorer::{last_error, B200Storage};
use crate::common::operation_error::{OperationError, OperationResult};

// qb_query_kind (include/qb200.h), passed as i32
const QB_QUERY_RECO_BEST_SCORE: i32 = 1;
const QB_QUERY_RECO_SUM_SCORES: i32 = 2;
const QB_QUERY_DISCOVER: i32 = 3;
const QB_QUERY_CONTEXT: i32 = 4;
const QB_QUERY_FEEDBACK_NAIVE: i32 = 5;

pub struct B200Hnsw<'a> { raw: *mut qb_hnsw, _storage: std::marker::PhantomData<&'a B200Storage> }
unsafe impl Send for B200Hnsw<'_> {}
unsafe impl Sync for B200Hnsw<'_> {}
impl Drop for B200Hnsw<'_> { fn drop(&mut self) { unsafe { qb_hnsw_destroy(self.raw) } } }

impl<'a> B200Hnsw<'a> {
    pub fn from_plain_links(storage: &'a B200Storage, links_bin: &[u8], m: usize, m0: usize) -> OperationResult<Self> {
        let mut raw = std::ptr::null_mut();
        let st = unsafe { qb_hnsw_create_plain(storage.raw, links_bin.as_ptr(), links_bin.len() as u64, m as u32, m0 as u32, &mut raw) };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        Ok(Self { raw, _storage: std::marker::PhantomData })
    }

    /// `links.bin` in GraphLinksFormat::CompressedWithVectors (inline storage), bound to the segment's SQ8 storage.
    pub fn from_compressed_links_with_vectors(quantized: &'a B200Storage, links_bin: &[u8]) -> OperationResult<Self> {
        let mut raw = std::ptr::null_mut();
        let st = unsafe { qb_hnsw_create_with_vectors(quantized.raw, links_bin.as_ptr(), links_bin.len() as u64, &mut raw) };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        Ok(Self { raw, _storage: std::marker::PhantomData })
    }

    /// `links.bin` (Compressed) of a multivector named vector: a graph over POINTS, point p being token rows
    /// [point_offsets[p], point_offsets[p + 1]) of `tokens` (dense f32 or SQ8).  Search it with `search_maxsim`.
    pub fn from_compressed_links_multivector(tokens: &'a B200Storage, point_offsets: &[u32], links_bin: &[u8]) -> OperationResult<Self> {
        let mut raw = std::ptr::null_mut();
        let n_points = point_offsets.len().saturating_sub(1) as u32;
        let st = unsafe {
            qb_hnsw_create_compressed_multivector(tokens.raw, point_offsets.as_ptr(), n_points, links_bin.as_ptr(), links_bin.len() as u64, &mut raw)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        Ok(Self { raw, _storage: std::marker::PhantomData })
    }

    /// `links.bin` in GraphLinksFormat::Compressed; m and m0 come from its header.  CompressedWithVectors is refused (see
    /// `from_compressed_links_with_vectors`).
    pub fn from_compressed_links(storage: &'a B200Storage, links_bin: &[u8]) -> OperationResult<Self> {
        let mut raw = std::ptr::null_mut();
        let st = unsafe { qb_hnsw_create_compressed(storage.raw, links_bin.as_ptr(), links_bin.len() as u64, &mut raw) };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        Ok(Self { raw, _storage: std::marker::PhantomData })
    }

    /// Builds the graph on the device, in place of `build_hnsw_on_gpu` (gpu/gpu_graph_builder.rs) and of the CPU
    /// `GraphLayersBuilder::link_new_point` pool (hnsw/build.rs:285-355) for a dense f32 or Uint8 storage.  The adapter keeps on the host:
    /// the level draw (`GraphLayersBuilder::get_random_layer`, one u8 per point), the mapping between point offsets and the
    /// storage's rows, the deleted flags (set on the storage beforehand), and writing `links.bin` in the compressed format from
    /// `export_plain` (GraphLinksSerializer).  Returns the graph and its entry point (id, level).
    pub fn build(storage: &'a B200Storage, m: usize, m0: usize, ef_construct: usize, levels: &[u8], batch: usize, serial_points: usize)
        -> OperationResult<(Self, (PointOffsetType, usize))> {
        let mut raw = std::ptr::null_mut();
        let (mut entry, mut level) = (0u32, 0u32);
        let st = unsafe {
            qb_hnsw_build(storage.raw, m as u32, m0 as u32, ef_construct as u32, levels.as_ptr(), batch as u32, serial_points as u32, &mut raw, &mut entry,
                          &mut level)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        Ok((Self { raw, _storage: std::marker::PhantomData }, (entry, level as usize)))
    }

    /// Builds the graph from the old segment's graph on the device (qb_hnsw_build_incremental), in place of the old-index path of
    /// `HNSWIndex::build` (hnsw/build.rs:225-357): `GraphLayersHealer` heals the lists that link to a removed point,
    /// `save_into_builder` renumbers them, and only the points the old graph did not have are inserted.  The adapter keeps on the
    /// host `OldIndexCandidate::evaluate` (whether to reuse `old`, and `old_to_new`: one per old point, `u32::MAX` = not carried
    /// over) and the level draw for the new points (`levels`: one per point, the reused ones keeping their old level).  `m` / `m0`
    /// are `old`'s.  Returns the graph and its entry point (id, level).
    pub fn build_incremental(storage: &'a B200Storage, old: &B200Hnsw<'_>, old_to_new: &[u32], ef_construct: usize, levels: &[u8], batch: usize,
                             serial_points: usize) -> OperationResult<(Self, (PointOffsetType, usize))> {
        let mut raw = std::ptr::null_mut();
        let (mut entry, mut level) = (0u32, 0u32);
        let st = unsafe {
            qb_hnsw_build_incremental(storage.raw, old.raw, old_to_new.as_ptr(), ef_construct as u32, levels.as_ptr(), batch as u32, serial_points as u32,
                                      &mut raw, &mut entry, &mut level)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        Ok((Self { raw, _storage: std::marker::PhantomData }, (entry, level as usize)))
    }

    /// Builds the graph over the POINTS of a multivector named vector on the device (qb_hnsw_build_multivector): `build`'s schedule
    /// with MaxSim between stored points, point p being token rows [point_offsets[p], point_offsets[p + 1]) of the dense f32 `tokens`.
    /// `levels`: one per point; `deleted`: a bitmap over points (not inserted), or None.  Search it with `search_maxsim`.  Returns the
    /// graph and its entry point (id, level).
    pub fn build_multivector(tokens: &'a B200Storage, point_offsets: &[u32], m: usize, m0: usize, ef_construct: usize, levels: &[u8],
                             deleted: Option<&[u64]>, batch: usize, serial_points: usize) -> OperationResult<(Self, (PointOffsetType, usize))> {
        if point_offsets.len() != levels.len() + 1 {
            return Err(OperationError::service_error("levels and point_offsets disagree on the point count"));
        }
        let mut raw = std::ptr::null_mut();
        let (mut entry, mut level) = (0u32, 0u32);
        let st = unsafe {
            qb_hnsw_build_multivector(tokens.raw, point_offsets.as_ptr(), levels.len() as u32, m as u32, m0 as u32, ef_construct as u32, levels.as_ptr(),
                                      deleted.map_or(std::ptr::null(), |d| d.as_ptr()), batch as u32, serial_points as u32, &mut raw, &mut entry, &mut level)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        Ok((Self { raw, _storage: std::marker::PhantomData }, (entry, level as usize)))
    }

    /// The graph as a plain `links.bin` (GraphLinksFormat::Plain), whichever way it was made.
    pub fn export_plain(&self) -> OperationResult<Vec<u8>> {
        let mut n = 0u64;
        if unsafe { qb_hnsw_export_plain(self.raw, std::ptr::null_mut(), 0, &mut n) } != QB_OK { return Err(OperationError::service_error(last_error())); }
        let mut out = vec![0u8; n as usize];
        if unsafe { qb_hnsw_export_plain(self.raw, out.as_mut_ptr(), n, &mut n) } != QB_OK { return Err(OperationError::service_error(last_error())); }
        Ok(out)
    }

    /// `entry` = GraphLayers::get_entry_point(filters, custom_entry_points) (it depends on the filter, so it stays host logic);
    /// `deleted` = the filter as a bitmap (bit = 1: check_vector fails), or None;
    /// `algorithm` = the level-0 algorithm GraphLayers::search dispatches on, as hnsw/read_view/search.rs:59-86 chooses it.
    pub fn search_batch(&self, queries: &[f32], n_queries: usize, top: usize, ef: usize, entry: (PointOffsetType, usize), deleted: Option<&[u64]>,
                        algorithm: SearchAlgorithm) -> Vec<Vec<ScoredPointOffset>> {
        let mut out = vec![qb_scored_point::default(); n_queries * top];
        let mut counts = vec![0u32; n_queries];
        let algo = match algorithm { SearchAlgorithm::Hnsw => QB_HNSW_ALGO_HNSW, SearchAlgorithm::Acorn => QB_HNSW_ALGO_ACORN };
        let st = unsafe {
            qb_hnsw_search_batch_algo(self.raw, queries.as_ptr(), n_queries as u32, top as u32, ef as u32, entry.0, entry.1 as u32,
                                      deleted.map_or(std::ptr::null(), |d| d.as_ptr()), std::ptr::null(), out.as_mut_ptr(), counts.as_mut_ptr(),
                                      std::ptr::null_mut(), algo)
        };
        assert!(st == QB_OK, "{}", last_error());
        (0..n_queries).map(|q| out[q * top..q * top + counts[q] as usize].iter().map(|p| ScoredPointOffset { idx: p.idx, score: p.score }).collect()).collect()
    }

    /// `GraphLayers::search_with_vectors` (graph_layers.rs:564-596) on a `from_compressed_links_with_vectors` graph.  The dispatch of
    /// hnsw/read_view/search.rs:88-178 stays with the caller: this search when the graph has inline vectors, the search is quantized
    /// and the algorithm is HNSW, with ef = max(ef, oversampled top); otherwise `search_batch` on the same handle.
    pub fn search_with_vectors(&self, queries: &[f32], n_queries: usize, top: usize, ef: usize, entry: (PointOffsetType, usize), deleted: Option<&[u64]>)
                               -> Vec<Vec<ScoredPointOffset>> {
        let mut out = vec![qb_scored_point::default(); n_queries * top];
        let mut counts = vec![0u32; n_queries];
        let st = unsafe {
            qb_hnsw_search_with_vectors_batch(self.raw, queries.as_ptr(), n_queries as u32, top as u32, ef as u32, entry.0, entry.1 as u32,
                                              deleted.map_or(std::ptr::null(), |d| d.as_ptr()), std::ptr::null(), out.as_mut_ptr(), counts.as_mut_ptr(),
                                              std::ptr::null_mut())
        };
        assert!(st == QB_OK, "{}", last_error());
        (0..n_queries).map(|q| out[q * top..q * top + counts[q] as usize].iter().map(|p| ScoredPointOffset { idx: p.idx, score: p.score }).collect()).collect()
    }

    /// `GraphLayers::search` with a MaxSim `FilteredScorer` (MultiMetricQueryScorer / QuantizedMultivectorStorage) on a
    /// `from_compressed_links_multivector` graph: query i = rows [query_offsets[i], query_offsets[i + 1]) of `query_vectors` (raw f32 x dim,
    /// 1..4096 vectors each); `deleted` is a bitmap over points.  Scores equal qb_score_maxsim bit for bit.
    pub fn search_maxsim(&self, query_vectors: &[f32], query_offsets: &[u32], top: usize, ef: usize, entry: (PointOffsetType, usize),
                         deleted: Option<&[u64]>, algorithm: SearchAlgorithm) -> Vec<Vec<ScoredPointOffset>> {
        let n_queries = query_offsets.len().saturating_sub(1);
        let mut out = vec![qb_scored_point::default(); n_queries * top];
        let mut counts = vec![0u32; n_queries];
        let algo = match algorithm { SearchAlgorithm::Hnsw => QB_HNSW_ALGO_HNSW, SearchAlgorithm::Acorn => QB_HNSW_ALGO_ACORN };
        let st = unsafe {
            qb_hnsw_search_maxsim_batch(self.raw, query_vectors.as_ptr(), query_offsets.as_ptr(), n_queries as u32, top as u32, ef as u32, entry.0,
                                        entry.1 as u32, deleted.map_or(std::ptr::null(), |d| d.as_ptr()), std::ptr::null(), out.as_mut_ptr(),
                                        counts.as_mut_ptr(), std::ptr::null_mut(), algo)
        };
        assert!(st == QB_OK, "{}", last_error());
        (0..n_queries).map(|q| out[q * top..q * top + counts[q] as usize].iter().map(|p| ScoredPointOffset { idx: p.idx, score: p.score }).collect()).collect()
    }

    /// `GraphLayers::search` with a MultiCustomQueryScorer on a multivector graph: custom queries whose examples are multivectors, one kind
    /// and shape per call (`kind`, `n_a`, `n_b` as qb_scorer_create_custom takes them, E examples per query in its order).  Example j of
    /// query q = rows [example_offsets[q * E + j], example_offsets[q * E + j + 1]) of `example_vectors` (raw f32 x dim, 1..4096 vectors
    /// each); `coef`: [a, partial...] per query for feedback.  QB_QUERY_DISCOVER runs both stages of discover_search_with_graph in one
    /// call (qb_hnsw_search_maxsim_discover_batch); the other kinds go through qb_hnsw_search_maxsim_custom_batch with
    /// `custom_entry_points` (n_queries x n_custom, `custom_counts[q]` valid).  `deleted` is a bitmap over points.  Scores equal
    /// qb_score_maxsim_custom bit for bit.
    pub fn search_maxsim_custom(&self, kind: i32, example_vectors: &[f32], example_offsets: &[u32], n_a: usize, n_b: usize, coef: Option<&[f32]>,
                                top: usize, ef: usize, entry: (PointOffsetType, usize), custom_entry_points: Option<(&[PointOffsetType], &[u32], usize)>,
                                deleted: Option<&[u64]>, algorithm: SearchAlgorithm, hc: &HardwareCounterCell)
                                -> OperationResult<Vec<Vec<ScoredPointOffset>>> {
        let n_ex = match kind { QB_QUERY_RECO_BEST_SCORE | QB_QUERY_RECO_SUM_SCORES => n_a + n_b, QB_QUERY_CONTEXT => 2 * n_a, _ => 1 + 2 * n_a };
        let n_queries = example_offsets.len().saturating_sub(1) / n_ex.max(1);
        let mut out = vec![qb_scored_point::default(); n_queries * top];
        let mut counts = vec![0u32; n_queries];
        let mut counters = qb_hw_counters::default();
        let algo = match algorithm { SearchAlgorithm::Hnsw => QB_HNSW_ALGO_HNSW, SearchAlgorithm::Acorn => QB_HNSW_ALGO_ACORN };
        let del = deleted.map_or(std::ptr::null(), |d| d.as_ptr());
        let st = unsafe {
            if kind == QB_QUERY_DISCOVER {
                qb_hnsw_search_maxsim_discover_batch(self.raw, example_vectors.as_ptr(), example_offsets.as_ptr(), n_a as u32, n_queries as u32, top as u32,
                                                     ef as u32, entry.0, entry.1 as u32, del, std::ptr::null(), out.as_mut_ptr(), counts.as_mut_ptr(),
                                                     &mut counters, algo)
            } else {
                let (cep, cep_counts, n_custom) = custom_entry_points.map_or((std::ptr::null(), std::ptr::null(), 0), |(c, n, w)| (c.as_ptr(), n.as_ptr(), w));
                qb_hnsw_search_maxsim_custom_batch(self.raw, kind, example_vectors.as_ptr(), example_offsets.as_ptr(), n_a as u32, n_b as u32,
                                                   coef.map_or(std::ptr::null(), |c| c.as_ptr()), n_queries as u32, top as u32, ef as u32, entry.0,
                                                   entry.1 as u32, cep, cep_counts, n_custom as u32, del, std::ptr::null(), out.as_mut_ptr(),
                                                   counts.as_mut_ptr(), &mut counters, algo)
            }
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        hc.cpu_counter().incr_delta(counters.cpu as usize);
        hc.vector_io_read().incr_delta(counters.vector_io_read as usize);
        Ok((0..n_queries).map(|q| out[q * top..q * top + counts[q] as usize].iter().map(|p| ScoredPointOffset { idx: p.idx, score: p.score }).collect()).collect())
    }

    /// `GraphLayers::search` with a custom `FilteredScorer` for ONE query vector of `search_vectors_with_graph`
    /// (hnsw/read_view/search.rs:181-208): RecommendBestScore / RecommendSumScores / Context through qb_hnsw_search_custom_batch,
    /// Discover through qb_hnsw_search_discover_batch (both stages of discover_search_with_graph, :314-349, in one call).
    /// Nearest goes through `search_batch`; a feedback query goes through `search_feedback` (its pairs and coefficients are computed
    /// by the caller's FeedbackQuery).  `custom_entry_points` is GraphLayers::search's argument (not used for discover).
    pub fn search_custom(&self, query: &QueryVector, top: usize, ef: usize, entry: (PointOffsetType, usize), deleted: Option<&[u64]>,
                         custom_entry_points: Option<&[PointOffsetType]>, algorithm: SearchAlgorithm, hc: &HardwareCounterCell)
                         -> OperationResult<Vec<ScoredPointOffset>> {
        let dense = |v: &VectorInternal| -> OperationResult<Vec<f32>> {
            match v { VectorInternal::Dense(d) => Ok(d.clone()), _ => Err(OperationError::service_error("device traversal: dense examples only")) }
        };
        let (kind, mut flat, n_a, n_b) = match query {
            QueryVector::RecommendBestScore(r) | QueryVector::RecommendSumScores(r) => {
                let kind = if matches!(query, QueryVector::RecommendBestScore(_)) { QB_QUERY_RECO_BEST_SCORE } else { QB_QUERY_RECO_SUM_SCORES };
                (kind, Vec::new(), r.positives.len(), r.negatives.len())
            }
            QueryVector::Context(c) => (QB_QUERY_CONTEXT, Vec::new(), c.pairs.len(), 0),
            QueryVector::Discover(d) => (QB_QUERY_DISCOVER, Vec::new(), d.pairs.len(), 0),
            _ => return Err(OperationError::service_error("search_custom: nearest / feedback queries have their own calls")),
        };
        match query {
            QueryVector::RecommendBestScore(r) | QueryVector::RecommendSumScores(r) => {
                for v in r.positives.iter().chain(r.negatives.iter()) { flat.extend(dense(v)?); }
            }
            QueryVector::Context(c) => { for p in &c.pairs { flat.extend(dense(&p.positive)?); flat.extend(dense(&p.negative)?); } }
            QueryVector::Discover(d) => {
                flat.extend(dense(&d.target)?);
                for p in &d.pairs { flat.extend(dense(&p.positive)?); flat.extend(dense(&p.negative)?); }
            }
            _ => unreachable!(),
        }
        let mut out = vec![qb_scored_point::default(); top];
        let mut count = 0u32;
        let mut counters = qb_hw_counters::default();
        let algo = match algorithm { SearchAlgorithm::Hnsw => QB_HNSW_ALGO_HNSW, SearchAlgorithm::Acorn => QB_HNSW_ALGO_ACORN };
        let del = deleted.map_or(std::ptr::null(), |d| d.as_ptr());
        let st = unsafe {
            if kind == QB_QUERY_DISCOVER {
                qb_hnsw_search_discover_batch(self.raw, flat.as_ptr(), n_a as u32, 1, top as u32, ef as u32, entry.0, entry.1 as u32, del, std::ptr::null(),
                                              out.as_mut_ptr(), &mut count, &mut counters, algo)
            } else {
                let n_custom = custom_entry_points.map_or(0, |c| c.len() as u32);
                qb_hnsw_search_custom_batch(self.raw, kind, flat.as_ptr(), n_a as u32, n_b as u32, std::ptr::null(), 1, top as u32, ef as u32, entry.0,
                                            entry.1 as u32, custom_entry_points.map_or(std::ptr::null(), |c| c.as_ptr()), &n_custom, n_custom.max(1),
                                            del, std::ptr::null(), out.as_mut_ptr(), &mut count, &mut counters, algo)
            }
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        hc.cpu_counter().incr_delta(counters.cpu as usize);
        hc.vector_io_read().incr_delta(counters.vector_io_read as usize);
        Ok(out[..count as usize].iter().map(|p| ScoredPointOffset { idx: p.idx, score: p.score }).collect())
    }

    /// A naive-feedback query (FeedbackQuery, feedback_query.rs:150-226) through the device traversal: `target`, then its context pairs
    /// as (positive, negative) rows in `pairs`, `a` and each pair's partial_computation.
    pub fn search_feedback(&self, target: &[f32], pairs: &[f32], a: f32, partial: &[f32], top: usize, ef: usize, entry: (PointOffsetType, usize),
                           deleted: Option<&[u64]>, algorithm: SearchAlgorithm, hc: &HardwareCounterCell) -> OperationResult<Vec<ScoredPointOffset>> {
        let mut flat = target.to_vec();
        flat.extend_from_slice(pairs);
        let mut coef = vec![a];
        coef.extend_from_slice(partial);
        let mut out = vec![qb_scored_point::default(); top];
        let mut count = 0u32;
        let mut counters = qb_hw_counters::default();
        let algo = match algorithm { SearchAlgorithm::Hnsw => QB_HNSW_ALGO_HNSW, SearchAlgorithm::Acorn => QB_HNSW_ALGO_ACORN };
        let st = unsafe {
            qb_hnsw_search_custom_batch(self.raw, QB_QUERY_FEEDBACK_NAIVE, flat.as_ptr(), partial.len() as u32, 0, coef.as_ptr(), 1, top as u32, ef as u32,
                                        entry.0, entry.1 as u32, std::ptr::null(), std::ptr::null(), 0, deleted.map_or(std::ptr::null(), |d| d.as_ptr()),
                                        std::ptr::null(), out.as_mut_ptr(), &mut count, &mut counters, algo)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        hc.cpu_counter().incr_delta(counters.cpu as usize);
        hc.vector_io_read().incr_delta(counters.vector_io_read as usize);
        Ok(out[..count as usize].iter().map(|p| ScoredPointOffset { idx: p.idx, score: p.score }).collect())
    }
}
