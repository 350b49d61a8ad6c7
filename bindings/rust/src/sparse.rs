//! Sparse vectors on the GPU: the inverted index of a sparse named vector and `SearchContext` over it
//! (lib/sparse/src/index/search_context.rs).  SOURCE ONLY (see ffi.rs).  The caller keeps the `IndicesTracker` remapping on the host and
//! passes internal dims; `search` replaces `SearchContext::search`, `plain_search` replaces `SearchContext::plain_search` over the
//! prefiltered points.  `Ram` may prune like `InvertedIndexRam`; `Compressed` never prunes, like the compressed indexes with f32 weights.
//! `B200SparseStorage` holds the segment's sparse vector storage in user dims and replaces `search_scored` for the queries that are not
//! Nearest (recommend, discover, context, feedback), which skip the inverted index, and the MMR rerank of sparse candidates (`mmr`), which
//! replaces `mmr_from_points_with_vector` for a sparse named vector.
use common::counter::hardware_counter::HardwareCounterCell;
use common::types::{PointOffsetType, ScoredPointOffset};

use super::ffi::*;
use super::raw_scorer::last_error;
use crate::common::operation_error::{OperationError, OperationResult};
use sparse::common::sparse_vector::{RemappedSparseVector, SparseVector};

pub enum B200SparseKind { Ram, Compressed }

pub struct B200SparseIndex { raw: *mut qb_sparse_index }

unsafe impl Send for B200SparseIndex {}
unsafe impl Sync for B200SparseIndex {}

fn flatten(v: &[&RemappedSparseVector]) -> (Vec<u64>, Vec<u32>, Vec<f32>) {
    let mut ptr = Vec::with_capacity(v.len() + 1);
    ptr.push(0u64);
    let (mut dims, mut w) = (Vec::new(), Vec::new());
    for x in v {
        dims.extend_from_slice(&x.indices);
        w.extend_from_slice(&x.values);
        ptr.push(dims.len() as u64);
    }
    (ptr, dims, w)
}

impl B200SparseIndex {
    /// Points 0..n in order (an empty vector for a point without one), internal dims < n_dims.
    pub fn new(device: i32, kind: B200SparseKind, points: &[&RemappedSparseVector], n_dims: u32) -> OperationResult<Self> {
        let (ptr, dims, w) = flatten(points);
        let k = match kind { B200SparseKind::Ram => QB_SPARSE_RAM, B200SparseKind::Compressed => QB_SPARSE_COMPRESSED };
        let mut raw = std::ptr::null_mut();
        let st = unsafe { qb_sparse_index_create(device, k, points.len() as u32, n_dims, ptr.as_ptr(), dims.as_ptr(), w.as_ptr(), &mut raw) };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        Ok(Self { raw })
    }

    fn lists(out: &[qb_scored_point], counts: &[u32], top: usize) -> Vec<Vec<ScoredPointOffset>> {
        (0..counts.len()).map(|q| out[q * top..q * top + counts[q] as usize].iter()
            .map(|p| ScoredPointOffset { idx: p.idx as PointOffsetType, score: p.score }).collect()).collect()
    }

    /// `SearchContext::search` per query; `deleted` holds ceil(n_points / 64) words, bit = 1 filtered out.
    pub fn search(&self, queries: &[&RemappedSparseVector], top: usize, deleted: Option<&[u64]>, hc: &HardwareCounterCell)
        -> OperationResult<Vec<Vec<ScoredPointOffset>>> {
        let (ptr, dims, w) = flatten(queries);
        let nq = queries.len();
        let mut out = vec![qb_scored_point { idx: 0, score: 0.0 }; nq * top.max(1)];
        let mut counts = vec![0u32; nq];
        let mut counters = qb_hw_counters::default();
        let st = unsafe {
            qb_sparse_search_batch(self.raw, ptr.as_ptr(), dims.as_ptr(), w.as_ptr(), nq as u32, top as u32, deleted.map_or(std::ptr::null(), |d| d.as_ptr()),
                                   std::ptr::null(), out.as_mut_ptr(), counts.as_mut_ptr(), &mut counters)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        hc.cpu_counter().incr_delta(counters.cpu as usize);
        Ok(Self::lists(&out, &counts, top))
    }

    /// `SearchContext::plain_search` per query over its own prefiltered ids.
    pub fn plain_search(&self, queries: &[&RemappedSparseVector], ids: &[&[PointOffsetType]], top: usize, hc: &HardwareCounterCell)
        -> OperationResult<Vec<Vec<ScoredPointOffset>>> {
        let (ptr, dims, w) = flatten(queries);
        let nq = queries.len();
        let mut iptr = vec![0u64];
        let mut flat_ids = Vec::new();
        for l in ids { flat_ids.extend_from_slice(l); iptr.push(flat_ids.len() as u64); }
        let mut out = vec![qb_scored_point { idx: 0, score: 0.0 }; nq * top.max(1)];
        let mut counts = vec![0u32; nq];
        let mut counters = qb_hw_counters::default();
        let st = unsafe {
            qb_sparse_search_plain_batch(self.raw, ptr.as_ptr(), dims.as_ptr(), w.as_ptr(), nq as u32, iptr.as_ptr(), flat_ids.as_ptr(), top as u32,
                                         std::ptr::null(), out.as_mut_ptr(), counts.as_mut_ptr(), &mut counters)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        hc.cpu_counter().incr_delta(counters.cpu as usize);
        Ok(Self::lists(&out, &counts, top))
    }
}

impl Drop for B200SparseIndex {
    fn drop(&mut self) { unsafe { qb_sparse_index_destroy(self.raw) } }
}

/// The sparse vector storage of a named vector (user dims) for `search_scored`: peek_top_iter with a SparseCustomQueryScorer.
pub struct B200SparseStorage { raw: *mut qb_sparse_storage }

unsafe impl Send for B200SparseStorage {}
unsafe impl Sync for B200SparseStorage {}

fn flatten_user(v: &[&SparseVector]) -> (Vec<u64>, Vec<u32>, Vec<f32>) {
    let mut ptr = Vec::with_capacity(v.len() + 1);
    ptr.push(0u64);
    let (mut dims, mut w) = (Vec::new(), Vec::new());
    for x in v {
        dims.extend_from_slice(&x.indices);
        w.extend_from_slice(&x.values);
        ptr.push(dims.len() as u64);
    }
    (ptr, dims, w)
}

impl B200SparseStorage {
    /// Points 0..n in order (an empty vector for a point without one); `on_disk` for an mmap storage (vector_io_read counted).
    pub fn new(device: i32, points: &[&SparseVector], on_disk: bool) -> OperationResult<Self> {
        let (ptr, dims, w) = flatten_user(points);
        let mut raw = std::ptr::null_mut();
        let st = unsafe { qb_sparse_storage_create(device, points.len() as u32, ptr.as_ptr(), dims.as_ptr(), w.as_ptr(), on_disk as i32, &mut raw) };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        Ok(Self { raw })
    }

    /// `search_scored` for a batch of queries of one kind and shape (`kind`, `n_a`, `n_b` as qb_scorer_create_custom takes them):
    /// `examples` holds E examples per query in its order; `coef` [a, partial...] per query for feedback.  `deleted`: ceil(n_points / 64)
    /// words, bit = 1 filtered out; `prefiltered`: the ids to score, shared by the batch.
    pub fn search_custom(&self, kind: i32, examples: &[&SparseVector], n_a: usize, n_b: usize, coef: Option<&[f32]>, top: usize, deleted: Option<&[u64]>,
                         prefiltered: Option<&[PointOffsetType]>, hc: &HardwareCounterCell) -> OperationResult<Vec<Vec<ScoredPointOffset>>> {
        let n_ex = match kind { 1 | 2 => n_a + n_b, 4 => 2 * n_a, _ => 1 + 2 * n_a };
        let nq = examples.len() / n_ex.max(1);
        let (ptr, dims, w) = flatten_user(examples);
        let mut out = vec![qb_scored_point { idx: 0, score: 0.0 }; nq * top.max(1)];
        let mut counts = vec![0u32; nq];
        let mut counters = qb_hw_counters::default();
        let (ids, n_ids) = prefiltered.map_or((std::ptr::null(), 0), |p| (p.as_ptr(), p.len() as u64));
        let st = unsafe {
            qb_sparse_search_custom_batch(self.raw, kind, n_a as u32, n_b as u32, ptr.as_ptr(), dims.as_ptr(), w.as_ptr(), coef.map_or(std::ptr::null(), |c| c.as_ptr()),
                                          nq as u32, top as u32, deleted.map_or(std::ptr::null(), |d| d.as_ptr()), ids, n_ids, std::ptr::null(),
                                          out.as_mut_ptr(), counts.as_mut_ptr(), &mut counters)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        hc.cpu_counter().incr_delta(counters.cpu as usize);
        hc.vector_io_read().incr_delta(counters.vector_io_read as usize);
        Ok(B200SparseIndex::lists(&out, &counts, top))
    }

    /// `score_stored_batch` of one query over `ids`.
    pub fn score_custom(&self, kind: i32, examples: &[&SparseVector], n_a: usize, n_b: usize, coef: Option<&[f32]>, ids: &[PointOffsetType],
                        hc: &HardwareCounterCell) -> OperationResult<Vec<f32>> {
        let (ptr, dims, w) = flatten_user(examples);
        let mut scores = vec![0f32; ids.len()];
        let mut counters = qb_hw_counters::default();
        let st = unsafe {
            qb_sparse_score_custom(self.raw, kind, n_a as u32, n_b as u32, ptr.as_ptr(), dims.as_ptr(), w.as_ptr(), coef.map_or(std::ptr::null(), |c| c.as_ptr()),
                                   ids.as_ptr(), ids.len() as u64, scores.as_mut_ptr(), &mut counters)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        hc.cpu_counter().incr_delta(counters.cpu as usize);
        hc.vector_io_read().incr_delta(counters.vector_io_read as usize);
        Ok(scores)
    }

    /// MMR over sparse candidates whose vectors are this storage's points: `queries[q]` in user dims (any order), `candidates[q]` are
    /// (point id, score) pairs (at most 16 384), `lambdas[q]` = 1 - diversity.  Returns each query's selection, in selection order, with
    /// the candidates' own scores.
    pub fn mmr(&self, queries: &[&SparseVector], candidates: &[&[ScoredPointOffset]], lambdas: &[f32], limit: usize,
               hc: &HardwareCounterCell) -> OperationResult<Vec<Vec<ScoredPointOffset>>> {
        let nq = queries.len();
        let (ptr, dims, w) = flatten_user(queries);
        let max_c = candidates.iter().map(|c| c.len()).max().unwrap_or(0);
        let mut cand = vec![qb_scored_point { idx: 0, score: 0.0 }; nq * max_c.max(1)];
        let mut counts = Vec::with_capacity(nq);
        for (q, c) in candidates.iter().enumerate() {
            for (i, p) in c.iter().enumerate() { cand[q * max_c + i] = qb_scored_point { idx: p.idx as PointOffsetType, score: p.score }; }
            counts.push(c.len() as u32);
        }
        let mut out = vec![qb_scored_point { idx: 0, score: 0.0 }; nq * limit.max(1)];
        let mut out_counts = vec![0u32; nq];
        let mut counters = qb_hw_counters::default();
        let st = unsafe {
            qb_mmr_sparse_batch(self.raw, ptr.as_ptr(), dims.as_ptr(), w.as_ptr(), nq as u32, lambdas.as_ptr(), cand.as_ptr(), counts.as_ptr(), max_c as u32,
                                limit as u32, out.as_mut_ptr(), out_counts.as_mut_ptr(), &mut counters)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        hc.cpu_counter().incr_delta(counters.cpu as usize);
        hc.vector_io_read().incr_delta(counters.vector_io_read as usize);
        Ok(B200SparseIndex::lists(&out, &out_counts, limit))
    }
}

impl Drop for B200SparseStorage {
    fn drop(&mut self) { unsafe { qb_sparse_storage_destroy(self.raw) } }
}
