//! Sparse vectors on the GPU: the inverted index of a sparse named vector and `SearchContext` over it
//! (lib/sparse/src/index/search_context.rs).  SOURCE ONLY (see ffi.rs).  The caller keeps the `IndicesTracker` remapping on the host and
//! passes internal dims; `search` replaces `SearchContext::search`, `plain_search` replaces `SearchContext::plain_search` over the
//! prefiltered points.  `Ram` may prune like `InvertedIndexRam`; `Compressed` never prunes, like the compressed indexes with f32 weights.
use common::counter::hardware_counter::HardwareCounterCell;
use common::types::{PointOffsetType, ScoredPointOffset};

use super::ffi::*;
use super::raw_scorer::last_error;
use crate::common::operation_error::{OperationError, OperationResult};
use sparse::common::sparse_vector::RemappedSparseVector;

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
