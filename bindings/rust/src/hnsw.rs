//! `GraphLayers::search` (lib/segment/src/index/hnsw_index/graph_layers.rs:530-561) for a batch of queries with the traversal on the GPU.
//! SOURCE ONLY (see ffi.rs).  The graph is handed over as the bytes of `links.bin`, either in GraphLinksFormat::Compressed (what
//! the reference writes for every index it builds, view.rs:137-163; decoded on the device) or in GraphLinksFormat::Plain (view.rs:121-135).
use common::types::{PointOffsetType, ScoredPointOffset};

use super::ffi::*;
use crate::index::hnsw_index::graph_layers::SearchAlgorithm;
use super::raw_scorer::{last_error, B200Storage};
use crate::common::operation_error::{OperationError, OperationResult};

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

    /// `links.bin` in GraphLinksFormat::Compressed; m and m0 come from its header.  CompressedWithVectors is refused.
    pub fn from_compressed_links(storage: &'a B200Storage, links_bin: &[u8]) -> OperationResult<Self> {
        let mut raw = std::ptr::null_mut();
        let st = unsafe { qb_hnsw_create_compressed(storage.raw, links_bin.as_ptr(), links_bin.len() as u64, &mut raw) };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        Ok(Self { raw, _storage: std::marker::PhantomData })
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
}
