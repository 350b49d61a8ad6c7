//! Maximal marginal relevance (lib/shard/src/query/mmr/mod.rs:42-279) for dense vectors on the GPU.  SOURCE ONLY (see ffi.rs).
//! Replaces `mmr_from_points_with_vector` for a dense named vector: the caller either fills a temporary f32 `B200Storage` of the
//! collection's distance with the candidates' vectors (ids = their positions), as the reference's volatile storage holds them, or passes
//! the resident f32 segment storage whose rows are the vectors `with_vector` returns.  The selection keeps the input scores.
//! `mmr_maxsim` is the same rerank for a multivector named vector: the storage holds the candidates' token rows, `point_offsets` says
//! which rows make up each point, and pair scores are MaxSim (candidate c's tokens against the pick's).
use common::counter::hardware_counter::HardwareCounterCell;
use common::types::{PointOffsetType, ScoredPointOffset};

use super::ffi::*;
use super::raw_scorer::{last_error, B200Storage};
use crate::common::operation_error::{OperationError, OperationResult};

impl B200Storage {
    /// One MMR rerank per query: `candidates[q]` are (id, score) pairs in the storage's numbering (at most 16 384), `lambdas[q]` = 1 -
    /// diversity.  Returns each query's selection, in selection order, with the candidates' own scores.
    pub fn mmr(&self, queries: &[&[f32]], candidates: &[&[ScoredPointOffset]], lambdas: &[f32], limit: usize, hc: &HardwareCounterCell)
        -> OperationResult<Vec<Vec<ScoredPointOffset>>> {
        let nq = queries.len();
        let dim = queries.first().map_or(0, |q| q.len());
        let max_c = candidates.iter().map(|c| c.len()).max().unwrap_or(0);
        let mut flat_q = Vec::with_capacity(nq * dim);
        for q in queries { flat_q.extend_from_slice(q); }
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
            qb_mmr_batch(self.raw, flat_q.as_ptr(), nq as u32, lambdas.as_ptr(), cand.as_ptr(), counts.as_ptr(), max_c as u32, limit as u32,
                         out.as_mut_ptr(), out_counts.as_mut_ptr(), &mut counters)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        hc.cpu_counter().incr_delta(counters.cpu as usize);
        hc.vector_io_read().incr_delta(counters.vector_io_read as usize);
        Ok((0..nq).map(|q| out[q * limit..q * limit + out_counts[q] as usize].iter()
            .map(|p| ScoredPointOffset { idx: p.idx, score: p.score }).collect()).collect())
    }

    /// MMR over multivector candidates: this storage holds dense f32 token rows, point p = rows [point_offsets[p], point_offsets[p + 1]);
    /// `queries[q]` is T_q x `dim` raw f32, row-major (1..4096 vectors), `candidates[q]` are (point offset, score) pairs (at most 16 384), `lambdas[q]` =
    /// 1 - diversity.  Returns each query's selection, in selection order, with the candidates' own scores.
    pub fn mmr_maxsim(&self, point_offsets: &[u32], dim: usize, queries: &[&[f32]], candidates: &[&[ScoredPointOffset]], lambdas: &[f32], limit: usize,
                      hc: &HardwareCounterCell) -> OperationResult<Vec<Vec<ScoredPointOffset>>> {
        let nq = queries.len();
        let n_points = point_offsets.len().saturating_sub(1);
        let max_c = candidates.iter().map(|c| c.len()).max().unwrap_or(0);
        let mut flat_q = Vec::new();
        let mut q_off = vec![0u32];
        for q in queries {
            flat_q.extend_from_slice(q);
            q_off.push((flat_q.len() / dim.max(1)) as u32);
        }
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
            qb_mmr_maxsim_batch(self.raw, point_offsets.as_ptr(), n_points as u32, flat_q.as_ptr(), q_off.as_ptr(), nq as u32, lambdas.as_ptr(),
                                cand.as_ptr(), counts.as_ptr(), max_c as u32, limit as u32, out.as_mut_ptr(), out_counts.as_mut_ptr(), &mut counters)
        };
        if st != QB_OK { return Err(OperationError::service_error(last_error())); }
        hc.cpu_counter().incr_delta(counters.cpu as usize);
        hc.vector_io_read().incr_delta(counters.vector_io_read as usize);
        Ok((0..nq).map(|q| out[q * limit..q * limit + out_counts[q] as usize].iter()
            .map(|p| ScoredPointOffset { idx: p.idx, score: p.score }).collect()).collect())
    }
}
