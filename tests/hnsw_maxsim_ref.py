"""The MaxSim scorer that drives the CPU traversals (tests/hnsw_acorn_ref.py, tests/hnsw_custom_ref.py) over a graph of multivector points:
every point's score is the oracle's per-row similarities of each query vector (score_rows_f32, or SQ8.score_all on the encoded query)
folded by oracle.maxsim_fold, the arithmetic of qb_score_maxsim.  The callable it returns maps ids -> scores."""
import numpy as np


def point_scores_f32(oracle, distance: int, rows_pre, offsets, query) -> np.ndarray:
    """MaxSim of one query (raw [Q, dim]) against every point of a dense f32 token storage (rows already preprocessed)"""
    qp = [oracle.preprocess_f32(distance, q) for q in np.atleast_2d(np.asarray(query, np.float32))]
    sims = np.stack([oracle.score_rows_f32(distance, rows_pre, q) for q in qp])
    return oracle.maxsim_fold(sims, offsets)


def point_scores_sq8(oracle, sq, distance: int, offsets, query) -> np.ndarray:
    """the same over an SQ8 token storage: each query vector preprocessed, then encoded (EncodedVectorsU8::encode_query)"""
    sims = []
    for q in np.atleast_2d(np.asarray(query, np.float32)):
        code, off = sq.encode_query(oracle.preprocess_f32(distance, q))
        sims.append(sq.score_all(code, off))
    return oracle.maxsim_fold(np.stack(sims), offsets)


def scorer(scores: np.ndarray):
    """ids -> the precomputed scores of those points"""
    return lambda ids: scores[np.asarray(ids, dtype=np.int64)]
