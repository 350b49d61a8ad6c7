"""The checker of qb_hnsw_search_maxsim_custom_batch / qb_hnsw_search_maxsim_discover_batch: custom queries whose examples are
multivectors, over a graph of multivector points.  A point's score is each example's MaxSim (tests/hnsw_maxsim_ref.py, the arithmetic of
qb_score_maxsim) folded by the oracle's Query::score_by (oracle.custom_combine; feedback: oracle.feedback_score), and the traversal is the
keyed CPU checker of tests/hnsw_custom_ref.py driven by those scores.  Discover is its two stages, restated as hnsw_custom_ref.discover
restates them (discover_search_with_graph, hnsw/read_view/search.rs:314-349)."""
import numpy as np

from tests import hnsw_custom_ref as cr
from tests import hnsw_maxsim_ref as mr

DISCOVER, CONTEXT = 3, 4


def per_example_f32(oracle, distance: int, rows_pre, offsets):
    """example (raw [V, dim]) -> its MaxSim against every point of a dense f32 token storage"""
    return lambda example: mr.point_scores_f32(oracle, distance, rows_pre, offsets, example)


def per_example_sq8(oracle, sq, distance: int, offsets):
    """the same over an SQ8 token storage"""
    return lambda example: mr.point_scores_sq8(oracle, sq, distance, offsets, example)


def point_scores(oracle, per_example, kind: int, n_a: int, n_b: int, examples, coef=None) -> np.ndarray:
    """the custom score of every point: examples in the qb_scorer_create_custom order; coef = [a, partial...] for feedback"""
    sims = np.stack([per_example(e) for e in examples])
    if kind == cr.FEEDBACK:
        c = np.asarray(coef, np.float32)
        return oracle.feedback_score(float(c[0]), c[1:], sims)
    return oracle.custom_combine(kind, n_a, n_b, sims)


def lazy_scores_f32(oracle, distance: int, rows_pre, offsets, kind: int, n_a: int, n_b: int, examples, coef=None):
    """ids -> point_scores of those points only, from their own token rows (a point's MaxSim reads nothing else): for collections too
    large to score every point per query"""
    qs = [np.stack([oracle.preprocess_f32(distance, v) for v in np.atleast_2d(np.asarray(e, np.float32))]) for e in examples]
    off = np.asarray(offsets, np.int64)

    def scores(ids):
        ids = np.asarray(ids, np.int64)
        runs = off[ids + 1] - off[ids]
        sub = np.concatenate([[0], np.cumsum(runs)]).astype(np.uint32)
        sel = np.concatenate([np.arange(off[i], off[i + 1]) for i in ids]) if runs.sum() else np.zeros(0, np.int64)
        rows = np.ascontiguousarray(rows_pre[sel]).reshape(-1, rows_pre.shape[1])
        sims = np.stack([oracle.maxsim_fold(np.stack([oracle.score_rows_f32(distance, rows, v) for v in q]), sub) for q in qs])
        if kind == cr.FEEDBACK:
            c = np.asarray(coef, np.float32)
            return oracle.feedback_score(float(c[0]), c[1:], sims)
        return oracle.custom_combine(kind, n_a, n_b, sims)

    return scores


class Scorer:
    """ids -> precomputed scores, recording the points each scorer call asked for (the counters' token rows)"""

    def __init__(self, scores):
        self.scores = scores
        self.seen = []

    def __call__(self, ids):
        self.seen.append(np.asarray(ids).copy())
        return self.scores[np.asarray(ids, dtype=np.int64)]

    def points(self) -> np.ndarray:
        return np.concatenate(self.seen).astype(np.int64) if self.seen else np.zeros(0, np.int64)


def search(graph: cr.Graph, oracle, per_example, kind: int, n_a: int, n_b: int, examples, top: int, ef: int, entry: int, entry_level: int,
           algo: int = cr.HNSW, filtered=None, coef=None, cep=None):
    """one custom search: (its list, the Scorer it ran with)"""
    sc = Scorer(point_scores(oracle, per_example, kind, n_a, n_b, examples, coef))
    return cr.search_cb(graph, sc, top, ef, entry, entry_level, algo, filtered, cep=cep, keyed=True), sc


def discover(graph: cr.Graph, oracle, per_example, examples, n_pairs: int, top: int, ef: int, entry: int, entry_level: int, algo: int = cr.HNSW,
             filtered=None):
    """a context search over the pairs (examples 1 .. 2 n_pairs) for the 10 best points, then the discover search from them as custom
    entry points: (the list, [stage-1 Scorer, stage-2 Scorer])"""
    stage1, s1 = search(graph, oracle, per_example, CONTEXT, n_pairs, 0, examples[1:], cr.DISCOVERY_ENTRY_POINT_COUNT, ef, entry, entry_level, algo,
                        filtered)
    got, s2 = search(graph, oracle, per_example, DISCOVER, n_pairs, 0, examples, top, ef, entry, entry_level, algo, filtered, cep=stage1["idx"].copy())
    return got, [s1, s2]
