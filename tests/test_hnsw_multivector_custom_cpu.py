"""The checker of the device custom queries with multivector examples (tests/hnsw_maxsim_custom_ref.py), pinned on the CPU: its per-point
scores equal the oracle's Query::score_by over the oracle's score_max_similarity per example, its traversal with one positive example is the
nearest MaxSim traversal, and its discover is the context search followed by the discover search from the context list."""
import numpy as np
import pytest

from tests import hnsw_custom_ref as cr
from tests import hnsw_maxsim_custom_ref as mc
from tests import hnsw_maxsim_ref as mr

# (kind, n_a, n_b): recommend best-score and sum-scores, discover, context, feedback
SHAPES = [(1, 2, 1), (2, 1, 2), (3, 2, 0), (4, 2, 0), (5, 2, 0)]


def _examples(rng, n, dim, lens=(1, 5)):
    return [rng.standard_normal((int(rng.integers(lens[0], lens[1] + 1)), dim)).astype(np.float32) for _ in range(n)]


@pytest.mark.parametrize("kind,n_a,n_b", SHAPES)
@pytest.mark.parametrize("dist", [0, 1, 2, 3])
def test_scores_equal_the_oracle_fold(oracle, kind, n_a, n_b, dist):
    """empty token runs, NaN tokens and exact zeros: each example's MaxSim by score_max_similarity, folded by score_by"""
    rng = np.random.default_rng(70 + 10 * kind + dist)
    n_points, dim = 200, 12
    off = np.concatenate([[0], np.cumsum(rng.choice([0, 1, 2, 5], n_points))]).astype(np.uint32)
    raw = rng.standard_normal((int(off[-1]), dim)).astype(np.float32)
    raw[rng.random(raw.shape[0]) < 0.05] = np.nan
    rows = oracle.preprocess_rows_f32(dist, raw)
    rows[rng.random(rows.shape[0]) < 0.05] = 0.0     # exact zero similarities (Dot / Cosine), so context plateaus and +-0 maxima occur
    examples = _examples(rng, cr.n_examples(kind, n_a, n_b), dim)
    coef = np.concatenate([[0.7], rng.standard_normal(n_a)]).astype(np.float32) if kind == cr.FEEDBACK else None
    got = mc.point_scores(oracle, mc.per_example_f32(oracle, dist, rows, off), kind, n_a, n_b, examples, coef)
    sims = np.array([[oracle.maxsim_f32(dist, np.stack([oracle.preprocess_f32(dist, v) for v in e]), rows[off[p] : off[p + 1]].reshape(-1, dim))
                      for p in range(n_points)] for e in examples], np.float32)
    want = oracle.feedback_score(float(coef[0]), coef[1:], sims) if kind == cr.FEEDBACK else oracle.custom_combine(kind, n_a, n_b, sims)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert (np.diff(off) == 0).any() and np.isnan(raw).any()
    ids = rng.permutation(n_points)[:37]
    lazy = mc.lazy_scores_f32(oracle, dist, rows, off, kind, n_a, n_b, examples, coef)(ids)
    assert np.array_equal(lazy.view(np.uint32), want[ids].view(np.uint32))


def _graph(oracle, rng, n_points, dim, dist, m=8):
    off = np.concatenate([[0], np.cumsum(rng.integers(1, 9, n_points))]).astype(np.uint32)
    rows = oracle.preprocess_rows_f32(dist, rng.standard_normal((int(off[-1]), dim)).astype(np.float32))
    means = np.stack([rows[off[p] : off[p + 1]].mean(0) for p in range(n_points)]).astype(np.float32)
    g = oracle.HNSW(oracle.preprocess_rows_f32(oracle.COSINE, means), oracle.COSINE, m=m, ef_construct=48, seed=7, threads=1)
    entry, lvl, m, m0 = g.entry()
    return cr.Graph(g.export_plain(), m, m0, n_points), off, rows, entry, lvl


@pytest.mark.parametrize("algo", [cr.HNSW, cr.ACORN])
def test_one_positive_is_the_nearest_maxsim_traversal(oracle, algo):
    """RecommendSumScores with one positive scores 0.0 + MaxSim, the MaxSim itself on tie-free data: the same lists, hops and scored points"""
    rng = np.random.default_rng(81 + algo)
    dist = oracle.DOT
    g, off, rows, entry, lvl = _graph(oracle, rng, 1200, 16, dist)
    filtered = (rng.random(1200) >= 0.3) if algo == cr.ACORN else None
    if filtered is not None:
        filtered[entry] = False
    pe = mc.per_example_f32(oracle, dist, rows, off)
    for i in range(4):
        ex = _examples(rng, 1, 16)
        for top, ef in ((10, 32), (5, 1)):
            got, sc = mc.search(g, oracle, pe, 2, 1, 0, ex, top, ef, entry, lvl, algo, filtered)
            got_stats = g.stats()[:2]
            want = cr.search_cb(g, mr.scorer(mr.point_scores_f32(oracle, dist, rows, off, ex[0])), top, ef, entry, lvl, algo, filtered, keyed=True)
            assert g.stats()[:2] == got_stats
            assert np.array_equal(got["idx"], want["idx"]) and np.array_equal(got["score"].view(np.uint32), want["score"].view(np.uint32)), (i, top, ef)
            assert sc.points().size > 0


def test_discover_is_context_then_discover(oracle):
    rng = np.random.default_rng(90)
    dist = oracle.COSINE
    g, off, rows, entry, lvl = _graph(oracle, rng, 1000, 16, dist)
    pe = mc.per_example_f32(oracle, dist, rows, off)
    n_pairs = 2
    for _ in range(3):
        ex = _examples(rng, 1 + 2 * n_pairs, 16)
        got, (s1, s2) = mc.discover(g, oracle, pe, ex, n_pairs, 10, 32, entry, lvl)
        ctx = mc.point_scores(oracle, pe, mc.CONTEXT, n_pairs, 0, ex[1:])
        stage1 = cr.search_cb(g, mr.scorer(ctx), cr.DISCOVERY_ENTRY_POINT_COUNT, 32, entry, lvl, keyed=True)
        disc = mc.point_scores(oracle, pe, mc.DISCOVER, n_pairs, 0, ex)
        want = cr.search_cb(g, mr.scorer(disc), 10, 32, entry, lvl, cep=stage1["idx"], keyed=True)
        assert np.array_equal(got, want)
        assert s1.points().size > 0 and s2.points().size > 0
        # the discover stage starts from the stage-1 list: its first scored point is the entry get_entry_point picks from it
        e, _, taken = cr.get_entry_point(g, stage1["idx"], entry, lvl)
        assert taken and s2.seen[0][0] == e
