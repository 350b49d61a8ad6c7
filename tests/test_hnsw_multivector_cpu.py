"""The checker of the device MaxSim traversal, pinned on the CPU: the MaxSim callback (tests/hnsw_maxsim_ref.py) equals the oracle's
score_max_similarity point by point, and the traversals that take it (oracle HNSW.search, the ACORN checker's HNSW mode, the keyed
custom-query checker) give the same lists, hops and scored points on the same graph of multivector points."""
import numpy as np
import pytest

from tests import hnsw_acorn_ref as ar
from tests import hnsw_custom_ref as cr
from tests import hnsw_maxsim_ref as mr


def _offsets(rng, n_points, lens=(0, 1, 2, 3, 7)):
    return np.concatenate([[0], np.cumsum(rng.choice(lens, n_points))]).astype(np.uint32)


def test_callback_reference_kat(oracle):
    """query_scorer/mod.rs:168-184: Euclid, score(a, a) == -0.0, score(a, b) == -19 (compared as values: the fold sums from +0.0, as
    qb_score_maxsim does, so every maximum being -0.0 gives +0.0)"""
    a = np.array([[1.0, 2.0, 3.0], [3.0, 3.0, 3.0], [4.0, 5.0, 6.0]], np.float32)
    b = np.array([[3.0, 3.0, 3.0], [4.0, 2.0, 1.0]], np.float32)
    got = mr.point_scores_f32(oracle, oracle.EUCLID, np.concatenate([a, b]), np.array([0, 3, 5], np.uint32), a)
    np.testing.assert_array_equal(got, np.array([-0.0, -19.0], np.float32))


@pytest.mark.parametrize("dist", [0, 1, 2, 3])
def test_callback_equals_maxsim_f32(oracle, dist):
    """empty runs stay -inf, NaN tokens never win, -0.0 / +0.0 keep the earlier token's bits"""
    rng = np.random.default_rng(40 + dist)
    n_points, dim = 300, 12
    off = _offsets(rng, n_points)
    raw = rng.standard_normal((int(off[-1]), dim)).astype(np.float32)
    raw[rng.random(raw.shape[0]) < 0.05] = np.nan
    rows = oracle.preprocess_rows_f32(dist, raw)
    rows[rng.random(rows.shape[0]) < 0.05] = 0.0       # exact zero similarities (Dot / Cosine) against any query
    for nq in (1, 5):
        query = rng.standard_normal((nq, dim)).astype(np.float32)
        qp = np.stack([oracle.preprocess_f32(dist, q) for q in query])
        got = mr.point_scores_f32(oracle, dist, rows, off, query)
        want = np.array([oracle.maxsim_f32(dist, qp, rows[off[p] : off[p + 1]].reshape(-1, dim)) for p in range(n_points)], np.float32)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        assert np.all(np.isneginf(got[np.diff(off) == 0]))


def _graph(oracle, rng, n_points, dim, dist, m=8):
    """a graph over the points' normalised mean tokens, as the probe builds one (no MaxSim graph builder exists)"""
    off = np.concatenate([[0], np.cumsum(rng.integers(1, 9, n_points))]).astype(np.uint32)
    rows = oracle.preprocess_rows_f32(dist, rng.standard_normal((int(off[-1]), dim)).astype(np.float32))
    means = np.stack([rows[off[p] : off[p + 1]].mean(0) for p in range(n_points)]).astype(np.float32)
    g = oracle.HNSW(oracle.preprocess_rows_f32(oracle.COSINE, means), oracle.COSINE, m=m, ef_construct=48, seed=7, threads=1)
    return g, off, rows


@pytest.mark.parametrize("dist", [0, 1])
def test_traversals_agree_with_the_maxsim_callback(oracle, dist):
    rng = np.random.default_rng(50 + dist)
    n_points, dim = 1200, 16
    g, off, rows = _graph(oracle, rng, n_points, dim, dist)
    entry, lvl, m, m0 = g.entry()
    blob = g.export_plain()
    ag = ar.Graph(blob, m, m0, n_points)
    cg = cr.Graph(blob, m, m0, n_points)
    dummy = np.zeros(dim, np.float32)
    for i in range(6):
        query = rng.standard_normal((int(rng.integers(1, 6)), dim)).astype(np.float32)
        cb = mr.scorer(mr.point_scores_f32(oracle, dist, rows, off, query))
        for top, ef in ((10, 32), (5, 1)):
            g.stats(reset=True)
            want = g.search(dummy, top, ef, score_points=cb)
            want_stats = g.stats(reset=True)
            a = ag.search(cb, top, ef, entry, lvl, ar.HNSW)
            c = cr.search_cb(cg, cb, top, ef, entry, lvl, cr.HNSW, keyed=True)
            assert ag.stats()[:2] == want_stats and cg.stats()[:2] == want_stats
            assert np.array_equal(a, want) and np.array_equal(c, want), (i, top, ef)


def test_acorn_checker_filters_points(oracle):
    """ACORN-1 through the MaxSim callback: no filtered-out point is returned or scored, and the keyed checker agrees"""
    rng = np.random.default_rng(60)
    n_points, dim = 1500, 16
    g, off, rows = _graph(oracle, rng, n_points, dim, oracle.DOT)
    entry, lvl, m, m0 = g.entry()
    blob = g.export_plain()
    ag = ar.Graph(blob, m, m0, n_points)
    cg = cr.Graph(blob, m, m0, n_points)
    filtered = rng.random(n_points) >= 0.1
    filtered[entry] = False
    query = rng.standard_normal((4, dim)).astype(np.float32)
    scores = mr.point_scores_f32(oracle, oracle.DOT, rows, off, query)
    seen = []
    cb = lambda ids: (seen.extend(ids.tolist()), scores[ids.astype(np.int64)])[1]   # noqa: E731
    a = ag.search(cb, 10, 64, entry, lvl, ar.ACORN, filtered)
    c = cr.search_cb(cg, mr.scorer(scores), 10, 64, entry, lvl, cr.ACORN, filtered, keyed=True)
    assert np.array_equal(a, c)
    assert not filtered[a["idx"]].any() and not filtered[np.array(seen, np.int64)].any()
