"""GPU parity: multivector MaxSim (score_max_similarity, vector_storage/query_scorer/mod.rs:77-98) through the C ABI vs the
CPU oracle — bit-exact.  A point is a run of consecutive vectors of a token-level storage."""
import numpy as np
import pytest

from tests.util import assert_topk_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def make_points(rng, n_points, max_len):
    lens = rng.integers(1, max_len + 1, n_points)
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)


def test_maxsim_reference_kat_on_gpu(qb, oracle):
    """query_scorer/mod.rs:168-184: Euclid, score(a, a) == -0.0, score(a, b) == -19."""
    a = np.array([[1.0, 2.0, 3.0], [3.0, 3.0, 3.0], [4.0, 5.0, 6.0]], np.float32)
    b = np.array([[3.0, 3.0, 3.0], [4.0, 2.0, 1.0]], np.float32)
    st = qb.DenseVectorStorage(np.concatenate([a, b]), qb.Distance.Euclid)
    mv = qb.MultiVectorView(st, [0, 3, 5])
    got = mv.score_points(a, [0, 1])
    np.testing.assert_array_equal(got, np.array([-0.0, -19.0], np.float32))
    st.close()


@pytest.mark.parametrize("dist", ["Cosine", "Dot", "Euclid", "Manhattan"])
@pytest.mark.parametrize("n_points,max_len,dim,nq", [(300, 7, 64, 5), (2000, 12, 128, 32)])
def test_maxsim_dense_f32(qb, oracle, dist, n_points, max_len, dim, nq):
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(21)
    off = make_points(rng, n_points, max_len)
    rows = oracle.preprocess_rows_f32(int(d), rng.standard_normal((int(off[-1]), dim)).astype(np.float32))
    st = qb.DenseVectorStorage(rows, d)
    mv = qb.MultiVectorView(st, off)
    query = rng.standard_normal((nq, dim)).astype(np.float32)
    qp = np.stack([oracle.preprocess_f32(int(d), q) for q in query])
    want = np.array([oracle.maxsim_f32(int(d), qp, rows[off[p] : off[p + 1]]) for p in range(n_points)], np.float32)
    ids = np.arange(n_points, dtype=np.uint32)
    np.testing.assert_array_equal(mv.score_points(query, ids), want)
    sub = np.array([7, 0, n_points - 1, 7], np.uint32)
    np.testing.assert_array_equal(mv.score_points(query, sub), want[sub])
    for top in (1, 10):
        got = mv.search(query, top)
        order = np.argsort(-want, kind="stable")[:top]
        ref = np.zeros(order.size, dtype=got.dtype)
        ref["idx"], ref["score"] = order, want[order]
        assert_topk_equal(got, ref, want, f"maxsim {dist} top{top}")
    deleted = rng.random(n_points) < 0.3
    got = mv.search(query, 10, point_deleted=deleted)
    live = np.flatnonzero(~deleted)
    order = live[np.argsort(-want[live], kind="stable")[:10]]
    ref = np.zeros(order.size, dtype=got.dtype)
    ref["idx"], ref["score"] = order, want[order]
    assert_topk_equal(got, ref, want, f"maxsim {dist} deleted")
    assert not np.any(deleted[got["idx"]])
    st.close()


@pytest.mark.parametrize("dist", ["Cosine", "Dot", "Euclid", "Manhattan"])
@pytest.mark.parametrize("dt", ["f16", "u8"])
def test_maxsim_dense_f16_u8(qb, oracle, dt, dist):
    """The MaxSim fold over f16 / u8 token similarities: each query vector converted as a plain query is, scored with the storage's metric."""
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(23)
    n_points, dim, nq = 300, 48, 5
    off = make_points(rng, n_points, 7)
    n_rows = int(off[-1])
    if dt == "u8":
        rows = rng.integers(0, 256, (n_rows, dim), dtype=np.uint8)
        st = qb.DenseVectorStorage(rows, d, qb.VectorStorageDatatype.Uint8)
        query = rng.uniform(-20.0, 300.0, (nq, dim)).astype(np.float32)
        sims = np.stack([oracle.score_rows_u8(int(d), rows, oracle.to_u8_query(q)) for q in query])
    else:
        rows = oracle.preprocess_rows_f32(int(d), rng.standard_normal((n_rows, dim)).astype(np.float32)).astype(np.float16)
        st = qb.DenseVectorStorage(rows, d, qb.VectorStorageDatatype.Float16)
        query = rng.standard_normal((nq, dim)).astype(np.float32)
        sims = np.stack([oracle.score_rows_f16(int(d), rows, oracle.to_f16_query(int(d), q)) for q in query])
    want = oracle.maxsim_fold(sims, off)
    mv = qb.MultiVectorView(st, off)
    np.testing.assert_array_equal(mv.score_points(query, np.arange(n_points, dtype=np.uint32)).view(np.uint32), want.view(np.uint32))
    sub = np.array([7, 0, n_points - 1, 7], np.uint32)
    np.testing.assert_array_equal(mv.score_points(query, sub).view(np.uint32), want[sub].view(np.uint32))
    for top in (1, 10):
        got = mv.search(query, top)
        order = np.argsort(-want, kind="stable")[:top]
        ref = np.zeros(order.size, dtype=got.dtype)
        ref["idx"], ref["score"] = order, want[order]
        assert_topk_equal(got, ref, want, f"maxsim {dt} {dist} top{top}")
    deleted = rng.random(n_points) < 0.3
    got = mv.search(query, 10, point_deleted=deleted)
    live = np.flatnonzero(~deleted)
    order = live[np.argsort(-want[live], kind="stable")[:10]]
    ref = np.zeros(order.size, dtype=got.dtype)
    ref["idx"], ref["score"] = order, want[order]
    assert_topk_equal(got, ref, want, f"maxsim {dt} {dist} deleted")
    assert not np.any(deleted[got["idx"]])
    st.close()


def test_maxsim_sq8(qb, oracle):
    """Quantized multivectors: the same fold over SQ8 similarities (quantized_multivector_storage)."""
    d = qb.Distance.Dot
    rng = np.random.default_rng(22)
    n_points, dim, nq = 200, 96, 6
    off = make_points(rng, n_points, 9)
    base = rng.standard_normal((int(off[-1]), dim)).astype(np.float32)
    sq = oracle.SQ8.encode(base, oracle.QD_DOT, False)
    st = qb.ScalarQuantizedVectors(sq.rows, dim, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, d)
    mv = qb.MultiVectorView(st, off)
    query = rng.standard_normal((nq, dim)).astype(np.float32)
    sims = []
    for q in query:
        code, qoff = sq.encode_query(q)
        sims.append(sq.score_all(code, qoff))
    want = oracle.maxsim_fold(np.stack(sims), off)
    np.testing.assert_array_equal(mv.score_points(query, np.arange(n_points, dtype=np.uint32)), want)
    got = mv.search(query, 5)
    order = np.argsort(-want, kind="stable")[:5]
    ref = np.zeros(5, dtype=got.dtype)
    ref["idx"], ref["score"] = order, want[order]
    assert_topk_equal(got, ref, want, "maxsim sq8")
    st.close()


def test_maxsim_rejects_bad_offsets(qb):
    from qdrant_b200._capi import QbError

    st = qb.DenseVectorStorage(np.ones((10, 8), np.float32), qb.Distance.Dot)
    with pytest.raises(QbError):
        qb.MultiVectorView(st, [0, 5, 3]).search(np.ones((1, 8), np.float32), 1)
    with pytest.raises(QbError):
        qb.MultiVectorView(st, [0, 5, 11]).search(np.ones((1, 8), np.float32), 1)
    with pytest.raises(QbError):
        qb.MultiVectorView(st, [0, 5, 10]).score_points(np.ones((1, 8), np.float32), [2])
    st.close()


@pytest.mark.parametrize("dist", ["Cosine", "Euclid"])
def test_custom_queries_over_multivectors(qb, oracle, dist):
    """MultiCustomQueryScorer (multi_custom_query_scorer.rs:88-104): the examples of a recommend / discover / context / feedback query are
    multivectors; similarity(example, point) = MaxSim; Query::score_by folds them."""
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(33)
    n_points, dim = 400, 48
    off = make_points(rng, n_points, 6)
    rows = oracle.preprocess_rows_f32(int(d), rng.standard_normal((int(off[-1]), dim)).astype(np.float32))
    st = qb.DenseVectorStorage(rows, d)
    mv = qb.MultiVectorView(st, off)
    mvec = lambda: rng.standard_normal((int(rng.integers(1, 5)), dim)).astype(np.float32)  # noqa: E731
    pos, neg, part = oracle.feedback_pairs(np.array([0.9, 0.2, 0.5], np.float32), 1.2, 0.7)
    items = [mvec() for _ in range(3)]
    queries = [
        qb.RecoBestScoreQuery(qb.RecoQuery([mvec(), mvec()], [mvec()])),
        qb.RecoSumScoresQuery(qb.RecoQuery([mvec()], [mvec(), mvec()])),
        qb.DiscoverQuery(mvec(), [qb.ContextPair(mvec(), mvec()), qb.ContextPair(mvec(), mvec())]),
        qb.ContextQuery([qb.ContextPair(mvec(), mvec())]),
        qb.FeedbackQuery(mvec(), [qb.ContextPair(items[i], items[j]) for i, j in zip(pos, neg)], part, 0.8),
    ]
    # the query classes hold 1-D vectors by default: store the matrices as given
    for q in queries:
        ex, n_a, n_b = q.flat()
        sims = np.stack([np.array([oracle.maxsim_f32(int(d), np.stack([oracle.preprocess_f32(int(d), t) for t in np.atleast_2d(e)]), rows[off[p] : off[p + 1]])
                                   for p in range(n_points)], np.float32) for e in ex])
        want = oracle.feedback_score(q.a, q.partial, sims) if int(q.kind) == 5 else oracle.custom_combine(int(q.kind), n_a, n_b, sims)
        ids = np.arange(n_points, dtype=np.uint32)
        np.testing.assert_array_equal(mv.score_points_custom(q, ids), want)
        got = mv.search_custom(q, 10)
        order = np.argsort(-want, kind="stable")[:10]
        ref = np.zeros(order.size, dtype=got.dtype)
        ref["idx"], ref["score"] = order, want[order]
        assert_topk_equal(got, ref, want, f"multi custom {dist} kind {int(q.kind)}")
    st.close()
