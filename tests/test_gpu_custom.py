"""GPU parity: custom-query scorers (recommend / discover / context) through the C ABI vs the CPU oracle — bit-exact.

The reference evaluates `Query::score_by(|example| similarity(example, stored))` per candidate
(vector_storage/query_scorer/custom_query_scorer.rs:78-122; quantized: quantized_custom_query_scorer.rs).  The oracle side
computes the per-example similarities with the SAME restatements the plain-query tests use, folds them with
oracle.custom_combine (pinned against the reference's rstest tables in tests/test_oracle_kat.py) and compares.
"""
import numpy as np
import pytest

from tests.util import assert_topk_equal, pack_bitmap

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def make_queries(qb, rng, dim, scale=1.0, shift=0.0):
    """scale / shift: example vectors on the scale of the stored values (u8 storages convert them with `x as u8`)"""
    v = lambda: (rng.standard_normal(dim) * scale + shift).astype(np.float32)  # noqa: E731
    return [
        qb.RecoBestScoreQuery(qb.RecoQuery([v(), v(), v()], [v(), v()])),
        qb.RecoBestScoreQuery(qb.RecoQuery([v()], [])),
        qb.RecoBestScoreQuery(qb.RecoQuery([], [v(), v()])),
        qb.RecoSumScoresQuery(qb.RecoQuery([v(), v()], [v(), v(), v()])),
        qb.DiscoverQuery(v(), [qb.ContextPair(v(), v()), qb.ContextPair(v(), v()), qb.ContextPair(v(), v())]),
        qb.DiscoverQuery(v(), []),
        qb.ContextQuery([qb.ContextPair(v(), v()), qb.ContextPair(v(), v())]),
        qb.RecoSumScoresQuery(qb.RecoQuery([v() for _ in range(12)], [v() for _ in range(9)])),   # 21 examples: beyond the fused-fold scan's 16
        feedback_query(qb, rng, dim, 4, v),
        feedback_query(qb, rng, dim, 1, v),  # fewer than two feedback items: no pairs, score = a * sim(target)
    ]


def feedback_query(qb, rng, dim, n_items, v):
    """NaiveFeedbackQuery -> FeedbackQuery the way the reference builds it (feedback_query.rs:121-172): every ordered pair of feedback
    items whose score difference is positive becomes a context pair with partial_computation = confidence^b * c."""
    from oracle import oracle as o

    items = [v() for _ in range(n_items)]
    scores = rng.random(n_items).astype(np.float32)
    a, b, c = 0.9, 1.5, 0.4
    pos, neg, part = o.feedback_pairs(scores, b, c)
    return qb.FeedbackQuery(v(), [qb.ContextPair(items[i], items[j]) for i, j in zip(pos, neg)], part, a)


def oracle_scores(oracle, query, sim_rows):
    """sim_rows(example_vector) -> similarities of every candidate to that example (np.float32 array)."""
    vecs, n_a, n_b = query.flat()
    sims = np.stack([sim_rows(v) for v in vecs])
    if int(query.kind) == 5:   # FeedbackQuery::score_by (feedback_query.rs:204-226)
        return oracle.feedback_score(query.a, query.partial, sims)
    return oracle.custom_combine(int(query.kind), n_a, n_b, sims)


def check_storage(qb, oracle, st, queries, sim_rows, n, what):
    ids = np.arange(n, dtype=np.uint32)
    rng = np.random.default_rng(5)
    deleted = rng.random(n) < 0.2
    some = np.sort(rng.choice(n, n // 3, replace=False)).astype(np.uint32)
    for qi, query in enumerate(queries):
        want = oracle_scores(oracle, query, sim_rows)
        sc = st.raw_scorer_custom(query)
        np.testing.assert_array_equal(sc.score_points(ids), want, err_msg=f"{what} q{qi} score_points")
        assert sc.score_point(3) == want[3]
        sub = np.array([5, 1, 77 % n, 5], np.uint32)
        np.testing.assert_array_equal(sc.score_points(sub), want[sub])
        from qdrant_b200._capi import QB_ERR_UNSUPPORTED, QbError

        with pytest.raises(QbError) as ei:  # custom_query_scorer.rs:111-113: unimplemented!()
            sc.score_internal(0, 1)
        assert ei.value.status == QB_ERR_UNSUPPORTED
        sc.close()
        # fused scan: all rows / soft-deleted rows / explicit id list
        for top in (1, 10):
            got = st.search_custom(query, top)
            order = np.argsort(-want, kind="stable")[:top]
            ref = np.zeros(order.size, dtype=got.dtype)
            ref["idx"], ref["score"] = order, want[order]
            assert_topk_equal(got, ref, want, f"{what} q{qi} top{top}")
        got = st.search_custom(query, 10, point_deleted=deleted)
        live = np.flatnonzero(~deleted)
        order = live[np.argsort(-want[live], kind="stable")[:10]]
        ref = np.zeros(order.size, dtype=got.dtype)
        ref["idx"], ref["score"] = order, want[order]
        assert_topk_equal(got, ref, want, f"{what} q{qi} deleted")
        assert not np.any(deleted[got["idx"]])
        got = st.search_custom(query, 7, id_list=some)
        order = some[np.argsort(-want[some], kind="stable")[:7]]
        ref = np.zeros(order.size, dtype=got.dtype)
        ref["idx"], ref["score"] = order, want[order]
        assert_topk_equal(got, ref, want, f"{what} q{qi} id_list")
        assert set(got["idx"].tolist()) <= set(some.tolist())


@pytest.mark.parametrize("dist", ["Cosine", "Dot", "Euclid", "Manhattan"])
@pytest.mark.parametrize("n,dim", [(300, 70), (2000, 768)])
def test_custom_dense_f32(qb, oracle, dist, n, dim):
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(11)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    stored = oracle.preprocess_rows_f32(int(d), base)  # Distance::preprocess_vector at insert time
    st = qb.DenseVectorStorage(stored, d)
    sim = lambda v: oracle.score_rows_f32(int(d), stored, oracle.preprocess_f32(int(d), v))  # noqa: E731
    check_storage(qb, oracle, st, make_queries(qb, rng, dim), sim, n, f"dense {dist}")
    st.close()


@pytest.mark.parametrize("dist", ["Cosine", "Dot", "Euclid", "Manhattan"])
@pytest.mark.parametrize("dt", ["f16", "u8"])
def test_custom_dense_f16_u8(qb, oracle, dt, dist):
    """Every example is converted the way a plain query is (f16: preprocess, then f16::from_f32; u8: `x as u8`), then scored with the
    storage's own metric."""
    d = getattr(qb.Distance, dist)
    n, dim = 300, 70
    rng = np.random.default_rng(15)
    if dt == "u8":
        stored = rng.integers(0, 256, (n, dim), dtype=np.uint8)
        st = qb.DenseVectorStorage(stored, d, qb.VectorStorageDatatype.Uint8)
        sim = lambda v: oracle.score_rows_u8(int(d), stored, oracle.to_u8_query(v))  # noqa: E731
        queries = make_queries(qb, rng, dim, scale=90.0, shift=120.0)              # some examples saturate or truncate to 0
    else:
        stored = oracle.preprocess_rows_f32(int(d), rng.standard_normal((n, dim)).astype(np.float32)).astype(np.float16)
        st = qb.DenseVectorStorage(stored, d, qb.VectorStorageDatatype.Float16)
        sim = lambda v: oracle.score_rows_f16(int(d), stored, oracle.to_f16_query(int(d), v))  # noqa: E731
        queries = make_queries(qb, rng, dim)
    check_storage(qb, oracle, st, queries, sim, n, f"dense {dt} {dist}")
    st.close()


@pytest.mark.parametrize("dist", ["Cosine", "Euclid"])
def test_custom_sq8(qb, oracle, dist):
    d = getattr(qb.Distance, dist)
    dt, inv = (int(x) for x in qb.construct_vector_parameters(d))
    n, dim = 400, 200
    rng = np.random.default_rng(12)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    if d == qb.Distance.Cosine:
        base = oracle.preprocess_rows_f32(oracle.COSINE, base)
    sq = oracle.SQ8.encode(base, dt, bool(inv))
    st = qb.ScalarQuantizedVectors(sq.rows, dim, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, d)

    def sim(v):
        code, off = sq.encode_query(oracle.preprocess_f32(int(d), v))
        return np.array([sq.score(code, off, i) for i in range(n)], np.float32)

    check_storage(qb, oracle, st, make_queries(qb, rng, dim), sim, n, f"sq8 {dist}")
    st.close()


def test_custom_pq(qb, oracle):
    d = qb.Distance.Dot
    n, dim, chunk = 300, 64, 8
    rng = np.random.default_rng(13)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    cents = oracle.kmeans_pq_centroids(base, chunk, n_centroids=256, iters=2)
    pq = oracle.PQ.encode(base, chunk, cents, oracle.QD_DOT, False)
    st = qb.ProductQuantizedVectors(pq.codes, cents, chunk, dim, d)

    def sim(v):
        lut = pq.encode_query(oracle.preprocess_f32(int(d), v))
        return np.array([pq.score(lut, i) for i in range(n)], np.float32)

    check_storage(qb, oracle, st, make_queries(qb, rng, dim), sim, n, "pq")
    st.close()


@pytest.mark.parametrize("qenc", ["SameAsStorage", "Scalar8bits"])
def test_custom_bq(qb, oracle, qenc):
    d = qb.Distance.Dot
    n, dim = 300, 256
    rng = np.random.default_rng(14)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    qe = int(getattr(qb.BQQueryEncoding, qenc))
    bq = oracle.BQ.encode(base, oracle.BQ_ONE, qe, oracle.QD_DOT, False, None)
    st = qb.BinaryQuantizedVectors(bq.rows, dim, d, qb.BQEncoding.OneBit, qb.BQQueryEncoding(qe), None)

    def sim(v):
        enc = bq.encode_query(oracle.preprocess_f32(int(d), v))
        return np.array([bq.score(enc, i) for i in range(n)], np.float32)

    check_storage(qb, oracle, st, make_queries(qb, rng, dim), sim, n, f"bq {qenc}")
    st.close()


def test_custom_rejects_bad_arguments(qb):
    from qdrant_b200._capi import QbError

    st = qb.DenseVectorStorage(np.ones((10, 8), np.float32), qb.Distance.Dot)
    with pytest.raises(ValueError):
        st.raw_scorer_custom(qb.RecoBestScoreQuery(qb.RecoQuery([], [])))
    with pytest.raises(ValueError):
        st.raw_scorer_custom(qb.ContextQuery([qb.ContextPair(np.ones(7), np.ones(7))]))
    with pytest.raises((QbError, ValueError)):
        st.search_custom(qb.ContextQuery([]), 5)
    st.close()
