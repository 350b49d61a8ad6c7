"""CPU pins for the oracle's whole-storage quantized scoring (SQ8 / PQ / BQ score_rows): bit for bit the per-row score it loops over,
with and without an id list, at dims on both sides of the 16-byte SQ8 padding and the 128-bit BQ word, for every BQ encoding x query
encoding and for PQ with a short last chunk."""
import numpy as np
import pytest

IDS = np.array([0, 5, 3, 3, 1], np.uint32)     # out of order, repeated


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def data(oracle, n, dim, seed, cosine=False):
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    if cosine:
        base = oracle.preprocess_rows_f32(oracle.COSINE, base)
    return base, rng.standard_normal((2, dim)).astype(np.float32)


@pytest.mark.parametrize("qd", ["QD_COSINE", "QD_DOT", "QD_L1", "QD_L2"])
@pytest.mark.parametrize("dim", [1, 15, 16, 17, 31, 32, 33, 65, 128])
def test_sq8_score_rows(oracle, qd, dim):
    dt = getattr(oracle, qd)
    base, queries = data(oracle, 40, dim, dim, cosine=qd == "QD_COSINE")
    for invert in (False, True):
        sq = oracle.SQ8.encode(base, dt, invert)
        for q in queries:
            code, off = sq.encode_query(q)
            want = np.array([sq.score(code, off, i) for i in range(base.shape[0])], np.float32)
            np.testing.assert_array_equal(bits(sq.score_rows(code, off)), bits(want))
            np.testing.assert_array_equal(bits(sq.score_all(code, off)), bits(want))
            np.testing.assert_array_equal(bits(sq.score_rows(code, off, IDS)), bits(want[IDS]))
            assert sq.score_rows(code, off, np.zeros(0, np.uint32)).size == 0


def test_sq8_score_rows_nonfinite_metadata(oracle):
    """Rows holding +inf: alpha is inf, every offset is 0 * inf = NaN, every score NaN."""
    base, queries = data(oracle, 30, 20, 3)
    base[4, 2] = np.inf
    sq = oracle.SQ8.encode(base, oracle.QD_DOT, False)
    assert np.isinf(sq.meta.alpha)
    code, off = sq.encode_query(queries[0])
    s = sq.score_rows(code, off)
    assert np.isnan(s).all() and np.isnan(sq.score(code, off, 7))


@pytest.mark.parametrize("qd", ["QD_DOT", "QD_L1", "QD_L2"])
@pytest.mark.parametrize("dim,chunk", [(65, 2), (70, 16), (128, 4), (96, 3), (7, 8)])
def test_pq_score_rows(oracle, qd, dim, chunk):
    """(70, 16): m = 5 with a last chunk of 6; (65, 2): m = 33 with a last chunk of 1; (7, 8): one short chunk."""
    dt = getattr(oracle, qd)
    base, queries = data(oracle, 60, dim, dim + chunk)
    cents = oracle.kmeans_pq_centroids(base, chunk, n_centroids=32, iters=2)
    for invert in (False, True):
        pq = oracle.PQ.encode(base, chunk, cents, dt, invert)
        assert pq.m == -(-dim // chunk)
        for q in queries:
            lut = pq.encode_query(q)
            want = np.array([pq.score(lut, i) for i in range(base.shape[0])], np.float32)
            np.testing.assert_array_equal(bits(pq.score_rows(lut)), bits(want))
            np.testing.assert_array_equal(bits(pq.score_rows(lut, IDS)), bits(want[IDS]))


@pytest.mark.parametrize("enc", ["BQ_ONE", "BQ_TWO", "BQ_ONE_AND_HALF"])
@pytest.mark.parametrize("qenc", ["BQQ_SAME", "BQQ_SCALAR4", "BQQ_SCALAR8"])
@pytest.mark.parametrize("dim", [1, 43, 63, 64, 65, 85, 86, 127, 128, 129, 300])
def test_bq_score_rows(oracle, enc, qenc, dim):
    """43 / 85 / 86: TwoBits and OneAndHalfBits rows end just below / at / above a 128-bit word; 127..129 the plain word edge."""
    e, qe = getattr(oracle, enc), getattr(oracle, qenc)
    base, queries = data(oracle, 50, dim, 7 * dim + e)
    ms = oracle.bq_mean_std(base) if e != oracle.BQ_ONE else None
    for dt, invert in ((oracle.QD_DOT, False), (oracle.QD_L2, True), (oracle.QD_L1, True)):
        bq = oracle.BQ.encode(base, e, qe, dt, invert, ms)
        for q in queries:
            qe_bytes = bq.encode_query(q)
            want = np.array([bq.score(qe_bytes, i) for i in range(base.shape[0])], np.float32)
            np.testing.assert_array_equal(bits(bq.score_rows(qe_bytes)), bits(want))
            np.testing.assert_array_equal(bits(bq.score_rows(qe_bytes, IDS)), bits(want[IDS]))
