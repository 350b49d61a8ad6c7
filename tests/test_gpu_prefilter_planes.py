"""Single-query prefilter (qb_prefilter.cu) on each integer shadow plane: option prefilter_plane 0 (the 6-bit plane, the default) and 2 (the
int8 plane).  Results must equal the exact f32 scan bit for bit; overflowing lists and undecidable queries fall back on the device."""
import numpy as np
import pytest

from tests.util import assert_topk_equal, pack_bitmap

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def search_both_ways(qb, st, queries, top, plane, deleted=None):
    """(prefilter results on `plane`, (searches, fallback reruns), exact-scan results)"""
    qb.set_option("prefilter_plane", plane)
    st.search_stats(reset=True)
    try:
        got = [st.search_batch(q, top, point_deleted=deleted)[0] for q in queries]
    finally:
        qb.set_option("prefilter_plane", 0)
    stats = st.search_stats(reset=True)
    qb.set_option("disable_prefilter", 1)
    try:
        exact = [st.search_batch(q, top, point_deleted=deleted)[0] for q in queries]
    finally:
        qb.set_option("disable_prefilter", 0)
    for i, (a, b) in enumerate(zip(got, exact)):
        np.testing.assert_array_equal(a["idx"], b["idx"], err_msg=f"query {i}")
        np.testing.assert_array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32), err_msg=f"query {i}")
    return got, stats


@pytest.mark.parametrize("dist,n,dim,top", [("Dot", 560_001, 200, 16), ("Cosine", 540_000, 1000, 10), ("Cosine", 524_289, 40, 5)])
@pytest.mark.parametrize("plane", [0, 2])
def test_integer_plane_prefilter_is_exact(qb, oracle, dist, n, dim, top, plane):
    """Odd row counts (a padded last tile on the 6-bit plane), dims that are not a multiple of 32 (zero-padded codes), deletions, zero and
    denormal rows: bit-identical to the exact scan, no fallback, and equal to the oracle."""
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(dim * 7 + plane)
    base = rng.standard_normal((n, dim), dtype=np.float32) * (1.0 if dist == "Cosine" else rng.uniform(0.2, 3.0, (n, 1)).astype(np.float32))
    if d == qb.Distance.Cosine:
        base = oracle.preprocess_rows_f32(oracle.COSINE, base)
    else:
        base[1000:1010] = 0.0
        base[2000:2010] *= np.float32(1e-38)
    queries = rng.standard_normal((4, dim)).astype(np.float32)
    queries[1] = base[n - 1] * 2.0                    # best match in the very last row (the odd one)
    deleted = rng.random(n) < 0.02
    deleted[n - 1] = False
    st = qb.DenseVectorStorage(base, d)
    got, (searches, reruns) = search_both_ways(qb, st, queries, top, plane, deleted)
    assert (searches, reruns) == (4, 0)
    qp = np.stack([oracle.preprocess_f32(int(d), q) for q in queries[:2]])
    want = oracle.scan_f32(int(d), base, qp, top, deleted=pack_bitmap(deleted))
    for i in range(2):
        assert_topk_equal(got[i], want[i], None, f"plane {plane} {dist} dim={dim} q={i}")
    st.close()


@pytest.mark.parametrize("plane", [0, 2])
def test_long_candidate_lists_are_rescored_without_fallback(qb, plane):
    """20 001 tied best rows on 2^20 rows: more than the lists of earlier builds held (16 384), fewer than n / 32.  Every CTA of the
    finish keeps its own top-k; the merge breaks the ties by ascending id, as the exact scan does."""
    rng = np.random.default_rng(11)
    n, dim = 1 << 20, 96
    base = rng.standard_normal((n, dim), dtype=np.float32)
    base[300_000:320_000] = base[299_999]
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    got, (searches, reruns) = search_both_ways(qb, st, [base[299_999] * 4.0, rng.standard_normal(dim).astype(np.float32)], 10, plane)
    assert (searches, reruns) == (2, 0)
    assert list(got[0]["idx"]) == list(range(299_999, 300_009))
    st.close()


def test_int8_plane_falls_back_on_the_device(qb):
    """The int8 plane keeps the device fallback: mass ties beyond n / 32 candidates, a NaN query, a sample without `top` live rows."""
    rng = np.random.default_rng(9)
    n, dim = 600_000, 96
    base = rng.standard_normal((n, dim), dtype=np.float32)
    base[100_000:120_000] = base[99_999]
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    q_nan = rng.standard_normal(dim).astype(np.float32); q_nan[5] = np.nan
    q_plain = rng.standard_normal(dim).astype(np.float32)
    del_prefix = np.zeros(n, bool); del_prefix[:200_000] = True; del_prefix[:4] = False
    for q, dl, expect in [(base[99_999] * 4.0, None, 1), (q_nan, None, 1), (q_plain, del_prefix, 1), (q_plain, None, 0)]:
        _, (s, r) = search_both_ways(qb, st, [q], 10, 2, dl)
        assert (s, r) == (1, expect)
    st.close()
