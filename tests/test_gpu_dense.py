"""GPU parity: f32 dense metrics through the C ABI vs the CPU oracle (bit-exact: assert_array_equal).

Mirrors the reference's two-backends-must-agree pattern (lib/segment/src/vector_storage/tests/async_raw_scorer.rs:41-114)
and its GPU-vs-CPU harness (index/hnsw_index/gpu/gpu_vector_storage/tests.rs:965-1060), with tolerance 0 instead of
get_precision (:790-802): the kernels reproduce the AVX2+FMA accumulation order.
"""
import ctypes as C

import numpy as np
import pytest

from tests.util import assert_topk_equal, pack_bitmap

pytestmark = pytest.mark.gpu

DISTS = ["Cosine", "Euclid", "Dot", "Manhattan"]


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def make_data(oracle, dist, n, dim, seed=42, nq=3):
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    if dist == oracle.COSINE:
        base = oracle.preprocess_rows_f32(oracle.COSINE, base)  # Distance::preprocess_vector at insert time
    return base, queries


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("dim", [1, 8, 15, 16, 31, 32, 33, 70, 128, 200, 768, 1000])
def test_score_points_bit_exact(qb, oracle, dist, dim):
    d = getattr(qb.Distance, dist)
    base, queries = make_data(oracle, int(d), 300, dim)
    st = qb.DenseVectorStorage(base, d)
    rng = np.random.default_rng(1)
    for q in queries:
        sc = st.build_raw_scorer(q)
        ids = rng.integers(0, base.shape[0], 77).astype(np.uint32)
        got = sc.score_points(ids)
        qp = oracle.preprocess_f32(int(d), q)
        want = oracle.score_points_f32(int(d), base, qp, ids)
        np.testing.assert_array_equal(got, want)
        assert sc.score_point(5) == want_one(oracle, int(d), base, qp, 5)
        # score_internal(a, b): TMetric::similarity(stored a, stored b)  (metric_query_scorer.rs:95-100)
        assert sc.score_internal(3, 9) == oracle.similarity_f32(int(d), base[3], base[9])
        cpu, io = sc.take_hardware_counters()
        assert cpu == (77 + 1 + 1) * dim * 4 and io == 0
        sc.close()
    st.close()


def want_one(oracle, d, base, qp, i):
    return oracle.similarity_f32(d, qp, base[i])


def test_metric_preprocess_bit_exact(qb, oracle):
    rng = np.random.default_rng(3)
    for dim in (4, 20, 32, 70, 768, 1500):
        v = rng.uniform(-1, 1, (50, dim)).astype(np.float32)
        v[0] = 0.0                                        # zero vector stays zero (simple.rs:248-252)
        v[1] = oracle.preprocess_f32(oracle.COSINE, v[1])  # already normalised -> unchanged (tools.rs:14-16)
        got = qb.metric_preprocess(qb.Distance.Cosine, v)
        np.testing.assert_array_equal(got, oracle.preprocess_rows_f32(oracle.COSINE, v))
        np.testing.assert_array_equal(qb.metric_preprocess(qb.Distance.Dot, v), v)


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("n,dim", [(1000, 32), (5000, 70), (20000, 128), (100_000, 128), (150_000, 48), (70_000, 768)])
def test_search_batch_matches_peek_top_iter(qb, oracle, dist, n, dim):
    d = getattr(qb.Distance, dist)
    base, queries = make_data(oracle, int(d), n, dim, nq=4)
    st = qb.DenseVectorStorage(base, d)
    qp = np.stack([oracle.preprocess_f32(int(d), q) for q in queries])
    for top in (1, 10, 100):
        got = st.search_batch(queries, top)
        want = oracle.scan_f32(int(d), base, qp, top)
        for i in range(len(queries)):
            assert_topk_equal(got[i], want[i], oracle.score_rows_f32(int(d), base, qp[i]), f"{dist} n={n} dim={dim} top={top} q={i}")
    # batched search == per-query search (lib/segment/tests/integration/batch_search_test.rs:33-223)
    single = [st.search_batch(q, 10)[0] for q in queries]
    batched = st.search_batch(queries, 10)
    for a, b in zip(single, batched):
        np.testing.assert_array_equal(a, b)
    st.close()


def test_config_c1_100k_x128_dot(qb, oracle):
    """BASELINE.json configs[0]: 100K x 128 f32 dot-product brute force (uniform(-1,1), seeds 42/43, top 10)."""
    base = np.random.default_rng(42).uniform(-1, 1, (100_000, 128)).astype(np.float32)
    queries = np.random.default_rng(43).uniform(-1, 1, (16, 128)).astype(np.float32)
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    got = st.search_batch(queries, 10)
    want = oracle.scan_f32(oracle.DOT, base, queries, 10)
    for i in range(len(queries)):
        assert_topk_equal(got[i], want[i], None, f"C1 q={i}")
    st.close()


def test_deleted_and_filtered(qb, oracle):
    d = qb.Distance.Dot
    base, queries = make_data(oracle, int(d), 90_000, 64, nq=2)
    st = qb.DenseVectorStorage(base, d)
    rng = np.random.default_rng(8)
    deleted = rng.random(base.shape[0]) < 0.3
    from tests.util import pack_bitmap

    bm = pack_bitmap(deleted)
    want = oracle.scan_f32(int(d), base, queries, 10, deleted=bm)
    got = st.search_batch(queries, 10, point_deleted=deleted)          # per-call bitslice
    for i in range(2):
        assert_topk_equal(got[i], want[i])
        assert not deleted[got[i]["idx"]].any()
    st.set_deleted(deleted)                                            # resident flags
    got2 = st.search_batch(queries, 10)
    for i in range(2):
        np.testing.assert_array_equal(got[i], got2[i])
    st.set_deleted(None)
    # explicit candidate ids (a payload filter's result), small and large
    for n_ids in (500, 80_000):
        ids = rng.choice(base.shape[0], n_ids, replace=False).astype(np.uint32)
        got = qb.BatchFilteredSearcher.new(queries, st, None, 10).peek_top_iter(ids)
        for i in range(2):
            sc = oracle.score_points_f32(int(d), base, queries[i], ids)
            want_i = oracle.topk(sc, 10, ids)
            assert_topk_equal(got[i], want_i)
    st.close()


def test_edges(qb, oracle):
    d = qb.Distance.Euclid
    rng = np.random.default_rng(0)
    # fewer points than top
    base = rng.standard_normal((7, 40)).astype(np.float32)
    st = qb.DenseVectorStorage(base, d)
    q = rng.standard_normal(40).astype(np.float32)
    got = st.search_batch(q, 10)[0]
    assert got.size == 7
    assert_topk_equal(got, oracle.scan_f32(int(d), base, q, 10)[0])
    # everything deleted -> empty result
    assert st.search_batch(q, 10, point_deleted=np.ones(7, bool))[0].size == 0
    # cancellation flag already set -> QB_ERR_CANCELLED (check_process_stopped)
    from qdrant_b200._capi import QbError, QB_ERR_CANCELLED, QB_ERR_INVALID

    with pytest.raises(QbError) as ei:
        st.search_batch(q, 10, is_stopped=True)
    assert ei.value.status == QB_ERR_CANCELLED
    # top == 0 panics in the reference (NonZeroUsize); here a construction error
    with pytest.raises(ValueError):
        qb.BatchFilteredSearcher(q, st, 0)
    # out-of-range ids
    sc = st.build_raw_scorer(q)
    with pytest.raises(QbError) as ei:
        sc.score_points([99])
    assert ei.value.status == QB_ERR_INVALID
    with pytest.raises(IndexError):
        sc.score_internal(0, 99)
    # wrong query dim -> error at construction only (OperationResult)
    with pytest.raises(ValueError):
        st.build_raw_scorer(np.zeros(3, np.float32))
    st.close()
    # empty storage
    st = qb.DenseVectorStorage(np.zeros((0, 16), np.float32), qb.Distance.Dot)
    assert st.search_batch(np.zeros(16, np.float32), 5)[0].size == 0
    st.close()
    # identical rows: mass ties must not break selection (overflow fallback path)
    base = np.tile(rng.standard_normal((1, 64)).astype(np.float32), (120_000, 1))
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    got = st.search_batch(base[0], 10)[0]
    assert got.size == 10 and np.all(got["score"] == got["score"][0])
    assert sorted(got["idx"].tolist()) == list(range(10))  # (score desc, id asc)
    st.close()


def test_filtered_scorer_like_hnsw_hop(qb, oracle):
    """FilteredScorer::score_points (point_scorer.rs:265-295): filter deleted, truncate to limit, one batch call."""
    d = qb.Distance.Cosine
    base, queries = make_data(oracle, int(d), 2000, 96, nq=1)
    st = qb.DenseVectorStorage(base, d)
    deleted = np.zeros(2000, bool)
    deleted[::3] = True
    fs = qb.FilteredScorer.new(queries[0], st, None, point_deleted=deleted)
    ids = list(range(100, 140))
    res = fs.score_points(ids, limit=16)
    assert len(ids) == 16 and all(not deleted[i] for i in ids)
    qp = oracle.preprocess_f32(int(d), queries[0])
    np.testing.assert_array_equal(res["score"], oracle.score_points_f32(int(d), base, qp, np.array(ids, np.uint32)))
    st.close()


# ------------------------------------------------------------------------------------------------ batched f32 on the tensor cores (J1)
@pytest.mark.parametrize("dist,n,dim,nq", [("Cosine", 150_000, 768, 200), ("Dot", 140_000, 100, 64), ("Cosine", 200_000, 128, 300), ("Dot", 131_072, 1536, 33)])
def test_f32_batch_tensor_core_prefilter_is_exact(qb, oracle, dist, n, dim, nq):
    """Batches of >= 32 f32 queries: bf16 wgmma prefilter + exact rescoring of the survivors == oracle peek_top_iter, bit-exact
    scores, no fallback rerun, and == the CUDA-core path (option disable_mma)."""
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(dim + nq)
    base = (rng.standard_normal((n, dim)) * (1.0 if dist == "Cosine" else rng.uniform(0.2, 3.0, (n, 1)))).astype(np.float32)   # Dot: rows of very different norms
    if d == qb.Distance.Cosine:
        base = oracle.preprocess_rows_f32(oracle.COSINE, base)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    queries[0] = base[12345] * 3.0                    # a query whose best match is exact: score far above the rest
    qp = np.stack([oracle.preprocess_f32(int(d), q) for q in queries])
    deleted = rng.random(n) < 0.03
    st = qb.DenseVectorStorage(base, d)
    st.search_stats(reset=True)
    got = st.search_batch(queries, 10, point_deleted=deleted)
    searches, reruns = st.search_stats(reset=True)
    assert (searches, reruns) == (1, 0), (searches, reruns)
    want = oracle.scan_f32(int(d), base, qp, 10, deleted=pack_bitmap(deleted))
    for i in range(nq):
        assert_topk_equal(got[i], want[i], None, f"f32-mma {dist} q={i}")
    qb.set_option("disable_mma", 1)
    try:
        got_cc = st.search_batch(queries[:40], 10, point_deleted=deleted)
    finally:
        qb.set_option("disable_mma", 0)
    for a, b in zip(got[:40], got_cc):
        np.testing.assert_array_equal(a, b)
    st.close()


def test_f32_batch_with_nan_rows_and_nan_queries_stays_exact(qb, oracle):
    rng = np.random.default_rng(3)
    n, dim, nq = 140_000, 64, 40
    base = rng.standard_normal((n, dim)).astype(np.float32)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    queries[5, 3] = np.nan                            # every score of query 5 is NaN: the prefilter cannot rank it -> exact rerun
    got = st.search_batch(queries, 5)
    want = oracle.scan_f32(oracle.DOT, base, queries, 5)
    for i in range(nq):
        if i != 5:
            assert_topk_equal(got[i], want[i], None, f"nan-query batch q={i}")
    assert np.isnan(got[5]["score"]).all()
    st.close()
    base[777, 1] = np.nan                             # a NaN row ranks first for every query (OrderedFloat): the storage opts out of the prefilter
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    got = st.search_batch(queries[:4].copy() * 0 + rng.standard_normal((4, dim)).astype(np.float32), 5)
    assert all(g["idx"][0] == 777 and np.isnan(g["score"][0]) for g in got)
    st.close()


# ------------------------------------------------------------------------------------------------ single query through the bf16 shadow plane
@pytest.mark.parametrize("dist,n,dim,top", [("Cosine", 600_000, 64, 10), ("Dot", 560_001, 200, 16), ("Cosine", 530_000, 264, 1), ("Dot", 524_288, 520, 10),
                                            ("Cosine", 540_000, 1000, 10)])
@pytest.mark.parametrize("plane", [0, 1])
def test_single_query_prefilter_is_exact(qb, oracle, dist, n, dim, top, plane):
    """Single-query top-k on >= 2^19 rows (dot / cosine): the scan streams a shadow plane — int8 codes with a per-row scale (plane 0) or
    bf16 (plane 1) —, keeps every row whose error bound reaches the exact sample threshold, re-scores the survivors in the AVX order —
    identical, bit for bit, to the exact f32 scan (option disable_prefilter) and to the oracle; no fallback on ordinary data; deletions and
    id_base honoured; all-zero and denormal rows in the storage."""
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(dim + top)
    base = (rng.standard_normal((n, dim), dtype=np.float32) * (1.0 if dist == "Cosine" else rng.uniform(0.2, 3.0, (n, 1)).astype(np.float32)))
    if d == qb.Distance.Cosine:
        base = oracle.preprocess_rows_f32(oracle.COSINE, base)
    queries = rng.standard_normal((5, dim)).astype(np.float32)
    queries[1] = base[n - 7] * 2.0                    # best match in the very last rows
    queries[2] = base[3] * 0.5                        # ... and inside the exactly-scored sample prefix
    if dist == "Dot":
        base[1000:1010] = 0.0
        base[2000:2010] *= np.float32(1e-38)          # denormal rows
        queries[3, ::2] = 0.0
    deleted = rng.random(n) < 0.02
    qb.set_option("prefilter_plane", plane)
    st = qb.DenseVectorStorage(base, d)
    from qdrant_b200._capi import check, lib
    check(lib().qb_storage_set_id_base(st._h, 1000))
    st.search_stats(reset=True)
    try:
        got = [st.search_batch(q, top, point_deleted=deleted)[0] for q in queries]
    finally:
        qb.set_option("prefilter_plane", 0)
    searches, reruns = st.search_stats(reset=True)
    assert (searches, reruns) == (5, 0), (searches, reruns)
    qb.set_option("disable_prefilter", 1)
    try:
        exact = [st.search_batch(q, top, point_deleted=deleted)[0] for q in queries]
    finally:
        qb.set_option("disable_prefilter", 0)
    for a, b in zip(got, exact):
        np.testing.assert_array_equal(a["idx"], b["idx"])
        np.testing.assert_array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32))
    qp = np.stack([oracle.preprocess_f32(int(d), q) for q in queries[:2]])
    want = oracle.scan_f32(int(d), base, qp, top, deleted=pack_bitmap(deleted))
    for i in range(2):
        g = got[i].copy()
        g["idx"] -= 1000
        assert_topk_equal(g, want[i], None, f"prefilter {dist} dim={dim} q={i}")
    st.close()


def test_single_query_prefilter_falls_back_on_the_device(qb, oracle):
    """Cases the prefilter cannot decide go to the exact scan WITHOUT a host round trip (the finish kernel raises a device flag, the
    always-enqueued exact scan runs): mass ties (more tied rows than candidate slots), a NaN query, a sample prefix that is almost
    entirely deleted.  Results == exact path; the fallbacks are counted by qb_search_stats."""
    rng = np.random.default_rng(9)
    n, dim = 600_000, 96
    base = rng.standard_normal((n, dim), dtype=np.float32)
    base[100_000:120_000] = base[99_999]              # 20 001 identical rows (more than the candidate list holds), the best match of query 0
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    q_ties = base[99_999] * 4.0
    q_nan = rng.standard_normal(dim).astype(np.float32); q_nan[5] = np.nan
    q_plain = rng.standard_normal(dim).astype(np.float32)
    del_prefix = np.zeros(n, bool); del_prefix[:200_000] = True; del_prefix[:4] = False    # 4 live rows in the sample < top
    cases = [(q_ties, None), (q_nan, None), (q_plain, del_prefix), (q_plain, None)]
    st.search_stats(reset=True)
    got = [st.search_batch(q, 10, point_deleted=dl)[0] for q, dl in cases]
    searches, reruns = st.search_stats(reset=True)
    assert searches == 4 and reruns == 3, (searches, reruns)
    qb.set_option("disable_prefilter", 1)
    try:
        exact = [st.search_batch(q, 10, point_deleted=dl)[0] for q, dl in cases]
    finally:
        qb.set_option("disable_prefilter", 0)
    for i, (a, b) in enumerate(zip(got, exact)):
        np.testing.assert_array_equal(a["idx"], b["idx"], err_msg=f"case {i}")
        np.testing.assert_array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32), err_msg=f"case {i}")
    assert list(got[0]["idx"]) == list(range(99_999, 100_009))          # ties broken by ascending id
    assert np.isnan(got[1]["score"]).all()
    st.close()
