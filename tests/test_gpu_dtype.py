"""GPU parity: Float16 and Uint8 dense storages vs the CPU oracle.

u8: bit-exact against the restated avx2 kernels (metric_uint/avx2/*.rs) incl. the reference's KAT vectors.
f16: the oracle restates metric_f16/avx/*.rs with F16C intrinsics; parity is bit-exact as well (the reference's own
     f16 test only asks for rel 5e-4, metric_f16/avx/dot.rs:124).

Neither datatype can use the in-kernel top-k, the shadow-plane prefilter or the tensor-core batch paths (all dense f32 only),
so every search here runs the generic planner: one dense pass + select up to 65 536 candidates, sample -> threshold ->
filter -> select above that, and a full rerun when the filter pass overflows."""
import numpy as np
import pytest

from tests.util import assert_topk_equal

pytestmark = pytest.mark.gpu

DISTS = ["Cosine", "Dot", "Euclid", "Manhattan"]


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


class Dt:
    """One storage datatype as the oracle sees it: row generation, query conversion, whole-storage scoring."""

    def __init__(self, qb, oracle, name, dist):
        self.o, self.name, self.d = oracle, name, getattr(qb.Distance, dist)
        self.cosine = self.d == qb.Distance.Cosine
        self.vdt = qb.VectorStorageDatatype.Uint8 if name == "u8" else qb.VectorStorageDatatype.Float16
        self.elem = 1 if name == "u8" else 2

    def rows(self, rng, n, dim):
        if self.name == "u8":
            return rng.integers(0, 256, (n, dim), dtype=np.uint8)
        base = rng.standard_normal((n, dim)).astype(np.float32)
        if self.cosine:   # Cosine: rows are stored normalised (Distance::preprocess_vector at insert time)
            base = self.o.preprocess_rows_f32(self.o.COSINE, base)
        return base.astype(np.float16)

    def queries(self, rng, nq, dim):
        if self.name == "u8":   # below 0 and above 255 on purpose: truncation and saturation of `x as u8`
            return rng.uniform(-20.0, 300.0, (nq, dim)).astype(np.float32)
        return rng.standard_normal((nq, dim)).astype(np.float32)

    def conv(self, q):
        return self.o.to_u8_query(q) if self.name == "u8" else self.o.to_f16_query(int(self.d), q)

    def raw(self, rows, q_conv, ids=None):
        """similarity of a query already in the storage datatype to every row (or the listed rows)"""
        f = self.o.score_rows_u8 if self.name == "u8" else self.o.score_rows_f16
        return f(int(self.d), rows, q_conv, ids)

    def scores(self, rows, q, ids=None):
        """similarity of the f32 query `q`, converted as the storage converts it, to every row (or the listed rows)"""
        return self.raw(rows, self.conv(q), ids)

    def scan(self, rows, queries, top, deleted=None):
        f = self.o.scan_u8 if self.name == "u8" else self.o.scan_f16
        return f(int(self.d), rows, np.stack([self.conv(q) for q in np.atleast_2d(queries)]), top, deleted)


def assert_scores_equal(got, want, what=""):
    """Score bits; a NaN only has to be NaN at the same position (x86 and the GPU produce different NaN payloads)."""
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN positions differ"
    np.testing.assert_array_equal(got.view(np.uint32)[~nan], want.view(np.uint32)[~nan], err_msg=what)


def check_all(got, want, all_scores, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert_topk_equal(g, w, all_scores[i] if all_scores is not None else None, f"{what} q{i}")


# ------------------------------------------------------------------------------------------------ scoring
@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("dim", [1, 8, 15, 16, 24, 31, 32, 33, 100, 300, 768, 1030, 2048, 2080, 4096, 65536])
def test_u8_bit_exact(qb, oracle, dist, dim):
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(dim)
    n = 400 if dim <= 4096 else 8
    base = rng.integers(0, 256, (n, dim), dtype=np.uint8)
    base[0] = 0
    base[1] = 255                                        # saturated: Dot / Cosine lane sums pass 2^24 from dim 2080 on
    base[2] = np.resize(np.array([0, 255], np.uint8), dim)
    base[3] = np.resize(np.array([255, 0], np.uint8), dim)
    hi = max(n // 2, n - 2)
    base[4:hi] = rng.integers(200, 256, (hi - 4, dim), dtype=np.uint8)   # large odd lane sums: rounded once at the end, not per block
    st = qb.DenseVectorStorage(base, d, qb.VectorStorageDatatype.Uint8)
    ids = np.arange(n, dtype=np.uint32)
    # `x as u8` edges: NaN -> 0, +-inf saturate, -0.0 / negatives / fractions truncate (data_types/primitive.rs:127-129)
    edge = np.resize(np.array([np.nan, np.inf, -np.inf, -0.0, -3.7, 255.5, 256.0, 1e30, 7.9, 200.2], np.float32), dim)
    for q in (rng.uniform(0, 255, dim).astype(np.float32), np.full(dim, 255.0, np.float32), np.full(dim, 300.7, np.float32),
              rng.uniform(-20, 40, dim).astype(np.float32), rng.uniform(200, 256, dim).astype(np.float32), edge, edge[::-1].copy()):
        want = oracle.score_rows_u8(int(d), base, oracle.to_u8_query(q))
        sc = st.build_raw_scorer(q)
        np.testing.assert_array_equal(sc.score_points(ids).view(np.uint32), want.view(np.uint32))
        sc.close()
    for r in (1, 4):
        isc = st.raw_internal_scorer(r)
        want = oracle.score_rows_u8(int(d), base, base[r])
        np.testing.assert_array_equal(isc.score_points(ids).view(np.uint32), want.view(np.uint32))
        assert isc.score_internal(r, 2).view(np.uint32) == want[2].view(np.uint32)
        isc.close()
    st.close()


def test_u8_reference_kat(qb, oracle):
    from tests.test_oracle_kat import u8_kat

    v1, v2 = u8_kat()
    for dist, name in ((qb.Distance.Dot, "dot"), (qb.Distance.Cosine, "cosine"), (qb.Distance.Euclid, "euclid"), (qb.Distance.Manhattan, "manhattan")):
        st = qb.DenseVectorStorage(v2[None, :], dist, qb.VectorStorageDatatype.Uint8)
        got = st.build_raw_scorer(v1.astype(np.float32)).score_point(0)
        assert got == oracle.raw_u8(name, "scalar", v1, v2) == oracle.raw_u8(name, "avx", v1, v2)
        st.close()


def test_u8_search(qb, oracle):
    rng = np.random.default_rng(5)
    base = rng.integers(0, 256, (70_000, 64), dtype=np.uint8)
    st = qb.DenseVectorStorage(base, qb.Distance.Euclid, qb.VectorStorageDatatype.Uint8)
    q = rng.uniform(0, 255, 64).astype(np.float32)
    got = st.search_batch(q, 10)[0]
    qu8 = np.trunc(q).astype(np.uint8)
    sc = np.array([oracle.similarity_u8(oracle.EUCLID, qu8, base[i]) for i in range(base.shape[0])], np.float32)
    assert_topk_equal(got, oracle.topk(sc, 10), sc)
    st.close()


@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("dim", [1, 8, 15, 16, 17, 20, 31, 32, 33, 70, 256, 768, 1000, 1536, 4096])
def test_f16_bit_exact(qb, oracle, dist, dim):
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(dim + 1)
    base32 = rng.standard_normal((300, dim)).astype(np.float32)
    if d == qb.Distance.Cosine:
        base32 = oracle.preprocess_rows_f32(oracle.COSINE, base32)
    base = base32.astype(np.float16)
    st = qb.DenseVectorStorage(base, d, qb.VectorStorageDatatype.Float16)
    ids = np.arange(300, dtype=np.uint32)
    # f16::from_f32 edges: 65519 rounds to 65504, 65520 and 1e6 overflow to inf (Dot / Euclid / Manhattan) but are normalised in
    # f32 first under Cosine; 2^-24 is the smallest subnormal, 2^-26 rounds to zero; one NaN makes every score NaN
    big = np.resize(np.array([65504.0, 65519.0, 65520.0, 1e6, -65520.0, 0.5, -2.0, 3.0], np.float32), dim)
    tiny = np.resize(np.array([2.0 ** -24, 2.0 ** -26, -(2.0 ** -24), 1.5 * 2.0 ** -24, 0.25], np.float32), dim)
    nan = rng.standard_normal(dim).astype(np.float32)
    nan[dim // 2] = np.nan
    queries = [rng.standard_normal(dim).astype(np.float32) for _ in range(3)] + [big, tiny, nan]
    for q in queries:
        want = oracle.score_rows_f16(int(d), base, oracle.to_f16_query(int(d), q))
        sc = st.build_raw_scorer(q)
        assert_scores_equal(sc.score_points(ids), want, f"{dist} dim {dim}")
        sc.close()
    # the internal scorer: a stored row is the query as it is (no conversion)
    for r in (0, 7):
        isc = st.raw_internal_scorer(r)
        want = oracle.score_rows_f16(int(d), base, base[r])
        np.testing.assert_array_equal(isc.score_points(ids).view(np.uint32), want.view(np.uint32))
        assert isc.score_internal(r, 11).view(np.uint32) == want[11].view(np.uint32)
        isc.close()
    st.close()


@pytest.mark.parametrize("dist", DISTS)
def test_f16_special_rows(qb, oracle, dist):
    """Rows holding +-inf, NaN, subnormals and signed zeros: score bits (NaN by position), NaN ranks first, -0.0 keeps its sign."""
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(40)
    n, dim = 3_000, 40
    base = rng.standard_normal((n, dim)).astype(np.float16)
    sub = np.float16(2.0 ** -24)
    base[10, 3], base[11, 39], base[12] = np.inf, -np.inf, np.inf
    base[20, 0], base[21, 35] = np.nan, np.nan
    base[30] = sub * rng.integers(-1023, 1024, dim)                      # subnormal rows
    base[31] = np.float16(0.0)
    base[32] = np.float16(-0.0)
    base[33, ::2] = np.float16(-0.0)
    ids = np.arange(n, dtype=np.uint32)
    st = qb.DenseVectorStorage(base, d, qb.VectorStorageDatatype.Float16)
    zero = np.zeros(dim, np.float32)
    neg_zero = np.full(dim, -0.0, np.float32)
    for q in (rng.standard_normal(dim).astype(np.float32), zero, neg_zero, base[32].astype(np.float32), base[30].astype(np.float32)):
        want = oracle.score_rows_f16(int(d), base, oracle.to_f16_query(int(d), q))
        sc = st.build_raw_scorer(q)
        assert_scores_equal(sc.score_points(ids), want, f"{dist} special rows")
        sc.close()
        for top in (1, 10):
            assert_topk_equal(st.search_batch(q, top)[0], oracle.topk(want, top), want, f"{dist} special rows top {top}")
    # identical vectors: Euclid / Manhattan give -0.0 (a negated +0.0), which must survive the top-k keys
    if dist in ("Euclid", "Manhattan"):
        g = st.search_batch(base[5].astype(np.float32), 5)[0]          # behind the NaN rows
        assert g["score"].view(np.uint32)[g["idx"] == 5].tolist() == [0x80000000]
    st.close()


@pytest.mark.parametrize("n", [3_000, 100_000])
def test_f16_nan_rows_rank_first(qb, oracle, n):
    """OrderedFloat: NaN is the greatest score, in the direct path (n <= 65 536) and through the threshold + filter passes."""
    rng = np.random.default_rng(2)
    base = rng.standard_normal((n, 64)).astype(np.float16)
    nan_rows = [17, n // 2, n - 5]
    base[nan_rows, 3] = np.nan
    q = rng.standard_normal((2, 64)).astype(np.float32)
    st = qb.DenseVectorStorage(base, qb.Distance.Dot, qb.VectorStorageDatatype.Float16)
    dt = Dt(qb, oracle, "f16", "Dot")
    for queries in (q[:1], q):
        got = st.search_batch(queries, 10)
        want = dt.scan(base, queries, 10)
        for g in got:
            assert np.isnan(g["score"][:3]).all() and sorted(g["idx"][:3].tolist()) == nan_rows
        check_all(got, want, None, f"NaN rows n={n} nq={len(queries)}")
    st.close()


# ------------------------------------------------------------------------------------------------ search
@pytest.mark.parametrize("n", [3_000, 150_001])
@pytest.mark.parametrize("dist", DISTS)
@pytest.mark.parametrize("dtn", ["f16", "u8"])
def test_search(qb, oracle, dtn, dist, n):
    """Direct path (n <= 65 536) and sample -> threshold -> filter path (odd row count): batches, single queries, deletions, id lists."""
    dt = Dt(qb, oracle, dtn, dist)
    dim = 40 if dtn == "f16" else 72
    rng = np.random.default_rng(100 + n + dim)
    base = dt.rows(rng, n, dim)
    queries = dt.queries(rng, 5, dim)
    st = qb.DenseVectorStorage(base, dt.d, dt.vdt)
    full = [dt.scores(base, q) for q in queries]
    for top in (1, 10, 100):
        got = st.search_batch(queries, top)
        check_all(got, [oracle.topk(s, top) for s in full], full, f"{dtn} {dist} n={n} top={top}")
        for i, q in enumerate(queries):                   # a batch answers exactly what its queries answer one at a time
            one = st.search_batch(q, top)[0]
            assert np.array_equal(one, got[i]), f"{dtn} {dist} n={n} top={top}: query {i} alone differs from the batch"
    # deletions: a per-call bitmap and the resident flags give the same answer
    deleted = rng.random(n) < 0.25
    deleted[np.argmax(full[0])] = True                    # the best row of query 0 goes
    live = np.flatnonzero(~deleted).astype(np.uint32)
    want = [oracle.topk(s[live], 10, live) for s in full]
    per_call = st.search_batch(queries, 10, point_deleted=deleted)
    check_all(per_call, want, full, f"{dtn} {dist} n={n} deleted (per call)")
    st.set_deleted(deleted)
    resident = st.search_batch(queries, 10)
    check_all(resident, want, full, f"{dtn} {dist} n={n} deleted (resident)")
    for a, b in zip(per_call, resident):
        assert np.array_equal(a, b)
    st.set_deleted(None)
    # id lists
    for k in (500, 80_000):
        if k > n:
            continue
        ids = rng.choice(n, k, replace=False).astype(np.uint32)
        got = st.search_batch(queries, 10, id_list=ids)
        check_all(got, [oracle.topk(s[ids], 10, ids) for s in full], full, f"{dtn} {dist} n={n} id list {k}")
        for g in got:
            assert set(g["idx"].tolist()) <= set(ids.tolist())
    if n > 65_536:
        # the select-large path (top > 4096)
        got = st.search_batch(queries[:2], 5000)
        check_all(got, [oracle.topk(s, 5000) for s in full[:2]], full, f"{dtn} {dist} top 5000")
        # the oracle's own scan agrees with the per-query scoring used above
        check_all(got[:1], dt.scan(base, queries[:1], 5000), full, f"{dtn} {dist} oracle scan")
    st.close()


@pytest.mark.parametrize("dtn,dist", [("f16", "Cosine"), ("u8", "Dot")])
def test_search_batch_device(qb, oracle, dtn, dist):
    """qb_search_batch_device with torch device tensors == the host search == the oracle."""
    import torch
    from qdrant_b200._capi import check, lib, vp

    dt = Dt(qb, oracle, dtn, dist)
    n, dim, nq, top = 120_000, 48, 6, 20
    rng = np.random.default_rng(9)
    base = dt.rows(rng, n, dim)
    queries = dt.queries(rng, nq, dim)
    st = qb.DenseVectorStorage(base, dt.d, dt.vdt)
    d_q = torch.from_numpy(queries).cuda()
    d_out = torch.zeros((nq, top), dtype=torch.int64, device="cuda")
    d_cnt = torch.zeros((nq,), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()                              # the library's stream does not wait for torch's copies
    for k in (1, nq):
        check(lib().qb_search_batch_device(st._h, vp(d_q.data_ptr()), k, top, vp(d_out.data_ptr()), vp(d_cnt.data_ptr())))
        torch.cuda.synchronize()
        out = d_out.cpu().numpy().view(qb.SCORED_POINT_OFFSET)
        cnt = d_cnt.cpu().numpy()
        got = [out[i, : cnt[i]].copy() for i in range(k)]
        host = st.search_batch(queries[:k], top)
        for g, h in zip(got, host):
            assert np.array_equal(g, h)
        full = [dt.scores(base, q) for q in queries[:k]]
        check_all(got, [oracle.topk(s, top) for s in full], full, f"{dtn} {dist} device nq={k}")
    st.close()


def test_u8_mass_ties(qb, oracle):
    """Whole blocks of equal scores overflow the filter pass's candidate buffer: the search reruns as one full materialisation and
    answers in (score desc, id asc) order."""
    rng = np.random.default_rng(12)
    # Cosine with an all-negative query: `x as u8` makes it the zero vector, every score is 0 (denominator 0)
    n, dim = 150_001, 40
    base = rng.integers(0, 256, (n, dim), dtype=np.uint8)
    st = qb.DenseVectorStorage(base, qb.Distance.Cosine, qb.VectorStorageDatatype.Uint8)
    q = -rng.uniform(0.5, 10.0, (2, dim)).astype(np.float32)
    assert not oracle.to_u8_query(q[0]).any()
    st.search_stats(reset=True)
    for g in st.search_batch(q, 10):
        assert g["idx"].tolist() == list(range(10)) and not g["score"].view(np.uint32).any()
    assert st.search_stats()[1] >= 1, "the filter pass should have overflowed and rerun"
    st.close()
    # ten distinct rows repeated to 200 000: every score value occurs 20 000 times, more than the ~8 K candidates the planner sizes
    n = 200_000
    distinct = rng.integers(0, 256, (10, dim), dtype=np.uint8)
    base = np.ascontiguousarray(distinct[np.arange(n) % 10])
    for dist in ("Dot", "Euclid"):
        dt = Dt(qb, oracle, "u8", dist)
        st = qb.DenseVectorStorage(base, dt.d, dt.vdt)
        queries = dt.queries(rng, 3, dim)
        st.search_stats(reset=True)
        for top in (10, 100):
            got = st.search_batch(queries, top)
            for g, qv in zip(got, queries):
                s = dt.scores(base, qv)
                order = np.lexsort((np.arange(n), -s.astype(np.float64)))[:top]
                assert np.array_equal(g["idx"], order.astype(np.uint32)) and np.array_equal(g["score"].view(np.uint32), s[order].view(np.uint32))
                assert_topk_equal(g, oracle.topk(s, top), s, f"ties {dist} top {top}")
        assert st.search_stats()[1] >= 1, "the filter pass should have overflowed and rerun"
        st.close()


@pytest.mark.parametrize("dtn,dist", [("f16", "Dot"), ("u8", "Euclid")])
def test_id_base(qb, oracle, dtn, dist):
    """Global ids (local row + id_base) through search, score_points, score_internal, rescore and id lists."""
    from qdrant_b200._capi import check, lib

    dt = Dt(qb, oracle, dtn, dist)
    rng = np.random.default_rng(6)
    n, dim, base_id = 20_000, 64, 1_000_000
    base = dt.rows(rng, n, dim)
    q = dt.queries(rng, 1, dim)[0]
    s = dt.scores(base, q)
    st = qb.DenseVectorStorage(base, dt.d, dt.vdt)
    check(lib().qb_storage_set_id_base(st._h, base_id))
    got = st.search_batch(q, 50)[0]
    want = oracle.topk(s, 50)
    assert np.array_equal(got["idx"], want["idx"] + base_id) and np.array_equal(got["score"].view(np.uint32), want["score"].view(np.uint32))
    sc = st.build_raw_scorer(q)
    np.testing.assert_array_equal(sc.score_points(got["idx"]).view(np.uint32), want["score"].view(np.uint32))
    with pytest.raises(qb.QbError):
        sc.score_points(np.array([5], np.uint32))          # a local id is out of range now
    cand = rng.choice(n, 300, replace=False).astype(np.uint32)
    res = qb.rescore(sc, cand + base_id, 10)
    order = np.lexsort((cand, -s[cand].astype(np.float64)))[:10]
    np.testing.assert_array_equal(res["idx"], cand[order] + base_id)
    np.testing.assert_array_equal(res["score"].view(np.uint32), s[cand[order]].view(np.uint32))
    ids = rng.choice(n, 3000, replace=False).astype(np.uint32)
    f = st.search_batch(q, 10, id_list=ids + base_id)[0]
    assert_topk_equal(f, oracle.topk(s[ids], 10, ids + base_id), None, "id list")
    assert set(f["idx"].tolist()) <= set((ids + base_id).tolist())
    internal = dt.raw(base, base[3], np.array([9], np.uint32))[0]
    assert sc.score_internal(base_id + 3, base_id + 9).view(np.uint32) == internal.view(np.uint32)
    sc.close(); st.close()


def test_rescore_with_f16_originals(qb, oracle):
    """Oversampled SQ8 candidates rescored with an f16 original storage (postprocess_search_result): oracle f16 scores, in order."""
    rng = np.random.default_rng(13)
    n, dim, top = 30_000, 64, 10
    rows16 = rng.standard_normal((n, dim)).astype(np.float16)
    dt = Dt(qb, oracle, "f16", "Dot")
    sq = oracle.SQ8.encode(rows16.astype(np.float32), oracle.QD_DOT, False)
    qs = qb.ScalarQuantizedVectors(sq.rows, dim, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, qb.Distance.Dot)
    orig = qb.DenseVectorStorage(rows16, qb.Distance.Dot, qb.VectorStorageDatatype.Float16)
    queries = rng.standard_normal((3, dim)).astype(np.float32)
    over_top = qb.get_oversampled_top(top, True, 4.0)
    got = qs.search_batch(queries, over_top)
    for q, cand in zip(queries, got):
        s = dt.scores(rows16, q, cand["idx"])
        order = np.lexsort((cand["idx"], -s.astype(np.float64)))[:top]
        for res in (qb.postprocess_search_result(cand, orig, q, top, rescore=True), qb.rescore(orig.build_raw_scorer(q), cand["idx"], top)):
            np.testing.assert_array_equal(res["idx"], cand["idx"][order])
            np.testing.assert_array_equal(res["score"].view(np.uint32), s[order].view(np.uint32))
    qs.close(); orig.close()


# ------------------------------------------------------------------------------------------------ storage plumbing
@pytest.mark.parametrize("dtn", ["f16", "u8"])
def test_storage_plumbing(qb, oracle, dtn):
    """write_rows on a sub-range, get_dense round trip, load_dense_file, and the hardware counters."""
    dist = "Euclid" if dtn == "f16" else "Manhattan"
    dt = Dt(qb, oracle, dtn, dist)
    rng = np.random.default_rng(14)
    n, dim, nq = 5_000, 48, 3
    base = dt.rows(rng, n, dim)
    if dtn == "f16":
        base[7, 1], base[8, 2], base[9, 3] = np.nan, -np.inf, np.float16(-0.0)
    queries = dt.queries(rng, nq, dim)
    st = qb.DenseVectorStorage(base, dt.d, dt.vdt)
    # get_dense: the stored bytes come back bit for bit, NaN payloads included
    ids = np.array([0, 7, 8, 9, n - 1, 7], np.uint32)
    np.testing.assert_array_equal(st.get_dense(ids).view(np.uint8), base[ids].view(np.uint8))
    # write_rows on [1000, 1700): searches see the new rows
    new = dt.rows(rng, 700, dim)
    st.write_rows(1000, new)
    upd = base.copy()
    upd[1000:1700] = new
    np.testing.assert_array_equal(st.get_dense(np.arange(990, 1710, dtype=np.uint32)).view(np.uint8), upd[990:1710].view(np.uint8))
    full = [dt.scores(upd, q) for q in queries]
    check_all(st.search_batch(queries, 10), [oracle.topk(s, 10) for s in full], full, f"{dtn} after write_rows")
    sc = st.build_raw_scorer(queries[0])
    pts = np.arange(995, 1010, dtype=np.uint32)
    assert_scores_equal(sc.score_points(pts), full[0][pts], f"{dtn} after write_rows")
    # counters: dim * size_of::<T>() per scored point (metric_query_scorer.rs:43-48); vector_io_read only once on disk
    assert sc.take_hardware_counters() == (pts.size * dim * dt.elem, 0)
    cnt = qb.HwCounters()
    st.search_batch(queries, 5, counters=cnt)
    assert (cnt.cpu, cnt.vector_io_read) == (n * nq * dim * dt.elem, 0)
    sc.close()
    st.set_on_disk(True)
    cnt = qb.HwCounters()
    st.search_batch(queries, 5, counters=cnt)
    assert (cnt.cpu, cnt.vector_io_read) == (n * nq * dim * dt.elem, n * nq * dim * dt.elem)
    sc = st.build_raw_scorer(queries[1])
    sc.score_points(np.arange(7, dtype=np.uint32))
    assert sc.take_hardware_counters() == (7 * dim * dt.elem, 7 * dim * dt.elem)
    sc.close(); st.close()
    # matrix.dat as it lies on disk (b"data" header, headerless rows, a trailing partial row ignored) == the oracle
    ld = qb.load_dense_file(b"data" + upd.tobytes() + b"\0" * 5, dt.d, dim, dt.vdt)
    assert (ld.count, ld.dim) == (n, dim)
    check_all(ld.search_batch(queries, 10), [oracle.topk(s, 10) for s in full], full, f"{dtn} load_dense_file")
    lsc = ld.raw_scorer(queries[1])
    assert_scores_equal(lsc.score_points(np.arange(n, dtype=np.uint32)), full[1], f"{dtn} load_dense_file")
    lsc.close(); ld.close()
