"""GPU search over SQ8 / PQ / BQ storages vs the CPU oracle, tolerance 0, through every search entry point.

tests/test_gpu_quant.py pins how these storages score (every distance, encoding and dim bit for bit); this file pins how they search:
the direct path (n <= 65 536) and the sample -> threshold -> filter path, batches against their queries one at a time, per-call and
resident deletions, id lists (which take SQ8 batches off the tensor cores and PQ / BQ onto their id-list kernels), id_base, the
device-resident entry point, tops above 4096 with rescoring against the original vectors, the three-level plan of large SQ8 batches
on the tensor cores, PQ shards, mass ties, and SQ8 storages whose metadata is not finite.

Storages are built from oracle-encoded rows (PQ codes drawn at random: scoring does not depend on how they were chosen), so both
sides score the same bytes.  Expected top-k lists come from oracle.topk over the oracle's whole-storage scores, and
assert_topk_equal gets those scores so that ties at the boundary may differ only between rows that really share the score."""
import numpy as np
import pytest

from tests.util import assert_topk_equal, pack_bitmap

pytestmark = pytest.mark.gpu

# (kind, distance, dim, kind parameter): PQ chunk (Dot: m = 32; Euclid: m = 18 with a last chunk of 2), BQ (encoding, query encoding)
SPECS = [
    ("sq8", "Cosine", 40, None), ("sq8", "Dot", 40, None), ("sq8", "Euclid", 40, None), ("sq8", "Manhattan", 40, None),
    ("pq", "Dot", 128, 4), ("pq", "Euclid", 70, 4),
    ("bq", "Dot", 100, ("OneBit", "SameAsStorage")), ("bq", "Euclid", 100, ("TwoBits", "Scalar8bits")),
    ("bq", "Manhattan", 100, ("OneAndHalfBits", "Scalar4bits")),
]


def spec_id(spec):
    kind, dist, _, par = spec
    return f"{kind}-{dist}" + (f"-{par[0]}-{par[1]}" if kind == "bq" else "")


def spec(name):
    return next(s for s in SPECS if spec_id(s) == name)


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


class Quant:
    """One quantized storage: the oracle's encoding of `base`, the library's storage over the same bytes, the oracle's scores."""

    def __init__(self, qb, oracle, spec, base, rng):
        self.qb, self.o = qb, oracle
        self.kind, dist, self.dim, self.par = spec
        self.d = getattr(qb.Distance, dist)
        dt, inv = qb.construct_vector_parameters(self.d)
        dt, inv = int(dt), bool(inv)
        if self.kind == "sq8":
            self.enc = oracle.SQ8.encode(base, dt, inv)
        elif self.kind == "pq":
            cents = (rng.standard_normal((256, self.dim)) * 0.5).astype(np.float32)
            m = -(-self.dim // self.par)
            self.enc = oracle.PQ(self.dim, self.par, cents, rng.integers(0, 256, (base.shape[0], m), dtype=np.uint8), dt, inv)
        else:
            self.e, self.qe = int(getattr(qb.BQEncoding, self.par[0])), int(getattr(qb.BQQueryEncoding, self.par[1]))
            self.ms = oracle.bq_mean_std(base) if self.e != oracle.BQ_ONE else None
            self.enc = oracle.BQ.encode(base, self.e, self.qe, dt, inv, self.ms)

    def storage(self, rows=None):
        """the library's storage over the oracle's bytes (or over a row slice of them)"""
        qb, enc = self.qb, self.enc
        if self.kind == "sq8":
            r = enc.rows if rows is None else enc.rows[rows]
            return qb.ScalarQuantizedVectors(r, self.dim, enc.meta.alpha, enc.meta.offset, enc.meta.multiplier, self.d)
        if self.kind == "pq":
            return qb.ProductQuantizedVectors(enc.codes if rows is None else enc.codes[rows], enc.centroids, self.par, self.dim, self.d)
        r = enc.rows if rows is None else enc.rows[rows]
        return qb.BinaryQuantizedVectors(r, self.dim, self.d, qb.BQEncoding(self.e), qb.BQQueryEncoding(self.qe), self.ms)

    def encode(self, q):
        qp = self.o.preprocess_f32(int(self.d), q)
        return self.enc.encode_query(qp)

    def scores(self, q, ids=None):
        """the oracle's score of the f32 query `q` (encoded as the storage encodes it) for every row, or every listed row"""
        e = self.encode(q)
        return self.enc.score_rows(*e, ids) if self.kind == "sq8" else self.enc.score_rows(e, ids)


def data(oracle, qb, dist, n, dim, rng, nq):
    base = rng.standard_normal((n, dim)).astype(np.float32)
    if dist == "Cosine":
        base = oracle.preprocess_rows_f32(oracle.COSINE, base)
    return base, rng.standard_normal((nq, dim)).astype(np.float32)


def shifted(res, delta):
    out = [r.copy() for r in res]
    for r in out:
        r["idx"] += np.uint32(delta % (1 << 32))
    return out


def check_all(got, want, all_scores, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert_topk_equal(g, w, all_scores[i] if all_scores is not None else None, f"{what} q{i}")


def device_search(st, queries, top):
    """qb_search_batch_device on torch device tensors -> list of SCORED arrays"""
    import torch
    from qdrant_b200 import scorer as qb
    from qdrant_b200._capi import check, lib, vp

    nq = queries.shape[0]
    d_q = torch.from_numpy(np.ascontiguousarray(queries, dtype=np.float32)).cuda()
    d_out = torch.zeros((nq, top), dtype=torch.int64, device="cuda")
    d_cnt = torch.zeros((nq,), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()                              # the library's stream does not wait for torch's copies
    check(lib().qb_search_batch_device(st._h, vp(d_q.data_ptr()), nq, top, vp(d_out.data_ptr()), vp(d_cnt.data_ptr())))
    torch.cuda.synchronize()
    out = d_out.cpu().numpy().view(qb.SCORED_POINT_OFFSET)
    cnt = d_cnt.cpu().numpy()
    return [out[i, : cnt[i]].copy() for i in range(nq)]


def set_id_base(st, base_id):
    from qdrant_b200._capi import check, lib

    check(lib().qb_storage_set_id_base(st._h, base_id))


def with_option(qb, name, value, fn):
    qb.set_option(name, value)
    try:
        return fn()
    finally:
        qb.set_option(name, 0)


# ------------------------------------------------------------------------------------------------ entry points
@pytest.mark.parametrize("n", [3_000, 150_001])
@pytest.mark.parametrize("spec", SPECS, ids=spec_id)
def test_entry_points(qb, oracle, spec, n):
    """Direct path (n <= 65 536) and sample -> threshold -> filter path (odd row count): tops, batch == one at a time, deletions,
    id lists at 1, 2 and 10 queries (PQ: pq_scan_kernel, pq_scan2_kernel; the four/eight/sixteen-query kernels take no ids), and id_base."""
    rng = np.random.default_rng(n + spec[2] + len(spec_id(spec)))
    base, queries = data(oracle, qb, spec[1], n, spec[2], rng, 10)
    k = Quant(qb, oracle, spec, base, rng)
    st = k.storage()
    full = [k.scores(q) for q in queries]
    what = f"{spec_id(spec)} n={n}"
    for top in (1, 10, 100):
        got = st.search_batch(queries, top)
        check_all(got, [oracle.topk(s, top) for s in full], full, f"{what} top={top}")
        for i, q in enumerate(queries):                   # a batch answers exactly what its queries answer one at a time
            assert np.array_equal(st.search_batch(q, top)[0], got[i]), f"{what} top={top}: query {i} alone differs from the batch"
    # deletions: a per-call bitmap and the resident flags give the same answer
    deleted = rng.random(n) < 0.25
    deleted[np.argmax(full[0])] = True                    # the best row of query 0 goes
    live = np.flatnonzero(~deleted).astype(np.uint32)
    want = [oracle.topk(s[live], 10, live) for s in full]
    per_call = st.search_batch(queries, 10, point_deleted=deleted)
    check_all(per_call, want, full, f"{what} deleted (per call)")
    st.set_deleted(deleted)
    resident = st.search_batch(queries, 10)
    check_all(resident, want, full, f"{what} deleted (resident)")
    for a, b in zip(per_call, resident):
        assert np.array_equal(a, b)
    st.set_deleted(None)
    # id lists, at the query counts that pick different kernels
    lists = {m: rng.choice(n, m, replace=False).astype(np.uint32) for m in (500, 80_000) if m <= n}
    for m, ids in lists.items():
        for nq in (1, 2, 10):
            sub = [k.scores(q, ids) for q in queries[:nq]]
            got = st.search_batch(queries[:nq], 10, id_list=ids)
            check_all(got, [oracle.topk(s, 10, ids) for s in sub], full, f"{what} id list {m} nq={nq}")
    # a top larger than the id list: exactly the live listed rows come back
    ids = lists[500]
    live_ids = ids[~deleted[ids]]
    for g, s in zip(st.search_batch(queries[:2], 600, point_deleted=deleted, id_list=ids), full):
        assert sorted(g["idx"].tolist()) == sorted(live_ids.tolist())
        assert_topk_equal(g, oracle.topk(s[live_ids], 600, live_ids), s, f"{what} top > id list")
    # id_base: search, id lists, score_points and rescore report and take global ids
    base_id = 6_250_000
    set_id_base(st, base_id)
    check_all(shifted(st.search_batch(queries[:3], 10), -base_id), [oracle.topk(s, 10) for s in full[:3]], full, f"{what} id_base")
    got = st.search_batch(queries[:3], 10, id_list=ids + base_id, point_deleted=deleted)
    check_all(shifted(got, -base_id), [oracle.topk(s[live_ids], 10, live_ids) for s in full[:3]], full, f"{what} id_base id list")
    sc = st.raw_scorer(queries[0])
    np.testing.assert_array_equal(sc.score_points(ids + base_id).view(np.uint32), full[0][ids].view(np.uint32))
    with pytest.raises(qb.QbError):
        sc.score_points(np.array([n - 1], np.uint32))      # a local id is out of range now
    if k.kind == "bq":       # BQ candidates are always rescored with the original vectors: its scorer refuses to rescore
        from qdrant_b200._capi import QB_ERR_UNSUPPORTED

        with pytest.raises(qb.QbError) as ei:
            qb.rescore(sc, ids + base_id, 10)
        assert ei.value.status == QB_ERR_UNSUPPORTED
    else:
        res = qb.rescore(sc, ids + base_id, 10)
        order = np.lexsort((ids, -full[0][ids].astype(np.float64)))[:10]
        np.testing.assert_array_equal(res["idx"], ids[order] + base_id)
        np.testing.assert_array_equal(res["score"].view(np.uint32), full[0][ids[order]].view(np.uint32))
    sc.close(); st.close()


@pytest.mark.parametrize("spec", SPECS, ids=spec_id)
def test_search_batch_device(qb, oracle, spec):
    """qb_search_batch_device at 1 and 40 queries (SQ8: the tensor-core path with its flag loop) == the host search == the oracle."""
    rng = np.random.default_rng(spec[2] + 77)
    n = 100_003
    base, queries = data(oracle, qb, spec[1], n, spec[2], rng, 40)
    k = Quant(qb, oracle, spec, base, rng)
    st = k.storage()
    for nq, top in ((1, 20), (40, 20)):
        got = device_search(st, queries[:nq], top)
        host = st.search_batch(queries[:nq], top)
        for g, h in zip(got, host):
            assert np.array_equal(g, h)
        full = [k.scores(q) for q in queries[:nq]]
        check_all(got, [oracle.topk(s, top) for s in full], full, f"{spec_id(spec)} device nq={nq}")
    st.close()


def test_sq8_device_flag_loop_on_mass_ties(qb, oracle):
    """Every row identical: the tensor-core path's candidate lists overflow; qb_search_batch_device must rerun like the host search
    until the answer is exact: ids 0..top-1 in order, all with the one score.  Then the ten best rows are the last ten."""
    rng = np.random.default_rng(12)
    n = 70_001
    base = np.tile(rng.standard_normal((1, 64)).astype(np.float32), (n, 1))
    queries = rng.standard_normal((40, 64)).astype(np.float32)
    sq = oracle.SQ8.encode(base, oracle.QD_DOT, False)
    st = qb.ScalarQuantizedVectors(sq.rows, 64, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, qb.Distance.Dot)
    st.search_stats(reset=True)
    got = device_search(st, queries, 10)
    assert st.search_stats()[1] >= 1, "the filter pass should have overflowed and rerun"
    for g, q in zip(got, queries):
        code, off = sq.encode_query(q)
        assert g["idx"].tolist() == list(range(10)) and np.all(g["score"] == sq.score(code, off, 0))
    for g, h in zip(got, st.search_batch(queries, 10)):
        assert np.array_equal(g, h)
    st.close()
    # the same ties, but the ten best rows are the last ones: an overflowed first attempt has dropped them, only the rerun finds them
    base[-10:] += np.float32(2.0)
    queries = np.abs(queries)                              # every query prefers the shifted rows
    sq = oracle.SQ8.encode(base, oracle.QD_DOT, False)
    st = qb.ScalarQuantizedVectors(sq.rows, 64, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, qb.Distance.Dot)
    st.search_stats(reset=True)
    got = device_search(st, queries, 10)
    assert st.search_stats()[1] >= 1, "the filter pass should have overflowed and rerun"
    for g, q in zip(got, queries):
        code, off = sq.encode_query(q)
        assert sq.score(code, off, n - 1) > sq.score(code, off, 0)
        assert g["idx"].tolist() == list(range(n - 10, n)) and np.all(g["score"] == sq.score(code, off, n - 1))
    for g, h in zip(got, st.search_batch(queries, 10)):
        assert np.array_equal(g, h)
    st.close()


# ------------------------------------------------------------------------------------------------ oversampling + rescoring
@pytest.mark.parametrize("name", ["sq8-Cosine", "pq-Dot", "bq-Euclid-TwoBits-Scalar8bits"])
def test_oversampled_top_and_rescore(qb, oracle, name):
    """get_oversampled_top(1000, True, 5.0) = 5000 candidates (qb_select_large_kernel), then postprocess_search_result rescoring them
    with the f32 originals: exact f32 scores in (score desc, id asc) order."""
    sp = spec(name)
    rng = np.random.default_rng(31)
    n = 150_001
    base, queries = data(oracle, qb, sp[1], n, sp[2], rng, 3)
    k = Quant(qb, oracle, sp, base, rng)
    st = k.storage()
    orig = qb.DenseVectorStorage(base, k.d)
    top = qb.get_oversampled_top(1000, True, 5.0)
    assert top == 5000
    got = st.search_batch(queries, top)
    full = [k.scores(q) for q in queries]
    check_all(got, [oracle.topk(s, top) for s in full], full, f"{name} top {top}")
    for q, cand in zip(queries, got):
        exact = oracle.score_points_f32(int(k.d), base, oracle.preprocess_f32(int(k.d), q), cand["idx"])
        order = np.lexsort((cand["idx"], -exact.astype(np.float64)))[:1000]
        res = qb.postprocess_search_result(cand, orig, q, 1000, rescore=True)
        np.testing.assert_array_equal(res["idx"], cand["idx"][order])
        np.testing.assert_array_equal(res["score"].view(np.uint32), exact[order].view(np.uint32))
    st.close(); orig.close()


# ------------------------------------------------------------------------------------------------ three-level plan (C3)
N3, DIM3 = 1_100_001, 64          # >= 2^20 rows: sample S1 -> level 2 (S2 = 1.5 sqrt(N S1) rows, <= N/4) -> full pass


@pytest.fixture(scope="module")
def sq8_large(oracle):
    rng = np.random.default_rng(2024)
    base = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((N3, DIM3)).astype(np.float32))
    sq = oracle.SQ8.encode(base, oracle.QD_DOT, False)
    return sq, rng.standard_normal((160, DIM3)).astype(np.float32)


def large_search(qb, oracle, sq, queries, top, deleted, base_id, what, rerun_ok):
    """tensor cores == the CUDA-core path bit for bit for every query, == the oracle's scan for the first 16; returns the reruns"""
    st = qb.ScalarQuantizedVectors(sq.rows, DIM3, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, qb.Distance.Cosine)
    set_id_base(st, base_id)
    st.search_stats(reset=True)
    got = st.search_batch(queries, top, point_deleted=deleted)
    searches, reruns = st.search_stats(reset=True)
    assert searches == 1
    if not rerun_ok:
        assert reruns == 0, f"{what}: the three-level plan should not rerun ({reruns})"
    cc = with_option(qb, "disable_mma", 1, lambda: st.search_batch(queries, top, point_deleted=deleted))
    for i in range(len(queries)):
        assert np.array_equal(got[i], cc[i]), f"{what}: query {i} differs from the CUDA-core path"
    enc = [sq.encode_query(oracle.preprocess_f32(oracle.COSINE, q)) for q in queries[:16]]
    codes, offs = np.stack([e[0] for e in enc]), np.array([e[1] for e in enc], np.float32)
    want = sq.scan(codes, offs, top, deleted=pack_bitmap(deleted))
    full = [sq.score_rows(c, o) for c, o in enc]
    check_all(shifted(got[:16], -base_id), want, full, what)
    st.close()
    return reruns


@pytest.mark.parametrize("nq", [64, 160])
def test_sq8_three_level_plan(qb, oracle, sq8_large, nq):
    """C3's plan: several query blocks at nq = 160, id_base, 3 % per-call deletions.  At top 5000 the per-(query, CTA) segments (256
    slots at most) may overflow by design, so the rerun count is reported there, not asserted."""
    sq, queries = sq8_large
    deleted = np.random.default_rng(nq).random(N3) < 0.03
    large_search(qb, oracle, sq, queries[:nq], 10, deleted, 3_000_000, f"three-level nq={nq} top=10", rerun_ok=False)
    r = large_search(qb, oracle, sq, queries[:nq], 5000, deleted, 3_000_000, f"three-level nq={nq} top=5000", rerun_ok=True)
    print(f"three-level nq={nq} top=5000: {r} rerun(s)")


@pytest.mark.parametrize("case", ["prefix_deleted", "prefix_top_minus_one"])
def test_sq8_three_level_deleted_prefix(qb, oracle, sq8_large, case):
    """The first 300 000 rows deleted (they cover S1 and S2 for any top), or all but top - 1 of them: still exact.  Whether the search
    reruns is reported, not assumed."""
    sq, queries = sq8_large
    rng = np.random.default_rng(5)
    for top in (10, 5000):
        deleted = np.zeros(N3, bool)
        deleted[:300_000] = True
        if case == "prefix_top_minus_one":
            deleted[rng.choice(300_000, top - 1, replace=False)] = False
        r = large_search(qb, oracle, sq, queries[:64], top, deleted, 0, f"{case} top={top}", rerun_ok=True)
        print(f"{case} top={top}: {r} rerun(s)")


def test_sq8_three_level_overflowing_level_two(qb, oracle):
    """Rows of the level-1 sample are much shorter than the rest, so its threshold admits about half of the level-2 prefix: the level-2
    candidate list overflows, the search must report the rerun, and the answer stays exact."""
    rng = np.random.default_rng(77)
    base = rng.standard_normal((N3, DIM3)).astype(np.float32)
    base[:8192] *= np.float32(0.05)
    sq = oracle.SQ8.encode(base, oracle.QD_DOT, False)
    del base
    queries = rng.standard_normal((64, DIM3)).astype(np.float32)
    st = qb.ScalarQuantizedVectors(sq.rows, DIM3, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, qb.Distance.Dot)
    st.search_stats(reset=True)
    got = st.search_batch(queries, 10)
    assert st.search_stats(reset=True)[1] >= 1, "the level-2 candidate list should have overflowed and rerun"
    got_dev = device_search(st, queries, 10)
    cc = with_option(qb, "disable_mma", 1, lambda: st.search_batch(queries, 10))
    enc = [sq.encode_query(q) for q in queries[:16]]
    want = sq.scan(np.stack([e[0] for e in enc]), np.array([e[1] for e in enc], np.float32), 10)
    full = [sq.score_rows(c, o) for c, o in enc]
    check_all(got[:16], want, full, "level-2 overflow")
    for i in range(len(queries)):
        assert np.array_equal(got[i], cc[i]) and np.array_equal(got[i], got_dev[i]), f"level-2 overflow: query {i}"
    st.close()


# ------------------------------------------------------------------------------------------------ PQ as a C4 shard
@pytest.mark.parametrize("qpp,nq", [(0, 12), (16, 12), (8, 7)])
def test_pq_shard_prefilter_kernels(qb, oracle, qpp, nq):
    """pq_scan16_kernel (nq >= 9) and pq_scan8_kernel on a shard: id_base 6 250 000 (the survivors' keys carry global ids and
    pq_rescore_kernel subtracts it again to find the codes) and resident deletions == the oracle == one query per pass."""
    rng = np.random.default_rng(qpp + nq)
    n, dim, chunk, base_id = 150_000, 128, 4, 6_250_000
    base, queries = data(oracle, qb, "Dot", n, dim, rng, nq)
    k = Quant(qb, oracle, ("pq", "Dot", dim, chunk), base, rng)
    st = k.storage()
    set_id_base(st, base_id)
    deleted = rng.random(n) < 0.05
    st.set_deleted(deleted)
    live = np.flatnonzero(~deleted).astype(np.uint32)
    full = [k.scores(q) for q in queries]
    st.search_stats(reset=True)
    got = with_option(qb, "pq_queries_per_pass", qpp, lambda: st.search_batch(queries, 10))
    assert st.search_stats(reset=True)[1] == 0
    one = with_option(qb, "pq_queries_per_pass", 1, lambda: st.search_batch(queries, 10))
    check_all(shifted(got, -base_id), [oracle.topk(s[live], 10, live) for s in full], full, f"pq shard qpp={qpp}")
    for a, b in zip(got, one):
        assert np.array_equal(a, b)
    st.close()


# ------------------------------------------------------------------------------------------------ mass ties
def test_bq_mass_ties(qb, oracle):
    """Ten distinct rows repeated to 200 000: every score value occurs 20 000 times, more than the filter pass's candidate buffer.
    The search must rerun and answer in (score desc, id asc) order."""
    rng = np.random.default_rng(12)
    n, dim = 200_000, 100
    distinct = rng.standard_normal((10, dim)).astype(np.float32)
    base = np.ascontiguousarray(distinct[np.arange(n) % 10])
    k = Quant(qb, oracle, spec("bq-Dot-OneBit-SameAsStorage"), base, rng)
    st = k.storage()
    queries = rng.standard_normal((3, dim)).astype(np.float32)
    st.search_stats(reset=True)
    for top in (10, 100):
        for g, q in zip(st.search_batch(queries, top), queries):
            s = k.scores(q)
            order = np.lexsort((np.arange(n), -s.astype(np.float64)))[:top]
            assert np.array_equal(g["idx"], order.astype(np.uint32)) and np.array_equal(g["score"].view(np.uint32), s[order].view(np.uint32))
            assert_topk_equal(g, oracle.topk(s, top), s, f"bq ties top {top}")
    assert st.search_stats()[1] >= 1, "the filter pass should have overflowed and rerun"
    st.close()


# ------------------------------------------------------------------------------------------------ non-finite SQ8 metadata
@pytest.mark.parametrize("dist", ["Dot", "Euclid"])
def test_sq8_nonfinite_metadata(qb, oracle, dist):
    """Rows holding +inf: alpha is inf, every row and query offset is 0 * inf = NaN, every score NaN.  One query, a batch of 40 (wide
    enough for the tensor cores, whose filter would drop NaN scores: the planner keeps such storages on the CUDA cores), the same batch
    through qb_search_batch_device and with the tensor cores disabled all return `top` NaN scores at ids 0..top-1, as the oracle does
    (NaN is the greatest score and all of them tie)."""
    rng = np.random.default_rng(8)
    n, dim, top = 70_001, 32, 10
    base = rng.standard_normal((n, dim)).astype(np.float32)
    base[rng.choice(n, 50, replace=False), rng.integers(0, dim, 50)] = np.inf
    d = getattr(qb.Distance, dist)
    dt, inv = qb.construct_vector_parameters(d)
    sq = oracle.SQ8.encode(base, int(dt), bool(inv))
    assert np.isinf(sq.meta.alpha)
    st = qb.ScalarQuantizedVectors(sq.rows, dim, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, d)
    queries = rng.standard_normal((40, dim)).astype(np.float32)
    code, off = sq.encode_query(queries[0])
    assert np.isnan(sq.score_rows(code, off)).all()
    want = sq.scan(code, off, top)[0]
    assert np.isnan(want["score"]).all() and sorted(want["idx"].tolist()) == list(range(top))
    runs = {"nq=1": lambda: st.search_batch(queries[:1], top),
            "nq=40": lambda: st.search_batch(queries, top),
            "nq=40 device": lambda: device_search(st, queries, top),
            "nq=40 disable_mma": lambda: with_option(qb, "disable_mma", 1, lambda: st.search_batch(queries, top))}
    for what, run in runs.items():
        for i, g in enumerate(run()):
            assert g["idx"].tolist() == list(range(top)) and np.isnan(g["score"]).all(), f"{dist} {what} q{i}: {g[:4]}"
    st.close()
