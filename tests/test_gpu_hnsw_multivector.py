"""GPU parity: the device HNSW search over a graph of multivector points (qb_hnsw_create_*_multivector + qb_hnsw_search_maxsim_batch)
against the CPU traversal driven by the oracle's MaxSim (tests/hnsw_maxsim_ref.py through the keyed checker of tests/hnsw_custom_ref.py):
the same lists (score bits included), hops, scored points and counters, and every score equal to qb_score_maxsim on its point."""
import numpy as np
import pytest

from tests import graph_links_compressed as gc
from tests import hnsw_custom_ref as cr
from tests import hnsw_maxsim_ref as mr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


class _Case:
    """a multivector collection (dense f32 or SQ8 tokens), its view and an oracle-built graph over the points' normalised mean tokens"""

    def __init__(self, qb, oracle, dist, dim, n_points, lens=(1, 12), m=16, sq8=False, seed=1, empty=0.0):
        self.qb, self.oracle = qb, oracle
        self.d = getattr(qb.Distance, dist)
        self.dim, self.n = dim, n_points
        rng = self.rng = np.random.default_rng(seed)
        runs = rng.integers(lens[0], lens[1] + 1, n_points)
        runs[rng.random(n_points) < empty] = 0
        self.off = np.concatenate([[0], np.cumsum(runs)]).astype(np.uint32)
        centers = rng.standard_normal((max(n_points // 8, 1), dim)).astype(np.float32)
        raw = (centers[np.repeat(rng.integers(0, centers.shape[0], n_points), runs)] + 0.5 * rng.standard_normal((int(self.off[-1]), dim))).astype(np.float32)
        self.rows = oracle.preprocess_rows_f32(int(self.d), raw)
        self.sq = None
        if sq8:
            dt, inv = qb.construct_vector_parameters(self.d)
            self.sq = oracle.SQ8.encode(self.rows, int(dt), bool(inv))
            self.st = qb.ScalarQuantizedVectors(self.sq.rows, dim, self.sq.meta.alpha, self.sq.meta.offset, self.sq.meta.multiplier, self.d)
        else:
            self.st = qb.DenseVectorStorage(self.rows, self.d)
        self.view = qb.MultiVectorView(self.st, self.off)
        means = np.stack([self.rows[self.off[p] : self.off[p + 1]].mean(0) if runs[p] else rng.standard_normal(dim) for p in range(n_points)])
        self.g = oracle.HNSW(oracle.preprocess_rows_f32(oracle.COSINE, means.astype(np.float32)), oracle.COSINE, m=m, ef_construct=64, seed=seed)
        self.entry, self.lvl, self.m, self.m0 = self.g.entry()
        self.blob = self.g.export_plain()
        self.cg = cr.Graph(self.blob, self.m, self.m0, n_points)
        self.units = dim if sq8 else dim * 4

    def queries(self, counts):
        return [self.rng.standard_normal((int(c), self.dim)).astype(np.float32) for c in counts]

    def scores(self, query):
        if self.sq is not None:
            return mr.point_scores_sq8(self.oracle, self.sq, int(self.d), self.off, query)
        return mr.point_scores_f32(self.oracle, int(self.d), self.rows, self.off, query)

    def check(self, hg, queries, top, ef, algorithm="hnsw", filtered=None):
        """device == checker: lists, hops, scored points, counters; every score == qb_score_maxsim"""
        algo = cr.ACORN if algorithm == "acorn" else cr.HNSW
        runs = np.diff(self.off).astype(np.uint64)
        want, cpu = [], 0
        self.cg.stats(reset=True)
        for q in queries:
            sc = self.scores(q)
            seen = []

            def cb(ids, sc=sc, seen=seen):
                seen.append(ids.copy())
                return sc[ids.astype(np.int64)]

            want.append(cr.search_cb(self.cg, cb, top, ef, self.entry, self.lvl, algo, filtered, keyed=True))
            cpu += int(runs[np.concatenate(seen).astype(np.int64)].sum()) * q.shape[0] * self.units
        want_stats = self.cg.stats()[:2]
        hg.stats(reset=True)
        c = self.qb.HwCounters()
        got = hg.search_maxsim(queries, top, ef, self.entry, self.lvl, point_deleted=filtered, counters=c, algorithm=algorithm)
        assert hg.stats() == want_stats
        assert c.cpu == cpu and c.vector_io_read == 0
        for i, (g, w) in enumerate(zip(got, want)):
            assert np.array_equal(g["idx"], w["idx"]) and np.array_equal(g["score"].view(np.uint32), w["score"].view(np.uint32)), (i, g, w)
            if g.size:
                direct = self.view.score_points(queries[i], g["idx"])
                assert np.array_equal(direct.view(np.uint32), g["score"].view(np.uint32)), i
        return got

    def close(self):
        self.st.close()


def _lists_equal(a, b):
    return all(np.array_equal(x["idx"], y["idx"]) and np.array_equal(x["score"].view(np.uint32), y["score"].view(np.uint32)) for x, y in zip(a, b))


@pytest.mark.parametrize("dist", ["Cosine", "Dot", "Euclid", "Manhattan"])
@pytest.mark.parametrize("dim", [8, 24, 48, 128])
def test_dense_f32_matches_checker(qb, oracle, dist, dim):
    c = _Case(qb, oracle, dist, dim, 500, seed=dim)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    qs = c.queries([1, 3, 32, 9, 1, 17])
    first = c.check(hg, qs, 10, 48)
    # a second identical batch: the visited state was cleaned
    assert _lists_equal(hg.search_maxsim(qs, 10, 48, c.entry, c.lvl), first)
    hg.close()
    c.close()


def test_dense_f32_768(qb, oracle):
    c = _Case(qb, oracle, "Cosine", 768, 300, lens=(1, 20), seed=768)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    c.check(hg, c.queries([1, 32, 5]), 10, 32)
    c.check(hg, c.queries([4, 2]), 5, 16, "acorn", c.rng.random(c.n) >= 0.3)
    hg.close()
    c.close()


@pytest.mark.parametrize("dist,dim", [("Dot", 64), ("Cosine", 96), ("Euclid", 64), ("Manhattan", 48), ("Dot", 1056)])
def test_sq8_matches_checker(qb, oracle, dist, dim):
    """dim 1056: actual_dim * 127^2 >= 2^24, the lane-exact SQ8 chain"""
    c = _Case(qb, oracle, dist, dim, 400, lens=(1, 10), sq8=True, seed=dim + 1)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    c.check(hg, c.queries([1, 32, 6]), 10, 32)
    c.check(hg, c.queries([3, 8]), 10, 32, "acorn", c.rng.random(c.n) >= 0.2)
    hg.close()
    c.close()


@pytest.mark.parametrize("algorithm", ["hnsw", "acorn"])
@pytest.mark.parametrize("sel", [0.01, 0.1, 0.5, 1.0])
def test_filters(qb, oracle, algorithm, sel):
    c = _Case(qb, oracle, "Dot", 64, 1500, lens=(1, 8), seed=int(sel * 100) + 7)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    for _ in range(2):   # a different filter per call
        filtered = c.rng.random(c.n) >= sel
        filtered[c.entry] = False
        got = c.check(hg, c.queries([2, 7, 1]), 10, 64, algorithm, filtered if sel < 1.0 else None)
        assert all(not filtered[g["idx"]].any() for g in got)
    hg.close()
    c.close()


@pytest.mark.parametrize("m", [4, 16, 32])
def test_loaders_and_m0(qb, oracle, m):
    """plain and compressed links.bin at m0 = 8 / 32 / 64: the same handle, the same results"""
    c = _Case(qb, oracle, "Euclid", 40, 700, lens=(1, 6), m=m, seed=m)
    assert c.m0 == 2 * m
    plain = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    comp = qb.HnswGraph.from_compressed_multivector(c.view, gc.plain_to_compressed(c.blob, c.m, c.m0))
    qs = c.queries([1, 5, 32])
    a = c.check(plain, qs, 10, 40)
    b = c.check(comp, qs, 10, 40, "acorn")
    assert len(a) == len(b)
    # the compressed format stores each list's first links sorted, so the two handles hold the same sets in their files' orders
    ids = np.arange(0, c.n, 97, dtype=np.uint32)
    assert all(np.array_equal(np.sort(x), np.sort(y)) for x, y in zip(comp.links(0, ids), plain.links(0, ids)))
    for h in (plain, comp):
        n, levels, hbm = h.info()
        assert n == c.n and hbm > 4 * (c.n + 1)
        again = qb.HnswGraph.multivector(c.view, h.export_plain(), c.m, c.m0)
        assert np.array_equal(again.export_plain(), h.export_plain())
        again.close()
    plain.close()
    comp.close()
    c.close()


def test_ef_extremes_and_top_above_ef(qb, oracle):
    c = _Case(qb, oracle, "Cosine", 32, 900, lens=(1, 5), seed=11)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    c.check(hg, c.queries([3, 1]), 1, 1)
    c.check(hg, c.queries([3, 1]), 10, 1)          # top > ef: max(ef, top)
    got = c.check(hg, c.queries([2, 30]), 20, 4096)
    assert all(g.size == 20 for g in got)
    c.check(hg, c.queries([2]), 5, 4096, "acorn", c.rng.random(c.n) >= 0.5)
    hg.close()
    c.close()


def test_many_query_vectors(qb, oracle):
    """a query beyond the shared-memory staging (read from HBM), up to 4096 vectors"""
    c = _Case(qb, oracle, "Dot", 128, 300, lens=(1, 6), seed=13)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    c.check(hg, c.queries([200, 1, 96, 97]), 10, 32)
    c.check(hg, c.queries([4096]), 5, 16)
    hg.close()
    c.close()
    s = _Case(qb, oracle, "Euclid", 8, 200, lens=(1, 4), seed=14)
    hg = qb.HnswGraph.multivector(s.view, s.blob, s.m, s.m0)
    s.check(hg, s.queries([4096, 3]), 5, 16, "acorn")
    hg.close()
    s.close()


@pytest.mark.parametrize("sq8", [False, True])
def test_token_runs_0_1_300(qb, oracle, sq8):
    """empty points score -inf (ties ordered by id), one-token points, and 300-token points (several batches of items); top = ef = the
    point count, so every point the search reaches is listed, the empty ones included"""
    c = _Case(qb, oracle, "Dot", 64, 300, lens=(0, 1), sq8=sq8, seed=17 + sq8, empty=0.2)
    long = c.rng.random(c.n) < 0.1
    runs = np.diff(c.off)
    runs[long] = 300
    c.off = np.concatenate([[0], np.cumsum(runs)]).astype(np.uint32)
    rows = oracle.preprocess_rows_f32(int(c.d), c.rng.standard_normal((int(c.off[-1]), c.dim)).astype(np.float32))
    c.st.close()
    c.rows = rows
    if sq8:
        dt, inv = qb.construct_vector_parameters(c.d)
        c.sq = oracle.SQ8.encode(rows, int(dt), bool(inv))
        c.st = qb.ScalarQuantizedVectors(c.sq.rows, c.dim, c.sq.meta.alpha, c.sq.meta.offset, c.sq.meta.multiplier, c.d)
    else:
        c.st = qb.DenseVectorStorage(rows, c.d)
    c.view = qb.MultiVectorView(c.st, c.off)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    got = c.check(hg, c.queries([1, 9, 32]), 300, 300)
    assert all(np.isneginf(g["score"]).sum() == (np.diff(c.off)[g["idx"]] == 0).sum() > 0 for g in got)
    hg.close()
    c.close()


def test_wide_mixed_batch(qb, oracle):
    """more queries than resident CTAs, with mixed vector counts"""
    c = _Case(qb, oracle, "Cosine", 32, 400, lens=(1, 6), seed=19)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    c.check(hg, c.queries(c.rng.integers(1, 41, 3000)), 10, 24)
    hg.close()
    c.close()


def test_device_entry(qb, oracle):
    import torch
    from qdrant_b200._capi import lib

    c = _Case(qb, oracle, "Dot", 64, 600, lens=(1, 8), seed=23)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    qs = c.queries([1, 32, 5, 12])
    want = hg.search_maxsim(qs, 10, 32, c.entry, c.lvl)
    off = np.concatenate([[0], np.cumsum([q.shape[0] for q in qs])]).astype(np.int32)
    dq = torch.from_numpy(np.concatenate(qs)).cuda()
    doff = torch.from_numpy(off).cuda()
    dout = torch.zeros((len(qs), 10, 2), dtype=torch.int32, device="cuda")
    dcnt = torch.zeros(len(qs), dtype=torch.int32, device="cuda")
    for algo in (0, 1):
        qb.check(lib().qb_hnsw_search_maxsim_batch_device(hg._h, dq.data_ptr(), dq.shape[0], doff.data_ptr(), len(qs), 32, 10, 32, c.entry, c.lvl,
                                                          dout.data_ptr(), dcnt.data_ptr(), algo))
        torch.cuda.synchronize()
        out = dout.cpu().numpy().view(np.uint32)
        cnt = dcnt.cpu().numpy()
        ref = want if algo == 0 else hg.search_maxsim(qs, 10, 32, c.entry, c.lvl, algorithm="acorn")
        for i, w in enumerate(ref):
            assert cnt[i] == w.size
            assert np.array_equal(out[i, : cnt[i], 0], w["idx"]) and np.array_equal(out[i, : cnt[i], 1], w["score"].view(np.uint32))
    hg.close()
    c.close()


def test_errors_leave_the_device_usable(qb, oracle):
    from qdrant_b200 import _capi

    c = _Case(qb, oracle, "Dot", 32, 300, lens=(1, 5), seed=29)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    qs = c.queries([3, 1])
    base = hg.search_maxsim(qs, 10, 32, c.entry, c.lvl)

    def status(f):
        with pytest.raises(qb.QbError) as ei:
            f()
        assert _lists_equal(hg.search_maxsim(qs, 10, 32, c.entry, c.lvl), base)
        return ei.value.status

    U, INV = _capi.QB_ERR_UNSUPPORTED, _capi.QB_ERR_INVALID
    # single-vector searches on a multivector handle
    assert status(lambda: hg.search(np.ones((1, 32), np.float32), 5, 16, c.entry, c.lvl)) == U
    assert status(lambda: hg.search(np.ones((1, 32), np.float32), 5, 16, c.entry, c.lvl, algorithm="acorn")) == U
    assert status(lambda: hg.search_custom(qb.QueryKind.RecommendBestScore, np.ones((1, 2, 32), np.float32), 1, 1, top=5, ef=16,
                                           entry_point=c.entry, entry_level=c.lvl)) == U
    assert status(lambda: hg.search_discover(np.ones((1, 3, 32), np.float32), 1, top=5, ef=16, entry_point=c.entry, entry_level=c.lvl)) == U
    assert status(lambda: hg.search_with_vectors(np.ones((1, 32), np.float32), 5, 16, c.entry, c.lvl)) == U
    # MaxSim search on a regular handle
    reg_st = qb.DenseVectorStorage(c.rows[: c.n], c.d)
    reg = qb.HnswGraph(reg_st, c.blob, c.m, c.m0)
    assert status(lambda: reg.search_maxsim(qs, 5, 16, c.entry, c.lvl)) == U
    reg.close()
    reg_st.close()
    # query shapes, ef
    assert status(lambda: hg.search_maxsim([np.zeros((0, 32), np.float32)], 5, 16, c.entry, c.lvl)) == INV
    assert status(lambda: hg.search_maxsim(c.queries([4097]), 5, 16, c.entry, c.lvl)) == INV
    assert status(lambda: hg.search_maxsim(qs, 5, 4097, c.entry, c.lvl)) == U
    assert status(lambda: hg.search_maxsim(qs, 5, 16, c.n, 0)) == INV
    # loaders
    bad = c.off.copy()
    bad[5], bad[6] = bad[6], bad[5] - 1
    assert status(lambda: qb.HnswGraph.multivector(qb.MultiVectorView(c.st, bad), c.blob, c.m, c.m0)) == INV
    over = c.off.copy()
    over[-1] = c.st.count + 1
    assert status(lambda: qb.HnswGraph.multivector(qb.MultiVectorView(c.st, over), c.blob, c.m, c.m0)) == INV
    assert status(lambda: qb.HnswGraph.multivector(qb.MultiVectorView(c.st, c.off[:-1]), c.blob, c.m, c.m0)) == INV   # point count
    comp = bytearray(gc.plain_to_compressed(c.blob, c.m, c.m0))
    comp[8:16] = (0xFFFFFFFFFFFFFF02).to_bytes(8, "little")
    assert status(lambda: qb.HnswGraph.from_compressed_multivector(c.view, bytes(comp))) == U
    f16 = qb.DenseVectorStorage(c.rows.astype(np.float16), c.d, qb.VectorStorageDatatype.Float16)
    assert status(lambda: qb.HnswGraph.multivector(qb.MultiVectorView(f16, c.off), c.blob, c.m, c.m0)) == U
    f16.close()
    hg.close()
    c.close()
