"""GPU parity: custom queries with multivector examples through the device HNSW traversal of a graph over multivector points
(qb_hnsw_search_maxsim_custom_batch / qb_hnsw_search_maxsim_discover_batch) against the keyed CPU checker driven by the oracle's MaxSim per
example folded by its Query::score_by (tests/hnsw_maxsim_custom_ref.py): the same lists (score bits included), hops, scored points and
counters, and every score equal to qb_score_maxsim_custom on its point."""
import ctypes as C

import numpy as np
import pytest

from tests import graph_links_compressed as gc
from tests import hnsw_custom_ref as cr
from tests import hnsw_maxsim_custom_ref as mc

pytestmark = pytest.mark.gpu

RECO_BEST, RECO_SUM, DISCOVER, CONTEXT, FEEDBACK = 1, 2, 3, 4, 5


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


class _Case:
    """a multivector collection (dense f32 or SQ8 tokens), its view and an oracle-built graph over the points' normalised mean tokens"""

    def __init__(self, qb, oracle, dist, dim, n_points, lens=(1, 12), m=16, sq8=False, seed=1, empty=0.0, long=0.0):
        self.qb, self.oracle = qb, oracle
        self.d = getattr(qb.Distance, dist)
        self.dim, self.n = dim, n_points
        rng = self.rng = np.random.default_rng(seed)
        runs = rng.integers(lens[0], lens[1] + 1, n_points)
        runs[rng.random(n_points) < empty] = 0
        runs[rng.random(n_points) < long] = 300
        self.off = np.concatenate([[0], np.cumsum(runs)]).astype(np.uint32)
        centers = rng.standard_normal((max(n_points // 8, 1), dim)).astype(np.float32)
        raw = (centers[np.repeat(rng.integers(0, centers.shape[0], n_points), runs)] + 0.5 * rng.standard_normal((int(self.off[-1]), dim))).astype(np.float32)
        self.rows = oracle.preprocess_rows_f32(int(self.d), raw)
        self.sq = None
        if sq8:
            dt, inv = qb.construct_vector_parameters(self.d)
            self.sq = oracle.SQ8.encode(self.rows, int(dt), bool(inv))
            self.st = qb.ScalarQuantizedVectors(self.sq.rows, dim, self.sq.meta.alpha, self.sq.meta.offset, self.sq.meta.multiplier, self.d)
            self.pe = mc.per_example_sq8(oracle, self.sq, int(self.d), self.off)
        else:
            self.st = qb.DenseVectorStorage(self.rows, self.d)
            self.pe = mc.per_example_f32(oracle, int(self.d), self.rows, self.off)
        self.view = qb.MultiVectorView(self.st, self.off)
        means = np.stack([self.rows[self.off[p] : self.off[p + 1]].mean(0) if runs[p] else rng.standard_normal(dim) for p in range(n_points)])
        self.g = oracle.HNSW(oracle.preprocess_rows_f32(oracle.COSINE, means.astype(np.float32)), oracle.COSINE, m=m, ef_construct=64, seed=seed)
        self.entry, self.lvl, self.m, self.m0 = self.g.entry()
        self.blob = self.g.export_plain()
        self.cg = cr.Graph(self.blob, self.m, self.m0, n_points)
        self.units = dim if sq8 else dim * 4
        self.io = 0

    def ex(self, lens=(1, 6)):
        return self.rng.standard_normal((int(self.rng.integers(lens[0], lens[1] + 1)), self.dim)).astype(np.float32)

    def query(self, kind, n_a, n_b=0, lens=(1, 6)):
        """one query object of this kind and shape with [vectors, dim] examples"""
        qb, ex = self.qb, lambda: self.ex(lens)
        pairs = lambda: [qb.ContextPair(ex(), ex()) for _ in range(n_a)]   # noqa: E731
        if kind in (RECO_BEST, RECO_SUM):
            r = qb.RecoQuery([ex() for _ in range(n_a)], [ex() for _ in range(n_b)])
            return qb.RecoBestScoreQuery(r) if kind == RECO_BEST else qb.RecoSumScoresQuery(r)
        if kind == CONTEXT:
            return qb.ContextQuery(pairs())
        if kind == DISCOVER:
            return qb.DiscoverQuery(ex(), pairs())
        return qb.FeedbackQuery(ex(), pairs(), self.rng.standard_normal(n_a).astype(np.float32), 0.75)

    def queries(self, kind, n_a, n_b=0, nq=3, lens=(1, 6)):
        return [self.query(kind, n_a, n_b, lens) for _ in range(nq)]

    def want(self, q, top, ef, algo, filtered, cep, fused):
        """the checker's list and its cpu units for one query"""
        examples, n_a, n_b = q.flat()
        runs = np.diff(self.off).astype(np.uint64)
        total = lambda exs: sum(e.shape[0] for e in exs)   # noqa: E731
        if fused:
            got, (s1, s2) = mc.discover(self.cg, self.oracle, self.pe, examples, n_a, top, ef, self.entry, self.lvl, algo, filtered)
            rows = [(s1, total(examples[1:])), (s2, total(examples))]
        else:
            coef = np.concatenate([[q.a], q.partial]).astype(np.float32) if int(q.kind) == FEEDBACK else None
            got, sc = mc.search(self.cg, self.oracle, self.pe, int(q.kind), n_a, n_b, examples, top, ef, self.entry, self.lvl, algo, filtered, coef, cep)
            rows = [(sc, total(examples))]
        cpu = sum(int(runs[s.points()].sum()) * v for s, v in rows)
        io = sum(int(runs[s.points()].sum()) for s, _ in rows)
        return got, cpu, io

    def check(self, hg, queries, top, ef, algorithm="hnsw", filtered=None, cep=None, fused=False):
        """device == checker: lists, hops, scored points, counters; every score == qb_score_maxsim_custom"""
        algo = cr.ACORN if algorithm == "acorn" else cr.HNSW
        want, cpu, io = [], 0, 0
        self.cg.stats(reset=True)
        for i, q in enumerate(queries):
            w, c, r = self.want(q, top, ef, algo, filtered, None if cep is None else np.asarray(cep[i], np.uint32), fused)
            want.append(w)
            cpu += c
            io += r
        want_stats = self.cg.stats()[:2]
        hg.stats(reset=True)
        c = self.qb.HwCounters()
        if fused:
            got = hg.search_maxsim_discover(queries, top, ef, self.entry, self.lvl, point_deleted=filtered, counters=c, algorithm=algorithm)
        else:
            got = hg.search_maxsim_custom(queries, top, ef, self.entry, self.lvl, point_deleted=filtered, counters=c, custom_entry_points=cep,
                                          algorithm=algorithm)
        assert hg.stats() == want_stats
        assert c.cpu == cpu * self.units and c.vector_io_read == io * self.io
        for i, (g, w) in enumerate(zip(got, want)):
            assert np.array_equal(g["idx"], w["idx"]) and np.array_equal(g["score"].view(np.uint32), w["score"].view(np.uint32)), (i, g, w)
            if g.size:
                direct = self.view.score_points_custom(queries[i], g["idx"])
                assert np.array_equal(direct.view(np.uint32), g["score"].view(np.uint32)), i
        return got

    def close(self):
        self.st.close()


SHAPES = [(RECO_BEST, 2, 1), (RECO_SUM, 1, 2), (CONTEXT, 2, 0), (FEEDBACK, 2, 0), (DISCOVER, 2, 0)]


def _all_kinds(c, hg, top=10, ef=32, algorithm="hnsw", filtered=None, nq=3, lens=(1, 6)):
    for kind, n_a, n_b in SHAPES:
        c.check(hg, c.queries(kind, n_a, n_b, nq, lens), top, ef, algorithm, filtered)
    c.check(hg, c.queries(DISCOVER, 2, 0, nq, lens), top, ef, algorithm, filtered, fused=True)


def _lists_equal(a, b):
    return all(np.array_equal(x["idx"], y["idx"]) and np.array_equal(x["score"].view(np.uint32), y["score"].view(np.uint32)) for x, y in zip(a, b))


@pytest.mark.parametrize("dist", ["Cosine", "Dot", "Euclid", "Manhattan"])
@pytest.mark.parametrize("dim", [8, 48, 128])
def test_dense_f32_all_kinds(qb, oracle, dist, dim):
    c = _Case(qb, oracle, dist, dim, 400, lens=(1, 8), seed=dim)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    _all_kinds(c, hg)
    hg.close()
    c.close()


@pytest.mark.parametrize("dist,dim", [("Dot", 64), ("Euclid", 48), ("Dot", 1056)])
def test_sq8_all_kinds(qb, oracle, dist, dim):
    """dim 1056: actual_dim * 127^2 >= 2^24, the lane-exact SQ8 chain"""
    c = _Case(qb, oracle, dist, dim, 300, lens=(1, 6), sq8=True, seed=dim + 1)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    _all_kinds(c, hg, nq=2)
    _all_kinds(c, hg, algorithm="acorn", filtered=c.rng.random(c.n) >= 0.3, nq=2)
    hg.close()
    c.close()


@pytest.mark.parametrize("algorithm", ["hnsw", "acorn"])
def test_filters_and_custom_entry_points(qb, oracle, algorithm):
    """a selective per-call filter; custom entry points that pass it, that it filters out (skipped), and none passing (entry_point)"""
    c = _Case(qb, oracle, "Dot", 64, 1500, lens=(1, 8), seed=31)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    c.st.set_on_disk(True)   # vector_io_read metered: token rows x dim * 4
    c.io = c.dim * 4
    for sel in (0.1, 0.5):
        filtered = c.rng.random(c.n) >= sel
        filtered[c.entry] = False
        _all_kinds(c, hg, algorithm=algorithm, filtered=filtered, nq=2)
        passing, failing = np.flatnonzero(~filtered), np.flatnonzero(filtered)
        cep = [c.rng.choice(passing, 3), np.concatenate([c.rng.choice(failing, 2), c.rng.choice(passing, 1)]), c.rng.choice(failing, 4), []]
        got = c.check(hg, c.queries(RECO_SUM, 2, 1, 4), 10, 48, algorithm, filtered, cep=cep)
        assert all(not filtered[g["idx"]].any() for g in got)
        c.check(hg, c.queries(CONTEXT, 1, 0, 4), 10, 48, algorithm, filtered, cep=cep)
    c.check(hg, c.queries(FEEDBACK, 2, 0, 3), 10, 48, algorithm, cep=[c.rng.integers(0, c.n, 5) for _ in range(3)])
    hg.close()
    c.close()


def test_examples_staged_and_from_hbm(qb, oracle):
    """dim 128 (512 B a vector): 4 examples of 20 vectors (40 KB, staged in shared memory), of 30 (60 KB, read from HBM), and one example of
    4096 vectors"""
    c = _Case(qb, oracle, "Cosine", 128, 300, lens=(1, 6), seed=37)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    c.check(hg, c.queries(RECO_SUM, 2, 2, 2, lens=(20, 20)), 10, 32)
    c.check(hg, c.queries(RECO_SUM, 2, 2, 2, lens=(30, 30)), 10, 32)
    c.check(hg, c.queries(CONTEXT, 2, 0, 2, lens=(30, 30)), 10, 32, "acorn", c.rng.random(c.n) >= 0.4)
    c.check(hg, c.queries(RECO_BEST, 1, 0, 2, lens=(1, 1)), 10, 32)
    c.check(hg, c.queries(RECO_BEST, 1, 1, 1, lens=(4096, 4096)), 5, 16)
    hg.close()
    c.close()


@pytest.mark.parametrize("n_a,n_b", [(40, 40), (100, 0), (4000, 96)])
def test_many_examples(qb, oracle, n_a, n_b):
    """E = 80 / 100 / 4096 examples: fewer points per scoring batch (51, 40, 1)"""
    c = _Case(qb, oracle, "Euclid", 8, 200, lens=(1, 4), seed=41 + n_a)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    ef = 16 if n_a + n_b == 4096 else 32
    c.check(hg, c.queries(RECO_BEST, n_a, n_b, 2, lens=(1, 2)), 5, ef)
    c.check(hg, c.queries(RECO_SUM, n_a, n_b, 1, lens=(1, 2)), 5, ef, "acorn", c.rng.random(c.n) >= 0.5)
    hg.close()
    c.close()


@pytest.mark.parametrize("sq8", [False, True])
def test_token_runs_0_1_300(qb, oracle, sq8):
    """points with no token rows (every MaxSim -inf), one-token points and 300-token points; top = ef = 300 lists every point reached.
    The kinds are those whose fold of -inf similarities is not NaN (a NaN's bits are the platform's, not the reference's)."""
    c = _Case(qb, oracle, "Dot", 64, 300, lens=(0, 1), sq8=sq8, seed=43 + sq8, empty=0.2, long=0.1)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    got = c.check(hg, c.queries(RECO_SUM, 2, 0, 3), 300, 300)
    assert all(np.isneginf(g["score"]).sum() == (np.diff(c.off)[g["idx"]] == 0).sum() > 0 for g in got)
    c.check(hg, c.queries(CONTEXT, 1, 0, 2), 300, 300)
    hg.close()
    c.close()


def test_ef_extremes_and_top_above_ef(qb, oracle):
    c = _Case(qb, oracle, "Cosine", 32, 900, lens=(1, 5), seed=47)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    c.check(hg, c.queries(RECO_BEST, 1, 1, 2), 1, 1)
    c.check(hg, c.queries(CONTEXT, 2, 0, 2), 10, 1)          # top > ef: max(ef, top)
    got = c.check(hg, c.queries(RECO_SUM, 2, 0, 2), 20, 4096)
    assert all(g.size == 20 for g in got)
    c.check(hg, c.queries(DISCOVER, 1, 0, 1), 20, 4096, fused=True)
    c.check(hg, c.queries(FEEDBACK, 1, 0, 1), 5, 4096, "acorn", c.rng.random(c.n) >= 0.5)
    hg.close()
    c.close()


@pytest.mark.parametrize("m", [4, 32])
def test_loaders_and_builds(qb, oracle, m):
    """plain and compressed links.bin and a build_multivector handle at m0 = 8 / 64, with MaxSim searches on the same handle in between"""
    c = _Case(qb, oracle, "Euclid", 40, 600, lens=(1, 6), m=m, seed=53 + m)
    assert c.m0 == 2 * m
    plain = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    comp = qb.HnswGraph.from_compressed_multivector(c.view, gc.plain_to_compressed(c.blob, c.m, c.m0))
    for hg, algorithm in ((plain, "hnsw"), (comp, "acorn")):
        mq = [c.ex() for _ in range(3)]
        nearest = hg.search_maxsim(mq, 10, 40, c.entry, c.lvl, algorithm=algorithm)
        _all_kinds(c, hg, 10, 40, algorithm, nq=2)
        assert _lists_equal(hg.search_maxsim(mq, 10, 40, c.entry, c.lvl, algorithm=algorithm), nearest)
    plain.close()
    comp.close()
    built = qb.HnswGraph.build_multivector(c.view, m=m, ef_construct=48, seed=m)
    c.cg = cr.Graph(built.export_plain(), m, 2 * m, c.n)
    c.entry, c.lvl = built.entry_point, built.entry_level
    _all_kinds(c, built, 10, 40, nq=2)
    built.close()
    c.close()


def test_fused_discover_is_context_then_discover(qb, oracle):
    c = _Case(qb, oracle, "Dot", 48, 800, lens=(1, 6), seed=59)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    for algorithm, filtered in (("hnsw", None), ("acorn", c.rng.random(c.n) >= 0.3)):
        if filtered is not None:
            filtered[c.entry] = False
        qs = c.queries(DISCOVER, 2, 0, 4)
        fused = hg.search_maxsim_discover(qs, 10, 32, c.entry, c.lvl, point_deleted=filtered, algorithm=algorithm)
        ctx = hg.search_maxsim_custom([qb.ContextQuery(q.pairs) for q in qs], 10, 32, c.entry, c.lvl, point_deleted=filtered, algorithm=algorithm)
        two = hg.search_maxsim_custom(qs, 10, 32, c.entry, c.lvl, point_deleted=filtered, custom_entry_points=[x["idx"] for x in ctx],
                                      algorithm=algorithm)
        assert _lists_equal(fused, two)
    hg.close()
    c.close()


def test_errors_leave_the_handle_usable(qb, oracle):
    from qdrant_b200 import _capi

    c = _Case(qb, oracle, "Dot", 32, 300, lens=(1, 5), seed=61)
    hg = qb.HnswGraph.multivector(c.view, c.blob, c.m, c.m0)
    qs = c.queries(RECO_SUM, 1, 1, 2)
    base = hg.search_maxsim_custom(qs, 10, 32, c.entry, c.lvl)
    mq = [c.ex() for _ in range(2)]
    base_mv = hg.search_maxsim(mq, 10, 32, c.entry, c.lvl)

    def status(f):
        with pytest.raises(qb.QbError) as ei:
            f()
        assert _lists_equal(hg.search_maxsim_custom(qs, 10, 32, c.entry, c.lvl), base)
        assert _lists_equal(hg.search_maxsim(mq, 10, 32, c.entry, c.lvl), base_mv)
        return ei.value.status

    U, INV = _capi.QB_ERR_UNSUPPORTED, _capi.QB_ERR_INVALID
    # the new entries on a regular handle
    reg_st = qb.DenseVectorStorage(c.rows[: c.n], c.d)
    reg = qb.HnswGraph(reg_st, c.blob, c.m, c.m0)
    assert status(lambda: reg.search_maxsim_custom(qs, 5, 16, c.entry, c.lvl)) == U
    assert status(lambda: reg.search_maxsim_discover(c.queries(DISCOVER, 1, 0, 1), 5, 16, c.entry, c.lvl)) == U
    reg.close()
    reg_st.close()
    # ef
    assert status(lambda: hg.search_maxsim_custom(qs, 5, 4097, c.entry, c.lvl)) == U
    # examples: empty, 4097 vectors
    e0 = qb.RecoSumScoresQuery(qb.RecoQuery([np.zeros((0, 32), np.float32)], [c.ex()]))
    assert status(lambda: hg.search_maxsim_custom([e0], 5, 16, c.entry, c.lvl)) == INV
    big = qb.RecoSumScoresQuery(qb.RecoQuery([c.rng.standard_normal((4097, 32)).astype(np.float32)], [c.ex()]))
    assert status(lambda: hg.search_maxsim_custom([big], 5, 16, c.entry, c.lvl)) == INV
    # custom entry points out of range
    assert status(lambda: hg.search_maxsim_custom(qs, 5, 16, c.entry, c.lvl, custom_entry_points=[[c.n], [0]])) == INV
    # the raw entry: a bad kind or shape, descending offsets, coef missing or extra
    L = _capi.lib()
    kind, n_a, n_b, vecs, off, _ = hg._multi_batch(qs)
    out = np.zeros((2, 5), dtype=qb.SCORED_POINT_OFFSET)
    cnt = np.zeros(2, np.uint32)
    coef = np.ones((2, 2), np.float32)

    def raw(kind, off, n_a, n_b, coef=None):
        qb.check(L.qb_hnsw_search_maxsim_custom_batch(hg._h, kind, vecs.ctypes.data_as(qb.f32p), off.ctypes.data_as(qb.u32p), n_a, n_b,
                                                      None if coef is None else coef.ctypes.data_as(qb.f32p), 2, 5, 16, c.entry, c.lvl, None, None, 0,
                                                      None, None, out.ctypes.data_as(C.POINTER(qb.ScoredPoint)), cnt.ctypes.data_as(qb.u32p), None, 0))

    assert status(lambda: raw(9, off, n_a, n_b)) == INV
    assert status(lambda: raw(CONTEXT, off, 1, 1)) == INV
    desc = off.copy()
    desc[2], desc[3] = desc[3], desc[2]
    assert status(lambda: raw(kind, desc, n_a, n_b)) == INV
    assert status(lambda: raw(kind, off, n_a, n_b, coef)) == INV
    assert status(lambda: raw(FEEDBACK, off[:3], 0, 0)) == INV   # one example per query, no coef
    raw(kind, off, n_a, n_b)   # the well-formed call answers as the wrapper does
    assert _lists_equal([out[i, : cnt[i]] for i in range(2)], hg.search_maxsim_custom(qs, 5, 16, c.entry, c.lvl))
    hg.close()
    c.close()
