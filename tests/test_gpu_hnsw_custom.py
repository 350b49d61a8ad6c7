"""Custom queries through the device traversal (qb_hnsw_search_custom_batch, qb_hnsw_search_discover_batch) vs the CPU checker
(tests/hnsw_custom_ref.c in keyed mode, the device's tie order; checked in tests/test_hnsw_custom_cpu.py): equal lists and score bit
patterns, hops and scored points (qb_hnsw_stats), and HwCounters, for every kind, both level-0 algorithms, dense f32 on every metric
and SQ8, both loaders, filters, custom entry points, example sets on both sides of the shared-memory budget, and the fused discover
against the Python two-stage restatement."""
import ctypes as C

import numpy as np
import pytest

from tests import graph_links_compressed as gl
from tests import hnsw_acorn_ref as ar
from tests import hnsw_custom_ref as cr

pytestmark = pytest.mark.gpu

# (kind, n_a, n_b): recommend best-score and sum-scores (3 positives, 2 negatives), context (2 pairs), discover as one search
# (target + 2 pairs, the reference's second stage), feedback (2 pairs)
KINDS = [(1, 3, 2), (2, 3, 2), (4, 2, 0), (3, 2, 0), (cr.FEEDBACK, 2, 0)]
ALGOS = {"hnsw": ar.HNSW, "acorn": ar.ACORN}


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _setup(oracle, qb, n, dim, dist, m, seed, threads=4):
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    if d == qb.Distance.Cosine:
        base = oracle.preprocess_rows_f32(oracle.COSINE, base)
    g = oracle.HNSW(base, int(d), m=m, ef_construct=64, seed=seed, threads=threads)
    entry, lvl, gm, gm0 = g.entry()
    plain = g.export_plain()
    g.close()
    return d, base, plain, entry, lvl, gm, gm0, rng


def _examples(oracle, d, rng, nq, ne, dim):
    raw = rng.standard_normal((nq, ne, dim)).astype(np.float32)
    pre = np.stack([[oracle.preprocess_f32(int(d), v) for v in q] for q in raw])
    return raw, pre


def _filter(rng, n, sel, entry):
    f = rng.random(n) >= sel
    f[entry] = False
    return f


def _same(got, want, what):
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a["idx"], b["idx"]), f"{what} query {i}: ids\n{a[:8]}\n{b[:8]}"
        assert np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)), f"{what} query {i}: score bits"


def _check(qb, hg, cg, oracle, base, d, kind, n_a, n_b, top, ef, entry, lvl, algo, filtered, nq=16, rng=None, cep=None, what="", **kw):
    """one device call vs the checker: lists, score bits, hops / scored points, counters; returns the device lists"""
    ne = cr.n_examples(kind, n_a, n_b)
    raw, pre = _examples(oracle, d, rng, nq, ne, base.shape[1])
    coef = rng.standard_normal((nq, 1 + n_a)).astype(np.float32) if kind == cr.FEEDBACK else None
    hg.stats(reset=True); cg.stats()
    cnt = qb.HwCounters()
    got = hg.search_custom(kind, raw, n_a, n_b, coef=coef, top=top, ef=ef, entry_point=entry, entry_level=lvl, counters=cnt,
                           custom_entry_points=cep, algorithm=algo, **kw)
    want = cr.search_custom_batch(cg, oracle, base, int(d), pre, kind, n_a, n_b, top, ef, entry, lvl, ALGOS[algo], filtered, coef=coef, cep=cep)
    _same(got, want, what)
    calls, scored = cg.stats()[:2]
    assert hg.stats(reset=True) == (calls, scored), what
    assert cnt.cpu == scored * ne * base.shape[1] * 4, what
    return got


@pytest.mark.parametrize("dist,dim,n,m", [("Cosine", 128, 8_000, 16), ("Euclid", 24, 6_000, 16), ("Dot", 8, 4_000, 8), ("Manhattan", 768, 3_000, 16)])
def test_every_kind_f32(qb, oracle, dist, dim, n, m):
    d, base, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, dist, m, seed=dim)
    st = qb.DenseVectorStorage(base, d)
    hg = qb.HnswGraph(st, plain, gm, gm0)
    cg = cr.Graph(plain, gm, gm0, n)
    for kind, n_a, n_b in KINDS:
        for algo, sel in (("hnsw", 1.0), ("hnsw", 0.5), ("acorn", 0.05)):
            f = None if sel == 1.0 else _filter(rng, n, sel, entry)
            got = _check(qb, hg, cg, oracle, base, d, kind, n_a, n_b, 10, 48, entry, lvl, algo, f, rng=rng, point_deleted=f,
                         what=f"{dist} {dim} kind {kind} {algo} sel {sel}")
            if kind == 4 and sel == 1.0:
                # context: the plateau of points that satisfy both pairs scores exactly 0.0
                assert any((g["score"].view(np.uint32) == 0).any() for g in got), "no compared score is 0.0"
    hg.close(); st.close(); cg.close()


def test_filters_large_ef_top_over_ef(qb, oracle):
    n, dim = 20_000, 32
    d, base, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Cosine", 16, seed=3)
    st = qb.DenseVectorStorage(base, d)
    hg = qb.HnswGraph(st, plain, gm, gm0)
    cg = cr.Graph(plain, gm, gm0, n)
    f1, f2 = _filter(rng, n, 0.3, entry), _filter(rng, n, 0.3, entry)
    for algo in ("hnsw", "acorn"):
        _check(qb, hg, cg, oracle, base, d, 1, 3, 2, 10, 1000, entry, lvl, algo, f1, nq=8, rng=rng, point_deleted=f1, what=f"ef 1000 {algo}")
        _check(qb, hg, cg, oracle, base, d, 2, 3, 2, 200, 40, entry, lvl, algo, f1, nq=8, rng=rng, point_deleted=f1, what=f"top > ef {algo}")
    st.set_deleted(f1)
    for algo, sel in (("hnsw", 0.5), ("acorn", 0.02)):
        f3 = _filter(rng, n, sel, entry)
        _check(qb, hg, cg, oracle, base, d, 4, 2, 0, 10, 64, entry, lvl, algo, f1, rng=rng, what=f"resident {algo}")
        _check(qb, hg, cg, oracle, base, d, cr.FEEDBACK, 2, 0, 10, 64, entry, lvl, algo, f1 | f3, rng=rng, point_deleted=f3, what=f"resident | call {algo}")
    hg.close(); st.close(); cg.close()


@pytest.mark.parametrize("m", [4, 32])
def test_m0_and_compressed_loader(qb, oracle, m):
    n, dim = 6_000, 48
    d, base, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Dot", m, seed=m)
    assert gm0 == 2 * m
    st = qb.DenseVectorStorage(base, d)
    hp = qb.HnswGraph(st, plain, gm, gm0)
    hc = qb.HnswGraph.from_compressed(st, gl.plain_to_compressed(plain, gm, gm0))
    cg = cr.Graph(plain, gm, gm0, n)
    for algo, sel in (("hnsw", 1.0), ("acorn", 0.1)):
        f = None if sel == 1.0 else _filter(rng, n, sel, entry)
        seed = int(rng.integers(1 << 30))
        a = _check(qb, hp, cg, oracle, base, d, 1, 3, 2, 10, 64, entry, lvl, algo, f, rng=np.random.default_rng(seed), point_deleted=f, what=f"plain m0 {gm0}")
        b = _check(qb, hc, cg, oracle, base, d, 1, 3, 2, 10, 64, entry, lvl, algo, f, rng=np.random.default_rng(seed), point_deleted=f, what=f"compressed m0 {gm0}")
        _same(a, b, "loaders")
    hp.close(); hc.close(); st.close(); cg.close()


def test_examples_in_shared_and_global_memory(qb, oracle):
    """E = 1 up to past the 48 KB staging budget (768 f32 = 3 KB per example: 16 fit, 20 do not); same arithmetic on both paths"""
    n, dim = 3_000, 768
    d, base, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Cosine", 16, seed=11)
    st = qb.DenseVectorStorage(base, d)
    hg = qb.HnswGraph(st, plain, gm, gm0)
    cg = cr.Graph(plain, gm, gm0, n)
    for n_a, n_b in ((1, 0), (8, 8), (12, 8), (40, 9)):
        for kind in (1, 2):
            _check(qb, hg, cg, oracle, base, d, kind, n_a, n_b, 10, 32, entry, lvl, "hnsw", None, nq=6, rng=rng, what=f"E {n_a + n_b}")
    f = _filter(rng, n, 0.2, entry)
    _check(qb, hg, cg, oracle, base, d, 3, 12, 0, 10, 32, entry, lvl, "acorn", f, nq=6, rng=rng, point_deleted=f, what="discover E 25")
    hg.close(); st.close(); cg.close()


@pytest.mark.parametrize("dim", [96, 1100])
def test_sq8(qb, oracle, dim):
    """SQ8 through the callback route: the checker scores with qb_score_points on a qb_scorer_create_custom scorer (pinned to the
    oracle by tests/test_gpu_custom.py); dim 1100 is the lane-exact kind"""
    n = 4_000
    d, base, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Cosine", 16, seed=dim)
    dt, inv = qb.construct_vector_parameters(d)
    sq = oracle.SQ8.encode(base, int(dt), bool(inv))
    qst = qb.ScalarQuantizedVectors(sq.rows, dim, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, d)
    hg = qb.HnswGraph(qst, plain, gm, gm0)
    cg = cr.Graph(plain, gm, gm0, n)
    nq = 6
    for kind, n_a, n_b, algo, sel in ((1, 3, 2, "hnsw", 1.0), (4, 2, 0, "acorn", 0.05), (2, 3, 2, "acorn", 0.3)):
        f = None if sel == 1.0 else _filter(rng, n, sel, entry)
        ne = cr.n_examples(kind, n_a, n_b)
        raw = rng.standard_normal((nq, ne, dim)).astype(np.float32)
        hg.stats(reset=True); cg.stats()
        got = hg.search_custom(kind, raw, n_a, n_b, top=10, ef=64, entry_point=entry, entry_level=lvl, point_deleted=f, algorithm=algo)
        for q in range(nq):
            h = C.c_void_p()
            qb.check(qb.lib().qb_scorer_create_custom(qst._h, kind, raw[q].ctypes.data_as(C.POINTER(C.c_float)), n_a, n_b, C.byref(h)))
            sc = qb.RawScorer(qst, h.value)
            want = cr.search_cb(cg, lambda ids, sc=sc: sc.score_points(ids.astype(np.uint32)), 10, 64, entry, lvl, ALGOS[algo], f)
            sc.close()
            _same([got[q]], [want], f"sq8 {dim} kind {kind}")
        assert hg.stats(reset=True) == cg.stats()[:2]
    hg.close(); qst.close(); cg.close()


@pytest.mark.parametrize("algo", ["hnsw", "acorn"])
def test_discover_fused_equals_two_stages(qb, oracle, algo):
    n, dim, n_pairs, nq = 10_000, 64, 2, 24
    d, base, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Cosine", 16, seed=21)
    st = qb.DenseVectorStorage(base, d)
    hg = qb.HnswGraph(st, plain, gm, gm0)
    cg = cr.Graph(plain, gm, gm0, n)
    for sel in (1.0, 0.05 if algo == "acorn" else 0.5):
        f = None if sel == 1.0 else _filter(rng, n, sel, entry)
        raw, pre = _examples(oracle, d, rng, nq, 1 + 2 * n_pairs, dim)
        hg.stats(reset=True); cg.stats()
        cnt = qb.HwCounters()
        got = hg.search_discover(raw, n_pairs, top=10, ef=48, entry_point=entry, entry_level=lvl, point_deleted=f, counters=cnt, algorithm=algo)
        want = cr.discover(cg, oracle, base, int(d), pre, n_pairs, 10, 48, entry, lvl, ALGOS[algo], f)
        _same(got, want, f"discover {algo} sel {sel}")
        calls, scored = cg.stats()[:2]
        assert hg.stats(reset=True) == (calls, scored)
        # counters: stage 1 scores 2 n_pairs examples per point, stage 2 1 + 2 n_pairs
        cr.search_custom_batch(cg, oracle, base, int(d), pre[:, 1:], 4, n_pairs, 0, 10, 48, entry, lvl, ALGOS[algo], f)
        s1 = cg.stats()[1]
        assert cnt.cpu == (s1 * 2 * n_pairs + (scored - s1) * (1 + 2 * n_pairs)) * dim * 4
        # stage 1 really lands on the context plateau sometimes: some stage-1 score is exactly 0.0
    ctx = cr.search_custom_batch(cg, oracle, base, int(d), pre[:, 1:], 4, n_pairs, 0, 10, 48, entry, lvl, ALGOS[algo], None)
    cg.stats()
    assert any((c["score"].view(np.uint32) == 0).any() for c in ctx)
    hg.close(); st.close(); cg.close()


def test_custom_entry_points(qb, oracle):
    n, dim = 8_000, 32
    d, base, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Euclid", 4, seed=7)
    st = qb.DenseVectorStorage(base, d)
    hg = qb.HnswGraph(st, plain, gm, gm0)
    cg = cr.Graph(plain, gm, gm0, n)
    lv = np.array([cr.get_entry_point(cg, [i], entry, lvl)[1] for i in range(n)])
    assert lv.max() >= 2
    hi, mid, low = np.flatnonzero(lv == lv.max()), np.flatnonzero(lv == 1), np.flatnonzero(lv == 0)
    nq = 8
    f = _filter(rng, n, 0.7, entry)
    f[hi[0]] = True          # a filtered-out candidate of the highest level
    f[mid[:4]] = False
    cep = [[hi[0], mid[0], low[0], mid[1]], [low[1], low[2], low[3]], [mid[2], hi[0]], [], [hi[0]], [mid[3], mid[0], mid[2], mid[1]],
           [low[4]], list(rng.choice(n, 30, replace=False))]
    for algo in ("hnsw", "acorn"):
        _check(qb, hg, cg, oracle, base, d, 1, 2, 1, 10, 32, entry, lvl, algo, f, nq=nq, rng=rng, cep=cep, point_deleted=f, what=f"cep {algo}")
        _check(qb, hg, cg, oracle, base, d, 4, 1, 0, 10, 32, entry, lvl, algo, None, nq=nq, rng=rng, cep=cep, what=f"cep unfiltered {algo}")
    hg.close(); st.close(); cg.close()


def test_alternating_custom_and_nearest_searches(qb, oracle):
    n, dim = 10_000, 32
    d, base, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Cosine", 16, seed=6)
    f = _filter(rng, n, 0.05, entry)
    st = qb.DenseVectorStorage(base, d)
    queries = rng.standard_normal((200, dim)).astype(np.float32)
    raw = rng.standard_normal((200, 5, dim)).astype(np.float32)
    disc = rng.standard_normal((100, 5, dim)).astype(np.float32)
    runs = {
        "nearest": lambda g: g.search(queries, 10, 64, entry, lvl, point_deleted=f, algorithm="acorn"),
        "reco": lambda g: g.search_custom(1, raw, 3, 2, top=10, ef=64, entry_point=entry, entry_level=lvl, point_deleted=f, algorithm="acorn"),
        "discover": lambda g: g.search_discover(disc, 2, top=10, ef=64, entry_point=entry, entry_level=lvl),
    }
    fresh = {}
    for k, run in runs.items():
        hg = qb.HnswGraph(st, plain, gm, gm0)
        fresh[k] = run(hg)
        hg.close()
    hg = qb.HnswGraph(st, plain, gm, gm0)
    for k in ("reco", "nearest", "discover", "reco", "discover", "nearest"):
        _same(runs[k](hg), fresh[k], k)
    hg.close(); st.close()


def test_invalid_arguments(qb, oracle):
    from qdrant_b200 import _capi

    n, dim = 2_000, 16
    d, base, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Dot", 8, seed=1)
    st = qb.DenseVectorStorage(base, d)
    hg = qb.HnswGraph(st, plain, gm, gm0)
    ex = rng.standard_normal((2, 5, dim)).astype(np.float32)

    def status(fn):
        with pytest.raises(_capi.QbError) as e:
            fn()
        return e.value.status

    E = _capi.QB_ERR_INVALID
    assert status(lambda: hg.search_custom(9, ex, 3, 2, entry_point=entry, entry_level=lvl)) == E                  # unknown kind
    assert status(lambda: hg.search_custom(4, ex[:, :4], 2, 1, entry_point=entry, entry_level=lvl)) == E           # context with n_b
    assert status(lambda: hg.search_custom(1, ex, 3, 2, entry_point=n, entry_level=0)) == E                        # entry out of range
    assert status(lambda: hg.search_custom(1, ex, 3, 2, entry_point=entry, entry_level=60)) == E                   # entry level
    assert status(lambda: hg.search_custom(1, ex, 3, 2, top=0, entry_point=entry, entry_level=lvl)) == E           # top
    assert status(lambda: hg.search_custom(cr.FEEDBACK, ex, 2, 0, entry_point=entry, entry_level=lvl)) == E        # feedback without coef
    assert status(lambda: hg.search_custom(1, ex, 3, 2, coef=np.ones((2, 4), np.float32), entry_point=entry, entry_level=lvl)) == E   # coef
    assert status(lambda: hg.search_custom(1, ex, 3, 2, entry_point=entry, entry_level=lvl, custom_entry_points=[[0], [n]])) == E     # cep
    assert status(lambda: hg.search_custom(1, ex, 3, 2, entry_point=entry, entry_level=lvl, algorithm="hnsw", ef=5000)) == _capi.QB_ERR_UNSUPPORTED
    assert status(lambda: hg.search_discover(ex[:, :1], 0, entry_point=entry, entry_level=lvl)) == E               # discover without a pair
    assert _capi.lib().qb_hnsw_search_custom_batch(hg._h, 1, ex.ctypes.data_as(_capi.f32p), 3, 2, None, 2, 10, 64, entry, lvl,
                                                   np.zeros(2, np.uint32).ctypes.data_as(_capi.u32p), None, 1, None, None,
                                                   (qb.ScoredPoint * 20)(), (C.c_uint32 * 2)(), None, 0) == E       # cep without counts
    with pytest.raises(ValueError):
        hg.search_custom(1, ex, 3, 2, entry_point=entry, entry_level=lvl, algorithm="nsg")
    # the device is still usable
    a = hg.search_custom(1, ex, 3, 2, entry_point=entry, entry_level=lvl)
    assert len(a) == 2 and all(len(x) == 10 for x in a)
    hg.close(); st.close()
