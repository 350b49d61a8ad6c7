"""Device ACORN-1 traversal (qb_hnsw_search_batch_algo with QB_HNSW_ALGO_ACORN) vs the CPU ACORN traversal of the SAME graph
(tests/hnsw_acorn_ref.c, checked against an independent restatement in tests/test_hnsw_acorn_cpu.py): tie-aware lists with equal
score bits, hops and scored points (qb_hnsw_stats), and HwCounters.  Also: unfiltered ACORN equals HNSW on the device, HNSW and
ACORN batches alternating on one graph leave the visited state clean, and a search that overflows the visited logs still answers
correctly."""
import numpy as np
import pytest

from tests import graph_links_compressed as gl
from tests import hnsw_acorn_ref as ar
from tests.util import assert_topk_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _setup(oracle, qb, n, dim, dist, m, seed, nq=48, threads=4):
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    if d == qb.Distance.Cosine:
        base = oracle.preprocess_rows_f32(oracle.COSINE, base)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    qp = np.stack([oracle.preprocess_f32(int(d), q) for q in queries])
    g = oracle.HNSW(base, int(d), m=m, ef_construct=64, seed=seed, threads=threads)
    entry, lvl, gm, gm0 = g.entry()
    plain = g.export_plain()
    g.close()
    return d, base, queries, qp, plain, entry, lvl, gm, gm0, rng


def _filter(rng, n, sel, entry):
    f = rng.random(n) >= sel
    f[entry] = False          # get_entry_point picks a point that passes the filter
    return f


def _check(qb, hg, cg, oracle, base, d, dim, queries, qp, entry, lvl, top, ef, filtered, what, per_point=None, **kw):
    hg.stats(reset=True); cg.stats()
    cnt = qb.HwCounters()
    got = hg.search(queries, top, ef, entry, lvl, counters=cnt, algorithm="acorn", **kw)
    want = cg.search_batch(oracle, base, int(d), qp, top, ef, entry, lvl, ar.ACORN, filtered, threads=4)
    for i, (a, b) in enumerate(zip(got, want)):
        assert_topk_equal(a, b, what=f"{what} query {i}")
    calls, scored = cg.stats()[:2]
    assert hg.stats(reset=True) == (calls, scored), what
    assert cnt.cpu == scored * (per_point if per_point is not None else dim * 4), what
    return got


@pytest.mark.parametrize("dist,dim,n,m", [("Cosine", 96, 20_000, 16), ("Euclid", 100, 6_000, 16), ("Dot", 8, 4_000, 4), ("Manhattan", 40, 4_000, 32),
                                          ("Cosine", 768, 4_000, 16), ("Dot", 20, 5_000, 32)])
def test_acorn_equals_cpu_f32(qb, oracle, dist, dim, n, m):
    d, base, queries, qp, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, dist, m, seed=dim + m)
    st = qb.DenseVectorStorage(base, d)
    hg = qb.HnswGraph(st, plain, gm, gm0)
    cg = ar.Graph(plain, gm, gm0, n)
    for sel, top, ef in ((0.01, 10, 64), (0.05, 10, 128), (0.2, 40, 20), (0.5, 5, 16), (1.0, 10, 64)):
        f = _filter(rng, n, sel, entry)
        _check(qb, hg, cg, oracle, base, d, dim, queries, qp, entry, lvl, top, ef, f, f"{dist} dim {dim} m0 {gm0} sel {sel}", point_deleted=f)
    hg.close(); st.close(); cg.close()


def test_acorn_large_ef_and_filter_sources(qb, oracle):
    """ef 1000 and top > ef; the filter per call, resident (set_deleted), and both OR-ed"""
    n, dim = 30_000, 32
    d, base, queries, qp, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Cosine", 16, seed=3, nq=24)
    st = qb.DenseVectorStorage(base, d)
    hg = qb.HnswGraph(st, plain, gm, gm0)
    cg = ar.Graph(plain, gm, gm0, n)
    f1, f2 = _filter(rng, n, 0.3, entry), _filter(rng, n, 0.3, entry)
    _check(qb, hg, cg, oracle, base, d, dim, queries, qp, entry, lvl, 10, 1000, f1, "ef 1000", point_deleted=f1)
    _check(qb, hg, cg, oracle, base, d, dim, queries, qp, entry, lvl, 300, 50, f1, "top > ef", point_deleted=f1)
    st.set_deleted(f1)
    _check(qb, hg, cg, oracle, base, d, dim, queries, qp, entry, lvl, 10, 64, f1, "resident")
    _check(qb, hg, cg, oracle, base, d, dim, queries, qp, entry, lvl, 10, 64, f1 | f2, "resident | per call", point_deleted=f2)
    hg.close(); st.close(); cg.close()


def test_acorn_m0_64_and_compressed_loader(qb, oracle):
    n, dim = 8_000, 48
    d, base, queries, qp, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Dot", 32, seed=8)
    assert gm0 == 64
    st = qb.DenseVectorStorage(base, d)
    hp = qb.HnswGraph(st, plain, gm, gm0)
    hc = qb.HnswGraph.from_compressed(st, gl.plain_to_compressed(plain, gm, gm0))
    cg = ar.Graph(plain, gm, gm0, n)
    for sel in (0.02, 0.1, 0.4):
        f = _filter(rng, n, sel, entry)
        a = _check(qb, hg=hp, cg=cg, oracle=oracle, base=base, d=d, dim=dim, queries=queries, qp=qp, entry=entry, lvl=lvl, top=10, ef=100,
                   filtered=f, what=f"plain m0 64 sel {sel}", point_deleted=f)
        b = _check(qb, hg=hc, cg=cg, oracle=oracle, base=base, d=d, dim=dim, queries=queries, qp=qp, entry=entry, lvl=lvl, top=10, ef=100,
                   filtered=f, what=f"compressed m0 64 sel {sel}", point_deleted=f)
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
    hp.close(); hc.close(); st.close(); cg.close()


@pytest.mark.parametrize("dim", [96, 1100])
def test_acorn_equals_cpu_sq8(qb, oracle, dim):
    """SQ8 scored through the oracle's quantized scorer; dim 1100: actual_dim > 1040, the lane-exact kind"""
    n = 5_000
    d, base, queries, qp, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Cosine", 16, seed=dim, nq=12)
    dt, inv = qb.construct_vector_parameters(d)
    sq = oracle.SQ8.encode(base, int(dt), bool(inv))
    qst = qb.ScalarQuantizedVectors(sq.rows, dim, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, d)
    hg = qb.HnswGraph(qst, plain, gm, gm0)
    cg = ar.Graph(plain, gm, gm0, n)
    for sel in (0.03, 0.3):
        f = _filter(rng, n, sel, entry)
        hg.stats(reset=True)
        got = hg.search(queries, 10, 64, entry, lvl, point_deleted=f, algorithm="acorn")
        for q, a in zip(qp, got):
            code, off = sq.encode_query(q)
            want = cg.search(lambda ids, code=code, off=off: np.array([sq.score(code, off, int(i)) for i in ids], np.float32), 10, 64, entry, lvl,
                             ar.ACORN, f)
            assert_topk_equal(a, want, what=f"sq8 dim {dim} sel {sel}")
        assert hg.stats(reset=True) == cg.stats()[:2]
    hg.close(); qst.close(); cg.close()


def test_unfiltered_acorn_equals_hnsw_on_device(qb, oracle):
    n, dim = 20_000, 64
    d, base, queries, qp, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Euclid", 16, seed=4, nq=100)
    st = qb.DenseVectorStorage(base, d)
    hg = qb.HnswGraph(st, plain, gm, gm0)
    for top, ef in ((10, 64), (100, 200)):
        hg.stats(reset=True)
        h = hg.search(queries, top, ef, entry, lvl)
        hs = hg.stats(reset=True)
        a = hg.search(queries, top, ef, entry, lvl, algorithm="acorn")
        assert hg.stats(reset=True) == hs
        for x, y in zip(h, a):
            assert np.array_equal(x, y)
    hg.close(); st.close()


def test_alternating_algorithms_leave_visited_state_clean(qb, oracle):
    n, dim = 10_000, 32
    d, base, queries, qp, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Cosine", 16, seed=6, nq=300)
    f = _filter(rng, n, 0.05, entry)
    st = qb.DenseVectorStorage(base, d)
    fresh = {}
    for algo in ("hnsw", "acorn"):
        hg = qb.HnswGraph(st, plain, gm, gm0)
        fresh[algo] = hg.search(queries, 10, 64, entry, lvl, point_deleted=f, algorithm=algo)
        hg.close()
    hg = qb.HnswGraph(st, plain, gm, gm0)
    for algo in ("acorn", "hnsw", "acorn", "hnsw", "hnsw", "acorn"):
        for x, y in zip(hg.search(queries, 10, 64, entry, lvl, point_deleted=f, algorithm=algo), fresh[algo]):
            assert np.array_equal(x, y), algo
    with pytest.raises(ValueError):
        hg.search(queries[:1], 10, 64, entry, lvl, algorithm="nsg")
    hg.close(); st.close()


def test_visited_log_overflow(qb, oracle):
    """searches that mark more points than the visited log holds (32768 entries; ACORN also marks filtered-out 1-hop links) clear
    the whole bitmap instead, and the next batch still answers correctly"""
    n, dim = 100_000, 24
    d, base, queries, qp, plain, entry, lvl, gm, gm0, rng = _setup(oracle, qb, n, dim, "Cosine", 16, seed=12, nq=16, threads=8)
    f = _filter(rng, n, 0.5, entry)
    st = qb.DenseVectorStorage(base, d)
    hg = qb.HnswGraph(st, plain, gm, gm0)
    cg = ar.Graph(plain, gm, gm0, n)
    cg.search_batch(oracle, base, int(d), qp[:4], 10, 4096, entry, lvl, ar.ACORN, f)
    max_hop1_marks = cg.stats()[2]
    assert max_hop1_marks > 32768, max_hop1_marks
    _check(qb, hg, cg, oracle, base, d, dim, queries, qp, entry, lvl, 10, 4096, f, "overflow", point_deleted=f)
    f2 = _filter(rng, n, 0.1, entry)
    _check(qb, hg, cg, oracle, base, d, dim, queries, qp, entry, lvl, 10, 64, f2, "after overflow", point_deleted=f2)
    hg.close(); st.close(); cg.close()
