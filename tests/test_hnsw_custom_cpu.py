"""The CPU checker of the device's custom-query traversal (tests/hnsw_custom_ref.c through tests/hnsw_custom_ref.py): unkeyed, it traverses
exactly as the ACORN checker (tests/hnsw_acorn_ref.c) does, its custom scorer is the oracle's fold, the keyed tie order changes nothing on
tie-free inputs and does change a context plateau, get_entry_point follows graph_layers.rs:506-528, and the Python discover restatement is
the reference's two stages."""
import numpy as np
import pytest

from tests import hnsw_acorn_ref as ar
from tests import hnsw_custom_ref as cr

DOT = 2   # oracle DOT (qb_distance)


def _graph(oracle, n=3000, dim=24, m=8, seed=5, distance=None):
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    d = oracle.DOT if distance is None else distance
    g = oracle.HNSW(base, d, m=m, ef_construct=48, seed=seed, threads=4)
    entry, lvl, gm, gm0 = g.entry()
    plain = g.export_plain()
    g.close()
    return base, d, plain, entry, lvl, gm, gm0, rng


def _point_levels(plain, n):
    """point_level of every point from a plain links.bin (view.rs:354-369), independently of the checker"""
    hdr = np.frombuffer(plain[:40].tobytes(), np.uint64)
    levels, n_off = int(hdr[1]), int(hdr[3])
    lo = np.frombuffer(plain[64: 64 + 8 * levels].tobytes(), np.uint64).astype(np.int64).tolist() + [n_off - 1]
    reindex = np.frombuffer(plain[64 + 8 * levels: 64 + 8 * levels + 4 * n].tobytes(), np.uint32).astype(np.int64)
    out = np.full(n, levels - 1, np.int64)
    done = np.zeros(n, bool)
    for l in range(1, levels):
        hit = ~done & (reindex >= lo[l + 1] - lo[l])
        out[hit] = l - 1
        done |= hit
    return out


def _sims(oracle, d, ex, row):
    return np.array([oracle.similarity_f32(d, e, row) for e in ex], np.float32)


@pytest.mark.parametrize("algo", [ar.HNSW, ar.ACORN])
def test_unkeyed_traversal_is_the_acorn_checkers(oracle, algo):
    """sum-scores with one positive and no negative scores 0.0 + sim = sim, so the custom checker, unkeyed, must give the nearest-query
    lists, hops and scored points of tests/hnsw_acorn_ref.c on the same graph, filter and entry point"""
    base, d, plain, entry, lvl, gm, gm0, rng = _graph(oracle)
    q = rng.standard_normal((32, 1, base.shape[1])).astype(np.float32)
    f = rng.random(base.shape[0]) >= 0.3
    f[entry] = False
    cg, ag = cr.Graph(plain, gm, gm0, base.shape[0]), ar.Graph(plain, gm, gm0, base.shape[0])
    for filt, top, ef in ((None, 10, 64), (f, 10, 48), (f, 100, 40)):
        got = cr.search_custom_batch(cg, oracle, base, d, q, 2, 1, 0, top, ef, entry, lvl, algo, filt, keyed=False)
        want = ag.search_batch(oracle, base, d, q[:, 0], top, ef, entry, lvl, algo, filt, threads=4)
        for a, b in zip(got, want):
            assert np.array_equal(a, b)
        assert cg.stats()[:2] == ag.stats()[:2]
    cg.close(); ag.close()


@pytest.mark.parametrize("kind,n_a,n_b", [(1, 3, 2), (2, 3, 2), (3, 2, 0), (4, 2, 0), (cr.FEEDBACK, 2, 0)])
def test_custom_scorer_is_the_oracle_fold(oracle, kind, n_a, n_b):
    """ef >= n keeps every scored point in `nearest`, so the list holds all of them: each score is the oracle's fold of its sims"""
    base, d, plain, entry, lvl, gm, gm0, rng = _graph(oracle, n=800)
    ne = cr.n_examples(kind, n_a, n_b)
    ex = rng.standard_normal((3, ne, base.shape[1])).astype(np.float32)
    coef = rng.standard_normal((3, 1 + n_a)).astype(np.float32) if kind == cr.FEEDBACK else None
    cg = cr.Graph(plain, gm, gm0, base.shape[0])
    got = cr.search_custom_batch(cg, oracle, base, d, ex, kind, n_a, n_b, 800, 800, entry, lvl, coef=coef)
    scored = cg.stats()[1]
    assert sum(len(g) for g in got) > 0.5 * scored
    for qi, lst in enumerate(got):
        for p in lst:
            s = _sims(oracle, d, ex[qi], base[p["idx"]])
            if kind == cr.FEEDBACK:
                want = oracle.lib().qo_feedback_score(n_a, float(coef[qi, 0]), coef[qi, 1:].ctypes.data_as(oracle.C.POINTER(oracle.C.c_float)),
                                                      s.ctypes.data_as(oracle.C.POINTER(oracle.C.c_float)), 1)
                want = np.float32(want)
            else:
                want = oracle.custom_combine(kind, n_a, n_b, s[:, None])[0]
            assert np.float32(p["score"]).view(np.uint32) == np.float32(want).view(np.uint32), (kind, qi, p)
    cg.close()


@pytest.mark.parametrize("algo", [ar.HNSW, ar.ACORN])
def test_keyed_equals_default_without_ties(oracle, algo):
    base, d, plain, entry, lvl, gm, gm0, rng = _graph(oracle)
    ex = rng.standard_normal((24, 5, base.shape[1])).astype(np.float32)
    f = rng.random(base.shape[0]) >= 0.3
    f[entry] = False
    cg = cr.Graph(plain, gm, gm0, base.shape[0])
    runs = []
    for keyed in (False, True):
        lists = cr.search_custom_batch(cg, oracle, base, d, ex, 2, 3, 2, 10, 64, entry, lvl, algo, f, keyed=keyed)
        runs.append((lists, cg.stats()[:2]))
    for a, b in zip(runs[0][0], runs[1][0]):
        assert len(np.unique(a["score"])) == len(a)          # tie-free
        assert np.array_equal(a, b)
    assert runs[0][1] == runs[1][1]
    cg.close()


def test_keyed_differs_on_a_context_plateau(oracle):
    """a context pair (p, -p) under Dot: every point with x.p > 0 scores exactly 0.0, half the graph on one plateau"""
    base, d, plain, entry, lvl, gm, gm0, rng = _graph(oracle, n=4000)
    nq = 32
    p = rng.standard_normal((nq, base.shape[1])).astype(np.float32)
    ex = np.stack([p, -p], axis=1)
    cg = cr.Graph(plain, gm, gm0, base.shape[0])
    a = cr.search_custom_batch(cg, oracle, base, d, ex, 4, 1, 0, 20, 32, entry, lvl, keyed=False)
    sa = cg.stats()[:2]
    b = cr.search_custom_batch(cg, oracle, base, d, ex, 4, 1, 0, 20, 32, entry, lvl, keyed=True)
    sb = cg.stats()[:2]
    assert all((x["score"] == 0.0).all() for x in b)
    assert sa != sb or any(not np.array_equal(x["idx"], y["idx"]) for x, y in zip(a, b))
    # keyed: the plateau is ranked by id, so each list is its lowest ids among the points visited
    for x in b:
        assert np.all(np.diff(x["idx"].astype(np.int64)) > 0)
    cg.close()


def test_get_entry_point(oracle):
    base, d, plain, entry, lvl, gm, gm0, rng = _graph(oracle, n=6000, m=4)
    n = base.shape[0]
    levels = _point_levels(plain, n)
    assert levels.max() >= 2
    cg = cr.Graph(plain, gm, gm0, n)
    hi = np.flatnonzero(levels == levels.max())
    mid = np.flatnonzero(levels == 1)[:3]
    low = np.flatnonzero(levels == 0)[:3]
    # the highest level wins, wherever it is in the list
    assert cr.get_entry_point(cg, [low[0], hi[0], mid[0]], entry, lvl) == (hi[0], levels.max(), True)
    # equal top levels: the LAST one wins (Iterator::max_by_key)
    assert cr.get_entry_point(cg, [mid[0], low[0], mid[1], low[1], mid[2]], entry, lvl) == (mid[2], 1, True)
    assert cr.get_entry_point(cg, [low[0], low[1], low[2]], entry, lvl) == (low[2], 0, True)
    # a filtered-out candidate is skipped even if its level is the highest
    f = np.zeros(n, bool)
    f[hi[0]] = True
    assert cr.get_entry_point(cg, [low[0], hi[0], mid[0]], entry, lvl, f) == (mid[0], 1, True)
    # every candidate filtered out: the caller's entry point
    f[[low[0], mid[0]]] = True
    assert cr.get_entry_point(cg, [low[0], hi[0], mid[0]], entry, lvl, f) == (entry, lvl, False)
    assert cr.get_entry_point(cg, [], entry, lvl) == (entry, lvl, False)
    # the search starts there: a list of one custom entry point equals a search from that point and its level
    ex = rng.standard_normal((4, 2, base.shape[1])).astype(np.float32)
    a = cr.search_custom_batch(cg, oracle, base, d, ex, 1, 1, 1, 10, 32, entry, lvl, cep=[[mid[1]]] * 4)
    b = cr.search_custom_batch(cg, oracle, base, d, ex, 1, 1, 1, 10, 32, int(mid[1]), 1)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    cg.close()


@pytest.mark.parametrize("algo", [ar.HNSW, ar.ACORN])
def test_discover_restatement_is_two_checker_calls(oracle, algo):
    """discover() against stage 1 and stage 2 run by hand, stage 2 per query through the callback route with the oracle's scorer"""
    base, d, plain, entry, lvl, gm, gm0, rng = _graph(oracle, n=2500)
    n_pairs = 2
    ex = rng.standard_normal((6, 1 + 2 * n_pairs, base.shape[1])).astype(np.float32)
    f = rng.random(base.shape[0]) >= 0.5
    f[entry] = False
    cg = cr.Graph(plain, gm, gm0, base.shape[0])
    got = cr.discover(cg, oracle, base, d, ex, n_pairs, 10, 40, entry, lvl, algo, f)
    s1 = cr.search_custom_batch(cg, oracle, base, d, ex[:, 1:], 4, n_pairs, 0, 10, 40, entry, lvl, algo, f)
    for qi in range(ex.shape[0]):
        def score(ids, qi=qi):
            return np.array([oracle.custom_combine(3, n_pairs, 0, _sims(oracle, d, ex[qi], base[i])[:, None])[0] for i in ids], np.float32)

        want = cr.search_cb(cg, score, 10, 40, entry, lvl, algo, f, cep=s1[qi]["idx"])
        assert np.array_equal(got[qi], want), qi
    cg.close()
