"""CPU checks of the restatement of the device graph build over multivector points (tests/hnsw_build_mv_ref.c), the checker
qb_hnsw_build_multivector is held to.

(a) With one point per batch the batched schedule is the serial MaxSim builder in the sorted order: every list on every level equal.
(b) A batched graph keeps the invariants under deletions: lists <= level_m, no self-links, no duplicates, every link on its level and
    not deleted; a deleted point has no links.
(c) The two-phase rule does not depend on the order the targets are processed in.
(d) With one token per point, MaxSim is the single-vector similarity (no score is -0.0 on these rows), so the graph is the
    single-vector restatement's (tests/hnsw_build_ref.c) over the same rows.
(e) The stored cosine tokens of the fixtures are what Metric::preprocess makes of them again, so the build's internal query (the
    stored rows as they are) is the reference's."""
import numpy as np
import pytest

from tests.hnsw_build_mv_ref import MvRefGraph, PlainGraph, clustered_tokens
from tests.hnsw_build_ref import RefGraph

COSINE, EUCLID, DOT, MANHATTAN = 0, 1, 2, 3


def _levels(n, m, seed):
    u = 1.0 - np.random.default_rng(seed).random(n)
    return np.minimum(np.round(-np.log(u) / np.log(m)), 30).astype(np.uint8)


def _order(levels):
    return np.lexsort((np.arange(levels.size), -levels.astype(np.int64))).astype(np.uint32)


@pytest.mark.parametrize("dist,dim,n,lens,m,m0,ef,serial", [(COSINE, 24, 300, (1, 6), 8, 16, 32, 1), (EUCLID, 40, 250, (0, 5), 4, 8, 16, 64),
                                                            (DOT, 8, 200, (2, 4), 16, 32, 40, 256), (MANHATTAN, 33, 160, (1, 3), 8, 64, 64, 7)])
def test_batch_of_one_is_the_serial_build(oracle, dist, dim, n, lens, m, m0, ef, serial):
    rows, off = clustered_tokens(oracle, dist, n, dim, lens, seed=1)
    lv = _levels(n, m, 2)
    a = MvRefGraph.batched(rows, off, dist, m, m0, ef, lv, batch=1, serial_points=serial)
    b = MvRefGraph.serial(rows, off, dist, m, m0, max(ef, m0), lv, order=_order(lv))
    assert a.entry() == b.entry()
    assert np.array_equal(a.export_plain(), b.export_plain())
    a.close(); b.close()


@pytest.mark.parametrize("dist", [COSINE, EUCLID, DOT, MANHATTAN])
def test_invariants_with_deletions(oracle, dist):
    n, m, m0 = 400, 6, 12
    rows, off = clustered_tokens(oracle, dist, n, 16, (0, 7), seed=3, empty=0.05)
    lv = _levels(n, m, 4)
    deleted = np.random.default_rng(5).random(n) < 0.2
    g = MvRefGraph.batched(rows, off, dist, m, m0, 24, lv, deleted=deleted, batch=16, serial_points=20)
    pg = PlainGraph(g.export_plain())
    entry, _ = g.entry()
    assert not deleted[entry]
    for p in range(n):
        assert pg.point_level[p] == lv[p]
        for lvl in range(int(lv[p]) + 1):
            links = pg.links(lvl, p)
            if deleted[p]:
                assert links.size == 0
                continue
            assert links.size <= (m0 if lvl == 0 else m)
            assert p not in links and np.unique(links).size == links.size
            assert all(lv[q] >= lvl and not deleted[q] for q in links)
    g.close()


def test_target_order_does_not_matter(oracle):
    rows, off = clustered_tokens(oracle, COSINE, 500, 12, (1, 5), seed=6)
    lv = _levels(500, 8, 7)
    a = MvRefGraph.batched(rows, off, COSINE, 8, 16, 32, lv, batch=32, serial_points=8)
    b = MvRefGraph.batched(rows, off, COSINE, 8, 16, 32, lv, batch=32, serial_points=8, shuffle=12345)
    assert np.array_equal(a.export_plain(), b.export_plain())
    a.close(); b.close()


@pytest.mark.parametrize("dist", [COSINE, EUCLID, DOT, MANHATTAN])
def test_one_token_per_point_is_the_single_vector_build(oracle, dist):
    n, dim = 600, 20
    rng = np.random.default_rng(8)
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    rows = oracle.preprocess_rows_f32(dist, rows) if dist == COSINE else rows
    lv = _levels(n, 8, 9)
    a = MvRefGraph.batched(rows, np.arange(n + 1, dtype=np.uint32), dist, 8, 16, 32, lv, batch=40, serial_points=30)
    b = RefGraph.batched(rows, dist, 8, 16, 32, lv, batch=40, serial_points=30)
    assert a.entry() == b.entry()
    assert np.array_equal(a.export_plain(), b.export_plain())
    a.close(); b.close()


def test_fixture_cosine_tokens_are_already_preprocessed(oracle):
    for n, dim, lens, seed in ((300, 24, (1, 6), 1), (500, 12, (1, 5), 6), (64, 128, (0, 120), 11)):
        rows, _ = clustered_tokens(oracle, COSINE, n, dim, lens, seed=seed)
        again = oracle.preprocess_rows_f32(COSINE, rows)
        assert np.array_equal(again.view(np.uint32), rows.view(np.uint32))
