"""CPU checks of the restatement of the device graph build (tests/hnsw_build_ref.c), the checker qb_hnsw_build is held to.

(a) With one point per batch the batched schedule is the serial builder in the sorted order, whatever the serial prefix (the
    reference's own equivalence claim, test_gpu_hnsw_equivalency, gpu_graph_builder.rs:164-183): every list on every level equal.
(b) The serial builder with the levels qo_hnsw_build drew, in id order, is qo_hnsw_build with one thread: byte-equal links.bin.
(c) A batched graph keeps the invariants: lists <= level_m, no self-links, no duplicates, every link on its level and not deleted.
(d) The two-phase rule does not depend on the order the targets are processed in."""
import numpy as np
import pytest

from tests.hnsw_build_ref import PlainGraph, RefGraph

COSINE, EUCLID, DOT, MANHATTAN = 0, 1, 2, 3


def _levels(n, m, seed):
    rng = np.random.default_rng(seed)
    u = 1.0 - rng.random(n)
    return np.minimum(np.round(-np.log(u) / np.log(m)), 30).astype(np.uint8)


def _order(levels):
    return np.lexsort((np.arange(levels.size), -levels.astype(np.int64))).astype(np.uint32)


def _data(n, dim, dist, seed, oracle):
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    return oracle.preprocess_rows_f32(dist, base) if dist == COSINE else base


@pytest.mark.parametrize("dist,dim,n,m,m0,ef,serial", [(COSINE, 24, 1500, 8, 16, 32, 1), (EUCLID, 40, 1200, 4, 8, 16, 64),
                                                       (DOT, 8, 1000, 16, 32, 40, 256), (MANHATTAN, 33, 800, 8, 64, 64, 7)])
def test_batch_of_one_is_the_serial_build(oracle, dist, dim, n, m, m0, ef, serial):
    base = _data(n, dim, dist, 1, oracle)
    lv = _levels(n, m, 2)
    a = RefGraph.batched(base, dist, m, m0, ef, lv, batch=1, serial_points=serial)
    b = RefGraph.serial(base, dist, m, m0, max(ef, m0), lv, order=_order(lv))
    assert a.entry() == b.entry()
    ea, eb = a.export_plain(), b.export_plain()
    assert np.array_equal(ea, eb)
    ga = PlainGraph(ea)
    assert ga.levels == int(lv.max()) + 1
    a.close(); b.close()


@pytest.mark.parametrize("dist,m", [(COSINE, 16), (EUCLID, 8)])
def test_serial_levels_equal_the_oracle_builder(oracle, dist, m):
    base = _data(1200, 32, dist, 3, oracle)
    o = RefGraph.oracle_build(base, dist, m, 40, seed=11)
    lv = o.levels()
    s = RefGraph.serial(base, dist, m, 2 * m, 40, lv)
    assert o.entry() == s.entry()
    assert np.array_equal(o.export_plain(), s.export_plain())
    o.close(); s.close()


@pytest.mark.parametrize("batch,serial,deleted_frac", [(7, 1, 0.0), (64, 256, 0.1), (512, 16, 0.3)])
def test_batched_invariants(oracle, batch, serial, deleted_frac):
    n, m, m0 = 3000, 8, 16
    base = _data(n, 20, COSINE, 4, oracle)
    lv = _levels(n, m, 5)
    rng = np.random.default_rng(6)
    deleted = rng.random(n) < deleted_frac
    g = RefGraph.batched(base, COSINE, m, m0, 32, lv, deleted=deleted if deleted_frac else None, batch=batch, serial_points=serial)
    pg = PlainGraph(g.export_plain())
    entry, elev = g.entry()
    assert not deleted[entry] and elev == int(lv[~deleted].max())
    assert np.array_equal(pg.point_level, lv.astype(np.int64))
    n_links = 0
    for p in range(n):
        for l in range(int(lv[p]) + 1):
            k = pg.links(l, p)
            n_links += k.size
            assert k.size <= (m0 if l == 0 else m)
            assert p not in k and np.unique(k).size == k.size
            if k.size:
                assert (lv[k] >= l).all() and not deleted[k].any()
            if deleted[p]:
                assert k.size == 0
    assert n_links > n * m // 2
    g.close()


def test_target_order_does_not_matter(oracle):
    n = 2500
    base = _data(n, 16, EUCLID, 7, oracle)
    lv = _levels(n, 8, 8)
    ref = RefGraph.batched(base, EUCLID, 8, 16, 24, lv, batch=64, serial_points=32).export_plain()
    for seed in (1, 2, 3):
        g = RefGraph.batched(base, EUCLID, 8, 16, 24, lv, batch=64, serial_points=32, shuffle=seed)
        assert np.array_equal(g.export_plain(), ref)
        g.close()
