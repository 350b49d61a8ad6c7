"""The keyed build restatements (tests/hnsw_build_ref.c and tests/hnsw_build_incr_ref.c over tests/hnsw_keyed_oracle.c, driven by
tests/hnsw_build_keyed_ref.py), which check the device builds over Uint8 storages: on tie-free f32 data they build and heal exactly the
graphs of the score-only restatements the f32 device builds are checked with, and on tie-heavy u8 data (tests/hnsw_build_u8_ref.c) they
build other graphs, so the tie order is exercised.  No GPU."""
import numpy as np
import pytest

from tests import hnsw_build_keyed_ref as kr
from tests.hnsw_build_incr_ref import GONE, build_incremental
from tests.hnsw_build_ref import RefGraph


def _levels(rng, n, m):
    return np.minimum(np.round(-np.log(1.0 - rng.random(n)) / np.log(m)), 30).astype(np.uint8)


def _incremental_case(rng, rows_old, new_extra):
    n_old = rows_old.shape[0]
    keep = rng.random(n_old) >= 0.15
    o2n = np.full(n_old, GONE, np.uint32)
    o2n[keep] = np.arange(int(keep.sum()), dtype=np.uint32)
    return o2n, keep, np.concatenate([rows_old[keep], new_extra])


@pytest.mark.parametrize("dist_name", ["COSINE", "EUCLID", "DOT", "MANHATTAN"])
def test_keyed_equals_score_only_on_f32(oracle, dist_name):
    dist = getattr(oracle, dist_name)
    rng = np.random.default_rng(21)
    n, dim = 1200, 24
    x = rng.standard_normal((n, dim)).astype(np.float32)
    base = oracle.preprocess_rows_f32(dist, x) if dist == oracle.COSINE else x
    lv = _levels(rng, n, 8)
    for batch, serial_points in ((1, 1), (64, 32)):
        a = RefGraph.batched(base, dist, 8, 16, 32, lv, batch=batch, serial_points=serial_points)
        b = kr.batched(base, dist, 8, 16, 32, lv, batch=batch, serial_points=serial_points, dtype="f32")
        assert np.array_equal(a.export_plain(), b.export_plain()) and a.entry() == b.entry()
        b.close()
    s = RefGraph.serial(base, dist, 8, 16, 32, lv)
    sk = kr.serial(base, dist, 8, 16, 32, lv, dtype="f32")
    assert np.array_equal(s.export_plain(), sk.export_plain())
    s.close(); sk.close()
    extra = rng.standard_normal((300, dim)).astype(np.float32)
    o2n, keep, new_base = _incremental_case(rng, base, oracle.preprocess_rows_f32(dist, extra) if dist == oracle.COSINE else extra)
    nl = np.concatenate([lv[keep], _levels(rng, 300, 8)])
    g0, e0 = build_incremental(base, a.export_plain(), dist, 8, 16, new_base, o2n, nl, ef_construct=32, batch=64, serial_points=32)
    g1, e1 = kr.build_incremental(base, a.export_plain(), dist, 8, 16, new_base, o2n, nl, ef_construct=32, batch=64, serial_points=32, dtype="f32")
    assert e0 == e1 and np.array_equal(g0.export_plain(), g1.export_plain())
    g0.close(); g1.close(); a.close()


@pytest.mark.parametrize("dim", [96, 20])
@pytest.mark.parametrize("dist_name", ["COSINE", "EUCLID", "DOT", "MANHATTAN"])
def test_keyed_differs_on_tie_heavy_u8(oracle, dist_name, dim):
    dist = getattr(oracle, dist_name)
    rng = np.random.default_rng(23)
    n = 1000
    rows = rng.integers(0, 2, (n, dim), dtype=np.uint8)
    rows[4::5] = rows[rng.integers(0, n // 2, n // 5)]
    lv = _levels(rng, n, 8)
    k = kr.batched(rows, dist, 8, 16, 32, lv, batch=64, serial_points=32)
    u = kr.batched(rows, dist, 8, 16, 32, lv, batch=64, serial_points=32, keyed=False)
    assert not np.array_equal(k.export_plain(), u.export_plain())
    o2n, keep, new_rows = _incremental_case(rng, rows, rng.integers(0, 2, (200, dim), dtype=np.uint8))
    nl = np.concatenate([lv[keep], _levels(rng, 200, 8)])
    gk, _ = kr.build_incremental(rows, k.export_plain(), dist, 8, 16, new_rows, o2n, nl, ef_construct=32, batch=64, serial_points=32)
    gu, _ = kr.build_incremental(rows, k.export_plain(), dist, 8, 16, new_rows, o2n, nl, ef_construct=32, batch=64, serial_points=32, keyed=False)
    assert not np.array_equal(gk.export_plain(), gu.export_plain())
    gk.close(); gu.close(); k.close(); u.close()
