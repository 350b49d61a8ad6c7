"""Device graph build over multivector points (qb_hnsw_build_multivector) vs its CPU restatement (tests/hnsw_build_mv_ref.c: the
oracle's HNSW code under qb_hnsw_build's schedule, every pair score the oracle's MaxSim): the same links.bin byte for byte and the same
entry point, across the four distances, build shapes, token runs of 0 up to a query larger than the 48 KB staging, and deleted points.
The built handle searches like a loaded multivector graph, and its recall is close to that of a graph over mean tokens."""
import numpy as np
import pytest

from tests import hnsw_custom_ref as cr
from tests import hnsw_maxsim_ref as mr
from tests.hnsw_build_mv_ref import MvRefGraph, clustered_tokens

pytestmark = pytest.mark.gpu

COSINE, EUCLID, DOT, MANHATTAN = 0, 1, 2, 3
_DIST = {COSINE: "Cosine", EUCLID: "Euclid", DOT: "Dot", MANHATTAN: "Manhattan"}


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _levels(n, m, seed):
    u = 1.0 - np.random.default_rng(seed).random(n)
    return np.minimum(np.round(-np.log(u) / np.log(max(m, 2))), 30).astype(np.uint8)


def _build_both(qb, oracle, dist, rows, off, m, m0, ef, batch, serial, lv, deleted=None):
    st = qb.DenseVectorStorage(rows, getattr(qb.Distance, _DIST[dist]))
    view = qb.MultiVectorView(st, off)
    g = qb.HnswGraph.build_multivector(view, m=m, m0=m0, ef_construct=ef, levels=lv, batch=batch, serial_points=serial, point_deleted=deleted)
    ref = MvRefGraph.batched(rows, off, dist, m, m0, ef, lv, deleted=deleted, batch=batch or 512, serial_points=serial or 256)
    return st, view, g, ref


# (distance, dim, points, token runs, m, m0, ef_construct, batch, serial_points, empty share, deleted share).  A point with no token rows
# scores -inf as a candidate and +0.0 against everything as the query, so such points make equal scores.  The device orders them by id,
# the oracle's heaps by arrival; the two graphs are the same whenever equal scores never compete for the last places of a full beam,
# which ef_construct >= points guarantees, so the cases with empty points use it.
CASES = [
    (COSINE, 64, 1500, (1, 8), 8, 16, 32, 64, 32, 0.0, 0.0),
    (EUCLID, 40, 300, (0, 6), 16, 32, 300, 128, 0, 0.05, 0.0),
    (DOT, 8, 800, (1, 5), 6, 12, 20, 1, 1, 0.0, 0.0),
    (MANHATTAN, 33, 700, (2, 4), 12, 64, 80, 0, 0, 0.0, 0.0),
    (COSINE, 128, 90, (0, 120), 8, 16, 96, 16, 4, 0.05, 0.0),      # a query of 120 x 512 B: read in place, not staged
    (DOT, 48, 1200, (1, 10), 10, 20, 40, 100, 50, 0.0, 0.15),
    (EUCLID, 16, 600, (1, 3), 1, 1, 1, 32, 8, 0.0, 0.3),
]


@pytest.mark.parametrize("dist,dim,n,lens,m,m0,ef,batch,serial,empty,dfrac", CASES)
def test_device_build_equals_cpu_restatement(qb, oracle, dist, dim, n, lens, m, m0, ef, batch, serial, empty, dfrac):
    rows, off = clustered_tokens(oracle, dist, n, dim, lens, seed=n + dim, empty=empty)
    lv = _levels(n, m, 3)
    deleted = (np.random.default_rng(4).random(n) < dfrac) if dfrac else None
    st, view, g, ref = _build_both(qb, oracle, dist, rows, off, m, m0, ef, batch, serial, lv, deleted)
    assert (g.entry_point, g.entry_level) == ref.entry()
    got = g.export_plain()
    assert np.array_equal(got, ref.export_plain())
    again = qb.HnswGraph.build_multivector(view, m=m, m0=m0, ef_construct=ef, levels=lv, batch=batch, serial_points=serial, point_deleted=deleted)
    assert np.array_equal(again.export_plain(), got)                    # two builds are identical
    again.close(); g.close(); ref.close(); st.close()


@pytest.mark.parametrize("dist,dim", [(COSINE, 48), (EUCLID, 20), (DOT, 64), (MANHATTAN, 33)])
def test_one_token_per_point_is_the_single_vector_build(qb, oracle, dist, dim):
    n, m = 2000, 8
    rows = np.random.default_rng(5).standard_normal((n, dim)).astype(np.float32)
    rows = oracle.preprocess_rows_f32(dist, rows) if dist == COSINE else rows
    lv = _levels(n, m, 6)
    st = qb.DenseVectorStorage(rows, getattr(qb.Distance, _DIST[dist]))
    mv = qb.HnswGraph.build_multivector(qb.MultiVectorView(st, np.arange(n + 1, dtype=np.uint32)), m=m, ef_construct=32, levels=lv, batch=64)
    sv = qb.HnswGraph.build(st, m=m, ef_construct=32, levels=lv, batch=64)
    assert (mv.entry_point, mv.entry_level) == (sv.entry_point, sv.entry_level)
    assert np.array_equal(mv.export_plain(), sv.export_plain())
    mv.close(); sv.close(); st.close()


def _mean_token_graph(qb, oracle, st, rows, off, m, ef, lv):
    """today's stand-in: qb_hnsw_build over each point's normalised mean token, bound to the token storage"""
    n = off.size - 1
    runs = np.diff(off)
    means = np.stack([rows[off[p]:off[p + 1]].mean(0) if runs[p] else np.zeros(rows.shape[1], np.float32) for p in range(n)]).astype(np.float32)
    means = oracle.preprocess_rows_f32(oracle.COSINE, means)
    ms = qb.DenseVectorStorage(means, qb.Distance.Cosine)
    mg = qb.HnswGraph.build(ms, m=m, ef_construct=ef, levels=lv, batch=256)
    blob, e, el = mg.export_plain(), mg.entry_point, mg.entry_level
    mg.close(); ms.close()
    return qb.HnswGraph.multivector(qb.MultiVectorView(st, off), blob, m, 2 * m), e, el


def test_built_graph_searches_like_the_cpu_and_recalls_like_mean_tokens(qb, oracle):
    n, dim, m, ef_c = 3000, 32, 16, 100
    rows, off = clustered_tokens(oracle, COSINE, n, dim, (1, 12), seed=21)
    lv = _levels(n, m, 22)
    st, view, g, ref = _build_both(qb, oracle, COSINE, rows, off, m, 2 * m, ef_c, 256, 64, lv)
    blob = g.export_plain()
    assert np.array_equal(blob, ref.export_plain())
    cg = cr.Graph(blob, m, 2 * m, n)
    rng = np.random.default_rng(23)
    # queries that resemble stored points: a random point's token rows plus noise
    queries = [(rows[off[p]:off[p + 1]] + 0.5 * rng.standard_normal((int(off[p + 1] - off[p]), dim))).astype(np.float32)
               for p in rng.integers(0, n, 48)]
    keep = rng.random(n) < 0.3
    keep[g.entry_point] = True
    for algo, filtered in (("hnsw", None), ("acorn", ~keep)):
        want = []
        cg.stats(reset=True)
        for q in queries:
            sc = mr.point_scores_f32(oracle, COSINE, rows, off, q)
            want.append(cr.search_cb(cg, mr.scorer(sc), 10, 48, g.entry_point, g.entry_level, cr.ACORN if algo == "acorn" else cr.HNSW, filtered,
                                     keyed=True))
        g.stats(reset=True)
        got = g.search_maxsim(queries, 10, 48, g.entry_point, g.entry_level, point_deleted=filtered, algorithm=algo)
        assert g.stats() == cg.stats()[:2]
        for a, b in zip(got, want):
            assert np.array_equal(a["idx"], b["idx"]) and np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)), (algo, a, b)
    cg.close()

    # recall@10 at ef = 128 against the brute-force MaxSim search, next to the mean-token graph over the same points
    exact = [view.search(q, 10)["idx"] for q in queries]
    mean_g, me, ml = _mean_token_graph(qb, oracle, st, rows, off, m, ef_c, lv)

    def recall(res):
        return float(np.mean([len(set(r["idx"].tolist()) & set(x.tolist())) / 10 for r, x in zip(res, exact)]))

    r_built = recall(g.search_maxsim(queries, 10, 128, g.entry_point, g.entry_level))
    r_mean = recall(mean_g.search_maxsim(queries, 10, 128, me, ml))
    print(f"recall@10 ef 128: MaxSim-built graph {r_built:.4f}, mean-token graph {r_mean:.4f}")
    # on these points (each point's tokens share one cluster, which suits the mean-token stand-in) the two are close: measured on an H100
    # 80GB HBM3 at 700 W, 0.9958 for the MaxSim-built graph and 0.9979 for the mean-token graph
    assert r_built >= 0.98 and r_built >= r_mean - 0.01
    mean_g.close(); g.close(); ref.close(); st.close()


def test_rejections_leave_the_device_usable(qb, oracle):
    n, dim, m = 400, 32, 8
    rows, off = clustered_tokens(oracle, EUCLID, n, dim, (1, 4), seed=31)
    lv = _levels(n, m, 32)

    def usable():
        st, _, g, ref = _build_both(qb, oracle, EUCLID, rows, off, m, 16, 32, 64, 16, lv)
        assert np.array_equal(g.export_plain(), ref.export_plain())
        g.close(); ref.close(); st.close()

    def rejects(status, view, **kw):
        args = dict(m=m, ef_construct=32, levels=lv)
        args.update(kw)
        with pytest.raises(qb.QbError) as e:
            qb.HnswGraph.build_multivector(view, **args)
        assert e.value.status == status, e.value
        usable()

    UNSUPPORTED, INVALID = -3, -1
    nr = int(off[-1])
    rng = np.random.default_rng(33)
    stores = [
        qb.DenseVectorStorage(rows, qb.Distance.Euclid, datatype=qb.VectorStorageDatatype.Float16),
        qb.DenseVectorStorage(np.clip(np.round(np.abs(rows) * 40), 0, 255).astype(np.float32), qb.Distance.Euclid, datatype=qb.VectorStorageDatatype.Uint8),
        qb.ScalarQuantizedVectors(np.zeros((nr, 4 + dim), np.uint8), dim, 0.01, 0.0, 1.0, qb.Distance.Dot),
        qb.ProductQuantizedVectors(rng.integers(0, 256, (nr, dim // 8), dtype=np.uint8), rng.standard_normal((256, dim)).astype(np.float32), 8, dim,
                                   qb.Distance.Euclid),
        qb.BinaryQuantizedVectors(rng.integers(0, 256, (nr, dim // 8), dtype=np.uint8), dim, qb.Distance.Dot),
    ]
    for s in stores:
        rejects(UNSUPPORTED, qb.MultiVectorView(s, off))
        s.close()
    st = qb.DenseVectorStorage(rows, qb.Distance.Euclid)
    view = qb.MultiVectorView(st, off)
    rejects(UNSUPPORTED, view, m=65)
    rejects(UNSUPPORTED, view, m0=65)
    rejects(UNSUPPORTED, view, ef_construct=4097)
    bad = lv.copy(); bad[17] = 31
    rejects(INVALID, view, levels=bad)                                          # a level > 30
    down = off.copy(); down[5] = down[6] + 1
    rejects(INVALID, qb.MultiVectorView(st, down))                              # offsets not ascending
    past = off.copy(); past[-1] = nr + 1
    rejects(INVALID, qb.MultiVectorView(st, past))                              # beyond the stored rows
    rejects(INVALID, qb.MultiVectorView(st, np.zeros(1, np.uint32)), levels=np.zeros(0, np.uint8))   # no points
    rejects(INVALID, view, point_deleted=np.ones(n, dtype=bool))                # every point deleted
    st.close()
