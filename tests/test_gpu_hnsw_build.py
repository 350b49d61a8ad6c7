"""Device graph build (qb_hnsw_build) vs its CPU restatement (tests/hnsw_build_ref.c, the oracle's HNSW code under the same schedule).
Gate: the device graph is the restated graph exactly — every list on every level, and the exported plain links.bin byte for byte;
with one point per batch it is the serial CPU build (the reference's test_gpu_hnsw_equivalency); a built handle searches like the CPU
traversal of the same graph; the batched graph's recall is within 2 % of the serially built graph's."""
import numpy as np
import pytest

from tests.hnsw_build_ref import PlainGraph, RefGraph
from tests.util import assert_topk_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _levels(n, m, seed):
    u = 1.0 - np.random.default_rng(seed).random(n)
    return np.minimum(np.round(-np.log(u) / np.log(m)), 30).astype(np.uint8)


def _data(qb, oracle, dist, n, dim, seed):
    """the rows as the storage holds them (cosine: normalised, Metric::preprocess), handed to the device and the CPU alike"""
    d = getattr(qb.Distance, dist)
    base = np.random.default_rng(seed).standard_normal((n, dim)).astype(np.float32)
    return d, oracle.preprocess_rows_f32(int(d), base) if d == qb.Distance.Cosine else base


def _same_lists(hg, pg, levels, sample=None):
    ids = np.arange(levels.size, dtype=np.uint32) if sample is None else sample
    for l in range(int(levels.max()) + 1):
        on = ids[levels[ids] >= l]
        got = hg.links(l, on)
        for p, g in zip(on, got):
            assert np.array_equal(g, pg.links(l, int(p))), f"level {l} point {p}"


CASES = [  # dist, dim, n, m, m0, ef_construct, batch, serial_points, deleted fraction
    ("Cosine", 100, 20_000, 16, 32, 100, 512, 256, 0.0),
    ("Euclid", 40, 6_000, 8, 16, 64, 64, 1, 0.0),
    ("Dot", 8, 5_000, 4, 8, 32, 7, 256, 0.0),
    ("Manhattan", 40, 4_000, 8, 16, 48, 64, 256, 0.0),
    ("Cosine", 768, 3_000, 16, 32, 64, 512, 1, 0.0),
    ("Euclid", 100, 4_000, 16, 64, 64, 64, 256, 0.0),
    ("Cosine", 40, 6_000, 8, 16, 64, 7, 16, 0.2),
    ("Dot", 768, 2_000, 4, 8, 16, 1, 1, 0.0),
]


@pytest.mark.parametrize("dist,dim,n,m,m0,ef,batch,serial,dfrac", CASES)
def test_device_build_equals_cpu_restatement(qb, oracle, dist, dim, n, m, m0, ef, batch, serial, dfrac):
    d, stored = _data(qb, oracle, dist, n, dim, 1)
    lv = _levels(n, m, 2)
    deleted = np.random.default_rng(3).random(n) < dfrac if dfrac else None
    st = qb.DenseVectorStorage(stored, d)
    if deleted is not None:
        st.set_deleted(deleted)
    hg = qb.HnswGraph.build(st, m=m, m0=m0, ef_construct=ef, levels=lv, batch=batch, serial_points=serial)
    ref = RefGraph.batched(stored, int(d), m, m0, ef, lv, deleted=deleted, batch=batch, serial_points=serial)
    assert (hg.entry_point, hg.entry_level) == ref.entry()
    want = ref.export_plain()
    got = hg.export_plain()
    assert got.size == want.size and np.array_equal(got, want), f"{dist} dim {dim} batch {batch}: exported graph differs"
    sample = np.random.default_rng(4).choice(n, size=min(n, 3000), replace=False).astype(np.uint32)
    _same_lists(hg, PlainGraph(want), lv, sample)
    # two builds give the same graph
    hg2 = qb.HnswGraph.build(st, m=m, m0=m0, ef_construct=ef, levels=lv, batch=batch, serial_points=serial)
    assert np.array_equal(hg2.export_plain(), want)
    hg2.close(); hg.close(); ref.close(); st.close()


@pytest.mark.parametrize("dist,dim,n,m,serial", [("Cosine", 64, 3_000, 8, 1), ("Euclid", 24, 2_000, 16, 256)])
def test_batch_of_one_is_the_serial_cpu_build(qb, oracle, dist, dim, n, m, serial):
    d, stored = _data(qb, oracle, dist, n, dim, 5)
    lv = _levels(n, m, 6)
    order = np.lexsort((np.arange(n), -lv.astype(np.int64))).astype(np.uint32)
    st = qb.DenseVectorStorage(stored, d)
    hg = qb.HnswGraph.build(st, m=m, ef_construct=48, levels=lv, batch=1, serial_points=serial)
    ref = RefGraph.serial(stored, int(d), m, 2 * m, 48, lv, order=order)
    assert (hg.entry_point, hg.entry_level) == ref.entry()
    assert np.array_equal(hg.export_plain(), ref.export_plain())
    hg.close(); ref.close(); st.close()


def test_built_graph_reloads_and_searches_like_the_cpu(qb, oracle):
    n, dim, m = 8_000, 96, 16
    d, stored = _data(qb, oracle, "Cosine", n, dim, 7)
    lv = _levels(n, m, 8)
    st = qb.DenseVectorStorage(stored, d)
    hg = qb.HnswGraph.build(st, m=m, ef_construct=64, levels=lv, batch=128)
    blob = hg.export_plain()
    again = qb.HnswGraph(st, blob, m, 2 * m)
    _same_lists(again, PlainGraph(blob), lv)
    assert np.array_equal(again.export_plain(), blob)
    ref = RefGraph.batched(stored, int(d), m, 2 * m, 64, lv, batch=128, serial_points=256)
    queries = np.random.default_rng(9).standard_normal((60, dim)).astype(np.float32)
    qp = np.stack([oracle.preprocess_f32(int(d), q) for q in queries])
    for top, ef in ((10, 64), (5, 16)):
        want = ref.search_batch(qp, top, ef)
        for g in (hg, again):
            for i, (a, b) in enumerate(zip(g.search(queries, top, ef, hg.entry_point, hg.entry_level), want)):
                assert_topk_equal(a, b, what=f"top {top} ef {ef} query {i}")
    again.close(); hg.close(); ref.close(); st.close()


def test_recall_against_the_serial_build(qb, oracle):
    n, dim, m, ef = 20_000, 96, 16, 64
    rng = np.random.default_rng(10)
    centers = rng.standard_normal((1000, dim)).astype(np.float32)
    base = (centers[rng.integers(0, 1000, n)] + 0.7 * rng.standard_normal((n, dim))).astype(np.float32)
    queries = (centers[rng.integers(0, 1000, 300)] + 0.7 * rng.standard_normal((300, dim))).astype(np.float32)
    stored = oracle.preprocess_rows_f32(oracle.COSINE, base)
    qp = np.stack([oracle.preprocess_f32(oracle.COSINE, q) for q in queries])
    exact = np.argsort(-(qp @ stored.T), axis=1, kind="stable")[:, :10]
    lv = _levels(n, m, 11)
    st = qb.DenseVectorStorage(stored, qb.Distance.Cosine)
    built = qb.HnswGraph.build(st, m=m, ef_construct=ef, levels=lv, batch=512)
    ser = RefGraph.serial(stored, oracle.COSINE, m, 2 * m, ef, lv)
    e, el = ser.entry()
    serial_g = qb.HnswGraph(st, ser.export_plain(), m, 2 * m)

    def recall(res):
        return float(np.mean([len(set(r["idx"].tolist()) & set(x.tolist())) / 10 for r, x in zip(res, exact)]))

    r_built = recall(built.search(queries, 10, ef, built.entry_point, built.entry_level))
    r_serial = recall(serial_g.search(queries, 10, ef, e, el))
    print(f"recall@10 ef {ef}: device batch-512 graph {r_built:.4f}, serial CPU graph {r_serial:.4f}")
    assert r_built >= 0.98 * r_serial
    serial_g.close(); built.close(); ser.close(); st.close()


def test_rejections_leave_the_device_usable(qb, oracle):
    n, dim = 1_000, 64
    rng = np.random.default_rng(12)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    lv = _levels(n, 8, 13)

    def usable():
        st = qb.DenseVectorStorage(base, qb.Distance.Euclid)
        g = qb.HnswGraph.build(st, m=8, ef_construct=32, levels=lv, batch=64)
        ref = RefGraph.batched(base, oracle.EUCLID, 8, 16, 32, lv, batch=64, serial_points=256)
        assert np.array_equal(g.export_plain(), ref.export_plain())
        g.close(); ref.close(); st.close()

    stores = [
        qb.DenseVectorStorage(base, qb.Distance.Euclid, datatype=qb.VectorStorageDatatype.Float16),
        qb.ScalarQuantizedVectors(np.zeros((n, 4 + dim), np.uint8), dim, 0.01, 0.0, 1.0, qb.Distance.Dot),
        qb.ProductQuantizedVectors(rng.integers(0, 256, (n, dim // 8), dtype=np.uint8), rng.standard_normal((256, dim)).astype(np.float32), 8, dim,
                                   qb.Distance.Euclid),
        qb.BinaryQuantizedVectors(rng.integers(0, 256, (n, dim // 8), dtype=np.uint8), dim, qb.Distance.Dot),
    ]
    for st in stores:
        with pytest.raises(qb.QbError) as e:
            qb.HnswGraph.build(st, m=8, levels=lv)
        assert e.value.status == -3                                           # QB_ERR_UNSUPPORTED
        st.close()
        usable()
    st = qb.DenseVectorStorage(base, qb.Distance.Euclid)
    with pytest.raises(qb.QbError):
        qb.HnswGraph.build(st, m=8, m0=65, levels=lv)                         # m0 > 64
    usable()
    bad = lv.copy(); bad[17] = 31
    with pytest.raises(qb.QbError):
        qb.HnswGraph.build(st, m=8, levels=bad)                               # a level > 30
    usable()
    st.set_deleted(np.ones(n, dtype=bool))
    with pytest.raises(qb.QbError):
        qb.HnswGraph.build(st, m=8, levels=lv)                                # nothing to insert
    st.close()
    usable()
    try:
        empty = qb.DenseVectorStorage(np.zeros((0, dim), np.float32), qb.Distance.Euclid)
    except qb.QbError:
        empty = None                                                          # no empty storage to build over
    if empty is not None:
        with pytest.raises(qb.QbError):
            qb.HnswGraph.build(empty, m=8, levels=np.zeros(0, np.uint8))
        empty.close()
    usable()
