"""Incremental device graph build (qb_hnsw_build_incremental) vs its CPU restatement (tests/hnsw_build_incr_ref.c: the oracle's HNSW
code under the same heal, renumbering and schedule).  The device graph is the restated graph exactly: the exported plain links.bin
byte for byte and the entry point, over the four distances, both scoring chains, old graphs from the device build, the oracle's builder
and a compressed links.bin, identity / permuted / compacted mappings, deletions from none to a whole cluster (deep searches, and the
stack-overflow rerun), new points from none to many (levels above the old top too), resident-deleted points and batch sizes 1 to 512.
Also: two runs agree, every rejected input leaves the device usable, the result searches like the CPU traversal of the same graph, and
its recall is within 0.01 of a from-scratch build's."""
import numpy as np
import pytest

from tests import graph_links_compressed as gl
from tests.hnsw_build_incr_ref import GONE, build_incremental
from tests.hnsw_build_ref import RefGraph
from tests.util import assert_topk_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _levels(n, m, seed):
    u = 1.0 - np.random.default_rng(seed).random(n)
    return np.minimum(np.round(-np.log(u) / np.log(max(m, 2))), 30).astype(np.uint8)


def _clustered(n, dim, seed, k=20):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((k, dim)).astype(np.float32) * 3
    lab = rng.integers(0, k, n)
    return (centres[lab] + rng.standard_normal((n, dim)).astype(np.float32)).astype(np.float32), lab


def _stored(qb, oracle, d, x):
    return oracle.preprocess_rows_f32(int(d), x) if d == qb.Distance.Cosine else x


def _run(qb, oracle, dist, dim, n, m, m0, ef, source, mapping, gone, n_new, high, resident, batch, serial, seed=1, stack=0):
    d = getattr(qb.Distance, dist)
    x, lab = _clustered(n + n_new, dim, seed)
    rows = _stored(qb, oracle, d, x)
    old_rows, fresh = rows[:n], rows[n:]
    lv = _levels(n, m, seed + 1)
    old_st = qb.DenseVectorStorage(old_rows, d)
    if source == "oracle":   # the oracle's own serial builder (m0 = 2m, its own levels), loaded plain
        ref = RefGraph.oracle_build(old_rows, int(d), m, ef, seed=seed)
        lv = ref.levels()
        old = qb.HnswGraph(old_st, ref.export_plain(), m, m0)
        ref.close()
    else:
        old = qb.HnswGraph.build(old_st, m=m, m0=m0, ef_construct=ef, levels=lv, batch=64, serial_points=32)
        if source == "compressed":   # the same graph through the compressed links.bin, whose lists are stored in another order
            blob = gl.plain_to_compressed(old.export_plain(), m, m0)
            old.close()
            old = qb.HnswGraph.from_compressed(old_st, blob)
    rng = np.random.default_rng(seed + 2)
    if gone == "cluster":
        dead = lab[:n] == lab[0]
    else:
        dead = rng.random(n) < gone
    keep = np.flatnonzero(~dead)
    ids = np.arange(keep.size + n_new)
    if mapping == "permutation":
        ids = rng.permutation(ids)
    o2n = np.full(n, GONE, dtype=np.uint32)
    o2n[keep] = ids[:keep.size]
    n_tot = keep.size + n_new
    new_rows = np.zeros((n_tot, dim), np.float32)
    new_rows[ids[:keep.size]] = old_rows[keep]
    new_rows[ids[keep.size:]] = fresh
    nlv = np.zeros(n_tot, np.uint8)
    nlv[ids[:keep.size]] = lv[keep]
    add = _levels(n_new, m, seed + 3)
    if high and n_new:
        add[: min(3, n_new)] = int(lv.max()) + np.array([1, 3, 2])[: min(3, n_new)]
    nlv[ids[keep.size:]] = add
    deleted = None
    if resident and n_new:
        deleted = np.zeros(n_tot, bool)
        deleted[ids[keep.size:][rng.random(n_new) < 0.2]] = True
    st = qb.DenseVectorStorage(new_rows, d)
    if deleted is not None:
        st.set_deleted(deleted)
    if stack:
        qb.set_option("hnsw_heal_stack", stack)
    try:
        hg = qb.HnswGraph.build_incremental(st, old, o2n, ef_construct=ef, levels=nlv, batch=batch, serial_points=serial)
    finally:
        if stack:
            qb.set_option("hnsw_heal_stack", 0)
    cpu, entry = build_incremental(old_rows, old.export_plain(), int(d), m, m0, new_rows, o2n, nlv, ef_construct=ef, deleted=deleted, batch=batch,
                                   serial_points=serial)
    return dict(hg=hg, cpu=cpu, entry=entry, st=st, old=old, old_st=old_st, rows=new_rows, o2n=o2n, nlv=nlv, d=d)


def _close(r):
    r["hg"].close(); r["cpu"].close(); r["old"].close(); r["st"].close(); r["old_st"].close()


CASES = [  # dist, dim, n, m, m0, ef, source, mapping, gone, new, high, resident, batch, serial
    ("Cosine", 100, 4000, 16, 32, 64, "device", "identity", 0.0, 0, False, False, 512, 256),
    ("Cosine", 100, 4000, 16, 32, 64, "device", "compact", 0.1, 400, False, False, 512, 256),
    ("Euclid", 20, 3000, 8, 16, 32, "oracle", "compact", 0.01, 1, False, True, 64, 256),
    ("Dot", 8, 3000, 4, 8, 16, "device", "permutation", 0.3, 257, True, False, 7, 256),
    ("Manhattan", 32, 2500, 8, 12, 48, "compressed", "compact", 0.1, 255, False, True, 7, 256),
    ("Cosine", 768, 1500, 8, 16, 32, "device", "compact", 0.1, 300, True, True, 64, 16),
    ("Euclid", 100, 3000, 8, 24, 40, "compressed", "permutation", "cluster", 500, False, False, 512, 1),
    ("Dot", 32, 2000, 8, 16, 32, "oracle", "permutation", 0.1, 2000, True, True, 1, 1),
    ("Manhattan", 8, 3000, 16, 32, 64, "device", "compact", 0.01, 3000, False, False, 512, 256),
    ("Cosine", 20, 3000, 8, 16, 32, "device", "compact", 0.0, 600, True, False, 64, 256),
]


@pytest.mark.parametrize("dist,dim,n,m,m0,ef,source,mapping,gone,new,high,resident,batch,serial", CASES)
def test_device_incremental_equals_cpu_restatement(qb, oracle, dist, dim, n, m, m0, ef, source, mapping, gone, new, high, resident, batch, serial):
    r = _run(qb, oracle, dist, dim, n, m, m0, ef, source, mapping, gone, new, high, resident, batch, serial)
    want = r["cpu"].export_plain()
    got = r["hg"].export_plain()
    assert (r["hg"].entry_point, r["hg"].entry_level) == r["entry"]
    assert got.size == want.size and np.array_equal(got, want), f"{dist} dim {dim} {source} {mapping} gone {gone} new {new}: graph differs"
    _close(r)


@pytest.mark.parametrize("dist,dim,stack", [("Cosine", 40, 8), ("Euclid", 768, 64)])
def test_deep_heal_reruns_with_a_larger_stack(qb, oracle, dist, dim, stack):
    """a whole cluster gone: deep searches through gone points; a tiny first stack sends items through the rerun path"""
    r = _run(qb, oracle, dist, dim, 3000, 8, 16, 32, "device", "compact", "cluster", 200, False, False, 64, 256, seed=4, stack=stack)
    assert np.array_equal(r["hg"].export_plain(), r["cpu"].export_plain())
    assert (r["hg"].entry_point, r["hg"].entry_level) == r["entry"]
    _close(r)


def test_two_runs_are_identical(qb, oracle):
    r = _run(qb, oracle, "Cosine", 64, 4000, 16, 32, 64, "device", "permutation", 0.1, 400, True, True, 512, 256)
    again = qb.HnswGraph.build_incremental(r["st"], r["old"], r["o2n"], ef_construct=64, levels=r["nlv"], batch=512, serial_points=256)
    assert np.array_equal(again.export_plain(), r["hg"].export_plain())
    again.close()
    _close(r)


def test_search_equals_cpu_traversal(qb, oracle):
    r = _run(qb, oracle, "Euclid", 48, 4000, 16, 32, 64, "device", "compact", 0.1, 400, False, False, 512, 256)
    q = np.random.default_rng(21).standard_normal((64, 48)).astype(np.float32)
    got = r["hg"].search(q, 10, 64, r["hg"].entry_point, r["hg"].entry_level)
    want = r["cpu"].search_batch(q, 10, 64)
    for g, w in zip(got, want):
        assert_topk_equal(g, w)
    _close(r)


def test_recall_is_that_of_a_full_build(qb, oracle):
    """clustered cosine data as the project's C5 setup makes it (centres plus 0.5 noise), 10 % deleted and 10 % new: recall@10 at ef 128
    within 0.01 of qb_hnsw_build over the same storage"""
    rng = np.random.default_rng(7)
    centres = rng.standard_normal((256, 64)).astype(np.float32)
    x = centres[rng.integers(0, 256, 22000)] + 0.5 * rng.standard_normal((22000, 64), dtype=np.float32)
    d = qb.Distance.Cosine
    rows0 = _stored(qb, oracle, d, x)
    lv0 = _levels(20000, 16, 8)
    old_st = qb.DenseVectorStorage(rows0[:20000], d)
    old = qb.HnswGraph.build(old_st, m=16, ef_construct=100, levels=lv0)
    keep = np.flatnonzero(rng.random(20000) >= 0.1)
    o2n = np.full(20000, GONE, np.uint32)
    o2n[keep] = np.arange(keep.size, dtype=np.uint32)
    rows = np.concatenate([rows0[keep], rows0[20000:]])
    nlv = np.concatenate([lv0[keep], _levels(2000, 16, 9)])
    st = qb.DenseVectorStorage(rows, d)
    hg = qb.HnswGraph.build_incremental(st, old, o2n, ef_construct=100, levels=nlv)
    full = qb.HnswGraph.build(st, m=16, ef_construct=100, levels=nlv)
    q = _stored(qb, oracle, d, centres[rng.integers(0, 256, 1000)] + 0.5 * rng.standard_normal((1000, 64), dtype=np.float32))
    exact = np.argsort(-(q @ rows.T), axis=1)[:, :10]

    def recall(g):
        res = g.search(q, 10, 128, g.entry_point, g.entry_level)
        return np.mean([len(set(int(i) for i in x["idx"]) & set(e.tolist())) / 10 for x, e in zip(res, exact)])

    ri, rf = recall(hg), recall(full)
    assert ri >= rf - 0.01, (ri, rf)
    full.close(); hg.close(); st.close(); old.close(); old_st.close()


def test_rejections_leave_the_device_usable(qb, oracle):
    from qdrant_b200._capi import QB_ERR_INVALID as INVALID, QB_ERR_UNSUPPORTED as UNSUPPORTED, QbError

    d = qb.Distance.Euclid
    x = np.random.default_rng(1).standard_normal((600, 16)).astype(np.float32)
    lv = _levels(600, 8, 2)
    st = qb.DenseVectorStorage(x, d)
    old = qb.HnswGraph.build(st, m=8, m0=16, ef_construct=32, levels=lv)
    ident = np.arange(600, dtype=np.uint32)

    def status(fn):
        with pytest.raises(QbError) as e:
            fn()
        return e.value.status

    inc = qb.HnswGraph.build_incremental
    o = ident.copy(); o[3] = 600
    assert status(lambda: inc(st, old, o, 32, levels=lv)) == INVALID                    # target out of range
    o = ident.copy(); o[3] = 4
    assert status(lambda: inc(st, old, o, 32, levels=lv)) == INVALID                    # two old points on one target
    assert status(lambda: inc(st, old, np.full(600, GONE, np.uint32), 32, levels=lv)) == INVALID   # nothing mapped
    bad = lv.copy(); bad[5] += 1
    assert status(lambda: inc(st, old, ident, 32, levels=bad)) == INVALID               # a reused point's level changed
    bad = lv.copy(); bad[5] = 31
    assert status(lambda: inc(st, old, ident, 32, levels=bad)) == INVALID               # level > 30
    dl = np.zeros(600, bool); dl[7] = True
    st.set_deleted(dl)
    assert status(lambda: inc(st, old, ident, 32, levels=lv)) == INVALID                # target deleted
    st.set_deleted(None)
    assert status(lambda: inc(st, old, ident, 5000, levels=lv)) == UNSUPPORTED          # ef > 4096
    other = qb.DenseVectorStorage(x, qb.Distance.Dot)
    assert status(lambda: inc(other, old, ident, 32, levels=lv)) == UNSUPPORTED         # another distance
    small = qb.DenseVectorStorage(x[:, :8].copy(), d)
    assert status(lambda: inc(small, old, ident, 32, levels=lv)) == UNSUPPORTED         # another dim
    f16 = qb.DenseVectorStorage(x, d, datatype=qb.VectorStorageDatatype.Float16)
    assert status(lambda: inc(f16, old, ident, 32, levels=lv)) == UNSUPPORTED           # not f32
    # the device is usable: a build and an incremental build succeed
    g = inc(st, old, ident, 32, levels=lv)
    assert np.array_equal(g.export_plain(), old.export_plain())
    g.close(); small.close(); other.close(); f16.close(); old.close(); st.close()
