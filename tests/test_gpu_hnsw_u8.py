"""Device HNSW over Uint8 storages: search (HNSW and ACORN-1 level 0, the host and the device-resident entries), custom queries, full
and incremental graph builds, each against a CPU checker that orders every level-0 comparison on (score desc, id asc) keys, the
device's tie order: tests/hnsw_custom_ref.c in keyed mode for the searches, the keyed u8 build restatements (tests/hnsw_build_keyed_ref.py)
for the builds.  u8 similarities are integers for Dot, Euclid and Manhattan, so the data here is tie-heavy on purpose: a narrow value
range and duplicated rows; the test asserts that the keyed and the score-only CPU lists really differ on it."""
import numpy as np
import pytest

from tests import hnsw_acorn_ref as ar
from tests import hnsw_build_keyed_ref as ur
from tests import hnsw_custom_ref as cr
from tests.hnsw_build_incr_ref import GONE

pytestmark = pytest.mark.gpu

DISTS = ["Cosine", "Dot", "Euclid", "Manhattan"]
DIMS = [96, 20]                       # the 8-lane chain (dim >= 32) and the one-thread integer tier
M, M0, EF_C, TOP, EF = 8, 16, 32, 10, 16   # a short beam: ties at its end change the lists
# (kind, n_a, n_b): recommend best-score and sum-scores, context, discover as one search, feedback
KINDS = [(1, 3, 2), (2, 3, 2), (4, 2, 0), (3, 2, 0), (cr.FEEDBACK, 2, 0)]


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def tie_rows(rng, n, dim):
    """values 0 and 1, and every fifth row a copy of an earlier one: equal similarities everywhere"""
    rows = rng.integers(0, 2, (n, dim), dtype=np.uint8)
    dup = np.arange(n) % 5 == 4
    rows[dup] = rows[rng.integers(0, n // 2, int(dup.sum()))]
    return rows


def raw_queries(rng, nq, dim):
    """raw f32 whose `as u8` lands in the stored range, with fractions to truncate"""
    return (rng.integers(0, 2, (nq, dim)) + rng.random((nq, dim)) * 0.99).astype(np.float32)


def levels_of(rng, n, m=M):
    return np.minimum(np.round(-np.log(1.0 - rng.random(n)) / np.log(m)), 30).astype(np.uint8)


class Env:
    """a tie-heavy u8 storage and a graph over it built by the keyed CPU restatement (independent of the device builder)"""

    def __init__(self, qb, oracle, dist, dim, n=1500, seed=3):
        self.d = getattr(qb.Distance, dist)
        self.rng = np.random.default_rng(seed)
        self.rows = tie_rows(self.rng, n, dim)
        self.n, self.dim = n, dim
        ref = ur.batched(self.rows, int(self.d), M, M0, EF_C, levels_of(self.rng, n), batch=64, serial_points=64)
        self.plain = ref.export_plain()
        self.entry, self.level = ref.entry()
        ref.close()
        self.st = qb.DenseVectorStorage(self.rows, self.d, qb.VectorStorageDatatype.Uint8)
        self.hg = qb.HnswGraph(self.st, self.plain, M, M0)
        self.cg = cr.Graph(self.plain, M, M0, n)

    def cpu(self, oracle, q_raw, algo, filtered, keyed=True):
        qu = oracle.to_u8_query(q_raw)
        return cr.search_cb(self.cg, lambda ids: oracle.score_rows_u8(int(self.d), self.rows, qu, ids), TOP, EF, self.entry, self.level, algo, filtered,
                            keyed=keyed)

    def close(self):
        self.cg.close(); self.hg.close(); self.st.close()


def _same(got, want, what):
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a["idx"], b["idx"]), f"{what} query {i}: ids\n{a}\n{b}"
        assert np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)), f"{what} query {i}: score bits"


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("dist", DISTS)
def test_search_equals_keyed_checker(qb, oracle, dist, dim):
    import torch

    from qdrant_b200._capi import HwCounters, check, lib, vp

    env = Env(qb, oracle, dist, dim)
    q = raw_queries(env.rng, 24, dim)
    filt = env.rng.random(env.n) >= 0.08        # a restrictive filter: 8 % of the points pass
    filt[env.entry] = False
    differ = False
    for algorithm, algo in (("hnsw", ar.HNSW), ("acorn", ar.ACORN)):
        for f in (None, filt):
            if algorithm == "acorn" and f is None:
                continue
            env.hg.stats(reset=True)
            hc = HwCounters()
            got = env.hg.search(q, TOP, EF, env.entry, env.level, point_deleted=f, counters=hc, algorithm=algorithm)
            want = [env.cpu(oracle, x, algo, f) for x in q]
            _same(got, want, f"{dist} dim {dim} {algorithm} filter {f is not None}")
            hops, scored = env.hg.stats(reset=True)
            assert (hops, scored) == env.cg.stats()[:2]
            assert hc.cpu == dim * scored and hc.vector_io_read == 0
            unkeyed = [env.cpu(oracle, x, algo, f, keyed=False) for x in q]
            env.cg.stats()
            differ |= any(not np.array_equal(a, b) for a, b in zip(want, unkeyed))
    assert differ, "the data has no ties that change a list"
    # the device-resident entry == the host entry
    dq = torch.from_numpy(q).cuda()
    out = torch.zeros((len(q), TOP), dtype=torch.int64, device="cuda")
    cnt = torch.zeros(len(q), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    check(lib().qb_hnsw_search_batch_device_algo(env.hg._h, vp(dq.data_ptr()), len(q), TOP, EF, env.entry, env.level, vp(out.data_ptr()),
                                                 vp(cnt.data_ptr()), 0))
    torch.cuda.synchronize()
    rec = out.cpu().numpy().view(qb.SCORED_POINT_OFFSET).reshape(len(q), TOP)
    c = cnt.cpu().numpy()
    _same([rec[i, : c[i]] for i in range(len(q))], env.hg.search(q, TOP, EF, env.entry, env.level), f"{dist} dim {dim} device entry")
    env.close()


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("dist", ["Dot", "Cosine"])
def test_custom_equals_keyed_checker(qb, oracle, dist, dim):
    env = Env(qb, oracle, dist, dim, seed=5)
    nq = 6
    for kind, n_a, n_b in KINDS:
        ne = cr.n_examples(kind, n_a, n_b)
        ex = np.stack([raw_queries(env.rng, ne, dim) for _ in range(nq)])
        coef = np.concatenate([env.rng.random((nq, 1)), env.rng.standard_normal((nq, n_a))], axis=1).astype(np.float32) if kind == cr.FEEDBACK else None
        for algorithm, algo in (("hnsw", ar.HNSW), ("acorn", ar.ACORN)):
            env.hg.stats(reset=True)
            got = env.hg.search_custom(qb.QueryKind(kind), ex, n_a, n_b, coef=coef, top=TOP, ef=EF, entry_point=env.entry, entry_level=env.level,
                                       algorithm=algorithm)
            want = []
            for i in range(nq):
                sc = _custom_scorer(qb, env.st, kind, ex[i], n_a, n_b, None if coef is None else coef[i])
                want.append(cr.search_cb(env.cg, sc.score_points, TOP, EF, env.entry, env.level, algo, keyed=True))
                sc.close()
            _same(got, want, f"{dist} dim {dim} kind {kind} {algorithm}")
            assert env.hg.stats(reset=True) == env.cg.stats()[:2]
    # discover, both stages in one call == a context search for 10 entry points, then the discover search from them
    ex = np.stack([raw_queries(env.rng, 5, dim) for _ in range(nq)])
    got = env.hg.search_discover(ex, 2, top=TOP, ef=EF, entry_point=env.entry, entry_level=env.level)
    for i in range(nq):
        ctx = _custom_scorer(qb, env.st, 4, ex[i, 1:], 2, 0, None)
        stage1 = cr.search_cb(env.cg, ctx.score_points, cr.DISCOVERY_ENTRY_POINT_COUNT, EF, env.entry, env.level, ar.HNSW, keyed=True)
        dsc = _custom_scorer(qb, env.st, 3, ex[i], 2, 0, None)
        want = cr.search_cb(env.cg, dsc.score_points, TOP, EF, env.entry, env.level, ar.HNSW, cep=stage1["idx"], keyed=True)
        _same([got[i]], [want], f"{dist} dim {dim} discover query {i}")
        ctx.close(); dsc.close()
    env.close()


def _custom_scorer(qb, st, kind, ex, n_a, n_b, coef):
    """qb_scorer_create_custom / _feedback over the examples in the device call's layout"""
    if kind == cr.FEEDBACK:
        q = qb.FeedbackQuery(ex[0], [qb.ContextPair(ex[1 + 2 * j], ex[2 + 2 * j]) for j in range(n_a)], coef[1:], coef[0])
    elif kind in (1, 2):
        q = (qb.RecoBestScoreQuery if kind == 1 else qb.RecoSumScoresQuery)(qb.RecoQuery(ex[:n_a], ex[n_a:n_a + n_b]))
    elif kind == 3:
        q = qb.DiscoverQuery(ex[0], [qb.ContextPair(ex[1 + 2 * j], ex[2 + 2 * j]) for j in range(n_a)])
    else:
        q = qb.ContextQuery([qb.ContextPair(ex[2 * j], ex[2 * j + 1]) for j in range(n_a)])
    return st.raw_scorer_custom(q)


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("dist", DISTS)
def test_build_equals_keyed_restatement(qb, oracle, dist, dim):
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(7)
    n = 1200
    rows = tie_rows(rng, n, dim)
    lv = levels_of(rng, n)
    st = qb.DenseVectorStorage(rows, d, qb.VectorStorageDatatype.Uint8)
    for batch, serial_points in ((1, 1), (64, 32)):
        g = qb.HnswGraph.build(st, m=M, m0=M0, ef_construct=EF_C, levels=lv, batch=batch, serial_points=serial_points)
        ref = ur.batched(rows, int(d), M, M0, EF_C, lv, batch=batch, serial_points=serial_points)
        assert (g.entry_point, g.entry_level) == ref.entry(), f"{dist} dim {dim} batch {batch}"
        assert np.array_equal(g.export_plain(), ref.export_plain()), f"{dist} dim {dim} batch {batch}"
        unkeyed = ur.batched(rows, int(d), M, M0, EF_C, lv, batch=batch, serial_points=serial_points, keyed=False)
        assert not np.array_equal(unkeyed.export_plain(), ref.export_plain()), "the data has no ties that change the graph"
        g2 = qb.HnswGraph.build(st, m=M, m0=M0, ef_construct=EF_C, levels=lv, batch=batch, serial_points=serial_points)
        assert np.array_equal(g2.export_plain(), g.export_plain())   # deterministic
        g.close(); g2.close(); ref.close(); unkeyed.close()
    # resident-deleted points are not inserted: no links from them, none to them
    dl = rng.random(n) < 0.1
    st.set_deleted(dl)
    g = qb.HnswGraph.build(st, m=M, m0=M0, ef_construct=EF_C, levels=lv, batch=64, serial_points=32)
    ref = ur.batched(rows, int(d), M, M0, EF_C, lv, deleted=dl, batch=64, serial_points=32)
    assert np.array_equal(g.export_plain(), ref.export_plain())
    links = g.links(0, np.arange(n))
    assert all(links[i].size == 0 for i in np.flatnonzero(dl))
    assert not np.isin(np.concatenate(links), np.flatnonzero(dl)).any()
    g.close(); ref.close(); st.close()


def test_build_recall_close_to_serial_build(qb, oracle):
    """recall@10 of a device-built graph against the exact scan, beside a graph built point by point by the oracle's own link_new_point
    with the u8 score (the score-only restatement)"""
    rng = np.random.default_rng(11)
    n, dim = 4000, 64
    centers = rng.integers(0, 200, (40, dim))
    rows = np.clip(centers[rng.integers(0, 40, n)] + rng.integers(-25, 26, (n, dim)), 0, 255).astype(np.uint8)
    lv = levels_of(rng, n, 16)
    d = qb.Distance.Euclid
    st = qb.DenseVectorStorage(rows, d, qb.VectorStorageDatatype.Uint8)
    g = qb.HnswGraph.build(st, m=16, ef_construct=100, levels=lv)
    ref = ur.batched(rows, int(d), 16, 32, 100, lv, batch=1, serial_points=n, keyed=False)
    q = (rows[rng.integers(0, n, 64)].astype(np.float32) + rng.integers(-20, 21, (64, dim))).clip(0, 255).astype(np.float32)
    exact = oracle.scan_u8(int(d), rows, np.stack([oracle.to_u8_query(x) for x in q]), 10)
    cg = cr.Graph(ref.export_plain(), 16, 32, n)
    e, el = ref.entry()
    qu = [oracle.to_u8_query(x) for x in q]
    cpu = [cr.search_cb(cg, lambda ids, qq=qq: oracle.score_rows_u8(int(d), rows, qq, ids), 10, 64, e, el, keyed=False) for qq in qu]
    dev = g.search(q, 10, 64, g.entry_point, g.entry_level)

    def recall(lists):
        return np.mean([np.isin(a["idx"], b["idx"]).mean() for a, b in zip(lists, exact)])

    r_dev, r_cpu = recall(dev), recall(cpu)
    assert r_dev >= r_cpu - 0.03, (r_dev, r_cpu)
    cg.close(); g.close(); ref.close(); st.close()


@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("dist", DISTS)
def test_incremental_equals_keyed_restatement(qb, oracle, dist, dim):
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(13)
    n_old, n_add = 1000, 300
    old_rows = tie_rows(rng, n_old, dim)
    old_lv = levels_of(rng, n_old)
    ost = qb.DenseVectorStorage(old_rows, d, qb.VectorStorageDatatype.Uint8)
    old = qb.HnswGraph.build(ost, m=M, m0=M0, ef_construct=EF_C, levels=old_lv, batch=64, serial_points=32)
    keep = rng.random(n_old) >= 0.15
    o2n = np.full(n_old, GONE, np.uint32)
    o2n[keep] = np.arange(int(keep.sum()), dtype=np.uint32)
    new_rows = np.concatenate([old_rows[keep], tie_rows(rng, n_add, dim)])
    new_lv = np.concatenate([old_lv[keep], levels_of(rng, n_add)])
    st = qb.DenseVectorStorage(new_rows, d, qb.VectorStorageDatatype.Uint8)
    g = qb.HnswGraph.build_incremental(st, old, o2n, ef_construct=EF_C, levels=new_lv, batch=64, serial_points=32)
    ref, entry = ur.build_incremental(old_rows, old.export_plain(), int(d), M, M0, new_rows, o2n, new_lv, ef_construct=EF_C, batch=64, serial_points=32)
    assert (g.entry_point, g.entry_level) == entry
    want = ref.export_plain()
    assert np.array_equal(g.export_plain(), want), f"{dist} dim {dim}"
    ref.close(); g.close()
    # mixed datatypes are rejected: a Uint8 old graph with an f32 storage, an f32 old graph with a Uint8 storage
    f32_new = qb.DenseVectorStorage(new_rows.astype(np.float32), d)
    f32_old_st = qb.DenseVectorStorage(old_rows.astype(np.float32), d)
    f32_old = qb.HnswGraph.build(f32_old_st, m=M, m0=M0, ef_construct=EF_C, levels=old_lv)
    for s_, o_ in ((f32_new, old), (st, f32_old)):
        with pytest.raises(qb.QbError) as e:
            qb.HnswGraph.build_incremental(s_, o_, o2n, ef_construct=EF_C, levels=new_lv, batch=64, serial_points=32)
        assert e.value.status == -3                                           # QB_ERR_UNSUPPORTED
    f32_old.close(); f32_old_st.close(); f32_new.close()
    # the device stays usable
    g = qb.HnswGraph.build_incremental(st, old, o2n, ef_construct=EF_C, levels=new_lv, batch=64, serial_points=32)
    assert np.array_equal(g.export_plain(), want)
    g.close(); st.close(); old.close(); ost.close()


def test_maxsim_over_u8_tokens_still_rejected(qb, oracle):
    rng = np.random.default_rng(17)
    tokens = rng.integers(0, 256, (400, 48), dtype=np.uint8)
    off = np.arange(0, 401, 4, dtype=np.uint32)
    st = qb.DenseVectorStorage(tokens, qb.Distance.Dot, qb.VectorStorageDatatype.Uint8)
    view = qb.MultiVectorView(st, off)
    with pytest.raises(qb.QbError) as e:
        qb.HnswGraph.build_multivector(view, m=8, ef_construct=32)
    assert e.value.status == -3
    st.close()
