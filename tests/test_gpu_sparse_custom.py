"""The custom queries over a device sparse vector storage (qb_sparse_storage_*, qb_sparse_search_custom_batch, qb_sparse_score_custom)
against the checker (tests/sparse_custom_ref.c, the fold by the oracle) bit for bit: ids, score bits, counts and both counters, for every
kind and several shapes, tops, filters and id lists, negative weights, user dims over the whole u32 range, empty rows and examples, points
sharing no dim, plateaus of equal scores, scores that reach +-inf and NaN, batches of several query groups, on-disk counters, the rescoring
entry, and every rejection."""
import sys

import numpy as np
import pytest

sys.dont_write_bytecode = True
from tests import sparse_custom_ref as scr  # noqa: E402

pytestmark = pytest.mark.gpu

N = 20_000
SHAPES = [(1, 1, 0), (1, 3, 2), (1, 0, 1), (2, 3, 2), (2, 0, 1), (3, 0, 0), (3, 1, 0), (3, 4, 0), (4, 1, 0), (4, 5, 0), (5, 2, 0)]


def _qb():
    from qdrant_b200 import _capi
    from qdrant_b200 import scorer as qb
    return qb, _capi


@pytest.fixture(scope="module")
def o():
    from oracle import oracle

    oracle.ensure_built()
    return oracle


@pytest.fixture(scope="module")
def pool():
    rng = np.random.default_rng(1)
    return np.unique(np.concatenate([[0, 1, 0xFFFFFFFE, 0xFFFFFFFF], rng.integers(0, 1 << 32, 400, dtype=np.uint64)]).astype(np.uint32))


@pytest.fixture(scope="module")
def corpus(pool):
    rng = np.random.default_rng(2)
    csr = scr.random_rows(rng, N, 12, pool, negative=0.2, empty=0.03)
    return csr, scr.Storage(*csr), scr.Storage(*csr, on_disk=True)


def n_examples(kind, n_a, n_b):
    return {1: n_a + n_b, 2: n_a + n_b, 3: 1 + 2 * n_a, 4: 2 * n_a, 5: 1 + 2 * n_a}[kind]


def make_batch(rng, o, kind, n_a, n_b, nq, pool, nnz=(1, 25)):
    """nq queries of E examples each (every 5th query's last example empty, some dims outside every row) and the feedback coefficients"""
    E = n_examples(kind, n_a, n_b)
    batch = []
    for q in range(nq):
        ex = []
        for j in range(E):
            k = 0 if (q % 5 == 4 and j == E - 1) else int(rng.integers(*nnz))
            d = rng.choice(pool, size=k, replace=False).astype(np.uint32)
            if k and q % 3 == 0:
                d[0] = np.uint32(1000 + j)            # a dim no stored row has
            ex.append((d, (rng.standard_normal(k) * 0.8).astype(np.float32)))
        batch.append(ex)
    coef = None
    if kind == 5:
        coef = []
        for _ in range(nq):
            _, _, part = o.feedback_pairs(rng.random(4).astype(np.float32), 1.5, 0.4)
            part = np.resize(part, n_a) if part.size else np.zeros(n_a, np.float32)
            coef.append(np.concatenate([[0.9], part]).astype(np.float32))
        coef = np.stack(coef)
    return batch, coef


def check(o, dev, ref, kind, n_a, n_b, batch, top, coef=None, deleted=None, id_list=None):
    from qdrant_b200._capi import HwCounters

    hw = HwCounters()
    got = dev.search_custom(kind, batch, n_a, n_b, coef=coef, top=top, point_deleted=deleted, id_list=id_list, counters=hw)
    bm = None if deleted is None else scr_bitmap(deleted)
    cpu = io = 0
    assert len(got) == len(batch)
    for q, (ex, g) in enumerate(zip(batch, got)):
        want, c, i = ref.search(o, kind, n_a, n_b, ex, top, None if coef is None else coef[q], bm, id_list)
        cpu += c
        io += i
        assert g.size == want.size, (q, g.size, want.size)
        assert np.array_equal(g["idx"], want["idx"]) and np.array_equal(g["score"].view(np.uint32), want["score"].view(np.uint32)), (q, g[:8], want[:8])
    assert (hw.cpu, hw.vector_io_read) == (cpu, io)
    return got


def scr_bitmap(mask):
    m = np.asarray(mask, bool)
    bits = np.zeros(((m.size + 63) // 64) * 64, bool)
    bits[: m.size] = m
    return np.packbits(bits, bitorder="little").view(np.uint64).copy()


@pytest.mark.parametrize("kind,n_a,n_b", SHAPES)
def test_shapes_and_filters_equal_checker(o, pool, corpus, kind, n_a, n_b):
    qb, _ = _qb()
    csr, ref, _ = corpus
    dev = qb.SparseVectorStorage(csr)
    rng = np.random.default_rng(kind * 100 + n_a * 10 + n_b)
    batch, coef = make_batch(rng, o, kind, n_a, n_b, 6, pool)
    deleted = rng.random(N) >= 0.08                            # 8 % pass
    listed = rng.choice(N, 3000, replace=False).astype(np.uint32)
    for top in (10, 100):
        check(o, dev, ref, kind, n_a, n_b, batch, top, coef)
        check(o, dev, ref, kind, n_a, n_b, batch, top, coef, deleted=deleted)
        check(o, dev, ref, kind, n_a, n_b, batch, top, coef, deleted=rng.random(N) >= 0.6)   # 60 % pass
        check(o, dev, ref, kind, n_a, n_b, batch, top, coef, deleted=deleted, id_list=listed)  # listed ids, most of them deleted
    dev.close()


@pytest.mark.parametrize("on_disk", [False, True])
def test_tops_and_on_disk(o, pool, corpus, on_disk):
    qb, _ = _qb()
    csr, ref, ref_disk = corpus
    dev = qb.SparseVectorStorage(csr, on_disk=on_disk)
    assert dev.info()[:2] == (N, csr[1].size)
    rng = np.random.default_rng(5)
    batch, _ = make_batch(rng, o, 1, 3, 2, 4, pool)
    for top in (1, 10, 100, 4096):
        check(o, dev, ref_disk if on_disk else ref, 1, 3, 2, batch, top)
    dev.close()


def test_several_query_groups_per_pass(o, pool, corpus):
    """300 recommend queries (64 per group), then queries whose examples fill a group's staging alone"""
    qb, _ = _qb()
    csr, ref, _ = corpus
    dev = qb.SparseVectorStorage(csr)
    rng = np.random.default_rng(6)
    batch, _ = make_batch(rng, o, 2, 3, 1, 300, pool)
    got = check(o, dev, ref, 2, 3, 1, batch, 10)
    assert sum(g.size for g in got) == 3000
    big, _ = make_batch(rng, o, 4, 2, 0, 5, pool, nnz=(300, 400))   # about 1400 example non-zeros per query
    check(o, dev, ref, 4, 2, 0, big, 20)
    dev.close()


def test_plateaus_ties_by_id(o):
    """context pairs most points satisfy: those points score exactly 0.0 and the top is decided by id; the points that share no dim
    score one equal negative value"""
    qb, _ = _qb()
    rng = np.random.default_rng(7)
    csr = scr.random_rows(rng, 5000, 6, np.arange(30, dtype=np.uint32))
    ref = scr.Storage(*csr)
    dev = qb.SparseVectorStorage(csr)
    ex = [[(np.arange(0, 30, dtype=np.uint32), np.full(30, 50.0, np.float32)), (np.array([7], np.uint32), np.array([1.0], np.float32)),
           (np.arange(10, 20, dtype=np.uint32), np.full(10, 9.0, np.float32)), (np.array([100], np.uint32), np.array([1.0], np.float32))]]
    got = check(o, dev, ref, 4, 2, 0, ex, 500)
    assert (got[0]["score"] == 0.0).sum() == 500 and np.all(np.diff(got[0]["idx"].astype(np.int64)) > 0)
    far = qb.SparseVectorStorage((np.array([0, 1, 2, 3], np.uint64), np.array([500, 501, 502], np.uint32), np.ones(3, np.float32)))
    fref = scr.Storage(np.array([0, 1, 2, 3], np.uint64), np.array([500, 501, 502], np.uint32), np.ones(3, np.float32))
    check(o, far, fref, 4, 2, 0, ex, 10)
    far.close(); fref.close(); dev.close(); ref.close()


def test_inf_and_nan_scores(o):
    """example weights near 3e38: sims reach +-inf, their sum NaN, and NaN ranks first"""
    qb, _ = _qb()
    rng = np.random.default_rng(8)
    indptr, dims, w = scr.random_rows(rng, 4000, 8, np.arange(20, dtype=np.uint32))
    # and a point whose similarities to the first query's examples are +inf and -inf
    csr = (np.append(indptr, indptr[-1] + 4).astype(np.uint64), np.append(dims, [4, 0, 3, 1]).astype(np.uint32), np.append(w, np.ones(4)).astype(np.float32))
    ref = scr.Storage(*csr)
    dev = qb.SparseVectorStorage(csr)
    big = np.float32(3e38)
    batch = [[(np.array([0, 1, 2], np.uint32), np.full(3, big, np.float32)), (np.array([3, 4, 5], np.uint32), np.full(3, -big, np.float32))],
             [(np.array([0, 5], np.uint32), np.array([big, -big], np.float32)), (np.array([9], np.uint32), np.array([1.0], np.float32))]]
    for kind in (1, 2):
        got = check(o, dev, ref, kind, 2, 0, batch, 50)
        if kind == 2:
            assert np.isnan(got[0]["score"][0])
    check(o, dev, ref, 4, 1, 0, batch, 50)
    dev.close(); ref.close()


def test_score_custom_equals_batch_scan(o, pool, corpus):
    from qdrant_b200._capi import HwCounters

    qb, _ = _qb()
    csr, ref, _ = corpus
    dev = qb.SparseVectorStorage(csr)
    rng = np.random.default_rng(9)
    for kind, n_a, n_b in ((1, 3, 2), (3, 2, 0), (5, 2, 0)):
        batch, coef = make_batch(rng, o, kind, n_a, n_b, 1, pool)
        c = None if coef is None else coef[0]
        top = dev.search_custom(kind, batch, n_a, n_b, coef=coef, top=200)[0]
        ids = rng.permutation(top["idx"])
        hw = HwCounters()
        sc = dev.score_points_custom(kind, batch[0], n_a, n_b, ids, coef=c, counters=hw)
        by_id = dict(zip(top["idx"].tolist(), top["score"].view(np.uint32).tolist()))
        assert sc.view(np.uint32).tolist() == [by_id[i] for i in ids.tolist()]
        sample = rng.choice(N, 500, replace=False).astype(np.uint32)
        want = ref.scores(o, kind, n_a, n_b, batch[0], sample, c)
        hw = HwCounters()
        got = dev.score_points_custom(kind, batch[0], n_a, n_b, sample, coef=c, counters=hw)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        assert (hw.cpu, hw.vector_io_read) == ref.counters(batch[0], sample)
    dev.close()


def test_user_dim_order_on_the_device(o):
    """products 1, 1e8, -1e8 at user dims 5, 7, 9 sum to 0.0 in user-dim order (1.0 in a tracker order that numbers 9 first)"""
    qb, _ = _qb()
    dev = qb.SparseVectorStorage([(np.array([9, 5, 7], np.uint32), np.array([1e4, 1.0, 1e4], np.float32))])
    ex = [(np.array([7, 9, 5], np.uint32), np.array([1e4, -1e4, 1.0], np.float32))]
    assert dev.score_points_custom(2, ex, 1, 0, np.array([0], np.uint32))[0] == 0.0
    got = dev.search_custom(2, [ex], 1, 0, top=1)[0]
    assert got["idx"].tolist() == [0] and got["score"].view(np.uint32).tolist() == [0]
    dev.close()


def test_rejections_leave_the_device_usable(o, pool, corpus):
    qb, capi = _qb()
    csr, ref, _ = corpus
    indptr, dims, w = csr

    def status(fn):
        with pytest.raises(capi.QbError) as e:
            fn()
        return e.value.status

    INV, UNS = capi.QB_ERR_INVALID, capi.QB_ERR_UNSUPPORTED
    r0 = int(np.nonzero(np.diff(indptr) >= 2)[0][0])
    dup = dims.copy(); dup[indptr[r0] + 1] = dup[indptr[r0]]
    bad_w = w.copy(); bad_w[3] = np.inf
    bad_ptr = indptr.copy(); bad_ptr[1] = indptr[2] + 1
    assert status(lambda: qb.SparseVectorStorage((indptr, dup, w))) == INV
    assert status(lambda: qb.SparseVectorStorage((indptr, dims, bad_w))) == INV
    assert status(lambda: qb.SparseVectorStorage((bad_ptr, dims, w))) == INV
    start = indptr.copy(); start[0] = 1
    assert status(lambda: qb.SparseVectorStorage((start, dims, w))) == INV
    dev = qb.SparseVectorStorage(csr)
    ex1 = (np.array([3, 1], np.uint32), np.array([1.0, 2.0], np.float32))
    q = [[ex1, ex1]]
    assert status(lambda: dev.search_custom(9, ([0, 0], np.zeros(0, np.uint32), np.zeros(0, np.float32)), 1, 0)) == INV   # unknown kind
    assert status(lambda: dev.search_custom(1, [], 0, 0)) == INV                                                      # no example
    assert status(lambda: dev.search_custom(3, [[ex1, ex1, ex1]], 1, 1)) == INV                                      # discover with n_b
    assert status(lambda: dev.search_custom(4, [[ex1, ex1]], 1, 1)) == INV                                            # context with n_b
    assert status(lambda: dev.search_custom(5, [[ex1, ex1, ex1]], 1, 0)) == INV                                      # feedback without coef
    assert status(lambda: dev.search_custom(1, q, 2, 0, top=0)) == INV
    assert status(lambda: dev.search_custom(1, q, 2, 0, top=4097)) == UNS
    desc = (np.array([0, 2, 1], np.uint64), np.array([1, 2], np.uint32), np.ones(2, np.float32))
    assert status(lambda: dev.search_custom(1, desc, 2, 0)) == INV                                                   # offsets descend
    nonzero = (np.array([1, 2, 2], np.uint64), np.array([1, 2], np.uint32), np.ones(2, np.float32))
    assert status(lambda: dev.search_custom(1, nonzero, 2, 0)) == INV                                                # offsets start at 1
    rep = [[(np.array([4, 4], np.uint32), np.ones(2, np.float32)), ex1]]
    assert status(lambda: dev.search_custom(1, rep, 2, 0)) == INV                                                    # a repeated dim
    assert status(lambda: dev.search_custom(1, q, 2, 0, id_list=np.array([N], np.uint32))) == INV
    assert status(lambda: dev.search_custom(1, q, 2, 0, id_list=np.array([4, 4], np.uint32))) == INV
    assert status(lambda: dev.score_points_custom(1, q[0], 2, 0, np.array([5, 5], np.uint32))) == INV
    assert status(lambda: dev.score_points_custom(1, q[0], 2, 0, np.array([N], np.uint32))) == INV
    wide = [[(np.arange(2049, dtype=np.uint32), np.ones(2049, np.float32))] * 2]
    assert status(lambda: dev.search_custom(1, wide, 2, 0)) == UNS                                                   # 4098 non-zeros
    many = [[ex1] * 257]
    assert status(lambda: dev.search_custom(2, many, 257, 0)) == UNS                                                 # E = 257
    assert status(lambda: dev.search_custom(2, [[ex1] * 4097], 4097, 0)) == INV                                      # E beyond 4096
    assert status(lambda: dev.search_custom(1, q, 2, 0, is_stopped=True)) == capi.QB_ERR_CANCELLED
    # and a search after them all equals the checker
    check(o, dev, ref, 1, 2, 0, q, 10)
    dev.close()
