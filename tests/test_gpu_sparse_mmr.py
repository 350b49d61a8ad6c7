"""MMR reranking over sparse vector candidates on the device (qb_mmr_sparse_batch) == the CPU checker (tests/mmr_sparse_ref.c) bit for
bit: selected ids in selection order, their input scores as bit patterns, counts and counters.  Lists of 2 .. 16 384 candidates (1, 2, 4
and 8 CTAs per cluster) in batches of mixed lengths; limits 1 / 10 / 100 / n; lambda 0 / 0.5 / 1; duplicate ids and lists of 0 or 1
unique candidates; empty rows and an empty query; a query and a pick row longer than the 4096-element staging; weights near 1e20 whose
products overflow to +-inf and sum to NaN; zero-score plateaus; user dims near 2^32 - 1; an on-disk storage (vector_io_read stays 0);
every rejection, each followed by a call that succeeds."""
import ctypes as C

import numpy as np
import pytest

from tests import mmr_sparse_ref as ms

pytestmark = pytest.mark.gpu

LAMBDAS = (0.0, 0.5, 1.0)


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _pool(rng, n):
    return np.concatenate([[0, 1, 0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFFFD], rng.choice(0xFFFFFFF0, n, replace=False)]).astype(np.uint32)


def _rows(rng, n_points, pool, mean_nnz, empty=0.1, weights=None):
    """CSR rows of distinct dims from pool in shuffled order; weights in [-1, 1) with a third from a few values (ties), or from `weights`"""
    counts = np.minimum(rng.poisson(mean_nnz, n_points), pool.size)
    counts[rng.random(n_points) < empty] = 0
    dims = np.concatenate([rng.choice(pool, size=c, replace=False) for c in counts]).astype(np.uint32)
    ip = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
    if weights is not None:
        w = rng.choice(np.asarray(weights, np.float32), dims.size)
    else:
        w = (rng.random(dims.size) * 2 - 1).astype(np.float32)
        tie = rng.random(dims.size) < 0.3
        w[tie] = rng.choice(np.array([0.5, 1.0, -0.25], np.float32), int(tie.sum()))
    return ip, dims, w.astype(np.float32)


def _query(rng, pool, n, weights=None):
    d = rng.choice(pool, size=min(n, pool.size), replace=False).astype(np.uint32)
    w = (rng.choice(np.asarray(weights, np.float32), d.size) if weights is not None else rng.random(d.size) * 2 - 1).astype(np.float32)
    return d, w


def _lists(rng, ns, n_points):
    out = []
    for n in ns:
        ids = rng.choice(n_points, size=n, replace=False).astype(np.uint32)
        if n > 3:
            for _ in range(max(1, n // 50)):   # duplicate ids: the first occurrence is kept
                ids[rng.integers(1, n)] = ids[rng.integers(0, n)]
        c = np.zeros(n, ms.SCORED)
        c["idx"] = ids
        c["score"] = rng.standard_normal(n).astype(np.float32)
        c["score"][rng.integers(0, n, max(1, n // 7))] = -0.0
        out.append(c)
    return out


def _check(qb, st, csr, queries, lams, lists, limit):
    hw = qb.HwCounters()
    got = st.mmr(queries, lists, lams, limit, counters=hw)
    want, cpu, io = ms.mmr_batch(csr, queries, lams, lists, limit)
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a["idx"], b["idx"]), (i, len(lists[i]), lams[i], a["idx"][:20], b["idx"][:20])
        assert np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)), i
    assert (hw.cpu, hw.vector_io_read) == (cpu, io)


@pytest.fixture(scope="module")
def corpus(qb):
    rng = np.random.default_rng(11)
    pool = _pool(rng, 400)
    csr = _rows(rng, 20_000, pool, 10)
    st = qb.SparseVectorStorage(csr)
    yield rng, pool, csr, st
    st.close()


@pytest.mark.parametrize("limit", [1, 10, 100, "n"])
def test_mmr_sparse_equals_checker(qb, corpus, limit):
    rng, pool, csr, st = corpus
    ns = (2, 3, 100, 300, 1500) if limit == "n" else (2, 3, 100, 300, 1500, 5000, 16384)
    if limit == "n":
        # limit = n: one call per list length, so the cluster is sized from it
        for n in ns:
            qs = [_query(rng, pool, int(k)) for k in rng.integers(0, 20, len(LAMBDAS))]
            _check(qb, st, csr, qs, np.array(LAMBDAS, np.float32), _lists(rng, [n] * len(LAMBDAS), 20_000), n)
    else:
        # one batch of every length and lambda: per-query counts differ, the cluster is sized from the longest
        qs = [_query(rng, pool, int(k)) for k in rng.integers(0, 20, len(ns) * len(LAMBDAS))]
        qs[0] = (qs[0][0][:0], qs[0][1][:0])   # an empty query: every relevance +0.0
        lams = np.array([l for _ in ns for l in LAMBDAS], np.float32)
        _check(qb, st, csr, qs, lams, _lists(rng, [n for n in ns for _ in LAMBDAS], 20_000), limit)


def test_short_and_duplicate_lists(qb, corpus):
    """lists of 0 and 1 unique candidates come back as they are, uncounted; a list of one id repeated, and of two ids repeated"""
    rng, pool, csr, st = corpus
    lists = [np.array([], ms.SCORED), np.array([(7, 0.5)], ms.SCORED), np.array([(9, 0.25), (9, 0.75), (9, 1.0)], ms.SCORED),
             np.array([(3, 1.0), (4, 2.0), (3, 3.0), (4, 4.0)], ms.SCORED)]
    qs = [_query(rng, pool, 5) for _ in lists]
    _check(qb, st, csr, qs, np.array([0.5, 0.5, 0.5, 0.2], np.float32), lists, 3)


def test_zero_plateaus(qb):
    """rows of 1..3 dims out of 20 000 and small queries: most relevances and pairs are exactly +0.0, so the swap_remove position order
    decides most picks; a third of the rows are empty"""
    rng = np.random.default_rng(21)
    pool = _pool(rng, 20_000)
    csr = _rows(rng, 8000, pool, 2, empty=0.3)
    st = qb.SparseVectorStorage(csr)
    qs = [_query(rng, pool, 3) for _ in range(6)]
    lams = np.array([0.0, 0.5, 1.0, 0.5, 0.3, 0.7], np.float32)
    _check(qb, st, csr, qs, lams, _lists(rng, [300, 2000, 4000, 257, 8000, 16], 8000), 100)
    st.close()


def test_non_finite_scores(qb):
    """weights near 1e20: products overflow to +-inf and sums of opposite infinities are NaN, so relevances and pair maxima are NaN
    (above everything under OrderedFloat); one query weight is NaN"""
    rng = np.random.default_rng(31)
    pool = _pool(rng, 30)
    csr = _rows(rng, 3000, pool, 6, weights=[1e20, -1e20, 3e19, 1.0, -0.5])
    st = qb.SparseVectorStorage(csr)
    qs = [_query(rng, pool, 6, weights=[1e20, -1e20, 1.0]) for _ in range(6)]
    qs[1][1][0] = np.nan
    lams = np.array([0.5, 0.5, 0.0, 1.0, 0.3, 0.9], np.float32)
    _check(qb, st, csr, qs, lams, _lists(rng, [200, 300, 1100, 2000, 50, 3], 3000), 30)
    st.close()


def test_rows_longer_than_the_stage(qb):
    """queries of 5 000 and 6 000 elements and pick rows of as many (the staging holds 4 096): read from global memory, same bits"""
    rng = np.random.default_rng(41)
    pool = _pool(rng, 9000)
    ip, d, w = _rows(rng, 3000, pool, 30)
    long_rows = [rng.choice(pool, 5000, replace=False), rng.choice(pool, 6000, replace=False)]
    parts_d = [d] + [x.astype(np.uint32) for x in long_rows]
    parts_w = [w] + [(rng.random(x.size) + 0.5).astype(np.float32) for x in long_rows]
    csr = (np.concatenate([ip, ip[-1] + np.cumsum([5000, 6000])]).astype(np.uint64), np.concatenate(parts_d), np.concatenate(parts_w))
    st = qb.SparseVectorStorage(csr)
    # each long point is the first pick of the query made of its dims (given in reverse order), and the second under lambda 1
    qs = [(x[::-1].astype(np.uint32).copy(), np.ones(x.size, np.float32)) for x in long_rows]
    qs = [qs[0], _query(rng, pool, 40), qs[1]]
    lists = _lists(rng, [500, 800, 1200], 3000)
    for c in lists:
        c["idx"][1], c["idx"][5] = 3000, 3001
    _check(qb, st, csr, qs, np.array([0.5, 0.5, 1.0], np.float32), lists, 20)
    st.close()


def test_on_disk_storage_counts_no_io(qb):
    rng = np.random.default_rng(51)
    pool = _pool(rng, 500)
    csr = _rows(rng, 5000, pool, 12)
    st = qb.SparseVectorStorage(csr, on_disk=True)
    qs = [_query(rng, pool, 10) for _ in range(4)]
    _check(qb, st, csr, qs, np.array([0.5, 0.1, 0.9, 1.0], np.float32), _lists(rng, [100, 1000, 4097, 2], 5000), 10)
    st.close()


def test_rejections_leave_the_device_usable(qb, corpus):
    from qdrant_b200._capi import ScoredPoint, f32p, lib, u32p, u64p

    rng, pool, csr, st = corpus
    qd = np.array([5, 1, 9, 1 << 31, 2, 7], np.uint32)
    qw = np.ones(6, np.float32)
    qp = np.array([0, 2, 6], np.uint64)
    ids0, ids1 = list(range(40)), list(range(50, 105))
    lists = [np.array([(i, 0.0) for i in ids0], ms.SCORED), np.array([(i, 1.0) for i in ids1], ms.SCORED)]
    cand = np.zeros((2, 60), ms.SCORED)
    cand[0, : len(ids0)], cand[1, : len(ids1)] = lists
    counts = np.array([len(ids0), len(ids1)], np.uint32)
    ok = np.array([0.5, 0.5], np.float32)

    def call(lams=ok, cand=cand, counts=counts, max_c=60, limit=5, qp=qp, qd=qd):
        out = np.zeros((2, max(limit, 1)), ms.SCORED)
        oc = np.zeros(2, np.uint32)
        return lib().qb_mmr_sparse_batch(st._h, qp.ctypes.data_as(u64p), qd.ctypes.data_as(u32p), qw.ctypes.data_as(f32p), 2, lams.ctypes.data_as(f32p),
                                         cand.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p), max_c, limit,
                                         out.ctypes.data_as(C.POINTER(ScoredPoint)), oc.ctypes.data_as(u32p), None)

    qs = [(qd[:2], qw[:2]), (qd[2:], qw[2:])]

    def still_usable():
        _check(qb, st, csr, qs, ok, lists, 5)

    INVALID, UNSUPPORTED = -1, -3
    bad = cand.copy()
    bad[1, 3]["idx"] = 20_000
    rep = qd.copy()
    rep[3] = rep[2]
    for rc, want in ((call(lams=np.array([0.5, np.nan], np.float32)), INVALID), (call(lams=np.array([-0.01, 0.5], np.float32)), INVALID),
                     (call(lams=np.array([0.5, 1.01], np.float32)), INVALID), (call(limit=0), INVALID),
                     (call(counts=np.array([39, 61], np.uint32)), INVALID), (call(cand=bad), INVALID),
                     (call(qp=np.array([1, 2, 6], np.uint64)), INVALID), (call(qp=np.array([0, 4, 2], np.uint64)), INVALID), (call(qd=rep), INVALID),
                     (call(cand=np.zeros((2, 16385), ms.SCORED), max_c=16385), UNSUPPORTED)):
        assert rc == want
        still_usable()
    assert lib().qb_mmr_sparse_batch(st._h, None, None, None, 2, ok.ctypes.data_as(f32p), None, None, 60, 5, None, None, None) == INVALID
    assert lib().qb_mmr_sparse_batch(None, qp.ctypes.data_as(u64p), qd.ctypes.data_as(u32p), qw.ctypes.data_as(f32p), 2, ok.ctypes.data_as(f32p),
                                     cand.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p), 60, 5,
                                     np.zeros((2, 5), ms.SCORED).ctypes.data_as(C.POINTER(ScoredPoint)), np.zeros(2, np.uint32).ctypes.data_as(u32p),
                                     None) == INVALID
    still_usable()
