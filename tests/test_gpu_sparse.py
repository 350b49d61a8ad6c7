"""The device sparse index (qb_sparse_*) against the checker (tests/sparse_ref.c) bit for bit: ids, score bits and counters of
SearchContext::search for both index kinds, filters, tops, negative weights, unknown dims, single-dim queries, lists ending in different
batches and ids over many batches; plain_search with its zero-score pushes; the device form; and every rejection."""
import ctypes as C
import sys

import numpy as np
import pytest

sys.dont_write_bytecode = True
from tests import sparse_ref as sr  # noqa: E402

pytestmark = pytest.mark.gpu


def _qb():
    from qdrant_b200 import _capi
    from qdrant_b200 import scorer as qb
    return qb, _capi


def _queries(rng, n, n_dims, unknown=0, negative=False, single=False):
    out = []
    for i in range(n):
        k = 1 if single else int(rng.integers(1, 30))
        d = rng.choice(n_dims + unknown, size=k, replace=False).astype(np.uint32)   # dims >= n_dims: unknown to the index
        w = (rng.random(k) + 0.05).astype(np.float32)
        if negative and i % 2 == 0:
            w[rng.integers(0, k)] *= -1
        out.append((d, w))
    return out


def _check(qb, dev, ref, queries, top, kind, deleted=None):
    from qdrant_b200._capi import HwCounters
    hw = HwCounters()
    got = dev.search(queries, top, point_deleted=deleted, counters=hw)
    cpu = 0
    bm = None if deleted is None else sr.deleted_bitmap(deleted)
    for (d, w), g in zip(queries, got):
        want, c = ref.search(d, w, top, reliable=kind == qb.SparseIndexKind.Ram, deleted=bm)
        cpu += c
        assert np.array_equal(g["idx"], want["idx"]) and np.array_equal(g["score"].view(np.uint32), want["score"].view(np.uint32)), (d, w, g[:8], want[:8])
    assert (hw.cpu, hw.vector_io_read) == (cpu, 0)


@pytest.fixture(scope="module")
def corpus():
    rng = np.random.default_rng(7)
    n_dims = 400
    csr = sr.random_csr(rng, 60_000, n_dims, 10, zipf=1.0)
    return n_dims, csr, sr.Index(*csr, n_dims)


@pytest.mark.parametrize("kind", ["Ram", "Compressed"])
@pytest.mark.parametrize("top", [1, 10, 100, 4096])
def test_search_equals_checker(corpus, kind, top):
    qb, _ = _qb()
    n_dims, csr, ref = corpus
    k = qb.SparseIndexKind[kind]
    dev = qb.SparseVectorIndex(csr, n_dims, k)
    rng = np.random.default_rng(top)
    qs = _queries(rng, 24, n_dims, unknown=20)
    for deleted in (None, rng.random(60_000) >= 0.08, rng.random(60_000) >= 0.6):   # no filter, 8 % and 60 % passing
        _check(qb, dev, ref, qs, top, k, deleted)
    _check(qb, dev, ref, _queries(rng, 16, n_dims, negative=True), top, k)        # negative weights: pruning off
    _check(qb, dev, ref, _queries(rng, 16, n_dims, single=True), top, k)          # one list from the start
    dev.close()


@pytest.mark.parametrize("kind", ["Ram", "Compressed"])
def test_many_batches_and_staggered_list_ends(kind):
    """ids over 25 batches (every 3rd row non-empty), and hot / cold dims whose lists end in different batches"""
    qb, _ = _qb()
    rng = np.random.default_rng(11)
    n_dims, n = 60, 250_000
    indptr, dims, w = sr.random_csr(rng, n, n_dims, 4, zipf=1.3, id_gap=3)
    # dim d's list stops at row 4000 * d: the lists run out in different batches
    rows = np.repeat(np.arange(n), np.diff(indptr).astype(np.int64))
    keep = rows < 4000 * (dims.astype(np.int64) + 1)
    indptr = np.concatenate([[0], np.cumsum(np.bincount(rows[keep], minlength=n))]).astype(np.uint64)
    dims, w = dims[keep], w[keep]
    ref = sr.Index(indptr, dims, w, n_dims)
    k = qb.SparseIndexKind[kind]
    dev = qb.SparseVectorIndex((indptr, dims, w), n_dims, k)
    for top in (1, 10, 100):
        _check(qb, dev, ref, _queries(rng, 12, n_dims), top, k)
        _check(qb, dev, ref, _queries(rng, 6, n_dims, negative=True), top, k, rng.random(n) >= 0.5)
    dev.close()
    ref.close()


def test_plain_search_equals_checker(corpus):
    qb, _ = _qb()
    from qdrant_b200._capi import HwCounters
    n_dims, csr, ref = corpus
    rng = np.random.default_rng(3)
    dev = qb.SparseVectorIndex(csr, n_dims)
    qs = _queries(rng, 20, n_dims, unknown=10, negative=True)
    lists = [rng.choice(60_000, size=int(rng.integers(0, 3000)), replace=False).astype(np.uint32) for _ in qs]
    for top in (1, 10, 100, 4096):
        hw = HwCounters()
        got = dev.search_plain(qs, lists, top, counters=hw)
        cpu = 0
        for (d, w), ids, g in zip(qs, lists, got):
            want, c = ref.plain(d, w, ids, top)
            cpu += c
            assert np.array_equal(g["idx"], want["idx"]) and np.array_equal(g["score"].view(np.uint32), want["score"].view(np.uint32))
        assert hw.cpu == cpu
    dev.close()
    # zero scores are pushed; ids without a shared dim are not
    small = qb.SparseVectorIndex((np.array([0, 2, 3, 4], np.uint64), np.array([1, 2, 1, 3], np.uint32), np.array([1.0, -1.0, 0.0, 5.0], np.float32)), 4)
    got = small.search_plain([(np.array([2, 1], np.uint32), np.array([1.0, 1.0], np.float32))], [np.array([0, 1, 2], np.uint32)], 10)[0]
    assert [(int(i), float(s)) for i, s in got] == [(0, 0.0), (1, 0.0)]
    assert small.search([(np.array([2, 1], np.uint32), np.array([1.0, 1.0], np.float32))], 10)[0].size == 0
    small.close()


def test_device_form_equals_host_form(corpus):
    import torch

    qb, capi = _qb()
    n_dims, csr, _ = corpus
    rng = np.random.default_rng(5)
    dev = qb.SparseVectorIndex(csr, n_dims)
    qs = _queries(rng, 40, n_dims, unknown=15, negative=True)
    deleted = rng.random(60_000) >= 0.3
    want = dev.search(qs, 50, point_deleted=deleted)
    # the device form takes queries as given: unsorted, unknown dims included
    qp = np.concatenate([[0], np.cumsum([d.size for d, _ in qs])]).astype(np.uint64)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
    d_qp, d_qd, d_qw = t(qp.view(np.int64)), t(np.concatenate([d for d, _ in qs]).view(np.int32)), t(np.concatenate([w for _, w in qs]))
    d_del = t(qb._bitmap(deleted, 60_000).view(np.int64))
    d_out = torch.zeros((40, 50, 2), dtype=torch.int32, device="cuda")
    d_cnt = torch.zeros(40, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    L = capi.lib()
    capi.check(L.qb_sparse_search_batch_device(dev._h, d_qp.data_ptr(), d_qd.data_ptr(), d_qw.data_ptr(), 40, max(d.size for d, _ in qs), 50,
                                               d_del.data_ptr(), d_out.data_ptr(), d_cnt.data_ptr()))
    torch.cuda.synchronize()
    assert C.c_void_p(L.qb_sparse_index_stream(dev._h)).value
    out = d_out.cpu().numpy().view(np.uint32).reshape(40, 50, 2)
    cnt = d_cnt.cpu().numpy()
    for q in range(40):
        assert cnt[q] == want[q].size
        assert np.array_equal(out[q, : cnt[q], 0], want[q]["idx"]) and np.array_equal(out[q, : cnt[q], 1], want[q]["score"].view(np.uint32))
    dev.close()


def test_rejections_leave_the_device_usable(corpus):
    qb, capi = _qb()
    n_dims, csr, ref = corpus
    indptr, dims, w = csr

    def status(fn):
        with pytest.raises(capi.QbError) as e:
            fn()
        return e.value.status

    bad_dims = dims.copy(); bad_dims[5] = n_dims
    bad_w = w.copy(); bad_w[7] = np.nan
    dup = dims.copy(); r0 = int(np.nonzero(np.diff(indptr) >= 2)[0][0]); dup[indptr[r0] + 1] = dup[indptr[r0]]
    bad_ptr = indptr.copy(); bad_ptr[1] = indptr[2] + 1
    assert status(lambda: qb.SparseVectorIndex((indptr, bad_dims, w), n_dims)) == capi.QB_ERR_INVALID
    assert status(lambda: qb.SparseVectorIndex((indptr, dims, bad_w), n_dims)) == capi.QB_ERR_INVALID
    assert status(lambda: qb.SparseVectorIndex((indptr, dup, w), n_dims)) == capi.QB_ERR_INVALID
    assert status(lambda: qb.SparseVectorIndex((bad_ptr, dims, w), n_dims)) == capi.QB_ERR_INVALID
    assert status(lambda: qb.SparseVectorIndex(csr, n_dims, qb.SparseIndexKind.CompressedF16)) == capi.QB_ERR_UNSUPPORTED
    assert status(lambda: qb.SparseVectorIndex(csr, n_dims, qb.SparseIndexKind.CompressedU8)) == capi.QB_ERR_UNSUPPORTED
    wide = qb.SparseVectorIndex((np.array([0, 1], np.uint64), np.array([0], np.uint32), np.ones(1, np.float32)), 5000)
    assert status(lambda: wide.search([(np.arange(4097, dtype=np.uint32), np.ones(4097, np.float32))], 10)) == capi.QB_ERR_UNSUPPORTED
    wide.close()
    dev = qb.SparseVectorIndex(csr, n_dims)
    n, d, e, b = dev.info()
    assert (n, d, e) == (60_000, n_dims, dims.size) and b >= dims.size * 20
    q = [(np.array([3, 1], np.uint32), np.array([1.0, 2.0], np.float32))]
    assert status(lambda: dev.search(q, 0)) == capi.QB_ERR_INVALID
    assert status(lambda: dev.search(q, 4097)) == capi.QB_ERR_UNSUPPORTED
    assert status(lambda: dev.search([(np.array([3, 3], np.uint32), np.array([1.0, 2.0], np.float32))], 10)) == capi.QB_ERR_INVALID
    assert status(lambda: dev.search(q, 10, is_stopped=True)) == capi.QB_ERR_CANCELLED
    assert status(lambda: dev.search_plain(q, [np.array([60_000], np.uint32)], 10)) == capi.QB_ERR_INVALID
    assert status(lambda: dev.search_plain(q, [np.array([4, 4], np.uint32)], 10)) == capi.QB_ERR_INVALID
    assert status(lambda: dev.search_plain(q, [np.array([4], np.uint32)], 10, is_stopped=True)) == capi.QB_ERR_CANCELLED
    # and a search after them all equals the checker
    want, _ = ref.search(*q[0], 10)
    got = dev.search(q, 10)[0]
    assert np.array_equal(got["idx"], want["idx"]) and np.array_equal(got["score"].view(np.uint32), want["score"].view(np.uint32))
    dev.close()
