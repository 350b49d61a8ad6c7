"""MMR reranking on the device (qb_mmr_batch / qb_mmr_batch_device) == the CPU checker (tests/mmr_ref.c) bit for bit: selected ids in
selection order, their input scores as bit patterns, counts and counters.  Tie-heavy rows (few distinct rows, many exact duplicates), NaN
rows, Cosine rows perturbed past the 1e-6 normalisation test, duplicate ids in the lists and a storage id_base != 0; every distance, the
AVX-tier dims 96 and 100 and the SSE tier at 20; list lengths that put the cluster at 1, 2, 4 and 8 CTAs; the device form chained after
the device searches on the storage's stream; every rejection leaves the device usable."""
import ctypes as C

import numpy as np
import pytest

from tests import mmr_ref as mr

pytestmark = pytest.mark.gpu

ID_BASE = 1000
COUNT = 20_000
NS = (2, 3, 257, 2048, 16384)
LAMBDAS = (0.0, 0.5, 1.0)


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _rows(oracle, distance, dim, seed):
    rng = np.random.default_rng(seed)
    rows = rng.standard_normal((COUNT, dim)).astype(np.float32)
    # tie-heavy block: a handful of distinct small-integer rows, each repeated many times
    distinct = rng.integers(-1, 2, (6, dim)).astype(np.float32)
    tie = rng.random(COUNT) < 0.4
    rows[tie] = distinct[rng.integers(0, 6, int(tie.sum()))]
    if distance == oracle.COSINE:
        rows = oracle.preprocess_rows_f32(oracle.COSINE, rows)
        bump = rng.random(COUNT) < 0.3
        rows[bump] *= np.float32(1.0 + 3e-5)   # |len^2 - 1| > 1e-6: preprocess renormalises these
    rows[rng.integers(0, COUNT, 4)] = np.nan
    rows[rng.integers(0, COUNT, 50)] = 0.0
    return np.ascontiguousarray(rows)


def _lists(rng, ns):
    out = []
    for n in ns:
        ids = rng.choice(COUNT, size=n, replace=False).astype(np.uint32) + ID_BASE
        if n > 3:
            for _ in range(max(1, n // 50)):   # duplicate ids: the first occurrence is kept
                ids[rng.integers(1, n)] = ids[rng.integers(0, n)]
        c = np.zeros(n, mr.SCORED)
        c["idx"] = ids
        c["score"] = rng.standard_normal(n).astype(np.float32)
        c["score"][rng.integers(0, n, max(1, n // 7))] = -0.0
        out.append(c)
    return out


def _queries(rng, rows, k):
    """half near tie rows (exact ties in the relevance), half random"""
    q = rng.standard_normal((k, rows.shape[1])).astype(np.float32)
    q[::2] = np.nan_to_num(rows[rng.integers(0, COUNT, (k + 1) // 2)])
    return q


def _check(qb, oracle, st, rows, distance, queries, lams, lists, limit):
    hw = qb.HwCounters()
    got = st.mmr(queries, lists, lams, limit, counters=hw)
    want, cpu, io = mr.mmr_batch(oracle, rows, distance, queries, lams, lists, limit, id_base=ID_BASE)
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a["idx"], b["idx"]), (i, len(lists[i]), lams[i], a["idx"][:20], b["idx"][:20])
        assert np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)), i
    assert (hw.cpu, hw.vector_io_read) == (cpu, io)


@pytest.mark.parametrize("limit", [1, 10, 100, "n"])
@pytest.mark.parametrize("dim", [96, 20, 100])
@pytest.mark.parametrize("dist", ["Cosine", "Euclid", "Dot", "Manhattan"])
def test_mmr_equals_checker(qb, oracle, dist, dim, limit):
    d = getattr(qb.Distance, dist)
    rows = _rows(oracle, int(d), dim, seed=dim + int(d))
    st = qb.DenseVectorStorage(rows, d)
    qb.lib().qb_storage_set_id_base(st._h, ID_BASE)
    rng = np.random.default_rng(7 * dim + int(d))
    if limit == "n":
        # limit = n: one call per list length, so the cluster is sized from it (1, 1, 2, 4 CTAs)
        for n in NS[:4]:
            lists = _lists(rng, [n] * len(LAMBDAS))
            _check(qb, oracle, st, rows, int(d), _queries(rng, rows, len(LAMBDAS)), np.array(LAMBDAS, np.float32), lists, n)
    else:
        ns = [n for n in NS for _ in LAMBDAS]
        lams = np.array([l for _ in NS for l in LAMBDAS], np.float32)
        _check(qb, oracle, st, rows, int(d), _queries(rng, rows, len(ns)), lams, _lists(rng, ns), limit)
    st.close()


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_device_form_chained_after_device_searches(qb, oracle):
    """qb_search_batch_device / qb_hnsw_search_batch_device -> qb_mmr_batch_device on the storage's stream, no host hop == the host form"""
    import torch

    from qdrant_b200._capi import lib, vp

    dim, top, limit, nq = 96, 600, 25, 12
    rows = _rows(oracle, oracle.COSINE, dim, seed=4)
    rows = np.nan_to_num(rows)
    st = qb.DenseVectorStorage(rows[:8000], qb.Distance.Cosine)
    g = oracle.HNSW(np.ascontiguousarray(rows[:8000]), oracle.COSINE, m=16, ef_construct=64, seed=3, threads=4)
    entry, lvl, m, m0 = g.entry()
    hg = qb.HnswGraph(st, g.export_plain(), m, m0)
    rng = np.random.default_rng(5)
    q = rng.standard_normal((nq, dim)).astype(np.float32)
    lams = rng.random(nq).astype(np.float32)
    dq, dl = _dev(torch, q), _dev(torch, lams)
    stream = torch.cuda.ExternalStream(st.stream_ptr())
    for search in ("scan", "hnsw"):
        dcand = torch.zeros((nq, top, 2), dtype=torch.int32, device="cuda")
        dcnt = torch.zeros(nq, dtype=torch.int32, device="cuda")
        dout = torch.zeros((nq, limit, 2), dtype=torch.int32, device="cuda")
        dout_cnt = torch.zeros(nq, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        if search == "scan":
            assert lib().qb_search_batch_device(st._h, vp(dq.data_ptr()), nq, top, vp(dcand.data_ptr()), vp(dcnt.data_ptr())) == 0
        else:
            assert lib().qb_hnsw_search_batch_device(hg._h, vp(dq.data_ptr()), nq, top, 700, entry, lvl, vp(dcand.data_ptr()), vp(dcnt.data_ptr())) == 0
        assert lib().qb_mmr_batch_device(st._h, vp(dq.data_ptr()), nq, vp(dl.data_ptr()), vp(dcand.data_ptr()), vp(dcnt.data_ptr()), top, limit,
                                         vp(dout.data_ptr()), vp(dout_cnt.data_ptr())) == 0
        stream.synchronize()
        cand = dcand.cpu().numpy().view(mr.SCORED).reshape(nq, top)
        counts = dcnt.cpu().numpy()
        lists = [cand[i, : counts[i]].copy() for i in range(nq)]
        host = st.mmr(q, lists, lams, limit)
        out = dout.cpu().numpy().view(mr.SCORED).reshape(nq, limit)
        oc = dout_cnt.cpu().numpy()
        for i in range(nq):
            assert oc[i] == host[i].size
            assert np.array_equal(out[i, : oc[i]].view(np.uint64), host[i].view(np.uint64)), (search, i)
        want = mr.mmr_batch(oracle, rows[:8000], oracle.COSINE, q, lams, lists, limit)[0]
        for a, b in zip(host, want):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    hg.close(); g.close(); st.close()


def test_rejections_leave_the_device_usable(qb, oracle):
    from qdrant_b200._capi import ScoredPoint, f32p, lib, u32p, vp

    rng = np.random.default_rng(9)
    rows = rng.standard_normal((500, 32)).astype(np.float32)
    st = qb.DenseVectorStorage(rows, qb.Distance.Dot)
    q = rng.standard_normal((2, 32)).astype(np.float32)
    lists = [np.array([(i, 0.0) for i in range(40)], mr.SCORED), np.array([(i, 1.0) for i in range(5, 60)], mr.SCORED)]

    def call(storage, lams, cand, counts, max_c, limit):
        out = np.zeros((2, max(limit, 1)), mr.SCORED)
        oc = np.zeros(2, np.uint32)
        return lib().qb_mmr_batch(storage._h, q.ctypes.data_as(f32p), 2, lams.ctypes.data_as(f32p), cand.ctypes.data_as(C.POINTER(ScoredPoint)),
                                  counts.ctypes.data_as(u32p), max_c, limit, out.ctypes.data_as(C.POINTER(ScoredPoint)), oc.ctypes.data_as(u32p), None)

    cand = np.zeros((2, 60), mr.SCORED)
    cand[0, :40], cand[1, :55] = lists
    counts = np.array([40, 55], np.uint32)
    ok = np.array([0.5, 0.5], np.float32)
    INVALID, UNSUPPORTED = -1, -3
    assert call(st, np.array([0.5, np.nan], np.float32), cand, counts, 60, 5) == INVALID
    assert call(st, np.array([-0.01, 0.5], np.float32), cand, counts, 60, 5) == INVALID
    assert call(st, np.array([0.5, 1.01], np.float32), cand, counts, 60, 5) == INVALID
    assert call(st, ok, cand, counts, 60, 0) == INVALID
    assert call(st, ok, cand, np.array([40, 61], np.uint32), 60, 5) == INVALID
    bad = cand.copy()
    bad[1, 3]["idx"] = 500
    assert call(st, ok, bad, counts, 60, 5) == INVALID
    big = np.zeros((2, 16385), mr.SCORED)
    assert call(st, ok, big, counts, 16385, 5) == UNSUPPORTED
    assert lib().qb_mmr_batch(st._h, None, 2, ok.ctypes.data_as(f32p), None, None, 60, 5, None, None, None) == INVALID
    u8 = qb.DenseVectorStorage(rng.integers(0, 4, (500, 32)).astype(np.uint8), qb.Distance.Dot, qb.VectorStorageDatatype.Uint8)
    assert call(u8, ok, cand, counts, 60, 5) == UNSUPPORTED
    assert lib().qb_mmr_batch_device(u8._h, None, 2, None, None, None, 60, 5, None, None) == INVALID
    assert lib().qb_mmr_batch_device(u8._h, vp(1), 2, vp(1), vp(1), vp(1), 60, 5, vp(1), vp(1)) == UNSUPPORTED
    assert lib().qb_mmr_batch_device(st._h, vp(1), 2, vp(1), vp(1), vp(1), 16385, 5, vp(1), vp(1)) == UNSUPPORTED
    assert lib().qb_mmr_batch_device(st._h, vp(1), 2, vp(1), vp(1), vp(1), 60, 0, vp(1), vp(1)) == INVALID
    u8.close()
    # the device is still usable: the same storage answers a valid batch == the checker
    got = st.mmr(q, lists, ok, 5)
    want = mr.mmr_batch(oracle, rows, oracle.DOT, q, ok, lists, 5)[0]
    for a, b in zip(got, want):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    st.close()
