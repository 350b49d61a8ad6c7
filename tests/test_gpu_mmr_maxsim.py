"""MMR reranking over multivector candidates on the device (qb_mmr_maxsim_batch / qb_mmr_maxsim_batch_device) == the CPU checker
(tests/mmr_maxsim_ref.c) bit for bit: selected ids in selection order, their input scores as bit patterns, counts and counters.  Every
distance; dims 128 and 100 (AVX tier, with and without a tail) and 20 (SSE tier); one token per point and 1..64 tokens; a pick too large to
stage in shared memory; query vectors 1 / 32 / 4096; lists that put the cluster at 1, 2, 4 and 8 CTAs; limits 1 / 10 / 100 / n; lambda
0 / 0.5 / 1; Cosine tokens perturbed past the 1e-6 normalisation test and a Cosine batch over more than one scratch chunk.  With one token
per point the path equals qb_mmr_batch over the same rows; the device form chained after qb_hnsw_search_maxsim_batch_device equals the
host form; every rejection leaves the device usable."""
import ctypes as C

import numpy as np
import pytest

from tests import mmr_maxsim_ref as mr
from tests import mmr_ref

pytestmark = pytest.mark.gpu

LAMBDAS = (0.0, 0.5, 1.0)


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _collection(oracle, distance, dim, n_points, lens, seed, nan=True):
    rng = np.random.default_rng(seed)
    runs = rng.integers(lens[0], max(lens[0], min(lens[1], 8)) + 1, n_points)   # mostly short runs, so the checker stays cheap; 5 % up to the maximum
    long = rng.random(n_points) < 0.05
    runs[long] = rng.integers(lens[0], lens[1] + 1, int(long.sum()))
    off = np.concatenate([[0], np.cumsum(runs)]).astype(np.uint32)
    n_rows = int(off[-1])
    rows = rng.standard_normal((n_rows, dim)).astype(np.float32)
    distinct = rng.integers(-1, 2, (5, dim)).astype(np.float32)   # tie-heavy tokens
    tie = rng.random(n_rows) < 0.3
    rows[tie] = distinct[rng.integers(0, 5, int(tie.sum()))]
    if distance == oracle.COSINE:
        rows = oracle.preprocess_rows_f32(oracle.COSINE, rows)
        bump = rng.random(n_rows) < 0.3
        rows[bump] *= np.float32(1.0 + 3e-5)   # |len^2 - 1| > 1e-6: preprocess renormalises these
    if nan:
        rows[rng.integers(0, n_rows, 3)] = np.nan
    rows[rng.integers(0, n_rows, 20)] = 0.0
    return np.ascontiguousarray(rows), off


def _lists(rng, ns, n_points):
    out = []
    for n in ns:
        ids = rng.choice(n_points, size=n, replace=False).astype(np.uint32)
        if n > 3:
            for _ in range(max(1, n // 50)):   # duplicate ids: the first occurrence is kept
                ids[rng.integers(1, n)] = ids[rng.integers(0, n)]
        c = np.zeros(n, mr.SCORED)
        c["idx"] = ids
        c["score"] = rng.standard_normal(n).astype(np.float32)
        c["score"][rng.integers(0, n, max(1, n // 7))] = -0.0
        out.append(c)
    return out


def _check(qb, oracle, view, rows, off, distance, queries, lams, lists, limit):
    hw = qb.HwCounters()
    got = view.mmr(queries, lists, lams, limit, counters=hw)
    want, cpu, io = mr.mmr_batch(oracle, rows, off, distance, queries, lams, lists, limit)
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a["idx"], b["idx"]), (i, len(lists[i]), lams[i], a["idx"][:20], b["idx"][:20])
        assert np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)), i
    assert (hw.cpu, hw.vector_io_read) == (cpu, io)


@pytest.mark.parametrize("limit", [1, 10, 100, "n"])
@pytest.mark.parametrize("dim,lens", [(128, (1, 64)), (128, (1, 1)), (20, (1, 64)), (100, (1, 16))])
@pytest.mark.parametrize("dist", ["Cosine", "Euclid", "Dot", "Manhattan"])
def test_mmr_maxsim_equals_checker(qb, oracle, dist, dim, lens, limit):
    d = getattr(qb.Distance, dist)
    n_points = 3000
    rows, off = _collection(oracle, int(d), dim, n_points, lens, seed=dim + int(d) + lens[1])
    st = qb.DenseVectorStorage(rows, d)
    view = qb.MultiVectorView(st, off)
    rng = np.random.default_rng(7 * dim + int(d) + lens[1])
    ns = (2, 3, 257) if limit == "n" else (2, 3, 257, 1100)
    qs = [rng.standard_normal((int(t), dim)).astype(np.float32) for t in rng.choice([1, 32, 3], len(ns) * len(LAMBDAS))]
    qs[0] = np.nan_to_num(rows[off[5] : off[6]])   # a query equal to a point: exact ties in the relevance
    lams = np.array([l for _ in ns for l in LAMBDAS], np.float32)
    if limit == "n":
        # limit = n: one call per list length, so the cluster is sized from it
        for k, n in enumerate(ns):
            sl = slice(k * len(LAMBDAS), (k + 1) * len(LAMBDAS))
            _check(qb, oracle, view, rows, off, int(d), qs[sl], lams[sl], _lists(rng, [n] * len(LAMBDAS), n_points), n)
    else:
        _check(qb, oracle, view, rows, off, int(d), qs, lams, _lists(rng, [n for n in ns for _ in LAMBDAS], n_points), limit)
    st.close()


@pytest.mark.parametrize("dist", ["Cosine", "Dot"])
def test_long_lists_and_wide_queries(qb, oracle, dist):
    """lists of 2 048 and 16 384 (4 and 8 CTAs) on few tokens and a small dim; a query of 4096 vectors; a pick of 64 x 1024-d (256 KB,
    read from global memory)"""
    d = getattr(qb.Distance, dist)
    rows, off = _collection(oracle, int(d), 20, 20_000, (1, 2), seed=31 + int(d))
    st = qb.DenseVectorStorage(rows, d)
    view = qb.MultiVectorView(st, off)
    rng = np.random.default_rng(3 + int(d))
    qs = [rng.standard_normal((t, 20)).astype(np.float32) for t in (1, 4096, 3)]
    lams = np.array([0.5, 1.0, 0.0], np.float32)
    lists = _lists(rng, [2048, 16384, 16384], 20_000)
    _check(qb, oracle, view, rows, off, int(d), qs, lams, lists, 10)
    st.close()
    rows, off = _collection(oracle, int(d), 1024, 40, (60, 64), seed=5, nan=False)
    st = qb.DenseVectorStorage(rows, d)
    view = qb.MultiVectorView(st, off)
    qs = [rng.standard_normal((t, 1024)).astype(np.float32) for t in (2, 32)]
    _check(qb, oracle, view, rows, off, int(d), qs, np.array([0.5, 0.3], np.float32), _lists(rng, [40, 17], 40), 8)
    st.close()


def test_cosine_scratch_chunks(qb, oracle):
    """16 384 candidates of up to 8 tokens x 1024-d: 512 MB of preprocessed rows per query, so every query is its own scratch chunk"""
    d = qb.Distance.Cosine
    rows, off = _collection(oracle, 0, 1024, 16_384, (1, 8), seed=41, nan=False)
    st = qb.DenseVectorStorage(rows, d)
    view = qb.MultiVectorView(st, off)
    rng = np.random.default_rng(43)
    qs = [rng.standard_normal((2, 1024)).astype(np.float32) for _ in range(3)]
    lists = _lists(rng, [16384, 300, 16384], 16_384)
    _check(qb, oracle, view, rows, off, 0, qs, np.array([0.5, 0.0, 1.0], np.float32), lists, 3)
    st.close()


@pytest.mark.parametrize("dist", ["Cosine", "Euclid", "Dot", "Manhattan"])
def test_one_token_per_point_equals_dense_mmr(qb, oracle, dist):
    """one token per point: qb_mmr_maxsim_batch == qb_mmr_batch over the same rows (NaN-free), list for list"""
    d = getattr(qb.Distance, dist)
    rows, off = _collection(oracle, int(d), 96, 4000, (1, 1), seed=50 + int(d), nan=False)
    st = qb.DenseVectorStorage(rows, d)
    view = qb.MultiVectorView(st, off)
    rng = np.random.default_rng(51)
    ns = [2, 3, 257, 2048]
    lists = _lists(rng, [n for n in ns for _ in LAMBDAS], 4000)
    q = rng.standard_normal((len(lists), 96)).astype(np.float32)
    lams = np.array([l for _ in ns for l in LAMBDAS], np.float32)
    for limit in (1, 10, 100):
        a = view.mmr([x[None] for x in q], lists, lams, limit)
        b = st.mmr(q, lists, lams, limit)
        for x, y in zip(a, b):
            assert np.array_equal(x.view(np.uint64), y.view(np.uint64))
    st.close()


def test_device_form_chained_after_device_hnsw(qb, oracle):
    """qb_hnsw_search_maxsim_batch_device -> qb_mmr_maxsim_batch_device on the token storage's stream, no host hop == the host form"""
    import torch

    from qdrant_b200._capi import lib, u32p, vp

    dim, n_points, top, limit = 64, 1500, 300, 20
    rows, off = _collection(oracle, oracle.COSINE, dim, n_points, (1, 12), seed=61, nan=False)
    st = qb.DenseVectorStorage(rows, qb.Distance.Cosine)
    view = qb.MultiVectorView(st, off)
    means = np.stack([rows[off[p] : off[p + 1]].mean(0) for p in range(n_points)]).astype(np.float32)
    g = oracle.HNSW(oracle.preprocess_rows_f32(oracle.COSINE, means), oracle.COSINE, m=16, ef_construct=64, seed=3)
    entry, lvl, m, m0 = g.entry()
    hg = qb.HnswGraph.multivector(view, g.export_plain(), m, m0)
    rng = np.random.default_rng(62)
    qs = [rng.standard_normal((t, dim)).astype(np.float32) for t in (1, 32, 5, 12)]
    nq = len(qs)
    q_off = np.concatenate([[0], np.cumsum([q.shape[0] for q in qs])]).astype(np.int32)
    lams = rng.random(nq).astype(np.float32)
    dq = torch.from_numpy(np.concatenate(qs)).cuda()
    doff = torch.from_numpy(q_off).cuda()
    dl = torch.from_numpy(lams).cuda()
    dcand = torch.zeros((nq, top, 2), dtype=torch.int32, device="cuda")
    dcnt = torch.zeros(nq, dtype=torch.int32, device="cuda")
    dout = torch.zeros((nq, limit, 2), dtype=torch.int32, device="cuda")
    dout_cnt = torch.zeros(nq, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    qb.check(lib().qb_hnsw_search_maxsim_batch_device(hg._h, dq.data_ptr(), dq.shape[0], doff.data_ptr(), nq, 32, top, 320, entry, lvl, dcand.data_ptr(),
                                                      dcnt.data_ptr(), 0))
    qb.check(lib().qb_mmr_maxsim_batch_device(st._h, view.offsets.ctypes.data_as(u32p), view.n_points, vp(dq.data_ptr()), dq.shape[0], vp(doff.data_ptr()), nq, 32,
                                              vp(dl.data_ptr()), vp(dcand.data_ptr()), vp(dcnt.data_ptr()), top, limit, vp(dout.data_ptr()),
                                              vp(dout_cnt.data_ptr())))
    torch.cuda.ExternalStream(st.stream_ptr()).synchronize()
    cand = dcand.cpu().numpy().view(mr.SCORED).reshape(nq, top)
    counts = dcnt.cpu().numpy()
    lists = [cand[i, : counts[i]].copy() for i in range(nq)]
    host = view.mmr(qs, lists, lams, limit)
    out = dout.cpu().numpy().view(mr.SCORED).reshape(nq, limit)
    oc = dout_cnt.cpu().numpy()
    want = mr.mmr_batch(oracle, rows, off, oracle.COSINE, qs, lams, lists, limit)[0]
    for i in range(nq):
        assert oc[i] == host[i].size == min(limit, counts[i]) and counts[i] > 0
        assert np.array_equal(out[i, : oc[i]].view(np.uint64), host[i].view(np.uint64)), i
        assert np.array_equal(host[i].view(np.uint64), want[i].view(np.uint64)), i
    hg.close(); g.close(); st.close()


def test_rejections_leave_the_device_usable(qb, oracle):
    from qdrant_b200._capi import ScoredPoint, f32p, lib, u32p, vp

    rng = np.random.default_rng(9)
    rows, off = _collection(oracle, oracle.DOT, 32, 200, (1, 4), seed=9, nan=False)
    off = off.copy()
    off[8] = off[7]   # point 7 has no token rows
    st = qb.DenseVectorStorage(rows, qb.Distance.Dot)
    view = qb.MultiVectorView(st, off)
    qv = rng.standard_normal((5, 32)).astype(np.float32)
    q_off = np.array([0, 2, 5], np.uint32)
    ids0, ids1 = [i for i in range(40) if i != 7], list(range(50, 105))
    lists = [np.array([(i, 0.0) for i in ids0], mr.SCORED), np.array([(i, 1.0) for i in ids1], mr.SCORED)]
    cand = np.zeros((2, 60), mr.SCORED)
    cand[0, : len(ids0)], cand[1, : len(ids1)] = lists
    counts = np.array([len(ids0), len(ids1)], np.uint32)
    ok = np.array([0.5, 0.5], np.float32)

    def call(storage, lams=ok, cand=cand, counts=counts, max_c=60, limit=5, offs=off, q_off=q_off, n_points=None):
        out = np.zeros((2, max(limit, 1)), mr.SCORED)
        oc = np.zeros(2, np.uint32)
        return lib().qb_mmr_maxsim_batch(storage._h, offs.ctypes.data_as(u32p), offs.size - 1 if n_points is None else n_points, qv.ctypes.data_as(f32p),
                                         q_off.ctypes.data_as(u32p), 2, lams.ctypes.data_as(f32p), cand.ctypes.data_as(C.POINTER(ScoredPoint)),
                                         counts.ctypes.data_as(u32p), max_c, limit, out.ctypes.data_as(C.POINTER(ScoredPoint)), oc.ctypes.data_as(u32p), None)

    INVALID, UNSUPPORTED = -1, -3
    assert call(st, lams=np.array([0.5, np.nan], np.float32)) == INVALID
    assert call(st, lams=np.array([-0.01, 0.5], np.float32)) == INVALID
    assert call(st, lams=np.array([0.5, 1.01], np.float32)) == INVALID
    assert call(st, limit=0) == INVALID
    assert call(st, counts=np.array([39, 61], np.uint32)) == INVALID
    bad = cand.copy()
    bad[1, 3]["idx"] = 200
    assert call(st, cand=bad) == INVALID
    empty = cand.copy()
    empty[0, 2]["idx"] = 7
    assert call(st, cand=empty) == INVALID
    desc = off.copy()
    desc[3] = desc[4] + 1
    assert call(st, offs=desc) == INVALID
    past = off.copy()
    past[-1] = rows.shape[0] + 1
    assert call(st, offs=past) == INVALID
    assert call(st, q_off=np.array([0, 0, 5], np.uint32)) == INVALID
    assert call(st, q_off=np.array([0, 2, 1], np.uint32)) == INVALID
    assert call(st, cand=np.zeros((2, 16385), mr.SCORED), max_c=16385) == UNSUPPORTED
    assert lib().qb_mmr_maxsim_batch(st._h, None, 200, None, None, 2, ok.ctypes.data_as(f32p), None, None, 60, 5, None, None, None) == INVALID
    too_many = np.zeros((4097, 32), np.float32)
    big_off = np.array([0, 4097, 4097], np.uint32)
    assert lib().qb_mmr_maxsim_batch(st._h, off.ctypes.data_as(u32p), 200, too_many.ctypes.data_as(f32p), big_off.ctypes.data_as(u32p), 1,
                                     ok.ctypes.data_as(f32p), cand.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p), 60, 5,
                                     np.zeros(5, mr.SCORED).ctypes.data_as(C.POINTER(ScoredPoint)), np.zeros(1, np.uint32).ctypes.data_as(u32p), None) == INVALID
    u8 = qb.DenseVectorStorage(rng.integers(0, 4, rows.shape).astype(np.uint8), qb.Distance.Dot, qb.VectorStorageDatatype.Uint8)
    f16 = qb.DenseVectorStorage(rows.astype(np.float16), qb.Distance.Dot, qb.VectorStorageDatatype.Float16)
    sq = oracle.SQ8.encode(rows, int(qb.construct_vector_parameters(qb.Distance.Dot)[0]), bool(qb.construct_vector_parameters(qb.Distance.Dot)[1]))
    sq8 = qb.ScalarQuantizedVectors(sq.rows, 32, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, qb.Distance.Dot)
    assert call(u8) == UNSUPPORTED and call(f16) == UNSUPPORTED and call(sq8) == UNSUPPORTED
    sq8.close()
    dev = lambda storage, offs=off, mq=4, max_c=60, limit=5: lib().qb_mmr_maxsim_batch_device(  # noqa: E731
        storage._h, offs.ctypes.data_as(u32p), offs.size - 1, vp(1), 5, vp(1), 2, mq, vp(1), vp(1), vp(1), max_c, limit, vp(1), vp(1))
    assert dev(u8) == UNSUPPORTED
    assert dev(st, max_c=16385) == UNSUPPORTED
    assert dev(st, limit=0) == INVALID
    assert dev(st, mq=0) == INVALID and dev(st, mq=4097) == INVALID
    assert dev(st, offs=desc) == INVALID and dev(st, offs=past) == INVALID
    assert lib().qb_mmr_maxsim_batch_device(st._h, None, 200, vp(1), 5, vp(1), 2, 4, vp(1), vp(1), vp(1), 60, 5, vp(1), vp(1)) == INVALID
    u8.close(); f16.close()
    # the device is still usable: the same storage answers a valid batch == the checker
    qs = [qv[:2], qv[2:]]
    got = view.mmr(qs, lists, ok, 5)
    want = mr.mmr_batch(oracle, rows, off, oracle.DOT, qs, ok, lists, 5)[0]
    for a, b in zip(got, want):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    st.close()
