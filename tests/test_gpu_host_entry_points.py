"""What the host search entry points share: a pre-set stop flag cancels each of them, the host and the device-resident form of a
search return the same lists (score bits included) for query batches whose raw bytes are not a multiple of 16, and a deleted
bitmap reaches every HNSW host form (an all-clear bitmap changes nothing; deleted points never come back)."""
import ctypes as C
import threading

import numpy as np
import pytest

from tests import graph_links_with_vectors as gv

pytestmark = pytest.mark.gpu

TOP, EF = 10, 64


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _same(got, want, what):
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a["idx"], b["idx"]), (what, i, a, b)
        assert np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)), (what, i, a, b)


class _Env:
    """Cosine rows of `dim` in a dense f32 and an SQ8 storage, one oracle-built graph over them bound to the dense storage (plain
    links) and to the SQ8 storage (inline vectors), and a multivector collection over the dense rows with a graph over its points."""

    def __init__(self, qb, oracle, dim, n=3000, seed=5):
        rng = self.rng = np.random.default_rng(seed)
        self.dim, self.n = dim, n
        d = qb.Distance.Cosine
        base = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((n, dim)).astype(np.float32))
        g = oracle.HNSW(base, oracle.COSINE, m=16, ef_construct=64, seed=11, threads=4)
        self.entry, self.level, m, m0 = g.entry()
        blob = g.export_plain()
        g.close()
        self.st = qb.DenseVectorStorage(base, d)
        self.hg = qb.HnswGraph(self.st, blob, m, m0)
        dt, inv = qb.construct_vector_parameters(d)
        sq = oracle.SQ8.encode(base, int(dt), bool(inv))
        self.sq = qb.ScalarQuantizedVectors(sq.rows, dim, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, d)
        inline = gv.serialize_with_vectors(gv.edges_of_plain(blob), m, m0, lambda i: base[i].tobytes(), lambda i: sq.rows[i].tobytes(), (dim * 4, 4),
                                           (sq.row_bytes, 1))
        self.hi = qb.HnswGraph.from_compressed_with_vectors(self.sq, inline)
        runs = rng.integers(1, 5, n // 4)   # point p = dense rows [off[p], off[p + 1])
        self.off = np.concatenate([[0], np.cumsum(runs)]).astype(np.uint32)
        self.n_points = runs.size
        self.view = qb.MultiVectorView(self.st, self.off)
        means = np.stack([base[self.off[p] : self.off[p + 1]].mean(0) for p in range(self.n_points)]).astype(np.float32)
        gm = oracle.HNSW(oracle.preprocess_rows_f32(oracle.COSINE, means), oracle.COSINE, m=16, ef_construct=64, seed=1)
        self.mv_entry, self.mv_level, mm, mm0 = gm.entry()
        self.hm = qb.HnswGraph.multivector(self.view, gm.export_plain(), mm, mm0)
        gm.close()

    def vectors(self, *shape):
        return np.ascontiguousarray(self.rng.standard_normal((*shape, self.dim)).astype(np.float32))

    def close(self):
        for h in (self.hm, self.hi, self.hg, self.sq, self.st):
            h.close()


@pytest.fixture(scope="module", params=[37, 40], ids=lambda d: f"dim{d}")
def env(request, qb, oracle):
    e = _Env(qb, oracle, request.param)
    yield e
    e.close()


# ------------------------------------------------------------------------------------------------ cancellation
def _cancel_calls(qb, e):
    """entry point -> call(stop): each host entry point that takes a stop flag, on a small valid request"""
    from qdrant_b200._capi import ScoredPoint, f32p, lib, u32p

    L, SP = lib(), C.POINTER(ScoredPoint)
    out = np.zeros((4, TOP), dtype=qb.SCORED_POINT_OFFSET)
    cnt = np.zeros(4, np.uint32)
    o, c = out.ctypes.data_as(SP), cnt.ctypes.data_as(u32p)
    reco, feedback, q = e.vectors(2), e.vectors(3), e.vectors(3)
    partial = np.array([0.25], np.float32)
    reco_b, discover_b = e.vectors(2, 2), e.vectors(2, 3)
    mv, mv_off = e.vectors(5), np.array([0, 2, 5], np.uint32)
    reco_kind = int(qb.QueryKind.RecommendBestScore)
    p = lambda a: a.ctypes.data_as(f32p)   # noqa: E731
    return {
        "search_custom": lambda stop: L.qb_search_custom(e.st._h, reco_kind, p(reco), 1, 1, TOP, None, None, 0, stop, o, c, None),
        "search_feedback": lambda stop: L.qb_search_feedback(e.st._h, p(feedback), 1, 0.5, p(partial), TOP, None, None, 0, stop, o, c, None),
        "hnsw_search_batch_algo-hnsw": lambda stop: L.qb_hnsw_search_batch_algo(e.hg._h, p(q), 3, TOP, EF, e.entry, e.level, None, stop, o, c, None, 0),
        "hnsw_search_batch_algo-acorn": lambda stop: L.qb_hnsw_search_batch_algo(e.hg._h, p(q), 3, TOP, EF, e.entry, e.level, None, stop, o, c, None, 1),
        "hnsw_search_maxsim_batch": lambda stop: L.qb_hnsw_search_maxsim_batch(e.hm._h, p(mv), mv_off.ctypes.data_as(u32p), 2, TOP, EF, e.mv_entry,
                                                                               e.mv_level, None, stop, o, c, None, 0),
        "hnsw_search_custom_batch": lambda stop: L.qb_hnsw_search_custom_batch(e.hg._h, reco_kind, p(reco_b), 1, 1, None, 2, TOP, EF, e.entry, e.level,
                                                                               None, None, 0, None, stop, o, c, None, 0),
        "hnsw_search_discover_batch": lambda stop: L.qb_hnsw_search_discover_batch(e.hg._h, p(discover_b), 1, 2, TOP, EF, e.entry, e.level, None, stop,
                                                                                   o, c, None, 0),
    }


CANCEL_ENTRIES = ["search_custom", "search_feedback", "hnsw_search_batch_algo-hnsw", "hnsw_search_batch_algo-acorn", "hnsw_search_maxsim_batch",
                  "hnsw_search_custom_batch", "hnsw_search_discover_batch"]


@pytest.mark.parametrize("entry", CANCEL_ENTRIES)
def test_preset_stop_flag_cancels(qb, env, entry):
    from qdrant_b200._capi import QB_ERR_CANCELLED, QB_OK, lib

    call = _cancel_calls(qb, env)[entry]
    assert call(None) == QB_OK, lib().qb_last_error()
    assert call(C.byref(C.c_int32(0))) == QB_OK, lib().qb_last_error()
    assert call(C.byref(C.c_int32(1))) == QB_ERR_CANCELLED
    assert lib().qb_last_error() == b"search cancelled"
    assert call(None) == QB_OK, lib().qb_last_error()   # the pooled context went back to the storage


def test_multi_search_cancelled_in_the_scan_still_joins_the_exchange(qb, oracle):
    """qb_multi_search_batch checks the flag only inside the scan (shards below 65 536 rows reach its chunk loop), so that a cancelled
    rank still joins the exchange: both ranks return QB_ERR_CANCELLED, and the next collective call equals the unsharded search."""
    from qdrant_b200._capi import QB_ERR_CANCELLED, QB_OK, ScoredPoint, check, f32p, lib, u32p, vp
    from qdrant_b200.sharded import shard_ranges

    world, n, dim, nq = 2, 40_000, 32, 3
    rng = np.random.default_rng(17)
    base = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((n, dim)).astype(np.float32))
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    single = qb.DenseVectorStorage(base, qb.Distance.Cosine)
    shards, comms = [], (vp * world)()
    for r, (b, e) in enumerate(shard_ranges(n, world)):
        st = qb.DenseVectorStorage(base[b:e], qb.Distance.Cosine)
        check(lib().qb_storage_set_id_base(st._h, b))
        shards.append(st)
        h = vp()
        check(lib().qb_comm_create(0, r, world, 64, 16, C.byref(h)))
        comms[r] = h
    check(lib().qb_comm_connect_local(comms, world))

    def collective(stop_value):
        res = [None] * world

        def task(r):
            stop = None if stop_value is None else C.c_int32(stop_value)
            out = np.zeros((nq, TOP), dtype=qb.SCORED_POINT_OFFSET)
            cnt = np.zeros(nq, np.uint32)
            st = lib().qb_multi_search_batch(comms[r], shards[r]._h, queries.ctypes.data_as(f32p), nq, TOP, None, None if stop is None else C.byref(stop),
                                             out.ctypes.data_as(C.POINTER(ScoredPoint)), cnt.ctypes.data_as(u32p), None)
            res[r] = (st, lib().qb_last_error(), [out[i, : cnt[i]].copy() for i in range(nq)])   # the error text is per thread

        th = [threading.Thread(target=task, args=(r,)) for r in range(world)]
        for t in th:
            t.start()
        for t in th:
            t.join(timeout=120)
        assert not any(t.is_alive() for t in th), "a rank did not return from the exchange"
        return res

    for r, (st, err, _) in enumerate(collective(1)):
        assert (st, err) == (QB_ERR_CANCELLED, b"search cancelled"), (r, st, err)
    want = single.search_batch(queries, TOP)
    for r, (st, err, got) in enumerate(collective(None)):
        assert st == QB_OK, (r, err)
        _same(got, want, f"rank {r} after a cancelled call")
    for r in range(world):
        lib().qb_comm_destroy(comms[r])
        shards[r].close()
    single.close()


# ------------------------------------------------------------------------------------------------ host form == device form
def _device_lists(qb, nq, call):
    """call(dev_out, dev_counts) on the device form; its lists back on the host"""
    import torch

    from qdrant_b200._capi import check, vp

    out = torch.zeros((nq, TOP), dtype=torch.int64, device="cuda")
    cnt = torch.zeros(nq, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    check(call(vp(out.data_ptr()), vp(cnt.data_ptr())))
    torch.cuda.synchronize()
    rec = out.cpu().numpy().view(qb.SCORED_POINT_OFFSET).reshape(nq, TOP)
    c = cnt.cpu().numpy()
    return [rec[i, : c[i]].copy() for i in range(nq)]


@pytest.mark.parametrize("kind", ["f32", "sq8"])
def test_search_batch_host_equals_device(qb, oracle, env, kind):
    """150 000 rows: the sampled threshold and the filter pass run, with the flags word read back by both forms"""
    import torch

    from qdrant_b200._capi import lib, vp

    dim, n = env.dim, 150_000
    rng = np.random.default_rng(dim)
    base = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((n, dim)).astype(np.float32))
    if kind == "sq8":
        dt, inv = qb.construct_vector_parameters(qb.Distance.Cosine)
        sq = oracle.SQ8.encode(base, int(dt), bool(inv))
        st = qb.ScalarQuantizedVectors(sq.rows, dim, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, qb.Distance.Cosine)
    else:
        st = qb.DenseVectorStorage(base, qb.Distance.Cosine)
    for nq in (3, 1):
        q = rng.standard_normal((nq, dim)).astype(np.float32)
        dq = torch.from_numpy(q).cuda()
        got = _device_lists(qb, nq, lambda o, c: lib().qb_search_batch_device(st._h, vp(dq.data_ptr()), nq, TOP, o, c))
        _same(got, st.search_batch(q, TOP), f"{kind} dim {dim} nq {nq}")
    st.close()


@pytest.mark.parametrize("algorithm", ["hnsw", "acorn"])
def test_hnsw_host_equals_device(qb, env, algorithm):
    import torch

    from qdrant_b200._capi import lib, vp

    q = env.vectors(3)
    dq = torch.from_numpy(q).cuda()
    algo = qb.HnswGraph.ALGORITHMS[algorithm]
    got = _device_lists(qb, 3, lambda o, c: lib().qb_hnsw_search_batch_device_algo(env.hg._h, vp(dq.data_ptr()), 3, TOP, EF, env.entry, env.level, o, c,
                                                                                    algo))
    _same(got, env.hg.search(q, TOP, EF, env.entry, env.level, algorithm=algorithm), f"dim {env.dim} {algorithm}")


def test_hnsw_with_vectors_host_equals_device(qb, env):
    import torch

    from qdrant_b200._capi import lib, vp

    q = env.vectors(3)
    dq = torch.from_numpy(q).cuda()
    got = _device_lists(qb, 3, lambda o, c: lib().qb_hnsw_search_with_vectors_batch_device(env.hi._h, vp(dq.data_ptr()), 3, TOP, EF, env.entry,
                                                                                            env.level, o, c))
    _same(got, env.hi.search_with_vectors(q, TOP, EF, env.entry, env.level), f"dim {env.dim}")


@pytest.mark.parametrize("algorithm", ["hnsw", "acorn"])
def test_hnsw_maxsim_host_equals_device(qb, env, algorithm):
    import torch

    from qdrant_b200._capi import lib, vp

    qs = [env.vectors(2), env.vectors(1)]   # three query vectors in all
    off = np.array([0, 2, 3], np.int32)
    dq = torch.from_numpy(np.concatenate(qs)).cuda()
    doff = torch.from_numpy(off).cuda()
    algo = qb.HnswGraph.ALGORITHMS[algorithm]
    got = _device_lists(qb, 2, lambda o, c: lib().qb_hnsw_search_maxsim_batch_device(env.hm._h, vp(dq.data_ptr()), 3, vp(doff.data_ptr()), 2, 2, TOP, EF,
                                                                                      env.mv_entry, env.mv_level, o, c, algo))
    _same(got, env.hm.search_maxsim(qs, TOP, EF, env.mv_entry, env.mv_level, algorithm=algorithm), f"dim {env.dim} {algorithm}")


# ------------------------------------------------------------------------------------------------ deleted bitmaps
def _hnsw_host_forms(qb, e):
    """form -> (search(point_deleted), number of items the bitmap covers, the graph's entry point)"""
    q, mq = e.vectors(3), [e.vectors(2), e.vectors(3), e.vectors(1)]
    reco, discover, feedback = e.vectors(3, 2), e.vectors(3, 3), e.vectors(3, 3)
    coef = np.array([[0.5, 0.25]] * 3, np.float32)
    at = dict(top=TOP, ef=EF, entry_point=e.entry, entry_level=e.level)
    return {
        "hnsw": (lambda pd: e.hg.search(q, TOP, EF, e.entry, e.level, point_deleted=pd), e.n, e.entry),
        "acorn": (lambda pd: e.hg.search(q, TOP, EF, e.entry, e.level, point_deleted=pd, algorithm="acorn"), e.n, e.entry),
        "with_vectors": (lambda pd: e.hi.search_with_vectors(q, TOP, EF, e.entry, e.level, point_deleted=pd), e.n, e.entry),
        "maxsim": (lambda pd: e.hm.search_maxsim(mq, TOP, EF, e.mv_entry, e.mv_level, point_deleted=pd), e.n_points, e.mv_entry),
        "maxsim-acorn": (lambda pd: e.hm.search_maxsim(mq, TOP, EF, e.mv_entry, e.mv_level, point_deleted=pd, algorithm="acorn"), e.n_points, e.mv_entry),
        "custom": (lambda pd: e.hg.search_custom(qb.QueryKind.RecommendBestScore, reco, 1, 1, point_deleted=pd, **at), e.n, e.entry),
        "feedback": (lambda pd: e.hg.search_custom(qb.QueryKind.FeedbackNaive, feedback, 1, coef=coef, point_deleted=pd, **at), e.n, e.entry),
        "discover": (lambda pd: e.hg.search_discover(discover, 1, point_deleted=pd, **at), e.n, e.entry),
    }


@pytest.mark.parametrize("form", ["hnsw", "acorn", "with_vectors", "maxsim", "maxsim-acorn", "custom", "feedback", "discover"])
def test_deleted_bitmap_on_every_hnsw_host_form(qb, env, form):
    search, n_items, entry = _hnsw_host_forms(qb, env)[form]
    plain = search(None)
    assert sum(a.size for a in plain) > 0
    _same(search(np.zeros(n_items, bool)), plain, f"{form}: all-clear bitmap")
    deleted = np.random.default_rng(3).random(n_items) < 0.3
    deleted[np.concatenate([a["idx"] for a in plain]).astype(np.int64)] = True   # every point of the unfiltered answer is gone
    deleted[entry] = False   # get_entry_point picks a point that passes the filter; the search takes the given one as it is
    got = search(deleted)
    assert sum(a.size for a in got) > 0, form
    for i, a in enumerate(got):
        assert not deleted[a["idx"].astype(np.int64)].any(), (form, i, a)
