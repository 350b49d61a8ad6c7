"""Sharded search through the C ABI (qb_comm_* / qb_multi_search_batch): W shards, one host thread per shard (the reference's
one-blocking-task-per-segment model, segments_searcher.rs:255), lists exchanged through peer-mapped buffers and merged on the
device.  Shards are spread over the visible GPUs; on a single-GPU box they share device 0, which exercises the same exchange
protocol (flags, parity slots, merge) through same-device pointers — so the sharded == single gate runs everywhere."""
import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _case(world, nq, top, n, dim, kind="f32"):
    return pytest.param(world, nq, top, n, dim, kind, id="-".join(map(str, (world, nq, top, n, dim))) + ("" if kind == "f32" else f"-{kind}"))


@pytest.mark.parametrize("world,nq,top,n,dim,kind", [_case(2, 1, 10, 150_003, 64), _case(3, 5, 10, 90_001, 96), _case(4, 40, 7, 70_000, 32),
                                                     _case(8, 1, 10, 80_000, 128),
                                                     _case(2, 1, 10, 1_200_001, 64),   # shards of >= 2^19 rows answer through the shadow-plane scan
                                                     _case(2, 12, 10, 150_002, 128, "pq"),   # pq_scan16_kernel + pq_rescore_kernel per shard
                                                     _case(2, 12, 10, 150_002, 64, "sq8")])  # SQ8 sample -> threshold -> filter per shard
def test_sharded_equals_single_through_the_c_abi(qb, oracle, world, nq, top, n, dim, kind):
    import torch

    from qdrant_b200._capi import ScoredPoint, check, f32p, lib, u32p, vp
    from qdrant_b200.sharded import shard_ranges

    n_dev = torch.cuda.device_count()
    if -(-world // n_dev) > 4:
        pytest.skip(f"{world} shards waiting for each other on {n_dev} GPU(s): more co-resident spinning kernels than is safe to schedule (one shard per GPU is the deployment)")
    rng = np.random.default_rng(world)
    base = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((n, dim)).astype(np.float32))
    queries = rng.standard_normal((6, nq, dim)).astype(np.float32)          # six consecutive collective calls (parity slots, seq)
    if kind == "pq":     # one codebook and one code array, split by rows: the shards and the single storage score the same bytes
        cents = (rng.standard_normal((256, dim)) * 0.5).astype(np.float32)
        codes = rng.integers(0, 256, (n, dim // 4), dtype=np.uint8)
        make = lambda lo, hi, dev: qb.ProductQuantizedVectors(codes[lo:hi], cents, 4, dim, qb.Distance.Cosine, device=dev)   # noqa: E731
    elif kind == "sq8":  # one alpha / offset for all shards, as a shard of one encoded storage has
        sq = oracle.SQ8.encode(base, oracle.QD_DOT, False)
        make = lambda lo, hi, dev: qb.ScalarQuantizedVectors(sq.rows[lo:hi], dim, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier,   # noqa: E731
                                                             qb.Distance.Cosine, device=dev)
    else:
        make = lambda lo, hi, dev: qb.DenseVectorStorage(base[lo:hi], qb.Distance.Cosine, device=dev)   # noqa: E731
    single = make(0, n, 0)
    shards, comms = [], (vp * world)()
    for r, (b, e) in enumerate(shard_ranges(n, world)):
        st = make(b, e, r % n_dev)
        check(lib().qb_storage_set_id_base(st._h, b))
        shards.append(st)
        h = vp()
        check(lib().qb_comm_create(r % n_dev, r, world, 64, 16, C.byref(h)))
        comms[r] = h
    check(lib().qb_comm_connect_local(comms, world))
    results = [[None] * 6 for _ in range(world)]
    errors = []

    def task(r):
        try:
            for it in range(6):
                q = np.ascontiguousarray(queries[it])
                out = np.zeros((nq, top), dtype=qb.SCORED_POINT_OFFSET); cnt = np.zeros(nq, np.uint32)
                check(lib().qb_multi_search_batch(comms[r], shards[r]._h, q.ctypes.data_as(f32p), nq, top, None, None,
                                                  out.ctypes.data_as(C.POINTER(ScoredPoint)), cnt.ctypes.data_as(u32p), None))
                results[r][it] = [out[i, : cnt[i]].copy() for i in range(nq)]
        except Exception as ex:   # noqa: BLE001
            errors.append((r, ex))

    th = [threading.Thread(target=task, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    assert not errors, errors
    for it in range(6):
        want = single.search_batch(queries[it], top)
        for r in range(world):
            for i in range(nq):
                np.testing.assert_array_equal(results[r][it][i], want[i], err_msg=f"world {world} rank {r} call {it} query {i}")
    for r in range(world):
        lib().qb_comm_destroy(comms[r])
        shards[r].close()
    single.close()


@pytest.mark.parametrize("world,nq,top,n,dim", [(2, 1, 10, 150_003, 64), (4, 3, 10, 120_000, 96), (8, 1, 10, 160_000, 128), (2, 1, 10, 1_200_001, 64)])
def test_pipelined_device_steps_equal_single(qb, oracle, world, nq, top, n, dim):
    """qb_multi_search_batch_device with dev_local = NULL: the exchange + merge of step i runs on the communicator's stream while the
    scan of step i + 1 is already enqueued (window of two steps, ring of four slots).  Fourteen back-to-back steps without any host
    synchronisation, every step's merged lists kept in its own buffer, all compared with the unsharded storage."""
    import torch

    from qdrant_b200._capi import check, lib, vp
    from qdrant_b200.sharded import shard_ranges

    steps = 14
    n_dev = torch.cuda.device_count()
    if -(-world // n_dev) > 2:
        # two streams per shard; a device has 8 hardware work queues by default (CUDA_DEVICE_MAX_CONNECTIONS): beyond that a waiting merge
        # kernel can sit in front of the scan it waits for.  One shard per GPU — the deployment — needs two.
        pytest.skip(f"{world} pipelined shards on {n_dev} GPU(s) oversubscribe the device's hardware queues")
    rng = np.random.default_rng(100 + world)
    base = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((n, dim)).astype(np.float32))
    queries = rng.standard_normal((steps, nq, dim)).astype(np.float32)
    single = qb.DenseVectorStorage(base, qb.Distance.Cosine)
    shards, comms = [], (vp * world)()
    for r, (b, e) in enumerate(shard_ranges(n, world)):
        st = qb.DenseVectorStorage(base[b:e], qb.Distance.Cosine, device=r % n_dev)
        check(lib().qb_storage_set_id_base(st._h, b))
        shards.append(st)
        h = vp()
        check(lib().qb_comm_create(r % n_dev, r, world, 64, 16, C.byref(h)))
        comms[r] = h
    check(lib().qb_comm_connect_local(comms, world))
    results = [None] * world
    errors = []

    def task(r):
        try:
            dev = torch.device("cuda", r % n_dev)
            torch.cuda.set_device(dev)
            d_q = torch.from_numpy(queries).to(dev)
            d_out = torch.zeros((steps, nq, top), dtype=torch.int64, device=dev)
            d_cnt = torch.zeros((steps, nq), dtype=torch.int32, device=dev)
            torch.cuda.synchronize(dev)
            for it in range(steps):
                check(lib().qb_multi_search_batch_device(comms[r], shards[r]._h, vp(d_q[it].data_ptr()), nq, top, None, None,
                                                         vp(d_out[it].data_ptr()), vp(d_cnt[it].data_ptr())))
            check(lib().qb_comm_check(comms[r]))             # drains the communicator's stream; a timed-out exchange is an error
            rec = d_out.cpu().numpy().view(qb.SCORED_POINT_OFFSET).reshape(steps, nq, top)
            cnt = d_cnt.cpu().numpy()
            results[r] = [[rec[it, i, : cnt[it, i]].copy() for i in range(nq)] for it in range(steps)]
        except Exception as ex:   # noqa: BLE001
            errors.append((r, ex))

    th = [threading.Thread(target=task, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=120)
    assert not errors, errors
    for it in range(steps):
        want = single.search_batch(queries[it], top)
        for r in range(world):
            for i in range(nq):
                np.testing.assert_array_equal(results[r][it][i], want[i], err_msg=f"world {world} rank {r} step {it} query {i}")
    for r in range(world):
        lib().qb_comm_destroy(comms[r])
        shards[r].close()
    single.close()
