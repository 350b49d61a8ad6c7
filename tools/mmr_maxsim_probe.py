#!/usr/bin/env python
"""MMR reranking over multivector candidates (qb_mmr_maxsim_batch) on clustered 128-d tokens, 32 per point: 256 queries of 32 vectors,
Cosine and Dot, lists of 100 / 1 000 / 16 384 candidates (each query's nearest points, from qb_search_maxsim), limit 10 / 100 / 10,
lambda 0.5.  One JSON line.
    python tools/mmr_maxsim_probe.py [points=20000] [out.json]
Per shape:
- device q/s: qb_mmr_maxsim_batch_device on device-resident queries, lambdas and candidate lists, timed with CUDA events on the token
  storage's stream, the median of 3 runs after a warm-up;
- host q/s: qb_mmr_maxsim_batch from host arrays (uploads, the kernels, the download), wall time, the median of 3 runs;
- checker q/s: the CPU checker (tests/mmr_maxsim_ref.c, one thread, the reference's arithmetic) on the first k queries of the batch on the
  same host, with the device's lists compared to its lists bit for bit (ids and score bits);
- FMAs per query (the cpu counter / 4: one FMA per dimension of a vector pair) and token bytes per query (the candidates' token rows the
  relevance pass and every step read: the row size x (sum of the candidates' tokens + the remaining candidates' tokens at each step))."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from oracle import oracle as o  # noqa: E402
from qdrant_b200 import scorer as qb  # noqa: E402
from qdrant_b200._capi import HwCounters, ScoredPoint, check, f32p, lib, u32p, vp  # noqa: E402
from tests import mmr_maxsim_ref as mr  # noqa: E402

n_points = int(sys.argv[1]) if len(sys.argv) > 1 else 20_000
DIM, TOK, NQ, QV, LAMBDA = 128, 32, 256, 32, 0.5
SHAPES = [(100, 10), (1000, 100), (16384, 10)]
CHECK_Q = {100: 4, 1000: 1, 16384: 1}
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def data(seed):
    """tokens and query vectors around 1024 centres (unit normal centres, sd 0.35 around them); a point's tokens share 4 centres"""
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((1024, DIM)).astype(np.float32)
    pc = rng.integers(0, 1024, (n_points, 4))
    tok_c = pc[np.repeat(np.arange(n_points), TOK), rng.integers(0, 4, n_points * TOK)]
    rows = centers[tok_c] + np.float32(0.35) * rng.standard_normal((n_points * TOK, DIM), dtype=np.float32)
    qc = rng.integers(0, 1024, (NQ, 4))
    q = centers[qc[np.repeat(np.arange(NQ), QV), rng.integers(0, 4, NQ * QV)]] + np.float32(0.35) * rng.standard_normal((NQ * QV, DIM), dtype=np.float32)
    return np.ascontiguousarray(rows), np.ascontiguousarray(q)


def median_of(f, runs=3):
    f()
    return float(np.median([f() for _ in range(runs)]))


def probe(dist_name):
    d = getattr(qb.Distance, dist_name)
    rows, qv = data(1)
    if d == qb.Distance.Cosine:
        rows = o.preprocess_rows_f32(o.COSINE, rows)
    off = np.arange(0, (n_points + 1) * TOK, TOK, dtype=np.uint32)
    st = qb.DenseVectorStorage(rows, d)
    view = qb.MultiVectorView(st, off)
    stream = torch.cuda.ExternalStream(st.stream_ptr())
    qs = [qv[i * QV : (i + 1) * QV] for i in range(NQ)]
    q_off = np.arange(0, (NQ + 1) * QV, QV, dtype=np.uint32)
    lams = np.full(NQ, LAMBDA, np.float32)
    dq, dqo, dl = torch.from_numpy(qv).cuda(), torch.from_numpy(q_off.view(np.int32)).cuda(), torch.from_numpy(lams).cuda()
    res = []
    for n_cand in sorted({s[0] for s in SHAPES}):
        lists = [view.search(q, n_cand) for q in qs]
        cand = np.ascontiguousarray(np.stack(lists))
        counts = np.full(NQ, n_cand, np.uint32)
        dc, dn = torch.from_numpy(cand.view(np.int32).reshape(NQ, n_cand, 2)).cuda(), torch.from_numpy(counts.view(np.int32)).cuda()
        for nc, limit in SHAPES:
            if nc != n_cand:
                continue
            dout = torch.zeros((NQ, limit, 2), dtype=torch.int32, device="cuda")
            doc = torch.zeros(NQ, dtype=torch.int32, device="cuda")

            def dev():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record(stream)
                check(lib().qb_mmr_maxsim_batch_device(st._h, off.ctypes.data_as(u32p), n_points, vp(dq.data_ptr()), NQ * QV, vp(dqo.data_ptr()), NQ, QV,
                                                       vp(dl.data_ptr()), vp(dc.data_ptr()), vp(dn.data_ptr()), n_cand, limit, vp(dout.data_ptr()),
                                                       vp(doc.data_ptr())))
                e1.record(stream)
                e1.synchronize()
                return e0.elapsed_time(e1) / 1e3

            out = np.zeros((NQ, limit), qb.SCORED_POINT_OFFSET)
            oc = np.zeros(NQ, np.uint32)
            hw = HwCounters()

            def host():
                t0 = time.perf_counter()
                check(lib().qb_mmr_maxsim_batch(st._h, off.ctypes.data_as(u32p), n_points, qv.ctypes.data_as(f32p), q_off.ctypes.data_as(u32p), NQ,
                                                lams.ctypes.data_as(f32p), cand.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p), n_cand,
                                                limit, out.ctypes.data_as(C.POINTER(ScoredPoint)), oc.ctypes.data_as(u32p), C.byref(hw)))
                return time.perf_counter() - t0

            t_dev, t_host = median_of(dev), median_of(host)
            dev_out = dout.cpu().numpy().view(qb.SCORED_POINT_OFFSET).reshape(NQ, limit)
            assert np.array_equal(dev_out.view(np.uint64), out.view(np.uint64))
            fmas = hw.cpu / 4 / 4 / NQ   # four host runs metered: the warm-up and three timed
            tok_reads = sum(TOK * n_cand + sum(TOK * (n_cand - k) for k in range(1, int(oc[i]))) for i in range(NQ)) / NQ
            k = CHECK_Q[n_cand]
            t0 = time.perf_counter()
            want = mr.mmr_batch(o, rows, off, int(d), qs[:k], lams[:k], lists[:k], limit)[0]
            t_ref = time.perf_counter() - t0
            equal = all(np.array_equal(out[i, : oc[i]].view(np.uint64), want[i].view(np.uint64)) for i in range(k))
            res.append({"distance": dist_name, "candidates": n_cand, "limit": limit, "device_qps": round(NQ / t_dev, 1),
                        "device_ms": round(t_dev * 1e3, 3), "host_qps": round(NQ / t_host, 1), "checker_qps_1thread": round(k / t_ref, 3),
                        "checker_queries": k, "equal_to_checker": bool(equal), "fmas_per_query": fmas, "token_bytes_per_query": tok_reads * DIM * 4,
                        "device_tflops": round(2 * fmas * NQ / t_dev / 1e12, 2), "device_token_tb_per_s": round(tok_reads * DIM * 4 * NQ / t_dev / 1e12, 2)})
            print(json.dumps(res[-1]), file=sys.stderr)
    st.close()
    return res


out = {"card_power_limit": card, "points": n_points, "tokens_per_point": TOK, "dim": DIM, "queries": NQ, "query_vectors": QV, "lambda": LAMBDA,
       "results": probe("Cosine") + probe("Dot")}
line = json.dumps(out)
print(line)
if len(sys.argv) > 2:
    with open(sys.argv[2], "w") as f:
        f.write(line + "\n")
