#!/usr/bin/env python
"""MMR reranking (qb_mmr_batch) on clustered 768-d data: 256 queries, Cosine and Euclid, lists of 100 / 1 000 / 16 384 candidates (each
query's nearest rows, from qb_search_batch), limit 10 / 100, lambda 0.5.  One JSON line.
    python tools/mmr_probe.py [rows=100000] [out.json]
Per shape:
- device q/s: qb_mmr_batch_device on device-resident queries, lambdas and candidate lists, timed with CUDA events on the storage's
  stream, the median of 3 runs after a warm-up;
- host q/s: qb_mmr_batch from host arrays (uploads, the kernels, the download), wall time, the median of 3 runs;
- checker q/s: the CPU checker (tests/mmr_ref.c, one thread, the reference's arithmetic) on the first k queries of the batch on the same
  host, with the device's lists compared to its lists bit for bit (ids and score bits)."""
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
from tests import mmr_ref as mr  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000
DIM, NQ, LAMBDA = 768, 256, 0.5
SHAPES = [(100, 10), (100, 100), (1000, 10), (1000, 100), (16384, 10), (16384, 100)]
CHECK_Q = {100: 256, 1000: 32, 16384: 2}
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def data(seed):
    """rows and queries around 512 centres (unit normal centres, sd 0.35 around them)"""
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((512, DIM)).astype(np.float32)
    rows = centers[rng.integers(0, 512, n)] + np.float32(0.35) * rng.standard_normal((n, DIM), dtype=np.float32)
    q = centers[rng.integers(0, 512, NQ)] + np.float32(0.35) * rng.standard_normal((NQ, DIM), dtype=np.float32)
    return np.ascontiguousarray(rows), np.ascontiguousarray(q)


def median_of(f, runs=3):
    f()
    ts = []
    for _ in range(runs):
        ts.append(f())
    return float(np.median(ts))


def probe(dist_name):
    d = getattr(qb.Distance, dist_name)
    rows, q = data(1)
    if d == qb.Distance.Cosine:
        rows = o.preprocess_rows_f32(o.COSINE, rows)
    st = qb.DenseVectorStorage(rows, d)
    stream = torch.cuda.ExternalStream(st.stream_ptr())
    lams = np.full(NQ, LAMBDA, np.float32)
    dq, dl = torch.from_numpy(q).cuda(), torch.from_numpy(lams).cuda()
    res = []
    for n_cand in sorted({s[0] for s in SHAPES}):
        lists = st.search_batch(q, n_cand)
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
                check(lib().qb_mmr_batch_device(st._h, vp(dq.data_ptr()), NQ, vp(dl.data_ptr()), vp(dc.data_ptr()), vp(dn.data_ptr()), n_cand, limit,
                                                vp(dout.data_ptr()), vp(doc.data_ptr())))
                e1.record(stream)
                e1.synchronize()
                return e0.elapsed_time(e1) / 1e3

            out = np.zeros((NQ, limit), qb.SCORED_POINT_OFFSET)
            oc = np.zeros(NQ, np.uint32)
            hw = HwCounters()

            def host():
                t0 = time.perf_counter()
                check(lib().qb_mmr_batch(st._h, q.ctypes.data_as(f32p), NQ, lams.ctypes.data_as(f32p), cand.ctypes.data_as(C.POINTER(ScoredPoint)),
                                         counts.ctypes.data_as(u32p), n_cand, limit, out.ctypes.data_as(C.POINTER(ScoredPoint)), oc.ctypes.data_as(u32p),
                                         C.byref(hw)))
                return time.perf_counter() - t0

            t_dev, t_host = median_of(dev), median_of(host)
            dev_out = dout.cpu().numpy().view(qb.SCORED_POINT_OFFSET).reshape(NQ, limit)
            assert np.array_equal(dev_out.view(np.uint64), out.view(np.uint64))
            k = CHECK_Q[n_cand]
            t0 = time.perf_counter()
            want = mr.mmr_batch(o, rows, int(d), q[:k], lams[:k], lists[:k], limit)[0]
            t_ref = time.perf_counter() - t0
            equal = all(np.array_equal(out[i, : oc[i]].view(np.uint64), want[i].view(np.uint64)) for i in range(k))
            res.append({"distance": dist_name, "candidates": n_cand, "limit": limit, "device_qps": round(NQ / t_dev, 1),
                        "device_ms": round(t_dev * 1e3, 3), "host_qps": round(NQ / t_host, 1), "checker_qps_1thread": round(k / t_ref, 2),
                        "checker_queries": k, "equal_to_checker": bool(equal)})
            print(json.dumps(res[-1]), file=sys.stderr)
    st.close()
    return res


out = {"card_power_limit": card, "rows": n, "dim": DIM, "queries": NQ, "lambda": LAMBDA,
       "results": probe("Cosine") + probe("Euclid")}
line = json.dumps(out)
print(line)
if len(sys.argv) > 2:
    with open(sys.argv[2], "w") as f:
        f.write(line + "\n")
