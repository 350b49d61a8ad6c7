#!/usr/bin/env python
"""MMR reranking over sparse candidates (qb_mmr_sparse_batch) on the corpus of tools/sparse_probe.py: 1M documents of about 91
non-zeros over 30 522 Zipf-distributed dims, 256 queries of about 22 non-zeros from the same distribution, lambda 0.5.  One JSON line.
    python tools/mmr_sparse_probe.py [docs=1000000] [out.json]
Each query's candidates are its top N by score_vectors: qb_sparse_search_batch over an inverted index of the same rows for N <= 4096
(the index's top limit), and for N = 16 384 the top N of an exact sparse x dense product on the device (torch), since the index caps top
at 4096.  Ids are shared by the index and the storage.  Per shape N x limit:
- device q/s: the summed device time of mmr_sparse_kernel per call, from torch.profiler over 3 calls run apart from the wall-time runs;
- host q/s: qb_mmr_sparse_batch from host arrays (query sorting, checks, uploads, the kernel, the download), wall time, the median of 3
  after a warm-up;
- row bytes: each step reads every remaining candidate's row once, 8 bytes per element (dim and weight), the relevance pass every
  candidate's row; their sum over the batch, over the kernel time, against the data sheet's 3.35 TB/s;
- the CPU checker (tests/mmr_sparse_ref.c) on one thread over the first queries, whose device lists are compared with the checker's
  (ids and score bits, and the counters of those queries)."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True
import torch  # noqa: E402

from qdrant_b200 import scorer as qb  # noqa: E402
from tests import mmr_sparse_ref as ms  # noqa: E402

N_DOCS = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
N_DIMS, DOC_NNZ, Q_NNZ, NQ, REPS, LAM = 30_522, 120, 25, 256, 3, 0.5
SHAPES = [(100, 10), (100, 100), (1000, 10), (1000, 100), (16384, 10), (16384, 100)]
CHECK_Q = {100: 32, 1000: 8, 16384: 2}
HBM_TBS = 3.35
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def corpus(n, nnz, seed):
    """tools/sparse_probe.py's corpus: Poisson(nnz) draws per row from a Zipf(1.0) CDF over N_DIMS, duplicates dropped"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    p = 1.0 / torch.arange(1, N_DIMS + 1, device="cuda", dtype=torch.float64)
    cdf = torch.cumsum(p / p.sum(), 0)
    counts = torch.poisson(torch.full((n,), float(nnz), device="cuda", dtype=torch.float64), generator=g).long()
    rows = torch.repeat_interleave(torch.arange(n, device="cuda"), counts)
    dims = torch.clamp(torch.searchsorted(cdf, torch.rand(rows.numel(), device="cuda", dtype=torch.float64, generator=g)), max=N_DIMS - 1)
    keys = torch.unique(rows * N_DIMS + dims)
    rows, dims = keys // N_DIMS, keys % N_DIMS
    indptr = torch.zeros(n + 1, dtype=torch.long, device="cuda")
    indptr[1:] = torch.cumsum(torch.bincount(rows, minlength=n), 0)
    w = torch.rand(dims.numel(), device="cuda", generator=g, dtype=torch.float32) + 0.01
    return indptr.cpu().numpy().astype(np.uint64), dims.cpu().numpy().astype(np.uint32), w.cpu().numpy()


def kernel_ms(fn):
    """device time of mmr_sparse_kernel in one call"""
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3):   # a profile that recorded no kernel is taken again
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(REPS):
                fn()
            torch.cuda.synchronize()
        t = sum(e.device_time for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "mmr_sparse_kernel" in e.name)
        if t > 0:
            return t / 1e3 / REPS
    return float("nan")


def row_bytes(lens, cand, picks):
    """bytes of candidate rows one query reads: the relevance pass, then one pass over the remaining candidates per pick but the last"""
    seen, uniq = set(), []
    for i in cand["idx"].tolist():
        if i not in seen:
            seen.add(i)
            uniq.append(i)
    if len(uniq) < 2:
        return 0
    left = int(lens[uniq].sum())
    total = left
    for p in picks[:-1].tolist():
        left -= int(lens[p])
        total += left
    return 8 * total


indptr, dims, w = corpus(N_DOCS, DOC_NNZ, 1)
qp, qd, qw = corpus(NQ, Q_NNZ, 2)
queries = [(qd[qp[i]: qp[i + 1]], qw[qp[i]: qp[i + 1]]) for i in range(NQ)]
lens = np.diff(indptr).astype(np.int64)
res = {"card_power_limit": card, "docs": N_DOCS, "dims": N_DIMS, "doc_nnz_mean": round(dims.size / N_DOCS, 1), "queries": NQ,
       "query_nnz_mean": round(qd.size / NQ, 1), "lambda": LAM, "results": []}
csr = (indptr, dims, w)
dev = qb.SparseVectorStorage(csr)
idx = qb.SparseVectorIndex(csr, N_DIMS, qb.SparseIndexKind.Ram)
cands = {n: idx.search(queries, n) for n in (100, 1000)}
idx.close()
# N = 16 384: the exact top N of the sparse x dense product (the index's top is capped at 4096)
mat = torch.sparse_csr_tensor(torch.from_numpy(indptr.astype(np.int64)), torch.from_numpy(dims.astype(np.int64)), torch.from_numpy(w),
                              (N_DOCS, N_DIMS)).cuda()
qdense = torch.zeros((N_DIMS, NQ), dtype=torch.float32, device="cuda")
for i, (d_, w_) in enumerate(queries):
    qdense[torch.from_numpy(d_.astype(np.int64)).cuda(), i] = torch.from_numpy(w_).cuda()
cands[16384] = []
for q0 in range(0, NQ, 32):
    sc = (mat @ qdense[:, q0: q0 + 32]).T
    top = torch.topk(sc, 16384, dim=1)
    for ids, s in zip(top.indices.cpu().numpy(), top.values.cpu().numpy()):
        c = np.zeros(16384, ms.SCORED)
        c["idx"], c["score"] = ids, s
        cands[16384].append(c)
del mat, qdense
lams = np.full(NQ, LAM, np.float32)
for n, limit in SHAPES:
    lists = cands[n]
    run = lambda: dev.mmr(queries, lists, lams, limit)   # noqa: E731
    run()
    host_s, got = [], None
    for _ in range(3):
        t0 = time.perf_counter()
        got = run()
        host_s.append(time.perf_counter() - t0)
    k_ms = kernel_ms(run)
    rb = sum(row_bytes(lens, c, g["idx"]) for c, g in zip(lists, got))
    kq = CHECK_Q[n]
    hw = qb.HwCounters()
    got_k = dev.mmr(queries[:kq], lists[:kq], lams[:kq], limit, counters=hw)
    t0 = time.perf_counter()
    want, cpu, io = ms.mmr_batch(csr, queries[:kq], lams[:kq], lists[:kq], limit)
    checker_qps = kq / (time.perf_counter() - t0)
    equal = all(np.array_equal(a["idx"], b["idx"]) and np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32))
                for a, b in zip(got[:kq] + got_k, want + want)) and (hw.cpu, hw.vector_io_read) == (cpu, io)
    tbs = rb / (k_ms / 1e3) / 1e12
    res["results"].append({"candidates": n, "limit": limit, "host_qps": round(NQ / float(np.median(host_s)), 1), "kernel_ms": round(k_ms, 3),
                           "device_qps": round(NQ / (k_ms / 1e3), 1), "row_bytes": rb, "row_read_tbs": round(tbs, 3),
                           "row_read_share_of_hbm": round(tbs / HBM_TBS, 3), "checker_qps_1thread": round(checker_qps, 2), "checker_queries": kq,
                           "equal_to_checker": bool(equal)})
    print(json.dumps(res["results"][-1]), file=sys.stderr)
dev.close()
line = json.dumps(res)
print(line)
if len(sys.argv) > 2:
    with open(sys.argv[2], "w") as f:
        f.write(line + "\n")
