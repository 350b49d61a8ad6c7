#!/usr/bin/env python
"""Sparse-vector search (qb_sparse_*) on a SPLADE-like corpus: 1M documents of about 120 non-zeros each over 30 522 dims (BERT's
vocabulary), the dims Zipf-distributed (exponent 1.0, so hot dims have lists of hundreds of thousands), and 10 000 queries of about 25
non-zeros from the same distribution.  One JSON line.
    python tools/sparse_probe.py [docs=1000000] [out.json]
- build s: qb_sparse_index_create from host arrays, wall time;
- device q/s: qb_sparse_search_batch_device on device-resident queries, CUDA events on the index's stream, the median of 3 runs after a
  warm-up, per index kind (RAM: pruning on; compressed: never prunes) and top 10 / 100;
- host q/s: qb_sparse_search_batch from host arrays (query preparation, uploads, the kernel, the download), wall time, the median of 3;
- plain q/s: qb_sparse_search_plain_batch over 2 000 random ids per query (host API, wall time), top 10;
- checker q/s: the CPU checker (tests/sparse_ref.c, the reference's SearchContext) on 16 host threads over the first queries, whose
  device lists are compared with the checker's bit for bit (ids and score bits).
The corpus is generated on the device with torch (inverse-CDF sampling, then duplicates dropped per row)."""
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True
import torch  # noqa: E402

from qdrant_b200 import scorer as qb  # noqa: E402
from qdrant_b200._capi import check, lib  # noqa: E402
from tests import sparse_ref as sr  # noqa: E402

N_DOCS = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
N_DIMS, DOC_NNZ, NQ, Q_NNZ, PLAIN_IDS, THREADS = 30_522, 120, 10_000, 25, 2_000, 16
CHECK_Q = {"search": 128, "plain": 256}
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def corpus(n, nnz, seed):
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


def median(xs):
    return float(np.median(xs))


indptr, dims, w = corpus(N_DOCS, DOC_NNZ, 1)
qp, qd, qw = corpus(NQ, Q_NNZ, 2)
queries = (qp, qd, qw)
qlist = [(qd[qp[i]: qp[i + 1]], qw[qp[i]: qp[i + 1]]) for i in range(NQ)]
rng = np.random.default_rng(3)
id_lists = [np.sort(rng.choice(N_DOCS, PLAIN_IDS, replace=False)).astype(np.uint32) for _ in range(NQ)]
res = {"card_power_limit": card, "docs": N_DOCS, "dims": N_DIMS, "doc_nnz_mean": round(dims.size / N_DOCS, 1), "queries": NQ,
       "query_nnz_mean": round(qd.size / NQ, 1), "longest_list": int(np.bincount(dims, minlength=N_DIMS).max()), "results": []}
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
d_qp, d_qd, d_qw = t(qp.view(np.int64)), t(qd.view(np.int32)), t(qw)
max_nnz = int(np.diff(qp).max())

ref = sr.Index(indptr, dims, w, N_DIMS)


def checker(kind_ram, top, n):
    def one(i):
        return ref.search(*qlist[i], top, reliable=kind_ram)[0]
    t0 = time.perf_counter()
    with ThreadPoolExecutor(THREADS) as ex:
        out = list(ex.map(one, range(n)))
    return out, n / (time.perf_counter() - t0)


for kind in (qb.SparseIndexKind.Ram, qb.SparseIndexKind.Compressed):
    t0 = time.perf_counter()
    idx = qb.SparseVectorIndex((indptr, dims, w), N_DIMS, kind)
    build_s = time.perf_counter() - t0
    stream = torch.cuda.ExternalStream(lib().qb_sparse_index_stream(idx._h))
    for top in (10, 100):
        d_out = torch.zeros((NQ, top, 2), dtype=torch.int32, device="cuda")
        d_cnt = torch.zeros(NQ, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()

        def dev_run():
            check(lib().qb_sparse_search_batch_device(idx._h, d_qp.data_ptr(), d_qd.data_ptr(), d_qw.data_ptr(), NQ, max_nnz, top, None,
                                                      d_out.data_ptr(), d_cnt.data_ptr()))
        dev_run()
        torch.cuda.synchronize()
        ms = []
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            dev_run()
            e1.record(stream)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        host_s, got = [], None
        for _ in range(3):
            t0 = time.perf_counter()
            got = idx.search(queries, top)
            host_s.append(time.perf_counter() - t0)
        want, cpu_qps = checker(kind == qb.SparseIndexKind.Ram, top, CHECK_Q["search"])
        equal = all(np.array_equal(a["idx"], b["idx"]) and np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)) for a, b in zip(got, want))
        dev_lists = d_out.cpu().numpy().view(np.uint32)
        equal = equal and all(np.array_equal(dev_lists[q, : got[q].size, 0], got[q]["idx"]) for q in range(NQ))
        res["results"].append({"op": "search", "kind": kind.name, "top": top, "build_s": round(build_s, 2), "device_ms": round(median(ms), 2),
                               "device_qps": round(NQ / (median(ms) / 1e3), 1), "host_qps": round(NQ / median(host_s), 1),
                               f"checker_qps_{THREADS}threads": round(cpu_qps, 1), "checker_queries": CHECK_Q["search"], "equal_to_checker": bool(equal)})
        print(json.dumps(res["results"][-1]), file=sys.stderr)
    if kind == qb.SparseIndexKind.Ram:
        idx.search_plain(qlist[:64], id_lists[:64], 10)
        host_s = []
        for _ in range(3):
            t0 = time.perf_counter()
            got = idx.search_plain(qlist, id_lists, 10)
            host_s.append(time.perf_counter() - t0)

        def one(i):
            return ref.plain(*qlist[i], id_lists[i], 10)[0]
        t0 = time.perf_counter()
        with ThreadPoolExecutor(THREADS) as ex:
            want = list(ex.map(one, range(CHECK_Q["plain"])))
        cpu_qps = CHECK_Q["plain"] / (time.perf_counter() - t0)
        equal = all(np.array_equal(a["idx"], b["idx"]) and np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)) for a, b in zip(got, want))
        res["results"].append({"op": "plain", "kind": kind.name, "ids_per_query": PLAIN_IDS, "top": 10, "host_qps": round(NQ / median(host_s), 1),
                               f"checker_qps_{THREADS}threads": round(cpu_qps, 1), "checker_queries": CHECK_Q["plain"], "equal_to_checker": bool(equal)})
        print(json.dumps(res["results"][-1]), file=sys.stderr)
    idx.close()
ref.close()
line = json.dumps(res)
print(line)
if len(sys.argv) > 2:
    with open(sys.argv[2], "w") as f:
        f.write(line + "\n")
