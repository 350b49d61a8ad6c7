#!/usr/bin/env python
"""Custom queries over a device sparse vector storage (qb_sparse_search_custom_batch) on the corpus of tools/sparse_probe.py: 1M documents
of about 91 non-zeros over 30 522 Zipf-distributed dims, examples of about 22 non-zeros from the same distribution.  One JSON line.
    python tools/sparse_custom_probe.py [docs=1000000] [out.json]
Per query shape (recommend 3 positives + 1 negative, discover with a target and 2 pairs, context with 3 pairs), unfiltered and over a 5 %
id list, top 10:
- host q/s: qb_sparse_search_custom_batch from host arrays (example preparation, uploads, the scan, the selection, the download), wall
  time, the median of 3 after a warm-up;
- device q/s: the summed device time of the scan (sparse_custom_kernel) and the selection kernels per call, from torch.profiler over 3
  calls run apart from the wall-time runs;
- pass bandwidth: each query group reads every scored row once, 8 bytes per stored element (dim and weight) and 8 per point (the row
  offset), so the bytes of a call are groups x that; over the scan kernel's time, against the data sheet's 3.35 TB/s;
- checker q/s: the CPU checker (tests/sparse_custom_ref.c with the oracle's fold) on 16 host threads over the first queries, whose device
  lists are compared with the checker's bit for bit (ids and score bits)."""
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

from oracle import oracle as o  # noqa: E402
from qdrant_b200 import scorer as qb  # noqa: E402
from tests import sparse_custom_ref as scr  # noqa: E402

N_DOCS = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
N_DIMS, DOC_NNZ, EX_NNZ, NQ, THREADS, CHECK_Q, TOP, REPS = 30_522, 120, 25, 512, 16, 32, 10, 3
SHAPES = [("recommend_best_score", qb.QueryKind.RecommendBestScore, 3, 1), ("discover", qb.QueryKind.Discover, 2, 0), ("context", qb.QueryKind.Context, 3, 0)]
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


def median(xs):
    return float(np.median(xs))


indptr, dims, w = corpus(N_DOCS, DOC_NNZ, 1)
ep, ed, ew = corpus(NQ * 6, EX_NNZ, 2)   # enough examples for the widest shape (context: 6 per query)
examples = [(ed[ep[i]: ep[i + 1]], ew[ep[i]: ep[i + 1]]) for i in range(NQ * 6)]
rng = np.random.default_rng(3)
id_list = np.sort(rng.choice(N_DOCS, N_DOCS // 20, replace=False)).astype(np.uint32)
lens = np.diff(indptr).astype(np.int64)
res = {"card_power_limit": card, "docs": N_DOCS, "dims": N_DIMS, "doc_nnz_mean": round(dims.size / N_DOCS, 1), "queries": NQ,
       "example_nnz_mean": round(ed.size / (NQ * 6), 1), "top": TOP, "results": []}
t0 = time.perf_counter()
dev = qb.SparseVectorStorage((indptr, dims, w))
res["build_s"] = round(time.perf_counter() - t0, 2)
ref = scr.Storage(indptr, dims, w)


def kernel_ms(fn):
    """device time of the scan and the selection kernels in one call"""
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3):   # a profile that recorded no scan kernel is taken again
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(REPS):
                fn()
            torch.cuda.synchronize()
        scan = sel = 0.0
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                if "sparse_custom_kernel" in e.name:
                    scan += e.device_time / 1e3 / REPS
                elif "qb_select" in e.name:
                    sel += e.device_time / 1e3 / REPS
        if scan > 0:
            break
    return scan, sel


for name, kind, n_a, n_b in SHAPES:
    E = {1: n_a + n_b, 3: 1 + 2 * n_a, 4: 2 * n_a}[int(kind)]
    batch = [examples[q * E: (q + 1) * E] for q in range(NQ)]
    # the groups the library forms: at most 64 queries and 512 / E of them, at most 72 KiB of staging at 16 bytes per example non-zero
    groups, cur, cur_nnz = 0, 0, 0
    for ex in batch:
        qn = sum(len(d) for d, _ in ex)
        if cur and (cur == min(64, 512 // E) or (cur_nnz + qn) * 16 + 8 > 72 * 1024):
            groups, cur, cur_nnz = groups + 1, 0, 0
        cur, cur_nnz = cur + 1, cur_nnz + qn
    groups += 1
    for filt in ("none", "id_list_5pct"):
        il = id_list if filt != "none" else None
        run = lambda: dev.search_custom(kind, batch, n_a, n_b, top=TOP, id_list=il)   # noqa: E731
        run()
        host_s, got = [], None
        for _ in range(3):
            t0 = time.perf_counter()
            got = run()
            host_s.append(time.perf_counter() - t0)
        scan_ms, sel_ms = kernel_ms(run)
        pts = N_DOCS if il is None else il.size
        elems = int(lens.sum()) if il is None else int(lens[il].sum())
        pass_bytes = 8 * elems + 8 * pts
        bw = groups * pass_bytes / (scan_ms / 1e3) / 1e12 if scan_ms > 0 else float("nan")

        def one(q):
            return ref.search(o, int(kind), n_a, n_b, batch[q], TOP, None, None, il)[0]
        t0 = time.perf_counter()
        with ThreadPoolExecutor(THREADS) as ex:
            want = list(ex.map(one, range(CHECK_Q)))
        cpu_qps = CHECK_Q / (time.perf_counter() - t0)
        equal = all(np.array_equal(a["idx"], b["idx"]) and np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32)) for a, b in zip(got, want))
        res["results"].append({"shape": name, "examples": E, "filter": filt, "scored_points": pts, "groups": groups, "host_qps": round(NQ / median(host_s), 1),
                               "device_ms": round(scan_ms + sel_ms, 2), "scan_ms": round(scan_ms, 2), "select_ms": round(sel_ms, 2),
                               "device_qps": round(NQ / ((scan_ms + sel_ms) / 1e3), 1) if scan_ms > 0 else float("nan"), "pass_bytes": pass_bytes, "scan_tbs": round(bw, 3),
                               "scan_share_of_hbm": round(bw / HBM_TBS, 3), f"checker_qps_{THREADS}threads": round(cpu_qps, 2),
                               "checker_queries": CHECK_Q, "equal_to_checker": bool(equal)})
        print(json.dumps(res["results"][-1]), file=sys.stderr)
dev.close()
ref.close()
line = json.dumps(res)
print(line)
if len(sys.argv) > 2:
    with open(sys.argv[2], "w") as f:
        f.write(line + "\n")
