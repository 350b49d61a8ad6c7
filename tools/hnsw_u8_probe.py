#!/usr/bin/env python
"""Device HNSW over a Uint8 storage beside the f32 storage of the same values: clustered Euclid rows whose values are integers in
0..255, stored once as u8 (VectorStorageDatatype::Uint8) and once as f32; M = 16, ef_construct = 100, levels from a seeded generator.
One JSON line.
    python tools/hnsw_u8_probe.py [rows=1000000] [dim=768] [out.json]
Per storage:
- build: wall time of qb_hnsw_build (batch 512) from the call to its synchronised return, and the kernel time of a second, traced build
  split into inserts (hnsw_search_kernel<..., ALGO_BUILD>), backlink sorts (cub radix sort) and backlinks (hnsw_backlink_kernel), from
  torch.profiler;
- search at ef = 128, top 10, on the built graph: q/s device-timed (qb_hnsw_search_batch_device on device-resident queries, the storage's
  profiling events around the traversal) and through the host API (qb_hnsw_search_batch, wall time with the uploads and downloads), the
  median of 3 runs after a warm-up; recall@10 against the exact scan (qb_search_batch) on 1000 queries."""
import json, os, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from qdrant_b200 import scorer as qb
from qdrant_b200._capi import check, lib, vp

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
dim = int(sys.argv[2]) if len(sys.argv) > 2 else 768
M, EF_C, EF, TOP, NQ_RECALL, NQ_RATE = 16, 100, 128, 10, 1000, 20000
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def data(rows, seed):
    """1024 centres in 0..255, rows and queries around them (sd 24), rounded and clipped to u8 values"""
    rng = np.random.default_rng(seed)
    centers = rng.integers(32, 224, (1024, dim)).astype(np.float32)
    out = np.empty((rows, dim), np.uint8)
    for a in range(0, rows, 1 << 18):
        b = min(rows, a + (1 << 18))
        out[a:b] = np.clip(np.rint(centers[rng.integers(0, 1024, b - a)] + 24.0 * rng.standard_normal((b - a, dim), dtype=np.float32)), 0, 255)
    q = np.clip(np.rint(centers[rng.integers(0, 1024, NQ_RATE)] + 24.0 * rng.standard_normal((NQ_RATE, dim))), 0, 255).astype(np.float32)
    return out, q


def recall(res, exact):
    return float(np.mean([len(set(r["idx"].tolist()) & set(e["idx"].tolist())) / TOP for r, e in zip(res, exact)]))


def build(st, lv):
    t0 = time.perf_counter()
    g = qb.HnswGraph.build(st, m=M, ef_construct=EF_C, levels=lv, batch=512)
    return g, time.perf_counter() - t0


def kernel_split(st, lv):
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            g, _ = build(st, lv)
        g.close()
        split = {"insert_ms": 0.0, "sort_ms": 0.0, "backlink_ms": 0.0, "other_ms": 0.0}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            k = "insert_ms" if "hnsw_search_kernel" in e.key else "backlink_ms" if "hnsw_backlink_kernel" in e.key else "sort_ms" if "RadixSort" in e.key else "other_ms"
            split[k] += t / 1e3
        return split
    except Exception as ex:   # noqa: BLE001 - the split is reported as missing, the rest stands
        return f"not measured: {ex!r}"


def rates(st, g, q):
    import torch

    nq = q.shape[0]
    dq = torch.from_numpy(q).cuda()
    out = torch.zeros((nq, TOP), dtype=torch.int64, device="cuda")
    cnt = torch.zeros(nq, dtype=torch.int32, device="cuda")

    def device_run():
        torch.cuda.synchronize()
        st.profile(True)
        st.profile_read(reset=True)
        check(lib().qb_hnsw_search_batch_device(g._h, vp(dq.data_ptr()), nq, TOP, EF, g.entry_point, g.entry_level, vp(out.data_ptr()), vp(cnt.data_ptr())))
        torch.cuda.synchronize()
        launches, ms = st.profile_read(reset=True)
        st.profile(False)
        return ms / 1e3

    def host_run():
        t0 = time.perf_counter()
        g.search(q, TOP, EF, g.entry_point, g.entry_level)
        return time.perf_counter() - t0

    device_run(); host_run()
    dev = sorted(device_run() for _ in range(3))[1]
    host = sorted(host_run() for _ in range(3))[1]
    return {"queries": nq, "device_qps": nq / dev, "device_s": dev, "host_api_qps": nq / host, "host_api_s": host}


rows, queries = data(n, 42)
lv = np.minimum(np.round(-np.log(1.0 - np.random.default_rng(7).random(n)) / np.log(M)), 30).astype(np.uint8)
out = {"card_power_limit": card, "rows": n, "dim": dim, "distance": "Euclid", "m": M, "m0": 2 * M, "ef_construct": EF_C, "ef": EF, "top": TOP}
for name, dt, values in (("u8", qb.VectorStorageDatatype.Uint8, rows), ("f32", qb.VectorStorageDatatype.Float32, None)):
    st = qb.DenseVectorStorage(rows if values is not None else rows.astype(np.float32), qb.Distance.Euclid, dt)
    exact = st.search_batch(queries[:NQ_RECALL], TOP)
    g, wall = build(st, lv)
    r = {"storage_bytes": st.hbm_bytes(), "device_build_s": wall}
    r["recall_at_10"] = recall(g.search(queries[:NQ_RECALL], TOP, EF, g.entry_point, g.entry_level), exact)
    r["search"] = rates(st, g, queries)
    g.close()
    r["device_kernel_ms"] = kernel_split(st, lv)
    st.close()
    out[name] = r
out["u8_over_f32"] = {"build": out["f32"]["device_build_s"] / out["u8"]["device_build_s"],
                      "device_qps": out["u8"]["search"]["device_qps"] / out["f32"]["search"]["device_qps"],
                      "host_api_qps": out["u8"]["search"]["host_api_qps"] / out["f32"]["search"]["host_api_qps"]}

line = json.dumps(out)
print(line)
if len(sys.argv) > 3:
    with open(sys.argv[3], "w") as fh:
        fh.write(line + "\n")
