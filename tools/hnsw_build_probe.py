#!/usr/bin/env python
"""Graph-build probe (qb_hnsw_build) on the C5 setup: clustered cosine rows, M = 16, ef_construct = 100, levels drawn from a seeded
generator.  One JSON line.
    python tools/hnsw_build_probe.py [rows=1000000] [dim=768] [big_rows=0] [out.json]      (rows = 0: the big leg only)
- device build: wall time from the call to its synchronised return (batch 512), and the kernel time of a second, traced build split into
  inserts (hnsw_search_kernel<..., ALGO_BUILD>), backlink sorts (cub radix sort) and backlinks (hnsw_backlink_kernel), from torch.profiler;
- the oracle's build on all host threads (its own level draw), wall time;
- recall@10 at ef = 128 of the device search on both graphs against the exact scan (qb_search_batch), 1000 queries;
- batch 256 / 512 / 1024 / 2048: build time and recall;
- big_rows > 0: the device build at that size (rows generated in chunks) and its recall on 1000 queries.  The CPU build is not run there."""
import json, os, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as o
from qdrant_b200 import scorer as qb

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
dim = int(sys.argv[2]) if len(sys.argv) > 2 else 768
big = int(sys.argv[3]) if len(sys.argv) > 3 else 0
M, EF_C, EF, TOP, NQ = 16, 100, 128, 10, 1000
threads = os.cpu_count() or 1
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def data(rows, seed):
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((1024, dim)).astype(np.float32)
    out = np.empty((rows, dim), np.float32)
    for a in range(0, rows, 1 << 18):   # chunked, so the big leg never holds a second copy
        b = min(rows, a + (1 << 18))
        out[a:b] = centers[rng.integers(0, 1024, b - a)] + 0.5 * rng.standard_normal((b - a, dim), dtype=np.float32)
        out[a:b] = o.preprocess_rows_f32(o.COSINE, out[a:b])   # the storage holds Metric::preprocess'd rows
    q = (centers[rng.integers(0, 1024, NQ)] + 0.5 * rng.standard_normal((NQ, dim))).astype(np.float32)
    return out, q


def levels_of(rows, seed):
    u = 1.0 - np.random.default_rng(seed).random(rows)
    return np.minimum(np.round(-np.log(u) / np.log(M)), 30).astype(np.uint8)


def recall(res, exact):
    return float(np.mean([len(set(r["idx"].tolist()) & set(e["idx"].tolist())) / TOP for r, e in zip(res, exact)]))


def timed_build(st, lv, batch):
    t0 = time.perf_counter()
    g = qb.HnswGraph.build(st, m=M, ef_construct=EF_C, levels=lv, batch=batch)
    return g, time.perf_counter() - t0


out = {"card_power_limit": card, "dim": dim, "m": M, "m0": 2 * M, "ef_construct": EF_C, "ef": EF, "queries": NQ, "host_threads": threads}
if n:
    base, queries = data(n, 42)
    lv = levels_of(n, 7)
    st = qb.DenseVectorStorage(base, qb.Distance.Cosine)
    exact = st.search_batch(queries, TOP)
    out["rows"] = n

    g, wall = timed_build(st, lv, 512)
    out["device_build_s"] = wall
    out["device_recall_at_10"] = recall(g.search(queries, TOP, EF, g.entry_point, g.entry_level), exact)
    g.close()

    # kernel time by kind, from a traced build (a run of its own: tracing slows the host)
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            g, _ = timed_build(st, lv, 512)
        g.close()
        split = {"insert_ms": 0.0, "sort_ms": 0.0, "backlink_ms": 0.0, "other_ms": 0.0}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            name = e.key
            k = "insert_ms" if "hnsw_search_kernel" in name else "backlink_ms" if "hnsw_backlink_kernel" in name else "sort_ms" if "RadixSort" in name else "other_ms"
            split[k] += t / 1e3
        out["device_kernel_ms"] = split
    except Exception as ex:   # noqa: BLE001 - the split is reported as missing, the rest stands
        out["device_kernel_ms"] = f"not measured: {ex!r}"

    # the oracle's build on every host thread (its own level draw)
    t0 = time.perf_counter()
    og = o.HNSW(base, o.COSINE, m=M, ef_construct=EF_C, seed=42, threads=threads)
    out["oracle_build_s"] = time.perf_counter() - t0
    out["oracle_build_threads"] = threads
    entry, elev, m, m0 = og.entry()
    cg = qb.HnswGraph(st, og.export_plain(), m, m0)
    og.close()
    out["oracle_graph_recall_at_10"] = recall(cg.search(queries, TOP, EF, entry, elev), exact)
    cg.close()

    out["batch_sweep"] = {}
    for batch in (256, 512, 1024, 2048):
        g, wall = timed_build(st, lv, batch)
        out["batch_sweep"][batch] = {"build_s": wall, "recall_at_10": recall(g.search(queries, TOP, EF, g.entry_point, g.entry_level), exact)}
        g.close()
    st.close()
    del base

if big:
    bb, bq = data(big, 43)
    bs = qb.DenseVectorStorage(bb, qb.Distance.Cosine)
    del bb
    bexact = bs.search_batch(bq, TOP)
    g, wall = timed_build(bs, levels_of(big, 8), 512)
    out["big"] = {"rows": big, "device_build_s": wall, "recall_at_10": recall(g.search(bq, TOP, EF, g.entry_point, g.entry_level), bexact),
                  "cpu_build": "not run at this size"}
    g.close(); bs.close()

line = json.dumps(out)
print(line)
if len(sys.argv) > 4:
    with open(sys.argv[4], "w") as fh:
        fh.write(line + "\n")
