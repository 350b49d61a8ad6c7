#!/usr/bin/env python
"""Incremental graph-build probe (qb_hnsw_build_incremental) on the C5 setup: clustered cosine rows, M = 16, ef_construct = 100, batch
512, the old graph built on the device.  One JSON line.
    python tools/hnsw_build_incremental_probe.py [rows=1000000] [dim=768] [out.json]
Scenarios, each a new storage made from the old one: (a) 0 % deleted, +1 % new; (b) 0 %, +10 %; (c) 1 %, +10 %; (d) 10 %, +10 %.
The kept rows are compacted in id order, the new rows appended.  For each:
- the incremental build and a full qb_hnsw_build of the same new storage, alternated over three rounds: wall time from the call to its
  synchronised return;
- the incremental build's kernel time split into heal (the heal kernels, their sorts and the old tables), insert (the build's insert,
  backlink and sort kernels) and finish (counts, scan, neighbours), from a separate torch.profiler run;
- recall@10 at ef = 128 of both graphs against the exact scan, 1000 queries."""
import json, os, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as o
from qdrant_b200 import scorer as qb

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
dim = int(sys.argv[2]) if len(sys.argv) > 2 else 768
M, EF_C, EF, TOP, NQ, ROUNDS = 16, 100, 128, 10, 1000, 3
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
rng = np.random.default_rng(42)
centers = rng.standard_normal((1024, dim)).astype(np.float32)


def rows_of(k):
    out = np.empty((k, dim), np.float32)
    for a in range(0, k, 1 << 18):
        b = min(k, a + (1 << 18))
        out[a:b] = centers[rng.integers(0, 1024, b - a)] + 0.5 * rng.standard_normal((b - a, dim), dtype=np.float32)
        out[a:b] = o.preprocess_rows_f32(o.COSINE, out[a:b])   # the storage holds Metric::preprocess'd rows
    return out


def levels_of(k, seed):
    u = 1.0 - np.random.default_rng(seed).random(k)
    return np.minimum(np.round(-np.log(u) / np.log(M)), 30).astype(np.uint8)


def recall(g, st, queries):
    exact = st.search_batch(queries, TOP)
    res = g.search(queries, TOP, EF, g.entry_point, g.entry_level)
    return float(np.mean([len(set(r["idx"].tolist()) & set(e["idx"].tolist())) / TOP for r, e in zip(res, exact)]))


def timed(fn):
    t0 = time.perf_counter()
    g = fn()
    return g, time.perf_counter() - t0


base = rows_of(n)
queries = (centers[rng.integers(0, 1024, NQ)] + 0.5 * rng.standard_normal((NQ, dim))).astype(np.float32)
lv = levels_of(n, 7)
old_st = qb.DenseVectorStorage(base, qb.Distance.Cosine)
old, t_old = timed(lambda: qb.HnswGraph.build(old_st, m=M, ef_construct=EF_C, levels=lv, batch=512))
out = {"card_power_limit": card, "rows": n, "dim": dim, "m": M, "m0": 2 * M, "ef_construct": EF_C, "ef": EF, "batch": 512, "queries": NQ,
       "rounds": ROUNDS, "old_build_s": t_old, "scenarios": {}}

for name, gone, new in (("a", 0.0, 0.01), ("b", 0.0, 0.10), ("c", 0.01, 0.10), ("d", 0.10, 0.10)):
    dead = np.random.default_rng(11).random(n) < gone
    keep = np.flatnonzero(~dead)
    n_new = int(n * new)
    o2n = np.full(n, 0xFFFFFFFF, np.uint32)
    o2n[keep] = np.arange(keep.size, dtype=np.uint32)
    new_rows = np.concatenate([base[keep], rows_of(n_new)])
    nlv = np.concatenate([lv[keep], levels_of(n_new, 13)])
    st = qb.DenseVectorStorage(new_rows, qb.Distance.Cosine)
    del new_rows
    incr = lambda: qb.HnswGraph.build_incremental(st, old, o2n, ef_construct=EF_C, levels=nlv, batch=512)
    full = lambda: qb.HnswGraph.build(st, m=M, ef_construct=EF_C, levels=nlv, batch=512)
    ti, tf = [], []
    for _ in range(ROUNDS):   # alternated, so both see the same machine
        g, t = timed(incr); ti.append(t); gi = g
        g, t = timed(full); tf.append(t); gf = g
    r = {"deleted": gone, "new_points": n_new, "kept": int(keep.size), "incremental_s": ti, "full_build_s": tf,
         "incremental_recall_at_10": recall(gi, st, queries), "full_recall_at_10": recall(gf, st, queries)}
    gi.close(); gf.close()
    try:   # kernel time by phase, from a traced run of its own (tracing slows the host)
        import torch
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            g = incr()
        g.close()
        split = {"heal_ms": 0.0, "insert_ms": 0.0, "finish_ms": 0.0, "other_ms": 0.0}
        for e in prof.events():
            if e.device_type.name != "CUDA":
                continue
            t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            k = e.name
            if "heal" in k:
                split["heal_ms"] += t / 1e3
            elif "hnsw_search_kernel" in k or "hnsw_backlink_kernel" in k:
                split["insert_ms"] += t / 1e3
            elif "build_counts" in k or "build_neighbors" in k or "Scan" in k:
                split["finish_ms"] += t / 1e3
            else:
                split["other_ms"] += t / 1e3   # radix sorts (heal and insert alike) and copies
        r["incremental_kernel_ms"] = split
    except Exception as ex:   # noqa: BLE001 - the split is reported as missing, the rest stands
        r["incremental_kernel_ms"] = f"not measured: {ex!r}"
    out["scenarios"][name] = r
    st.close()
    print(json.dumps({name: r}), file=sys.stderr, flush=True)

old.close(); old_st.close()
line = json.dumps(out)
print(line)
if len(sys.argv) > 3:
    with open(sys.argv[3], "w") as fh:
        fh.write(line + "\n")
