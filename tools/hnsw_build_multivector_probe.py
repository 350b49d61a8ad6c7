#!/usr/bin/env python
"""Graph build over multivector (MaxSim) points on the device (qb_hnsw_build_multivector) on a ColBERT-shaped collection.  One JSON line.
    python tools/hnsw_build_multivector_probe.py [points=100000] [out.json]
Setup: `points` points of 32 clustered 128-d cosine tokens each (points / 8 Gaussian clusters; a point's tokens share one cluster),
M = 16, ef_construct = 100, batch 512, levels drawn from a seeded generator.  Reports:
  - the device build's wall time (a host clock around the synchronous call), and its kernel time by kind from a traced build of its
    own (torch.profiler): MaxSim inserts (hnsw_build_mv_kernel), backlink sorts (cub radix sort), MaxSim backlinks
    (hnsw_backlink_mv_kernel), the rest;
  - recall@10 at ef = 128 of qb_hnsw_search_maxsim_batch on that graph against the brute-force qb_search_maxsim, for 256 queries of 32
    vectors, and the same for today's stand-in: qb_hnsw_build over each point's normalised mean token, bound to the token storage;
  - the CPU restatement (tests/hnsw_build_mv_ref.c, one thread) on the first `cpu_points` points, and the device on the same points.
The card's name and power limit are read in the same run."""
import json, os, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from oracle import oracle as o
from qdrant_b200 import scorer as qb
from tests.hnsw_build_mv_ref import MvRefGraph

n = int(sys.argv[1]) if len(sys.argv) > 1 else 100_000
dim, T, M, EF_C, EF, TOP, NQ, QV, N_CPU = 128, 32, 16, 100, 128, 10, 256, 32, 1000
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"card_power_limit": card, "points": n, "tokens_per_point": T, "dim": dim, "m": M, "m0": 2 * M, "ef_construct": EF_C, "batch": 512,
       "ef": EF, "top": TOP, "queries": NQ, "query_vectors": QV}

g = torch.Generator(device="cuda").manual_seed(42)
n_cl = max(n // 8, 1)
centers = torch.randn((n_cl, dim), device="cuda", generator=g)
cluster = torch.randint(0, n_cl, (n,), device="cuda", generator=g)
tok = centers[cluster.repeat_interleave(T)] + 0.5 * torch.randn((n * T, dim), device="cuda", generator=g)
rows = torch.nn.functional.normalize(tok, dim=1).cpu().numpy()
rows = o.preprocess_rows_f32(o.COSINE, rows)
off = np.arange(0, n * T + 1, T, dtype=np.uint32)
qcl = torch.randint(0, n_cl, (NQ,), device="cuda", generator=g)
queries = list((centers[qcl.repeat_interleave(QV)] + 0.5 * torch.randn((NQ * QV, dim), device="cuda", generator=g)).cpu().numpy().reshape(NQ, QV, dim))
levels = np.minimum(np.round(-np.log(1.0 - np.random.default_rng(7).random(n)) / np.log(M)), 30).astype(np.uint8)
del tok

st = qb.DenseVectorStorage(rows, qb.Distance.Cosine)
view = qb.MultiVectorView(st, off)


def timed_build(v, lv):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gr = qb.HnswGraph.build_multivector(v, m=M, ef_construct=EF_C, levels=lv, batch=512)
    return gr, time.perf_counter() - t0


exact = [view.search(q, TOP)["idx"] for q in queries]


def recall(res):
    return float(np.mean([len(set(r["idx"].tolist()) & set(x.tolist())) / TOP for r, x in zip(res, exact)]))


mg, wall = timed_build(view, levels)
out["device_build_s"] = wall
out["recall_at_10"] = recall(mg.search_maxsim(queries, TOP, EF, mg.entry_point, mg.entry_level))
mg.close()

# kernel time by kind, from a traced build (a run of its own: tracing slows the host)
try:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        mg, _ = timed_build(view, levels)
    mg.close()
    split = {"insert_ms": 0.0, "sort_ms": 0.0, "backlink_ms": 0.0, "other_ms": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        name = e.key
        k = "insert_ms" if "hnsw_build_mv_kernel" in name else "backlink_ms" if "hnsw_backlink_mv_kernel" in name else "sort_ms" if "RadixSort" in name else "other_ms"
        split[k] += t / 1e3
    out["device_kernel_ms"] = split
except Exception as ex:   # noqa: BLE001 - the split is reported as missing, the rest stands
    out["device_kernel_ms"] = f"not measured: {ex!r}"

# today's stand-in: a single-vector graph over the normalised mean tokens, bound to the token storage
means = o.preprocess_rows_f32(o.COSINE, rows.reshape(n, T, dim).mean(1).astype(np.float32))
ms = qb.DenseVectorStorage(means, qb.Distance.Cosine)
t0 = time.perf_counter()
sg = qb.HnswGraph.build(ms, m=M, ef_construct=EF_C, levels=levels, batch=512)
out["mean_token_build_s"] = time.perf_counter() - t0
plain, se, sl = sg.export_plain(), sg.entry_point, sg.entry_level
sg.close(); ms.close()
pg = qb.HnswGraph.multivector(view, plain, M, 2 * M)
out["mean_token_recall_at_10"] = recall(pg.search_maxsim(queries, TOP, EF, se, sl))
pg.close()

# the CPU restatement at a size it finishes, and the device on the same points
sub_rows, sub_off, sub_lv = rows[: N_CPU * T], off[: N_CPU + 1], levels[:N_CPU]
t0 = time.perf_counter()
ref = MvRefGraph.batched(sub_rows, sub_off, o.COSINE, M, 2 * M, EF_C, sub_lv, batch=512, serial_points=256)
out["cpu_restatement"] = {"points": N_CPU, "threads": 1, "build_s": time.perf_counter() - t0}
sst = qb.DenseVectorStorage(sub_rows, qb.Distance.Cosine)
sg, wall = timed_build(qb.MultiVectorView(sst, sub_off), sub_lv)
out["cpu_restatement"]["device_build_s"] = wall
out["cpu_restatement"]["device_equals_restatement"] = bool(np.array_equal(sg.export_plain(), ref.export_plain()))
sg.close(); sst.close(); ref.close()
st.close()

line = json.dumps(out)
print(line)
if len(sys.argv) > 2:
    with open(sys.argv[2], "w") as f:
        f.write(line + "\n")
