#!/usr/bin/env python
"""Compressed vs plain links.bin: file sizes, load time (host-to-device copy included), the device decode kernels' time, and
C5-shaped search throughput on one CPU-built graph loaded both ways (lists compared).
    python tools/hnsw_links_probe.py [--sizes 1000000,10000000] [--runs 3] [--search-rows 1000000] [--dim 768] [--queries 4096]"""
import argparse, json, os, re, subprocess, sys, time
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as o
from qdrant_b200 import scorer as qb
from tests import graph_links_compressed as gl

ap = argparse.ArgumentParser()
ap.add_argument("--sizes", default="1000000,10000000")
ap.add_argument("--runs", type=int, default=3)
ap.add_argument("--search-rows", type=int, default=1_000_000)
ap.add_argument("--dim", type=int, default=768)
ap.add_argument("--queries", type=int, default=4096)
args = ap.parse_args()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else torch.cuda.get_device_name(0)


out = {"card": card(), "graphs": [], "search": None}
for n in (int(x) for x in args.sizes.split(",")):
    rng = np.random.default_rng(n)
    lo, reindex, nb, off = gl.synthetic_graph(rng, n, 16, 32)            # m = 16, m0 = 32, geometric levels, full link lists
    plain = np.frombuffer(gl.serialize_plain(n, lo, reindex, nb, off), np.uint8)
    comp = np.frombuffer(gl.compress_plain_csr(n, lo, reindex, nb, off, 16, 32), np.uint8)
    del nb
    r = gl.CompressedLinks(comp)
    level0_bytes = gl.read_pair(r.offsets, r.params, n - 1)[1]          # byte offset where level 1's lists start
    del r
    st = qb.DenseVectorStorage(np.zeros((n, 1), np.float32), qb.Distance.Dot)
    t_plain, t_comp = [], []
    for _ in range(args.runs):                                           # alternated
        torch.cuda.synchronize(); t0 = time.perf_counter(); h = qb.HnswGraph(st, plain, 16, 32); torch.cuda.synchronize(); t_plain.append(time.perf_counter() - t0); h.close()
        torch.cuda.synchronize(); t0 = time.perf_counter(); h = qb.HnswGraph.from_compressed(st, comp); torch.cuda.synchronize(); t_comp.append(time.perf_counter() - t0); h.close()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        h = qb.HnswGraph.from_compressed(st, comp); torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        name = re.search(r"(hnsw_\w+|DeviceScan\w*)", e.key)
        if e.device_type == torch.autograd.DeviceType.CUDA and name:
            kernels[name.group(1)] = kernels.get(name.group(1), 0.0) + round(e.device_time_total / 1e3, 3)   # ms
    h.close(); st.close()
    out["graphs"].append({"points": n, "plain_bytes": int(plain.size), "compressed_bytes": int(comp.size),
                          "level0_bytes_per_point_plain": 4 * 32, "level0_bytes_per_point_compressed": round(level0_bytes / n, 2),
                          "load_s_plain": [round(x, 4) for x in t_plain], "load_s_compressed": [round(x, 4) for x in t_comp], "decode_kernels_ms": kernels})
    del plain, comp
    print(json.dumps(out["graphs"][-1]), flush=True)

# C5-shaped search (M = 16, ef = 128, top 10, clustered cosine data) on one CPU-built graph, loaded both ways
n, dim, nq = args.search_rows, args.dim, args.queries
rng = np.random.default_rng(42)
centers = rng.standard_normal((1024, dim)).astype(np.float32)
base = o.preprocess_rows_f32(o.COSINE, centers[rng.integers(0, 1024, n)] + 0.5 * rng.standard_normal((n, dim)).astype(np.float32))
queries = (centers[rng.integers(0, 1024, nq)] + 0.5 * rng.standard_normal((nq, dim))).astype(np.float32)
g = o.HNSW(base, o.COSINE, m=16, ef_construct=100, seed=42, threads=os.cpu_count() or 1)
entry, lvl, m, m0 = g.entry()
plain = g.export_plain()
comp = gl.plain_to_compressed(plain, m, m0)
st = qb.DenseVectorStorage(base, qb.Distance.Cosine)
hp = qb.HnswGraph(st, plain, m, m0)
hc = qb.HnswGraph.from_compressed(st, comp)
qps = {"plain": [], "compressed": []}
res = {}
hp.search(queries, 10, 128, entry, lvl); hc.search(queries, 10, 128, entry, lvl)
for _ in range(args.runs):
    for name, h in (("plain", hp), ("compressed", hc)):
        torch.cuda.synchronize(); t0 = time.perf_counter(); res[name] = h.search(queries, 10, 128, entry, lvl); qps[name].append(round(nq / (time.perf_counter() - t0), 1))
same = sum(int(np.array_equal(a, b)) for a, b in zip(res["plain"], res["compressed"]))
out["search"] = {"points": n, "dim": dim, "queries": nq, "ef": 128, "plain_bytes": int(plain.size), "compressed_bytes": len(comp),
                 "qps_plain": qps["plain"], "qps_compressed": qps["compressed"], "identical_lists": same}
hp.close(); hc.close(); st.close(); g.close()
print(json.dumps(out))
