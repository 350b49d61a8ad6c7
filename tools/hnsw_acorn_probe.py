#!/usr/bin/env python
"""ACORN probe: device traversal with SearchAlgorithm::Hnsw vs ::Acorn under filters, on the C5 setup (clustered cosine, M = 16,
ef = 128), against the exact filtered scan and the CPU ACORN traversal of the same graph on all host cores.  One JSON line.
    python tools/hnsw_acorn_probe.py [rows=1000000] [dim=768] [queries=4096] [ef=128] [out.json]
Filters: random at selectivity 0.01 / 0.05 / 0.1 / 0.4, and cluster-correlated (a cluster is kept or not, ~5 % of the points).
Per filter and algorithm: q/s through the host API (per-call bitmap) and device-timed (resident flags + qb_hnsw_search_batch_device_algo,
CUDA events), hops and scored points per query, recall@10 against qb_search_batch with the same bitmap, lists identical to the CPU
ACORN traversal, and the CPU ACORN q/s."""
import json, os, subprocess, sys, time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as o
from qdrant_b200 import scorer as qb
from qdrant_b200._capi import check, lib, vp
from tests import hnsw_acorn_ref as ar

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
dim = int(sys.argv[2]) if len(sys.argv) > 2 else 768
nq = int(sys.argv[3]) if len(sys.argv) > 3 else 4096
ef = int(sys.argv[4]) if len(sys.argv) > 4 else 128
top, threads = 10, os.cpu_count() or 1
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()

rng = np.random.default_rng(42)
centers = rng.standard_normal((1024, dim)).astype(np.float32)
label = rng.integers(0, 1024, n)
base = o.preprocess_rows_f32(o.COSINE, centers[label] + 0.5 * rng.standard_normal((n, dim)).astype(np.float32))
qr = np.random.default_rng(43)
queries = (centers[qr.integers(0, 1024, nq)] + 0.5 * qr.standard_normal((nq, dim))).astype(np.float32)
qp = o.preprocess_rows_f32(o.COSINE, queries)
t0 = time.perf_counter(); g = o.HNSW(base, o.COSINE, m=16, ef_construct=100, seed=42, threads=threads); build_s = time.perf_counter() - t0
entry0, lvl, m, m0 = g.entry()
blob = g.export_plain()
g.close()
hdr = np.frombuffer(blob[:40].tobytes(), np.uint64).astype(np.int64)      # point_count, levels_count, neighbours, offsets, padding
level_offsets = np.frombuffer(blob[64:64 + 8 * hdr[1]].tobytes(), np.uint64).astype(np.int64)
reindex = np.frombuffer(blob[64 + 8 * hdr[1]:64 + 8 * hdr[1] + 4 * n].tobytes(), np.uint32)
level_counts = np.diff(np.r_[level_offsets, hdr[3] - 1])
st = qb.DenseVectorStorage(base, qb.Distance.Cosine)
hg = qb.HnswGraph(st, blob, m, m0)
cg = ar.Graph(blob, m, m0, n)
dev = torch.device("cuda", 0)
d_q = torch.from_numpy(queries).to(dev)
d_out = torch.empty((nq, top), dtype=torch.int64, device=dev)
d_cnt = torch.empty((nq,), dtype=torch.int32, device=dev)
stream = torch.cuda.ExternalStream(st.stream_ptr(), device=dev)

filters = {f"random_{s}": rng.random(n) >= s for s in (0.01, 0.05, 0.1, 0.4)}
filters["clusters_5pct"] = ~np.isin(label, rng.choice(1024, 51, replace=False))
out = {"card_power_limit": card, "entry_rule": "graph entry if it passes, else highest-level passing point", "rows": n, "dim": dim, "queries": nq, "ef": ef, "m": m, "m0": m0, "build_s": build_s, "host_threads": threads, "filters": {}}
for name, filtered in filters.items():
    # Entry point: the graph's own if it passes the filter, else the highest-level point that passes (back_index order: a smaller reindex
    # is a higher level).  The reference's get_entry_point searches its EntryPoints list (and extra entry points) instead, so recall and
    # q/s here are for this rule; device and CPU traversal start from the same point either way.
    entry, elvl = entry0, lvl
    if filtered[entry0]:
        entry = int(np.flatnonzero(~filtered)[np.argmin(reindex[~filtered])])
        elvl = int(sum(reindex[entry] < c for c in level_counts[1:]))
    exact = st.search_batch(queries, top, point_deleted=filtered)
    row = {"selectivity": float(1 - filtered.mean()), "entry_level": elvl}
    cpu_t0 = time.perf_counter()
    cpu = cg.search_batch(o, base, o.COSINE, qp, top, ef, entry, elvl, ar.ACORN, filtered, threads=threads)
    row["cpu_acorn_qps_all_threads"] = nq / (time.perf_counter() - cpu_t0)
    cg.stats()
    st.set_deleted(filtered)
    for algo, code in (("hnsw", 0), ("acorn", 1)):
        hg.search(queries, top, ef, entry, elvl, point_deleted=filtered, algorithm=algo)          # scratch sized on first use
        hg.stats(reset=True)
        t0 = time.perf_counter(); got = hg.search(queries, top, ef, entry, elvl, point_deleted=filtered, algorithm=algo); api_s = time.perf_counter() - t0
        hops, evals = hg.stats(reset=True)
        step = lambda: check(lib().qb_hnsw_search_batch_device_algo(hg._h, vp(d_q.data_ptr()), nq, top, ef, entry, elvl, vp(d_out.data_ptr()),
                                                                    vp(d_cnt.data_ptr()), code))
        step(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(3):
            step()
        e1.record(stream); torch.cuda.synchronize()
        hg.stats(reset=True)
        rec = float(np.mean([len(set(a["idx"].tolist()) & set(e["idx"].tolist())) / max(len(e), 1) for a, e in zip(got, exact)]))
        r = {"qps_host_api": nq / api_s, "qps_device_timed": 3 * nq / (e0.elapsed_time(e1) / 1e3), "hops_per_query": hops / nq,
             "scored_per_query": evals / nq, "recall_at_10": rec}
        if algo == "acorn":
            r["identical_to_cpu_acorn"] = int(sum(np.array_equal(a, b) for a, b in zip(got, cpu)))
        row[algo] = r
    st.set_deleted(None)
    out["filters"][name] = row
line = json.dumps(out)
print(line)
if len(sys.argv) > 5:
    with open(sys.argv[5], "w") as f:
        f.write(line + "\n")
