#!/usr/bin/env python
"""Custom-query probe: recommend (best-score, sum-scores: 3 positives, 2 negatives), context (2 pairs), discover (target + 2 pairs, both
stages in one call) and naive feedback (2 pairs) through the device traversal, on the C5 setup (clustered cosine, M = 16, ef = 128, graph
built in the run as in tools/hnsw_acorn_probe.py), unfiltered (HNSW) and under one random 5 % filter (ACORN).  One JSON line.
    python tools/hnsw_custom_probe.py [rows=1000000] [dim=768] [queries=4096] [ef=128] [out.json]
Per kind and filter: lists identical to the CPU checker (keyed tie order) out of the query count, q/s through the host API, device-timed
q/s (the traversal kernels bracketed by CUDA events, qb_profile_read), hops and scored points per query, and the CPU checker's q/s on
all host threads."""
import json, os, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as o
from qdrant_b200 import scorer as qb
from tests import hnsw_acorn_ref as ar
from tests import hnsw_custom_ref as cr

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
t0 = time.perf_counter(); g = o.HNSW(base, o.COSINE, m=16, ef_construct=100, seed=42, threads=threads); build_s = time.perf_counter() - t0
entry, lvl, m, m0 = g.entry()
blob = g.export_plain()
g.close()
st = qb.DenseVectorStorage(base, qb.Distance.Cosine)
hg = qb.HnswGraph(st, blob, m, m0)
cg = cr.Graph(blob, m, m0, n)

# examples near the data: cluster centres plus noise, as a user's liked / disliked points would be
qr = np.random.default_rng(43)
KINDS = {"reco_best_score": (1, 3, 2), "reco_sum_scores": (2, 3, 2), "context": (4, 2, 0), "discover": (3, 2, 0), "feedback": (cr.FEEDBACK, 2, 0)}
filtered = rng.random(n) >= 0.05
filtered[entry] = False
out = {"card_power_limit": card, "rows": n, "dim": dim, "queries": nq, "ef": ef, "top": top, "m": m, "m0": m0, "build_s": build_s, "host_threads": threads,
       "filter_selectivity": float(1 - filtered.mean()), "kinds": {}}
for name, (kind, n_a, n_b) in KINDS.items():
    ne = cr.n_examples(kind, n_a, n_b)
    raw = (centers[qr.integers(0, 1024, (nq, ne))] + 0.5 * qr.standard_normal((nq, ne, dim))).astype(np.float32)
    pre = o.preprocess_rows_f32(o.COSINE, raw.reshape(-1, dim)).reshape(nq, ne, dim)
    coef = qr.standard_normal((nq, 1 + n_a)).astype(np.float32) if kind == cr.FEEDBACK else None
    res = {}
    for fname, algo, f in (("unfiltered", "hnsw", None), ("random_5pct", "acorn", filtered)):
        if kind == 3:
            run = lambda: hg.search_discover(raw, n_a, top=top, ef=ef, entry_point=entry, entry_level=lvl, point_deleted=f, algorithm=algo)
        else:
            run = lambda: hg.search_custom(kind, raw, n_a, n_b, coef=coef, top=top, ef=ef, entry_point=entry, entry_level=lvl, point_deleted=f,
                                           algorithm=algo)
        run()                                               # scratch sized on first use
        hg.stats(reset=True)
        st.profile(True); st.profile_read(reset=True)
        t0 = time.perf_counter(); got = run(); api_s = time.perf_counter() - t0
        launches, ms = st.profile_read(reset=True); st.profile(False)
        hops, evals = hg.stats(reset=True)
        t0 = time.perf_counter()
        if kind == 3:
            want = cr.discover(cg, o, base, o.COSINE, pre, n_a, top, ef, entry, lvl, ar.ACORN if algo == "acorn" else ar.HNSW, f, threads=threads)
        else:
            want = cr.search_custom_batch(cg, o, base, o.COSINE, pre, kind, n_a, n_b, top, ef, entry, lvl, ar.ACORN if algo == "acorn" else ar.HNSW, f,
                                          coef=coef, threads=threads)
        cpu_s = time.perf_counter() - t0
        cpu_calls, cpu_scored = cg.stats()[:2]
        res[fname] = {"algorithm": algo, "identical_to_cpu_checker": int(sum(np.array_equal(a, b) for a, b in zip(got, want))),
                      "qps_host_api": nq / api_s, "qps_device_timed": nq / (ms / 1e3) if launches else None, "hops_per_query": hops / nq,
                      "scored_per_query": evals / nq, "stats_equal_cpu": [hops, evals] == [cpu_calls, cpu_scored], "cpu_checker_qps_all_threads": nq / cpu_s,
                      "exact_zero_scores": int(sum(int((a["score"] == 0).sum()) for a in got))}
    out["kinds"][name] = {"examples": ne, **res}
line = json.dumps(out)
print(line)
if len(sys.argv) > 5:
    with open(sys.argv[5], "w") as fh:
        fh.write(line + "\n")
