#!/usr/bin/env python
"""Device HNSW search over multivector (MaxSim) points on a ColBERT-shaped collection, against the routes it replaces.  One JSON line.
    python tools/hnsw_multivector_probe.py [points=200000] [out.json]
Setup: `points` points of 16..128 clustered 128-d cosine tokens each (4096 Gaussian clusters; a point's tokens share one cluster), f32
and SQ8 (encoded on the device) storages of the same tokens, 32-token queries, top 10, ef 128.  No MaxSim graph builder exists, so the
graph is qb_hnsw_build (M = 16, ef_construct = 100) over each point's normalised mean token, exported plain and bound to the token
storage with qb_hnsw_create_plain_multivector: recall is that of this proxy graph.
Per storage: device q/s (qb_hnsw_search_maxsim_batch_device on HBM queries, a host clock around the call and a device synchronise),
host-API q/s (qb_hnsw_search_maxsim_batch), hops, scored points and token rows per query, token-row bytes per second against the
H100 SXM data-sheet HBM3 figure (3.35 TB/s, a data-sheet number, not a measured peak), recall@10 against qb_search_maxsim (exact
MaxSim over every point) and qb_search_maxsim's own q/s, and today's per-hop route on a few queries: the CPU traversal
(tests/hnsw_custom_ref.py) calling qb_score_maxsim once per hop.  The two storages are timed alternately, three rounds, after a
warm-up of every shape."""
import json, os, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from qdrant_b200 import scorer as qb
from qdrant_b200._capi import check, lib
from tests import hnsw_custom_ref as cr

n = int(sys.argv[1]) if len(sys.argv) > 1 else 200_000
dim, M, EF, TOP, QV, NQ, N_EXACT, N_HOP = 128, 16, 128, 10, 32, 4096, 64, 4
HBM_DATASHEET = 3.35e12
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"card_power_limit": card, "points": n, "dim": dim, "m": M, "ef_construct": 100, "ef": EF, "top": TOP, "query_vectors": QV, "queries": NQ}

g = torch.Generator(device="cuda").manual_seed(42)
centers = torch.randn((4096, dim), device="cuda", generator=g)
runs = torch.randint(16, 129, (n,), device="cuda", generator=g)
cluster = torch.randint(0, 4096, (n,), device="cuda", generator=g)
tok = centers[torch.repeat_interleave(cluster, runs)] + 0.5 * torch.randn((int(runs.sum()), dim), device="cuda", generator=g)
tok = torch.nn.functional.normalize(tok, dim=1).contiguous()
off = np.concatenate([[0], np.cumsum(runs.cpu().numpy())]).astype(np.uint32)
n_rows = int(off[-1])
qcl = torch.randint(0, 4096, (NQ,), device="cuda", generator=g)
d_queries = (centers[qcl.repeat_interleave(QV)] + 0.5 * torch.randn((NQ * QV, dim), device="cuda", generator=g)).contiguous()
queries = list(d_queries.cpu().numpy().reshape(NQ, QV, dim))
d_qoff = torch.arange(0, NQ * QV + 1, QV, dtype=torch.int32, device="cuda")
out["token_rows"] = n_rows

# the proxy graph over normalised mean tokens
pid = torch.repeat_interleave(torch.arange(n, device="cuda"), runs)
means = torch.zeros((n, dim), device="cuda").index_add_(0, pid, tok)
means = torch.nn.functional.normalize(means, dim=1).cpu().numpy()
mst = qb.DenseVectorStorage(means, qb.Distance.Cosine)
levels = np.minimum(np.round(-np.log(1.0 - np.random.default_rng(7).random(n)) / np.log(M)), 30).astype(np.uint8)
t0 = time.perf_counter()
mg = qb.HnswGraph.build(mst, m=M, ef_construct=100, levels=levels, batch=512)
out["graph_build_s"] = time.perf_counter() - t0
entry, elev = mg.entry_point, mg.entry_level
plain = mg.export_plain()
mg.close(); mst.close()

stores = {"f32": qb.DenseVectorStorage(tok.cpu().numpy(), qb.Distance.Cosine)}
alpha, offset = qb.sq8_find_alpha_offset(tok.data_ptr(), n_rows, dim)
d_rows = torch.zeros((n_rows, 4 + dim), dtype=torch.uint8, device="cuda")
qb.sq8_encode_rows(tok.data_ptr(), n_rows, dim, alpha, offset, qb.Distance.Cosine, d_rows.data_ptr())
torch.cuda.synchronize()
stores["sq8"] = qb.ScalarQuantizedVectors(None, dim, alpha, offset, qb.sq8_multiplier(alpha, qb.Distance.Cosine), qb.Distance.Cosine,
                                          rows_ptr=d_rows.data_ptr(), count=n_rows)
del tok
views = {k: qb.MultiVectorView(s, off) for k, s in stores.items()}
graphs = {k: qb.HnswGraph.multivector(v, plain, M, 2 * M) for k, v in views.items()}
row_bytes = {"f32": dim * 4, "sq8": 4 + dim}
units = {"f32": dim * 4, "sq8": dim}

d_out = torch.zeros((NQ, TOP, 2), dtype=torch.int32, device="cuda")
d_cnt = torch.zeros(NQ, dtype=torch.int32, device="cuda")


def device_run(k):
    torch.cuda.synchronize()
    t = time.perf_counter()
    check(lib().qb_hnsw_search_maxsim_batch_device(graphs[k]._h, d_queries.data_ptr(), NQ * QV, d_qoff.data_ptr(), NQ, QV, TOP, EF, entry, elev,
                                                   d_out.data_ptr(), d_cnt.data_ptr(), 0))
    torch.cuda.synchronize()
    return time.perf_counter() - t


def host_run(k):
    c = qb.HwCounters()
    t = time.perf_counter()
    res = graphs[k].search_maxsim(queries, TOP, EF, entry, elev, counters=c)
    return time.perf_counter() - t, res, c


for k in graphs:   # warm-up of every shape
    device_run(k)
    host_run(k)
res = {k: {"device_qps": [], "host_qps": []} for k in graphs}
lists = {}
for _ in range(3):
    for k in graphs:
        res[k]["device_qps"].append(NQ / device_run(k))
        graphs[k].stats(reset=True)
        dt, lists[k], c = host_run(k)
        res[k]["host_qps"].append(NQ / dt)
        hops, pts = graphs[k].stats(reset=True)
        res[k]["hops_per_query"], res[k]["scored_points_per_query"] = hops / NQ, pts / NQ
        res[k]["token_rows_per_query"] = c.cpu / (QV * units[k]) / NQ
for k in graphs:
    r = res[k]
    bps = r["token_rows_per_query"] * row_bytes[k] * max(r["device_qps"])
    r["token_row_bytes_per_s"] = bps
    r["share_of_hbm_datasheet"] = bps / HBM_DATASHEET
    # exact MaxSim over every point: recall reference and its own rate
    t = time.perf_counter()
    exact = [views[k].search(queries[i], TOP) for i in range(N_EXACT)]
    r["search_maxsim_qps"] = N_EXACT / (time.perf_counter() - t)
    r["recall_at_10"] = float(np.mean([len(set(a["idx"].tolist()) & set(e["idx"].tolist())) / TOP for a, e in zip(lists[k][:N_EXACT], exact)]))
    # today's route: the CPU traversal with one qb_score_maxsim call per hop
    cg = cr.Graph(plain, M, 2 * M, n)
    t = time.perf_counter()
    for i in range(N_HOP):
        cr.search_cb(cg, lambda ids, i=i: views[k].score_points(queries[i], ids), TOP, EF, entry, elev, keyed=True)
    r["per_hop_host_route_qps"] = N_HOP / (time.perf_counter() - t)
    cg.close()
out["results"] = res
line = json.dumps(out)
print(line)
if len(sys.argv) > 2:
    with open(sys.argv[2], "w") as f:
        f.write(line + "\n")
