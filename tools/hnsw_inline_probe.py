#!/usr/bin/env python
"""Search over a graph with inline vectors (qb_hnsw_search_with_vectors_batch) on the C5 setup, against the two searches it stands in
for.  One JSON line.
    python tools/hnsw_inline_probe.py [rows=1000000] [dim=768] [out.json]
Setup: clustered cosine rows (1024 Gaussian clusters, as bench.py's C5), M = 16, ef = 128, top 10, 4096 queries.  The graph is built
on the device (qb_hnsw_build, batch 512), exported as a plain links.bin, and written as CompressedWithVectors with f32 base vectors and
SQ8 link vectors encoded on the device (qb_sq8_encode_rows_device).
  (a) with_vectors: qb_hnsw_search_with_vectors_batch with ef = 128 (no rescoring);
  (b) sq8_rescore: the SQ8 traversal (qb_hnsw_search_batch on the same graph bound to the SQ8 storage) at the oversampled top
      (oversampling 2: top 20, ef 128), then qb_rescore of each list with the f32 scorer down to 10;
  (c) f32: the f32 traversal (qb_hnsw_search_batch on the dense storage).
Per run: device-resident q/s (the *_device entry on HBM queries, a host clock around the call and a device synchronise; (b) adds the
host rescoring time), host-API q/s (the host-facing call; (b) includes its rescoring), recall@10 against the exact scan, hops,
link-scored and base-scored points per query, the graph's HBM bytes (qb_hnsw_info) and its load time.  The three are timed
alternately, three rounds."""
import ctypes as C
import json, os, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from oracle import oracle as o
from qdrant_b200 import scorer as qb
from qdrant_b200._capi import check, lib, vp
from tests import graph_links_with_vectors as gv

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
dim = int(sys.argv[2]) if len(sys.argv) > 2 else 768
M, EF, TOP, NQ, OVERSAMPLED = 16, 128, 10, 4096, 20
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"card_power_limit": card, "rows": n, "dim": dim, "m": M, "m0": 2 * M, "ef": EF, "top": TOP, "queries": NQ, "oversampled_top": OVERSAMPLED}

rng = np.random.default_rng(42)
centers = rng.standard_normal((1024, dim)).astype(np.float32)
base = np.empty((n, dim), np.float32)
for a in range(0, n, 1 << 18):
    b = min(n, a + (1 << 18))
    base[a:b] = o.preprocess_rows_f32(o.COSINE, centers[rng.integers(0, 1024, b - a)] + 0.5 * rng.standard_normal((b - a, dim), dtype=np.float32))
queries = (centers[rng.integers(0, 1024, NQ)] + 0.5 * rng.standard_normal((NQ, dim))).astype(np.float32)
levels = np.minimum(np.round(-np.log(1.0 - np.random.default_rng(7).random(n)) / np.log(M)), 30).astype(np.uint8)

st = qb.DenseVectorStorage(base, qb.Distance.Cosine)
exact = st.search_batch(queries, TOP)
g = qb.HnswGraph.build(st, m=M, ef_construct=100, levels=levels, batch=512)
entry, elev = g.entry_point, g.entry_level
plain = g.export_plain()

# SQ8 rows encoded on the device
d_base = torch.from_numpy(base).cuda()
alpha, offset = qb.sq8_find_alpha_offset(d_base.data_ptr(), n, dim)
ad = (dim + 15) // 16 * 16
d_rows = torch.zeros((n, 4 + ad), dtype=torch.uint8, device="cuda")
qb.sq8_encode_rows(d_base.data_ptr(), n, dim, alpha, offset, qb.Distance.Cosine, d_rows.data_ptr())
torch.cuda.synchronize()
rows = d_rows.cpu().numpy()
del d_rows
qst = qb.ScalarQuantizedVectors(rows, dim, alpha, offset, qb.sq8_multiplier(alpha, qb.Distance.Cosine), qb.Distance.Cosine)
gq = qb.HnswGraph(qst, plain, M, 2 * M)

t0 = time.perf_counter()
blob = gv.serialize_plain_with_vectors(plain, M, 2 * M, base.view(np.uint8).reshape(n, dim * 4), rows)
out["file_write_s"] = time.perf_counter() - t0
out["file_bytes"] = int(blob.size)
t0 = time.perf_counter()
gw = qb.HnswGraph.from_compressed_with_vectors(qst, blob)
out["with_vectors_load_s"] = time.perf_counter() - t0
del blob
out["hbm_bytes"] = {"with_vectors": gw.info()[2], "sq8_graph": gq.info()[2], "sq8_rows": int(rows.nbytes), "f32_graph": g.info()[2],
                    "f32_rows": int(base.nbytes)}


def recall(lists):
    return float(np.mean([len(set(r["idx"].tolist()) & set(e["idx"].tolist())) / TOP for r, e in zip(lists, exact)]))



def rescore(lists):
    res = []
    for q, lst in zip(queries, lists):
        sc = st.build_raw_scorer(q)
        res.append(qb.rescore(sc, lst["idx"], TOP))
        sc.close()
    return res


dq = torch.from_numpy(queries).cuda()
d_out = torch.zeros((NQ, OVERSAMPLED, 2), dtype=torch.int32, device="cuda")
d_cnt = torch.zeros(NQ, dtype=torch.int32, device="cuda")


def device_call(kind):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if kind == "with_vectors":
        check(lib().qb_hnsw_search_with_vectors_batch_device(gw._h, vp(dq.data_ptr()), NQ, TOP, EF, entry, elev, vp(d_out.data_ptr()), vp(d_cnt.data_ptr())))
    elif kind == "sq8_rescore":
        check(lib().qb_hnsw_search_batch_device(gq._h, vp(dq.data_ptr()), NQ, OVERSAMPLED, EF, entry, elev, vp(d_out.data_ptr()), vp(d_cnt.data_ptr())))
    else:
        check(lib().qb_hnsw_search_batch_device(g._h, vp(dq.data_ptr()), NQ, TOP, EF, entry, elev, vp(d_out.data_ptr()), vp(d_cnt.data_ptr())))
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def host_call(kind):
    cnt = qb.HwCounters()
    t0 = time.perf_counter()
    if kind == "with_vectors":
        res = gw.search_with_vectors(queries, TOP, EF, entry, elev, counters=cnt)
        t_res = 0.0
    elif kind == "sq8_rescore":
        lists = gq.search(queries, OVERSAMPLED, EF, entry, elev, counters=cnt)
        t1 = time.perf_counter()
        res = rescore(lists)
        t_res = time.perf_counter() - t1
    else:
        res = g.search(queries, TOP, EF, entry, elev, counters=cnt)
        t_res = 0.0
    return time.perf_counter() - t0, t_res, res, cnt


handles = {"with_vectors": gw, "sq8_rescore": gq, "f32": g}
for k in handles:   # warm up every shape
    device_call(k); host_call(k)
runs = {k: {"device_qps": [], "host_qps": []} for k in handles}
for _ in range(3):
    for k, h in handles.items():
        t_dev = device_call(k)
        h.stats(reset=True)
        t_host, t_res, res, cnt = host_call(k)
        hops, scored = h.stats(reset=True)
        r = runs[k]
        r["device_qps"].append(NQ / (t_dev + t_res))
        r["host_qps"].append(NQ / t_host)
        if k == "sq8_rescore":
            r.setdefault("traversal_only_device_qps", []).append(NQ / t_dev)
            r.setdefault("rescore_host_s", []).append(t_res)
        r["recall_at_10"] = recall(res)
        r["hops_per_query"] = hops / NQ
        r["link_scored_per_query"] = scored / NQ   # with_vectors: SQ8 link scores; the others: the traversal's scored points
        if k == "with_vectors":
            r["base_scored_per_query"] = (cnt.cpu - scored * dim) / (4 * dim) / NQ
        elif k == "sq8_rescore":
            r["base_scored_per_query"] = OVERSAMPLED   # qb_rescore scores each list's ids with the f32 scorer
        else:
            r["base_scored_per_query"] = scored / NQ
out["runs"] = runs
line = json.dumps(out)
print(line)
if len(sys.argv) > 3:
    with open(sys.argv[3], "w") as fh:
        fh.write(line + "\n")
gw.close(); gq.close(); g.close(); qst.close(); st.close()
