#!/usr/bin/env python
"""Device HNSW traversal for custom queries with multivector examples on a ColBERT-shaped collection, against the routes it replaces.
One JSON line.
    python tools/hnsw_multivector_custom_probe.py [points=200000] [out.json]
Setup: `points` points of 16..48 clustered 128-d cosine tokens each (about 32; 4096 Gaussian clusters, a point's tokens share one
cluster), dense f32 tokens, examples of 32 vectors drawn near random clusters, top 10, ef 128.  The graph is qb_hnsw_build (M = 16,
ef_construct = 100) over each point's normalised mean token, built on the device, exported plain and bound to the token storage with
qb_hnsw_create_plain_multivector (the collection and graph of tools/hnsw_multivector_probe.py with shorter runs).
Kinds: recommend best-score and sum-scores (3 positives, 1 negative), context (2 pairs): 4 examples; feedback and discover (a target and
2 pairs): 5 examples; discover once as one search (qb_hnsw_search_maxsim_custom_batch) and once with both stages
(qb_hnsw_search_maxsim_discover_batch).  Per kind: host-API q/s (the call, queries in and lists out), device q/s (the traversal kernels
alone, CUDA events through qb_profile_*), hops and scored points per query, recall@10 against qb_search_maxsim_custom (MaxSim over
every point) and that scan's own q/s, how many lists equal the keyed CPU checker's (tests/hnsw_maxsim_custom_ref.py, scoring the points
it visits from their token rows), and the per-hop route this replaces on a few queries: the CPU traversal calling qb_score_maxsim_custom
once per hop.  Timed rounds alternate the kinds, three rounds after a warm-up of every shape."""
import json, os, subprocess, sys, time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from oracle import oracle as o
from qdrant_b200 import scorer as qb
from tests import hnsw_custom_ref as cr
from tests import hnsw_maxsim_custom_ref as mc

o.ensure_built()

n = int(sys.argv[1]) if len(sys.argv) > 1 else 200_000
dim, M, EF, TOP, QV, NQ, N_EXACT, N_CHECK, N_HOP = 128, 16, 128, 10, 32, 1024, 16, 16, 2
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"card_power_limit": card, "points": n, "dim": dim, "m": M, "ef_construct": 100, "ef": EF, "top": TOP, "example_vectors": QV, "queries": NQ}

g = torch.Generator(device="cuda").manual_seed(42)
centers = torch.randn((4096, dim), device="cuda", generator=g)
runs = torch.randint(16, 49, (n,), device="cuda", generator=g)
cluster = torch.randint(0, 4096, (n,), device="cuda", generator=g)
tok = centers[torch.repeat_interleave(cluster, runs)] + 0.5 * torch.randn((int(runs.sum()), dim), device="cuda", generator=g)
tok = torch.nn.functional.normalize(tok, dim=1).contiguous()
off = np.concatenate([[0], np.cumsum(runs.cpu().numpy())]).astype(np.uint32)
out["token_rows"] = int(off[-1])

# the proxy graph over normalised mean tokens, built on the device
pid = torch.repeat_interleave(torch.arange(n, device="cuda"), runs)
means = torch.zeros((n, dim), device="cuda").index_add_(0, pid, tok)
means = torch.nn.functional.normalize(means, dim=1).cpu().numpy()
mst = qb.DenseVectorStorage(means, qb.Distance.Cosine)
levels = np.minimum(np.round(-np.log(1.0 - np.random.default_rng(7).random(n)) / np.log(M)), 30).astype(np.uint8)
mg = qb.HnswGraph.build(mst, m=M, ef_construct=100, levels=levels, batch=512)
entry, elev = mg.entry_point, mg.entry_level
plain = mg.export_plain()
mg.close(); mst.close()

rows = tok.cpu().numpy()
del tok
st = qb.DenseVectorStorage(rows, qb.Distance.Cosine)
rows_pre = o.preprocess_rows_f32(o.COSINE, rows)   # the rows as the storage holds them, for the checker
view = qb.MultiVectorView(st, off)
hg = qb.HnswGraph.multivector(view, plain, M, 2 * M)
rng = np.random.default_rng(3)
cent = centers.cpu().numpy()


def ex():
    return (cent[rng.integers(0, 4096)] + 0.5 * rng.standard_normal((QV, dim))).astype(np.float32)


def pairs(k):
    return [qb.ContextPair(ex(), ex()) for _ in range(k)]


make = {
    "recommend_best_score": lambda: qb.RecoBestScoreQuery(qb.RecoQuery([ex(), ex(), ex()], [ex()])),
    "recommend_sum_scores": lambda: qb.RecoSumScoresQuery(qb.RecoQuery([ex(), ex(), ex()], [ex()])),
    "context": lambda: qb.ContextQuery(pairs(2)),
    "feedback": lambda: qb.FeedbackQuery(ex(), pairs(2), rng.random(2).astype(np.float32), 0.5),
    "discover_one_search": lambda: qb.DiscoverQuery(ex(), pairs(2)),
}
queries = {k: [f() for _ in range(NQ)] for k, f in make.items()}
queries["discover_two_stages"] = queries["discover_one_search"]


def run(k, qs):
    if k == "discover_two_stages":
        return hg.search_maxsim_discover(qs, TOP, EF, entry, elev)
    return hg.search_maxsim_custom(qs, TOP, EF, entry, elev)


for k, qs in queries.items():   # warm-up of every shape
    run(k, qs[:64])
res = {k: {"host_qps": [], "device_qps": []} for k in queries}
lists = {}
for _ in range(3):
    for k, qs in queries.items():
        hg.stats(reset=True)
        st.profile(True)
        st.profile_read(reset=True)
        t = time.perf_counter()
        lists[k] = run(k, qs)
        dt = time.perf_counter() - t
        _, ms = st.profile_read(reset=True)
        st.profile(False)
        hops, pts = hg.stats(reset=True)
        r = res[k]
        r["host_qps"].append(NQ / dt)
        r["device_qps"].append(NQ / (ms / 1e3))
        r["hops_per_query"], r["scored_points_per_query"] = hops / NQ, pts / NQ

cg = cr.Graph(plain, M, 2 * M, n)
for k, qs in queries.items():
    r = res[k]
    fused = k == "discover_two_stages"
    if not fused:   # exact: qb_search_maxsim_custom over every point (the two discover forms share it)
        t = time.perf_counter()
        exact = [view.search_custom(q, TOP) for q in qs[:N_EXACT]]
        r["search_maxsim_custom_qps"] = N_EXACT / (time.perf_counter() - t)
        ex_lists = exact
    r["recall_at_10"] = float(np.mean([len(set(a["idx"].tolist()) & set(e["idx"].tolist())) / TOP for a, e in zip(lists[k][:N_EXACT], ex_lists)]))
    # the keyed CPU checker, scoring only the points it visits
    same = 0
    for i, q in enumerate(qs[:N_CHECK]):
        examples, n_a, n_b = q.flat()
        coef = np.concatenate([[q.a], q.partial]).astype(np.float32) if k == "feedback" else None
        if fused:
            ctx = mc.lazy_scores_f32(o, o.COSINE, rows_pre, off, mc.CONTEXT, n_a, 0, examples[1:])
            s1 = cr.search_cb(cg, ctx, cr.DISCOVERY_ENTRY_POINT_COUNT, EF, entry, elev, keyed=True)
            w = cr.search_cb(cg, mc.lazy_scores_f32(o, o.COSINE, rows_pre, off, mc.DISCOVER, n_a, 0, examples), TOP, EF, entry, elev,
                             cep=s1["idx"].copy(), keyed=True)
        else:
            w = cr.search_cb(cg, mc.lazy_scores_f32(o, o.COSINE, rows_pre, off, int(q.kind), n_a, n_b, examples, coef), TOP, EF, entry, elev, keyed=True)
        a = lists[k][i]
        same += int(np.array_equal(a["idx"], w["idx"]) and np.array_equal(a["score"].view(np.uint32), w["score"].view(np.uint32)))
    r["lists_equal_to_checker"] = f"{same}/{N_CHECK}"
    if not fused:   # the route this replaces: the CPU traversal with one qb_score_maxsim_custom call per hop
        t = time.perf_counter()
        for q in qs[:N_HOP]:
            cr.search_cb(cg, lambda ids, q=q: view.score_points_custom(q, ids), TOP, EF, entry, elev, keyed=True)
        r["per_hop_host_route_qps"] = N_HOP / (time.perf_counter() - t)
cg.close()
out["results"] = res
line = json.dumps(out)
print(line)
if len(sys.argv) > 2:
    with open(sys.argv[2], "w") as f:
        f.write(line + "\n")
hg.close(); st.close()
