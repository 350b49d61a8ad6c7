"""BASELINE configs[0] (C1): 100 000 x 128 f32 dot product, single query, CPU only (SURVEY §8d).

The reference's own CPU-runnable case: the oracle's restatement of `dot_similarity_avx` + the `peek_top_iter` loop
(64-id chunks, binary heap) timed (i) on one thread = one segment, and (ii) on T threads over T equal segments + host
merge = how SegmentsSearcher parallelises.  With --gpu it also runs the same queries through the CUDA path on cuda:0 and
checks the results against the CPU scan (C1 is a parity case, not a GPU bench line: the whole data set is 51 MB).

    python tools/c1_cpu.py [--gpu] > c1_cpu.json
"""
import argparse
import concurrent.futures as cf
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpu", action="store_true")
    ap.add_argument("--queries", type=int, default=1000)
    args = ap.parse_args()
    from oracle import oracle as o
    from qdrant_b200.sharded import merge_topk_host, shard_ranges

    n, dim, top = 100_000, 128, 10
    base = np.random.default_rng(42).uniform(-1, 1, (n, dim)).astype(np.float32)
    queries = np.random.default_rng(43).uniform(-1, 1, (args.queries, dim)).astype(np.float32)

    def timed(fn, reps):
        for i in range(3):
            fn(i)
        ts = []
        for i in range(reps):
            t0 = time.perf_counter()
            fn(i)
            ts.append(time.perf_counter() - t0)
        return float(np.median(ts))

    one = timed(lambda i: o.scan_f32(o.DOT, base, queries[i % len(queries)][None, :], top), 200)
    threads = os.cpu_count() or 1
    pool = cf.ThreadPoolExecutor(max_workers=threads)
    rng = shard_ranges(n, threads)

    def multi(i):
        q = queries[i % len(queries)][None, :]
        parts = list(pool.map(lambda r: o.scan_f32(o.DOT, base, q, top, row_begin=r[0], row_end=r[1]), rng))
        return merge_topk_host([p[0] for p in parts], top)

    many = timed(multi, 200)
    out = {"config": "C1: 100000x128 f32 dot, single query, top 10 (BASELINE configs[0]); rng(42) uniform(-1,1) base, rng(43) queries",
           "cpu_1_thread": {"queries_per_s": 1.0 / one, "ms_per_query": one * 1e3, "gb_per_s": n * dim * 4 / one / 1e9},
           "cpu_all_threads": {"threads": threads, "queries_per_s": 1.0 / many, "ms_per_query": many * 1e3, "gb_per_s": n * dim * 4 / many / 1e9},
           "kind": "port (oracle: AVX2+FMA dot_similarity_avx + 64-id chunks + binary heap; not AVX-512)",
           "host": os.uname().nodename}
    if args.gpu:
        import torch

        from qdrant_b200 import scorer as qb

        st = qb.DenseVectorStorage(base, qb.Distance.Dot, device=0)
        bad = 0
        for b in range(0, len(queries), 100):
            got = st.search_batch(queries[b : b + 100], top)
            want = o.scan_f32(o.DOT, base, queries[b : b + 100], top)
            for g, w in zip(got, want):
                bad += 0 if np.array_equal(g["score"], w["score"]) else 1
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(200):
            st.search_batch(queries[i][None, :], top)
        gpu = (time.perf_counter() - t0) / 200
        out["gpu_e2e"] = {"queries_per_s": 1.0 / gpu, "ms_per_query": gpu * 1e3, "mismatching_queries": bad, "checked": len(queries),
                          "note": "host query in, host top-10 out through qb_search_batch; 51 MB fits L2, latency-bound"}
        st.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
