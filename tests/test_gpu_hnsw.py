"""Config #5 harness: HNSW (M=16, ef=128) graph search driven by the GPU RawScorer vs the same traversal driven by the
CPU scorer.  Traversal stays on the CPU exactly as in the reference (GraphLayers::search -> FilteredScorer::score_points,
<= 2M ids per hop); only the scorer behind the trait changes.  Gate: identical result lists => recall@10 difference 0
(north_star asks for |delta recall| <= 1e-4, tie-aware)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def recall(res, exact):
    hit = tot = 0
    for r, e in zip(res, exact):
        kth = e["score"][-1]
        hit += sum(1 for s in r["score"] if s >= kth)  # tie-aware: anything at least as good as the exact k-th counts
        tot += e.size
    return hit / tot


@pytest.mark.parametrize("dist,quant", [("Cosine", None), ("Euclid", None), ("Cosine", "sq8"), ("Dot", "f16"), ("Euclid", "u8")])
def test_hnsw_gpu_scorer_matches_cpu_scorer(qb, oracle, dist, quant):
    """quant f16 / u8: the graph is built from the f32 values the stored rows were converted from; both traversals score the stored
    rows (CPU: the oracle's f16 / u8 metric on the converted query, GPU: the storage's scorer)."""
    n, dim, nq, top, ef = 30_000, 96, 60, 10, 128
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(7)
    if quant == "u8":
        base = rng.uniform(0.0, 256.0, (n, dim)).astype(np.float32)
        queries = rng.uniform(0.0, 256.0, (nq, dim)).astype(np.float32)
    else:
        base = rng.standard_normal((n, dim)).astype(np.float32)
        if d == qb.Distance.Cosine:
            base = oracle.preprocess_rows_f32(oracle.COSINE, base)
        queries = rng.standard_normal((nq, dim)).astype(np.float32)
    graph = oracle.HNSW(base, int(d), m=16, ef_construct=100, seed=42)   # built once on the CPU (single-threaded, deterministic)
    stored = None
    if quant == "f16":
        stored = base.astype(np.float16)
        dense = qb.DenseVectorStorage(stored, d, qb.VectorStorageDatatype.Float16)
    elif quant == "u8":
        stored = oracle.to_u8_query(base.reshape(-1)).reshape(n, dim)
        dense = qb.DenseVectorStorage(stored, d, qb.VectorStorageDatatype.Uint8)
    else:
        dense = qb.DenseVectorStorage(base, d)
    sq = qst = None
    if quant == "sq8":
        dt, inv = qb.construct_vector_parameters(d)
        sq = oracle.SQ8.encode(base, int(dt), bool(inv))
        qst = qb.ScalarQuantizedVectors(sq.rows, dim, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, d)
    cpu_res, gpu_res, exact = [], [], []
    calls = []
    for q in queries:
        qp = oracle.preprocess_f32(int(d), q)
        if quant == "sq8":
            code, off = sq.encode_query(qp)
            cpu_scorer = lambda ids, code=code, off=off: np.array([sq.score(code, off, int(i)) for i in ids], np.float32)
            fs = qb.FilteredScorer.new(q, dense, qst)       # quantized scorer preferred (point_scorer.rs:172-175)
        elif stored is not None:
            qc = oracle.to_f16_query(int(d), q) if quant == "f16" else oracle.to_u8_query(q)
            score_rows = oracle.score_rows_f16 if quant == "f16" else oracle.score_rows_u8
            cpu_scorer = lambda ids, qc=qc, score_rows=score_rows: score_rows(int(d), stored, qc, ids)  # noqa: E731
            fs = qb.FilteredScorer.new(q, dense, None)
        else:
            cpu_scorer = None                                # oracle's built-in f32 scorer
            fs = qb.FilteredScorer.new(q, dense, None)
        graph.stats(reset=True)
        cpu_res.append(graph.search(qp, top, ef, score_points=cpu_scorer))
        gpu_res.append(graph.search(qp, top, ef, score_points=lambda ids, fs=fs: fs.raw_scorer.score_points(ids)))
        calls.append(graph.stats(reset=True))
        if quant == "f16":
            exact.append(oracle.scan_f16(int(d), stored, qc, top)[0])
        elif quant == "u8":
            exact.append(oracle.scan_u8(int(d), stored, qc, top)[0])
        else:
            exact.append(oracle.scan_f32(int(d), base, qp, top)[0])
    for a, b in zip(cpu_res, gpu_res):
        np.testing.assert_array_equal(a, b)                 # same traversal, same scores, same result
    r_cpu, r_gpu = recall(cpu_res, exact), recall(gpu_res, exact)
    assert abs(r_cpu - r_gpu) <= 1e-4
    assert r_cpu > (0.4 if quant == "sq8" else 0.6)  # graph quality on random 96-d data; the gate is CPU == GPU above
    hops = np.mean([c[0] for c in calls]); evals = np.mean([c[1] for c in calls])
    print(f"{dist} {quant}: recall@10 cpu={r_cpu:.4f} gpu={r_gpu:.4f}; {hops:.0f} score_points calls, {evals:.0f} evaluations per query")
    graph.close(); dense.close()
    if qst:
        qst.close()
