"""The CPU checker of qb_mmr_sparse_batch (tests/mmr_sparse_ref.c through tests/mmr_sparse_ref.py): it reproduces the reference's own
sparse MMR case with the order worked out by hand, equals an independent NumPy restatement of maximal_marginal_relevance over
score_vectors (full pair matrix, a Python list with swap-remove) on random, tie-heavy, duplicate-id, empty-row, short-list and non-finite
inputs, scores pairs symmetrically bit for bit, sums in ascending dim order observably, and meters the counters the reference meters."""
import json
import os

import numpy as np

from tests import mmr_sparse_ref as ms

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mmr_sparse_reference_cases.json")


def _key(x):
    """OrderedFloat: NaN above everything and equal to NaN; -0.0 == +0.0 (Python's float comparison)"""
    return (1, 0.0) if np.isnan(x) else (0, float(x))


def _argmax(vals):
    """max_by_key: the last maximal element"""
    best = 0
    for i in range(1, len(vals)):
        if _key(vals[i]) >= _key(vals[best]):
            best = i
    return best


def py_score(a, b, descending=False):
    """score_vectors: 0 + a_w * b_w over the shared dims in ascending dim order (descending: the negative control), f32 throughout"""
    wa = {int(d): np.float32(w) for d, w in zip(a[0], a[1])}
    wb = {int(d): np.float32(w) for d, w in zip(b[0], b[1])}
    s = np.float32(0.0)
    with np.errstate(all="ignore"):
        for d in sorted(set(wa) & set(wb), reverse=descending):
            s = np.float32(s + np.float32(wa[d] * wb[d]))
    return s


def _row(csr, p):
    ip, d, w = csr
    return d[int(ip[p]) : int(ip[p + 1])], w[int(ip[p]) : int(ip[p + 1])]


def py_mmr(csr, query, lam, cand, limit, descending=False):
    """maximal_marginal_relevance over the full pair matrix, the remaining candidates as a list with swap-remove -> (ids, cpu)"""
    uniq, seen = [], set()
    for c in cand:
        if int(c["idx"]) not in seen:
            seen.add(int(c["idx"]))
            uniq.append(c)
    n = len(uniq)
    if n < 2:
        return [int(c["idx"]) for c in uniq], 0
    rows = [_row(csr, int(c["idx"])) for c in uniq]
    ln = [len(r[0]) for r in rows]
    rel = [py_score(query, r, descending) for r in rows]
    mat = [[py_score(rows[c], rows[s], descending) for s in range(n)] for c in range(n)]
    lam = np.float32(lam)
    remaining, selected = list(range(n)), []

    def pick(vals):
        p = _argmax(vals)
        selected.append(remaining[p])
        remaining[p] = remaining[-1]
        remaining.pop()

    pick(rel)
    cpu = sum(min(len(query[0]), x) for x in ln)
    while len(selected) < limit and remaining:
        cpu += sum(min(ln[c], ln[selected[-1]]) for c in remaining)
        scores = []
        with np.errstate(all="ignore"):
            for c in remaining:
                sims = [mat[c][s] for s in selected]
                ms_ = sims[_argmax(sims)]
                scores.append(np.float32(np.float32(lam * rel[c]) - np.float32(np.float32(np.float32(1.0) - lam) * ms_)))
        pick(scores)
    return [int(uniq[s]["idx"]) for s in selected], cpu


def _rows(rng, n_points, dims, mean_nnz, weights=None, empty=0.0):
    """CSR rows of distinct dims drawn from `dims` in shuffled order; weights from `weights` when given, else in [-1, 1)"""
    counts = np.minimum(rng.poisson(mean_nnz, n_points), len(dims))
    counts[rng.random(n_points) < empty] = 0
    d = [rng.choice(dims, size=c, replace=False) for c in counts]
    ip = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
    dd = np.concatenate(d).astype(np.uint32) if counts.sum() else np.zeros(0, np.uint32)
    w = (rng.choice(weights, dd.size) if weights is not None else rng.random(dd.size) * 2 - 1).astype(np.float32)
    return ip, dd, w


def _cands(rng, n, n_points, dup_ids=0):
    ids = rng.choice(n_points, size=n, replace=n > n_points).astype(np.uint32)
    for _ in range(dup_ids if n > 1 else 0):
        ids[rng.integers(1, n)] = ids[rng.integers(0, n)]
    c = np.zeros(n, ms.SCORED)
    c["idx"] = ids
    c["score"] = rng.standard_normal(n).astype(np.float32)
    return c


def _check(csr, q, lam, cand, limit):
    got, cpu, io = ms.mmr(csr, q, lam, cand, limit)
    want, want_cpu = py_mmr(csr, q, lam, cand, limit)
    assert got["idx"].tolist() == want, (lam, limit, got["idx"].tolist(), want)
    first = {}
    for c in cand:
        first.setdefault(int(c["idx"]), c["score"])
    assert np.array_equal(got["score"].view(np.uint32), np.array([first[i] for i in want], np.float32).view(np.uint32))
    assert (cpu, io) == (want_cpu, 0)


def test_reference_case():
    with open(FIXTURE) as f:
        fx = json.load(f)
    pts = fx["points"]
    ip = np.concatenate([[0], np.cumsum([len(p["dims"]) for p in pts])]).astype(np.uint64)
    csr = (ip, np.concatenate([p["dims"] for p in pts]).astype(np.uint32), np.concatenate([p["weights"] for p in pts]).astype(np.float32))
    ids = [p["id"] for p in pts]   # point i holds reference id ids[i]
    cand = np.zeros(len(ids), ms.SCORED)
    cand["idx"] = np.arange(len(ids))
    q = (np.array(fx["query"]["dims"], np.uint32), np.array(fx["query"]["weights"], np.float32))
    assert [ms.score(q, _row(csr, i)) for i in range(3)] == [np.float32(x) for x in fx["relevance"]]
    got, cpu, io = ms.mmr(csr, q, fx["lambda"], cand, fx["limit"])
    assert [ids[i] for i in got["idx"]] == fx["expected"] and (cpu, io) == (fx["cpu"], 0)
    assert [ids[i] for i in py_mmr(csr, q, fx["lambda"], cand, fx["limit"])[0]] == fx["expected"]
    assert fx["expected"] != fx["expected_in_input_order"]


def test_checker_equals_numpy_restatement():
    rng = np.random.default_rng(3)
    dims = np.concatenate([[0, 0xFFFFFFFF, 0xFFFFFFFE], rng.choice(1 << 31, 40, replace=False)]).astype(np.uint32)
    cases = {
        "random": dict(csr=_rows(rng, 80, dims, 8), weights=None),
        "tie": dict(csr=_rows(rng, 80, dims[:8], 3, weights=[0.5, 1.0, 2.0], empty=0.1), weights=[0.5, 1.0, 2.0]),
        "empty": dict(csr=_rows(rng, 80, dims, 4, empty=0.4), weights=None),
        "huge": dict(csr=_rows(rng, 80, dims[:12], 5, weights=[1e20, -1e20, 3e19, 1.0]), weights=[1e20, -1e20, 1.0]),
    }
    for name, cs in cases.items():
        csr = cs["csr"]
        for n, limit, lam in ((0, 3, 0.5), (1, 3, 0.5), (2, 1, 0.5), (2, 5, 0.0), (3, 3, 1.0), (3, 2, 0.5), (20, 4, 0.5), (20, 30, 0.3),
                              (45, 45, 0.0), (45, 8, 1.0), (60, 12, 0.5)):
            cand = _cands(rng, n, 80, dup_ids=3 if n > 5 else 0)
            qn = int(rng.integers(0, 6))
            qd = rng.choice(dims[:12] if name in ("tie", "huge") else dims, qn, replace=False).astype(np.uint32)
            qw = (rng.choice(cs["weights"], qn) if cs["weights"] else rng.random(qn) * 2 - 1).astype(np.float32)
            if name == "huge" and qn:
                qw[0] = np.nan if n % 2 else np.inf   # NaN relevance, and +-inf products summing to NaN
            _check(csr, (qd, qw), lam, cand, limit)


def test_pair_is_symmetric_bit_for_bit():
    rng = np.random.default_rng(5)
    dims = rng.choice(1 << 32, 64, replace=False).astype(np.uint32)
    ip, d, w = _rows(rng, 200, dims, 20)
    w *= np.float32(1e3) ** rng.integers(-3, 4, w.size).astype(np.float32)   # magnitudes that make the summation order matter
    diff_order = 0
    for _ in range(400):
        a, b = rng.integers(0, 200, 2)
        ra, rb = _row((ip, d, w), a), _row((ip, d, w), b)
        x, y = ms.score(ra, rb), ms.score(rb, ra)
        assert np.float32(x).view(np.uint32) == np.float32(y).view(np.uint32)
        assert np.float32(x).view(np.uint32) == py_score(ra, rb).view(np.uint32)
        diff_order += py_score(ra, rb, descending=True).view(np.uint32) != np.float32(x).view(np.uint32)
    assert diff_order > 0


def test_summation_order_is_observable():
    """the products 1, 1e8, -1e8 sum to 0 in ascending dim order and to 1 in descending order: the pair's bits and the list differ"""
    q = (np.array([1, 5, 9], np.uint32), np.array([1.0, 1.0, 5.0], np.float32))
    pts = [([1, 2, 3, 9], [1.0, 1e4, 1e4, 1.0]),   # A: rel 6, picked first
           ([3, 1, 2], [-1e4, 1.0, 1e4]),          # c: rel 1, pair(c, A) = 1 + 1e8 - 1e8 (given out of order)
           ([5], [0.8])]                           # d: rel 0.8, pair(d, A) = +0.0
    ip = np.concatenate([[0], np.cumsum([len(p[0]) for p in pts])]).astype(np.uint64)
    csr = (ip, np.concatenate([p[0] for p in pts]).astype(np.uint32), np.concatenate([p[1] for p in pts]).astype(np.float32))
    assert ms.score(_row(csr, 1), _row(csr, 0)) == 0.0 and py_score(_row(csr, 1), _row(csr, 0), descending=True) == 1.0
    cand = np.zeros(3, ms.SCORED)
    cand["idx"] = [0, 1, 2]
    got = ms.mmr(csr, q, 0.5, cand, 2)[0]["idx"].tolist()
    assert got == [0, 1] == py_mmr(csr, q, 0.5, cand, 2)[0]
    assert py_mmr(csr, q, 0.5, cand, 2, descending=True)[0] == [0, 2]


def test_counters_by_hand():
    """lengths 1, 2, 3, 4 and a query of 2: relevance 1 + 2 + 2 + 2 = 7; pick 3 (rel 2) leaves [0, 1, 2]: 1 + 2 + 3 = 6; pick 1 (mmr
    0.5, the last of two maxima) leaves [0, 2]: min(1, 2) + min(3, 2) = 3; pick 0.  cpu 16, vector_io_read 0"""
    pts = [([0], [1.0]), ([0, 1], [1.0, 1.0]), ([1, 2, 3], [1.0, 1.0, 1.0]), ([4, 5, 6, 7], [1.0, 1.0, 1.0, 1.0])]
    ip = np.concatenate([[0], np.cumsum([len(p[0]) for p in pts])]).astype(np.uint64)
    csr = (ip, np.concatenate([p[0] for p in pts]).astype(np.uint32), np.concatenate([p[1] for p in pts]).astype(np.float32))
    cand = np.zeros(4, ms.SCORED)
    cand["idx"] = [0, 1, 2, 3]
    got, cpu, io = ms.mmr(csr, (np.array([0, 4], np.uint32), np.array([1.0, 2.0], np.float32)), 0.5, cand, 3)
    assert got["idx"].tolist() == [3, 1, 0] and (cpu, io) == (16, 0)


def test_short_lists_are_returned_as_they_are():
    csr = (np.array([0, 1, 2], np.uint64), np.array([0, 0], np.uint32), np.array([1.0, 2.0], np.float32))
    cand = np.zeros(3, ms.SCORED)
    cand["idx"] = [1, 1, 1]
    cand["score"] = [0.5, 0.7, 0.9]
    got, cpu, io = ms.mmr(csr, (np.array([0], np.uint32), np.array([1.0], np.float32)), 0.5, cand, 1)
    assert got.tolist() == [(1, np.float32(0.5))] and (cpu, io) == (0, 0)
    got, cpu, _ = ms.mmr(csr, (np.array([0], np.uint32), np.array([1.0], np.float32)), 0.5, cand[:0], 3)
    assert got.size == 0 and cpu == 0
