"""The CPU checker of qb_mmr_maxsim_batch (tests/mmr_maxsim_ref.c through tests/mmr_maxsim_ref.py): it reproduces the reference's own
multivector MMR case with the order worked out by hand, equals an independent Python restatement of maximal_marginal_relevance over the
oracle's MaxSim (full pair matrix, a Python list with swap-remove) on tie-heavy, NaN, +-0, duplicate-id and short-list inputs, meters the
counters the reference meters, and its pair order is observable: inputs exist where scoring pair(s, c) in place of pair(c, s) gives
another list."""
import json
import os

import numpy as np
import pytest

from tests import mmr_maxsim_ref as mr

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mmr_multivector_reference_cases.json")
DISTANCES = {"Cosine": 0, "Euclid": 1, "Dot": 2, "Manhattan": 3}


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


def py_mmr(o, rows, off, distance, query, lam, cand, limit, swapped=False):
    """maximal_marginal_relevance over the full MaxSim matrix of the oracle, remaining candidates as a list with swap-remove.
    swapped: the negative control, pair(c, s) scored as MaxSim(preprocess(P_s), P_c)"""
    uniq, seen = [], set()
    for c in cand:
        if int(c["idx"]) not in seen:
            seen.add(int(c["idx"]))
            uniq.append(c)
    n = len(uniq)
    dim = rows.shape[1]
    if n < 2:
        return [int(c["idx"]) for c in uniq], 0
    pts = [rows[off[int(c["idx"])] : off[int(c["idx"]) + 1]] for c in uniq]
    pre = [np.stack([o.preprocess_f32(distance, t) for t in p]) for p in pts]
    qp = np.stack([o.preprocess_f32(distance, v) for v in np.atleast_2d(query)])
    rel = [o.maxsim_f32(distance, qp, p) for p in pts]
    if swapped:
        mat = [[o.maxsim_f32(distance, pre[s], pts[c]) for s in range(n)] for c in range(n)]
    else:
        mat = [[o.maxsim_f32(distance, pre[c], pts[s]) for s in range(n)] for c in range(n)]
    lam = np.float32(lam)
    remaining, selected = list(range(n)), []

    def pick(vals):
        p = _argmax(vals)
        selected.append(remaining[p])
        remaining[p] = remaining[-1]
        remaining.pop()

    pick([rel[c] for c in remaining])
    cpu = dim * 4 * len(qp) * sum(len(p) for p in pts)
    while len(selected) < limit and remaining:
        cpu += dim * 4 * len(pts[selected[-1]]) * sum(len(pts[c]) for c in remaining)
        scores = []
        for c in remaining:
            sims = [mat[c][s] for s in selected]
            ms = sims[_argmax(sims)]
            scores.append(lam * rel[c] - (np.float32(1.0) - lam) * ms)
        pick(scores)
    return [int(uniq[s]["idx"]) for s in selected], cpu


def _points(rng, n_points, dim, distance, oracle, kind, lens=(1, 5)):
    """token rows and offsets.  tie: few distinct small-integer tokens, identical points; nan: some NaN tokens; zero: +-0 tokens"""
    runs = rng.integers(lens[0], lens[1] + 1, n_points)
    off = np.concatenate([[0], np.cumsum(runs)]).astype(np.uint32)
    n_rows = int(off[-1])
    if kind == "tie":
        base = rng.integers(-1, 2, (3, dim)).astype(np.float32)
        rows = base[rng.integers(0, 3, n_rows)]
        # identical points: a few copy the first point's run (same length and tokens)
        for p in rng.integers(1, n_points, 3):
            if runs[p] == runs[0]:
                rows[off[p] : off[p + 1]] = rows[off[0] : off[1]]
    else:
        rows = rng.standard_normal((n_rows, dim)).astype(np.float32)
    if kind == "nan":
        rows[rng.integers(0, n_rows, 3)] = np.nan
    if kind == "zero":
        rows[rng.integers(0, n_rows, n_rows // 3)] = 0.0
        rows[rng.integers(0, n_rows, 3)] = -0.0
    if distance == oracle.COSINE and kind not in ("tie",):
        rows = oracle.preprocess_rows_f32(oracle.COSINE, rows)
    return np.ascontiguousarray(rows), off


def _cands(rng, n, n_points, dup_ids=0):
    ids = rng.choice(n_points, size=n, replace=n > n_points).astype(np.uint32)
    if dup_ids and n > 1:
        for _ in range(dup_ids):
            ids[rng.integers(1, n)] = ids[rng.integers(0, n)]
    c = np.zeros(n, mr.SCORED)
    c["idx"] = ids
    c["score"] = rng.standard_normal(n).astype(np.float32)
    if n:
        c["score"][rng.integers(0, n, max(n // 4, 1))] = -0.0
    return c


def test_reference_case(oracle):
    with open(FIXTURE) as f:
        fx = json.load(f)
    rows = np.array([v for p in fx["points"] for v in p["vectors"]], np.float32)
    off = np.concatenate([[0], np.cumsum([len(p["vectors"]) for p in fx["points"]])]).astype(np.uint32)
    ids = [p["id"] for p in fx["points"]]   # point offset i holds reference id ids[i]
    cand = np.zeros(len(ids), mr.SCORED)
    cand["idx"] = np.arange(len(ids))
    q = np.array(fx["query"], np.float32)
    for name, d in DISTANCES.items():
        got, _, io = mr.mmr(oracle, rows, off, d, q, fx["lambda"], cand, fx["limit"])
        assert got.size == 3 and io == 0
        assert [ids[i] for i in got["idx"]] == fx["expected"][name], name
        assert [ids[i] for i in py_mmr(oracle, rows, off, d, q, fx["lambda"], cand, fx["limit"])[0]] == fx["expected"][name]


@pytest.mark.parametrize("kind", ["plain", "tie", "nan", "zero"])
@pytest.mark.parametrize("dim", [5, 20, 40])
def test_checker_equals_python_restatement(oracle, kind, dim):
    rng = np.random.default_rng(dim * 11 + len(kind))
    for distance in DISTANCES.values():
        rows, off = _points(rng, 40, dim, distance, oracle, kind)
        for n, limit, lam in ((0, 3, 0.5), (1, 3, 0.5), (2, 1, 0.5), (2, 5, 0.0), (3, 3, 1.0), (3, 2, 0.5), (12, 4, 0.5), (12, 20, 0.3), (25, 25, 0.0),
                              (25, 6, 1.0)):
            cand = _cands(rng, n, 40, dup_ids=2 if n > 5 else 0)
            q = rng.standard_normal((int(rng.integers(1, 4)), dim)).astype(np.float32)
            if kind == "tie":
                q = rng.integers(-1, 2, q.shape).astype(np.float32)
            got, cpu, io = mr.mmr(oracle, rows, off, distance, q, lam, cand, limit)
            want, want_cpu = py_mmr(oracle, rows, off, distance, q, lam, cand, limit)
            assert got["idx"].tolist() == want, (distance, n, limit, lam)
            first = {}
            for c in cand:
                first.setdefault(int(c["idx"]), c["score"])
            assert np.array_equal(got["score"].view(np.uint32), np.array([first[i] for i in want], np.float32).view(np.uint32))
            assert (cpu, io) == (want_cpu, 0)


def test_short_lists_are_returned_as_they_are(oracle):
    rows = np.eye(4, dtype=np.float32)
    off = np.array([0, 2, 4], np.uint32)
    cand = np.zeros(3, mr.SCORED)
    cand["idx"] = [1, 1, 1]
    cand["score"] = [0.5, 0.7, 0.9]
    got, cpu, io = mr.mmr(oracle, rows, off, 2, np.ones((2, 4), np.float32), 0.5, cand, 1)
    assert got.tolist() == [(1, np.float32(0.5))] and (cpu, io) == (0, 0)
    got, cpu, _ = mr.mmr(oracle, rows, off, 2, np.ones((2, 4), np.float32), 0.5, cand[:0], 3)
    assert got.size == 0 and cpu == 0


def test_counters_formula(oracle):
    """cpu = dim * 4 * (T_q * sum_i T_i + sum over picks k = 1 .. L-1 of T_pick_k * (tokens of the candidates remaining after pick k))"""
    rng = np.random.default_rng(5)
    dim = 24
    rows, off = _points(rng, 200, dim, 2, oracle, "plain", lens=(1, 9))
    T = np.diff(off).astype(np.int64)
    for n, limit, tq in ((2, 1, 1), (2, 2, 3), (50, 1, 2), (50, 10, 5), (50, 50, 1), (50, 80, 4)):
        cand = _cands(rng, n, 200)
        cand["idx"] = rng.choice(200, size=n, replace=False)
        got, cpu, io = mr.mmr(oracle, rows, off, 2, rng.standard_normal((tq, dim)), 0.5, cand, limit)
        L = got.size
        assert L == min(n, limit)
        picks = [int(i) for i in got["idx"]]
        left = int(T[cand["idx"]].sum())
        want = tq * left
        for k in range(L - 1):
            left -= int(T[picks[k]])
            want += int(T[picks[k]]) * left
        assert cpu == dim * 4 * want and io == 0


def test_pair_order_is_observable(oracle):
    """MaxSim is not symmetric: on varied token counts, scoring pair(s, c) in place of pair(c, s) changes some lists"""
    rng = np.random.default_rng(17)
    diff = 0
    for trial in range(30):
        d = list(DISTANCES.values())[trial % 4]
        rows, off = _points(rng, 30, 6, d, oracle, "plain", lens=(1, 6))
        cand = _cands(rng, 15, 30)
        q = rng.standard_normal((3, 6)).astype(np.float32)
        got = mr.mmr(oracle, rows, off, d, q, 0.3, cand, 8)[0]["idx"].tolist()
        assert got == py_mmr(oracle, rows, off, d, q, 0.3, cand, 8)[0]
        diff += py_mmr(oracle, rows, off, d, q, 0.3, cand, 8, swapped=True)[0] != got
    assert diff > 0
