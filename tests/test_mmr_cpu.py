"""The CPU checker of qb_mmr_batch (tests/mmr_ref.c through tests/mmr_ref.py): it reproduces the reference's own MMR cases, equals a plain
numpy restatement of maximal_marginal_relevance (full similarity matrix, a Python list with swap-remove) on tie-heavy, NaN and duplicate-id
inputs, meters the counters the reference meters, and its tie rules are observable: inputs exist where "first maximum wins" or ties broken by
candidate index instead of current position give another list."""
import json
import os

import numpy as np
import pytest

from tests import mmr_ref as mr

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mmr_reference_cases.json")


def _key(x):
    """OrderedFloat: NaN above everything and equal to NaN; -0.0 == +0.0 (Python's float comparison)"""
    return (1, 0.0) if np.isnan(x) else (0, float(x))


def _argmax(vals, first_wins=False, order=None):
    """max_by_key: the last maximal element (or the first, for the negative control); order: tie rank per element (default: list position)"""
    best = 0
    for i in range(1, len(vals)):
        a, b = _key(vals[i]), _key(vals[best])
        if order is not None and a == b:
            if order[i] > order[best]:
                best = i
        elif (a > b) if first_wins else (a >= b):
            best = i
    return best


def np_mmr(o, rows, distance, query, lam, cand, limit, id_base=0, first_wins=False, index_ties=False):
    """maximal_marginal_relevance over the full matrix of the oracle's similarities, remaining candidates as a list with swap-remove"""
    uniq, seen = [], set()
    for c in cand:
        if int(c["idx"]) not in seen:
            seen.add(int(c["idx"]))
            uniq.append(c)
    n = len(uniq)
    dim = rows.shape[1]
    if n < 2:
        return [int(c["idx"]) for c in uniq], 0
    vecs = [rows[int(c["idx"]) - id_base] for c in uniq]
    qp = o.preprocess_f32(distance, query)
    rel = [o.similarity_f32(distance, qp, v) for v in vecs]
    pre = [o.preprocess_f32(distance, v) for v in vecs]
    mat = [[o.similarity_f32(distance, pre[c], vecs[s]) for s in range(n)] for c in range(n)]
    lam = np.float32(lam)
    remaining, selected = list(range(n)), []

    def pick(vals):
        p = _argmax(vals, first_wins, remaining if index_ties else None)
        selected.append(remaining[p])
        remaining[p] = remaining[-1]
        remaining.pop()

    pick([rel[c] for c in remaining])
    while len(selected) < limit and remaining:
        scores = []
        for c in remaining:
            sims = [mat[c][s] for s in selected]
            ms = sims[_argmax(sims, first_wins)]
            scores.append(lam * rel[c] - (np.float32(1.0) - lam) * ms)
        pick(scores)
    L = len(selected)
    cpu = dim * 4 * (n + sum(n - k for k in range(1, L)))
    return [int(uniq[s]["idx"]) for s in selected], cpu


def _cands(rng, n, count, id_base=0, dup_ids=0):
    ids = rng.choice(count, size=n, replace=n > count).astype(np.uint32) + id_base
    if dup_ids and n > 1:
        for _ in range(dup_ids):
            ids[rng.integers(1, n)] = ids[rng.integers(0, n)]
    c = np.zeros(n, mr.SCORED)
    c["idx"] = ids
    c["score"] = rng.standard_normal(n).astype(np.float32)
    return c


def _rows(rng, count, dim, distance, oracle, kind):
    """tie: few distinct rows, many exact duplicates; nan: some rows NaN; zero: zero rows (+-0 similarities); plain"""
    if kind == "tie":
        base = rng.integers(-1, 2, (4, dim)).astype(np.float32)
        rows = base[rng.integers(0, 4, count)]
    else:
        rows = rng.standard_normal((count, dim)).astype(np.float32)
    if kind == "nan":
        rows[rng.integers(0, count, 3)] = np.nan
    if kind == "zero":
        rows[rng.integers(0, count, count // 3)] = 0.0
        rows[rng.integers(0, count, 2)] = -0.0
    if distance == oracle.COSINE and kind != "tie":
        rows = oracle.preprocess_rows_f32(oracle.COSINE, rows)
    return np.ascontiguousarray(rows)


def test_reference_cases(oracle):
    with open(FIXTURE) as f:
        fx = json.load(f)
    rows = np.array([p["vector"] for p in fx["points"]], np.float32)   # row k holds id k + 1: the storage's id_base is 1
    cand = np.zeros(len(fx["points"]), mr.SCORED)
    cand["idx"] = [p["id"] for p in fx["points"]]
    for case in fx["cases"]:
        got, _, io = mr.mmr(oracle, rows, oracle.EUCLID, fx["query"], case["lambda"], cand, fx["limit"], id_base=1)
        assert got["idx"].tolist() == case["expected"], case
        assert io == 0
        assert np_mmr(oracle, rows, oracle.EUCLID, np.array(fx["query"], np.float32), case["lambda"], cand, fx["limit"], id_base=1)[0] == case["expected"]


@pytest.mark.parametrize("kind", ["plain", "tie", "nan", "zero"])
@pytest.mark.parametrize("dim", [5, 20, 40])
def test_checker_equals_numpy_restatement(oracle, kind, dim):
    rng = np.random.default_rng(dim * 7 + len(kind))
    for distance in (oracle.COSINE, oracle.EUCLID, oracle.DOT, oracle.MANHATTAN):
        rows = _rows(rng, 60, dim, distance, oracle, kind)
        for n, limit, lam in ((0, 3, 0.5), (1, 3, 0.5), (2, 1, 0.5), (2, 5, 0.0), (3, 3, 1.0), (17, 5, 0.5), (17, 40, 0.3), (40, 40, 0.0), (40, 7, 1.0)):
            cand = _cands(rng, n, 60, id_base=100, dup_ids=2 if n > 5 else 0)
            q = rng.standard_normal(dim).astype(np.float32)
            if kind == "tie":
                q = rng.integers(-1, 2, dim).astype(np.float32)
            got, cpu, io = mr.mmr(oracle, rows, distance, q, lam, cand, limit, id_base=100)
            want, want_cpu = np_mmr(oracle, rows, distance, q, lam, cand, limit, id_base=100)
            assert got["idx"].tolist() == want, (distance, n, limit, lam)
            # original scores, as their bit patterns: the first occurrence of each selected id
            first = {}
            for c in cand:
                first.setdefault(int(c["idx"]), c["score"])
            assert np.array_equal(got["score"].view(np.uint32), np.array([first[i] for i in want], np.float32).view(np.uint32))
            assert (cpu, io) == (want_cpu, 0)


def test_short_lists_are_returned_as_they_are(oracle):
    rows = np.eye(4, dtype=np.float32)
    cand = np.zeros(3, mr.SCORED)
    cand["idx"] = [2, 2, 2]
    cand["score"] = [0.5, 0.7, 0.9]
    got, cpu, io = mr.mmr(oracle, rows, oracle.DOT, np.ones(4, np.float32), 0.5, cand, 1)
    assert got.tolist() == [(2, np.float32(0.5))] and (cpu, io) == (0, 0)
    got, cpu, _ = mr.mmr(oracle, rows, oracle.DOT, np.ones(4, np.float32), 0.5, cand[:0], 3)
    assert got.size == 0 and cpu == 0


def test_counters_formula(oracle):
    rng = np.random.default_rng(3)
    rows = rng.standard_normal((300, 24)).astype(np.float32)
    for n, limit in ((2, 1), (2, 2), (50, 1), (50, 10), (50, 50), (50, 80)):
        cand = _cands(rng, n, 300)
        got, cpu, io = mr.mmr(oracle, rows, oracle.DOT, rng.standard_normal(24), 0.5, cand, limit)
        L = got.size
        assert L == min(n, limit)
        assert cpu == 24 * 4 * (n + sum(n - k for k in range(1, L))) and io == 0


def test_tie_rules_are_observable(oracle):
    """On tie-heavy data the reference's rules (last maximum, current positions) pick other lists than first-maximum or by-index ties"""
    rng = np.random.default_rng(11)
    diff_first = diff_index = 0
    for trial in range(40):
        rows = _rows(rng, 30, 8, oracle.DOT, oracle, "tie")
        cand = _cands(rng, 20, 30)
        q = rng.integers(-1, 2, 8).astype(np.float32)
        lam = [0.0, 0.5, 1.0][trial % 3]
        got = mr.mmr(oracle, rows, oracle.DOT, q, lam, cand, 10)[0]["idx"].tolist()
        want = np_mmr(oracle, rows, oracle.DOT, q, lam, cand, 10)[0]
        assert got == want
        diff_first += np_mmr(oracle, rows, oracle.DOT, q, lam, cand, 10, first_wins=True)[0] != want
        diff_index += np_mmr(oracle, rows, oracle.DOT, q, lam, cand, 10, index_ties=True)[0] != want
    assert diff_first > 0 and diff_index > 0, (diff_first, diff_index)
