"""CPU checks of the sparse-vector checker (tests/sparse_ref.c), which the device index is compared with bit for bit: it reproduces the
reference's own SearchContext cases, agrees with a brute-force top-k, and exercises the parts of the state machine that make the
emulation necessary (pruning's swap changes score bits, the last of the longest lists is promoted)."""
import json
import os
import sys

import numpy as np

sys.dont_write_bytecode = True
from tests import sparse_ref as sr  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sparse_reference_cases.json")


def _index(points: dict, n_dims: int) -> sr.Index:
    n = max((int(k) for k in points), default=-1) + 1
    indptr = np.zeros(n + 1, np.uint64)
    dims, w = [], []
    for r in range(n):
        row = points.get(str(r), [])
        dims += [d for d, _ in row]
        w += [x for _, x in row]
        indptr[r + 1] = len(dims)
    return sr.Index(indptr, np.array(dims, np.uint32), np.array(w, np.float32), n_dims)


def test_reference_cases():
    doc = json.load(open(GOLDEN))
    prev_cpu = None
    for case in doc["cases"]:
        for reliable in (True, False):   # the RAM index and the compressed f32 indexes run every case of the reference's test module
            if case.get("reliable_only") and not reliable:
                continue
            idx = _index(case["points"], doc["n_dims"])
            qd, qw = case["query"]
            ctx = idx.context(*sr.remap(qd, qw, doc["n_dims"]), case["top"], reliable)
            if case["op"] == "search":
                got, cpu = ctx.search()
                assert [[int(i), float(s)] for i, s in got] == case["expected"], case["test"]
                if case["expected"]:
                    assert cpu > 0
                if case.get("same_cpu_as_previous"):
                    assert cpu == prev_cpu
                prev_cpu = cpu
            elif case["op"] == "plain":
                got, cpu = ctx.plain(np.array(case["ids"], np.uint32))
                assert [[int(i), float(s)] for i, s in got] == case["expected"], case["test"]
                assert cpu > 0
            elif case["op"] == "prune":
                for min_score, pruned in case["prune"]:
                    assert ctx.prune(min_score) == pruned, case["test"]
                assert ctx.list_len(0) == case["list0_len_after"]
            elif case["op"] == "promote":
                assert ctx.list_len(0) == case["list0_len_before"]
                ctx.promote()
                assert ctx.list_len(0) == case["list0_len_after"]
            ctx.close()
            idx.close()


def _brute(indptr, dims, w, qd, qw, top, deleted=None):
    """f64 scores of every point sharing a dim with the query; the points with a non-zero score, best first"""
    q = dict(zip(qd.tolist(), qw.tolist()))
    out = []
    for r in range(indptr.size - 1):
        if deleted is not None and deleted[r]:
            continue
        s, hit = 0.0, False
        for d, x in zip(dims[indptr[r]: indptr[r + 1]].tolist(), w[indptr[r]: indptr[r + 1]].tolist()):
            if d in q:
                s += float(x) * q[d]
                hit = True
        if hit and s != 0.0:
            out.append((s, r))
    out.sort(key=lambda t: (-t[0], t[1]))
    return out


def test_matches_brute_force_where_scores_are_distinct():
    rng = np.random.default_rng(1)
    n_dims = 300
    indptr, dims, w = sr.random_csr(rng, 30_000, n_dims, 12, id_gap=1)
    idx = sr.Index(indptr, dims, w, n_dims)
    checked = 0
    for t in range(12):
        qd = rng.choice(n_dims, size=int(rng.integers(1, 12)), replace=False).astype(np.uint32)
        qw = (rng.random(qd.size) + 0.05).astype(np.float32)
        if t % 3 == 2:
            qw[0] = -qw[0]                     # pruning off
        deleted = rng.random(indptr.size - 1) < 0.3 if t % 2 else None
        top = int(rng.choice([1, 10, 50]))
        want = _brute(indptr, dims, w, qd, qw, top, deleted)
        if len(want) > top and want[top - 1][0] - want[top][0] < 1e-4 * abs(want[top][0]):
            continue                           # a near-tie at the boundary: rounding may order it either way
        for reliable in (True, False):
            got, _ = idx.search(qd, qw, top, reliable, None if deleted is None else sr.deleted_bitmap(deleted))
            assert got["idx"].tolist() == [r for _, r in want[:top]]
            np.testing.assert_allclose(got["score"], [s for s, _ in want[:top]], rtol=1e-5)
        checked += 1
    assert checked >= 8
    idx.close()


def test_pruning_swap_changes_score_bits():
    """Points 0 and 1 fill TopK(1) in the first batch (threshold 0.5); dim 3 then has the longest list and is swapped to the front, so
    point 20000 of the second batch sums its three products in the order dim 3, 2, 1: (2^-24 + 2^-24) + 1 = 1 + 2^-23.  Without pruning
    it sums them in query order: (1 + 2^-24) + 2^-24 = 1."""
    tiny = float(np.float32(2.0 ** -24))
    rows = {0: [(1, 0.5)], 1: [(1, 0.5)], 20000: [(1, 1.0), (2, tiny), (3, tiny)]}
    rows.update({10001 + i: [(3, 0.1)] for i in range(5)})
    n = 20001
    indptr = np.zeros(n + 1, np.uint64)
    dims, w = [], []
    for r in range(n):
        for d, x in rows.get(r, []):
            dims.append(d)
            w.append(x)
        indptr[r + 1] = len(dims)
    idx = sr.Index(indptr, np.array(dims, np.uint32), np.array(w, np.float32), 4)
    q = (np.array([1, 2, 3], np.uint32), np.ones(3, np.float32))
    pruned, _ = idx.search(*q, 1, reliable=True)
    plain, _ = idx.search(*q, 1, reliable=False)
    assert pruned["idx"].tolist() == plain["idx"].tolist() == [20000]
    assert pruned["score"].view(np.uint32)[0] == np.float32(1.0 + 2.0 ** -23).view(np.uint32)
    assert plain["score"].view(np.uint32)[0] == np.float32(1.0).view(np.uint32)
    idx.close()


def test_last_longest_list_is_promoted():
    """dims 2 and 3 both have the longest list; max_by keeps the last, so dim 3's list is swapped to the front"""
    rows = [[(1, 1.0), (2, 1.0), (3, 1.0)], [(2, 1.0), (3, 1.0)], [(2, 1.0), (3, 1.0)]]
    indptr = np.array([0, 3, 5, 7], np.uint64)
    dims = np.array([d for r in rows for d, _ in r], np.uint32)
    w = np.array([x for r in rows for _, x in r], np.float32)
    idx = sr.Index(indptr, dims, w, 4)
    ctx = idx.context(np.array([1, 2, 3], np.uint32), np.ones(3, np.float32), 3)
    assert [ctx.list_dim(i) for i in range(3)] == [1, 2, 3]
    ctx.promote()
    assert [ctx.list_dim(i) for i in range(3)] == [3, 2, 1]
    assert ctx.list_len(0) == 3
    ctx.close()
    idx.close()


def test_tie_members_differ_but_scores_do_not():
    """Integer weights make many equal scores: keeping the larger ids among ties (another order the reference allows) returns the same
    score bits, and some lists keep other ids"""
    rng = np.random.default_rng(4)
    indptr, dims, w = sr.random_csr(rng, 5000, 40, 6)
    w = np.ceil(w * 3).astype(np.float32)
    idx = sr.Index(indptr, dims, w, 40)
    differ = 0
    for _ in range(10):
        qd = rng.choice(40, size=5, replace=False).astype(np.uint32)
        qw = np.ones(5, np.float32)
        a, _ = idx.search(qd, qw, 10, keyed=True)
        b, _ = idx.search(qd, qw, 10, keyed=False)
        assert np.array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32))
        differ += a["idx"].tolist() != b["idx"].tolist()
    assert differ > 0
    idx.close()


def test_plain_search_pushes_zero_scores_and_counts():
    """plain_search pushes a zero score (search would not), skips an id with no shared dim, and counts query.len + 4 per shared dim"""
    indptr = np.array([0, 2, 3, 4], np.uint64)
    dims = np.array([1, 2, 1, 3], np.uint32)
    w = np.array([1.0, -1.0, 0.0, 5.0], np.float32)
    idx = sr.Index(indptr, dims, w, 4)
    got, cpu = idx.plain(np.array([2, 1], np.uint32), np.array([1.0, 1.0], np.float32), np.array([0, 1, 2], np.uint32), 10)
    assert [(int(i), float(s)) for i, s in got] == [(0, 0.0), (1, 0.0)]
    assert cpu == (2 + 2 * 4) + (2 + 1 * 4)
    searched, _ = idx.search(np.array([2, 1], np.uint32), np.array([1.0, 1.0], np.float32), 10)
    assert searched.size == 0
    idx.close()
