"""CPU checks of the ACORN-1 reference traversal (tests/hnsw_acorn_ref.c), the checker of the device's ACORN variant.

The reference has no test of search_on_level_acorn, so parity rests on restating graph_layers.rs:154-243 twice, independently:
(a) a pure-Python restatement below, over its own parse of the plain links.bin, equals the C traversal — lists, scorer calls and
    scored points — on built graphs (m0 = 8 / 32 / 64, filters of selectivity 0.02-0.5) and on random graphs with lists wider
    than m0 and repeated ids, which reach the 1-hop break, a 2-hop break in the middle of a list, and a point explored as a
    2-hop neighbour that is met again later as a 1-hop link;
(b) unfiltered ACORN equals HNSW, and the C traversal's HNSW equals the oracle's own (oracle/hnsw.c), filtered or not;
(c) on clustered data under a 2 % filter, ACORN's recall@10 against the exact filtered scan is clearly above HNSW's."""
import heapq

import numpy as np
import pytest

from tests import graph_links_compressed as gl
from tests import hnsw_acorn_ref as ar
from tests.util import assert_topk_equal, pack_bitmap


# ------------------------------------------------------------------------------------------------ Python restatement
class PyGraph:
    """links.bin (GraphLinksFormat::Plain, header.rs:9-20) parsed field by field; links(p, level) = GraphLinks::links"""

    def __init__(self, blob, m, m0):
        b = bytes(np.ascontiguousarray(blob, dtype=np.uint8))
        n, levels, n_nb, n_off, pad = np.frombuffer(b, np.uint64, 5, 0).astype(np.int64)
        p = 64
        self.level_offsets = np.frombuffer(b, np.uint64, levels, p).astype(np.int64); p += 8 * levels
        self.reindex = np.frombuffer(b, np.uint32, n, p).astype(np.int64); p += 4 * n
        self.neighbors = np.frombuffer(b, np.uint32, n_nb, p); p += 4 * n_nb + pad
        self.offsets = np.frombuffer(b, np.uint64, n_off, p).astype(np.int64)
        self.n, self.m, self.m0 = int(n), m, m0

    def links(self, point, level):
        idx = point if level == 0 else self.level_offsets[level] + self.reindex[point]
        return [int(x) for x in self.neighbors[self.offsets[idx]:self.offsets[idx + 1]]]


class PySearch:
    def __init__(self, g, score_fn, filtered):
        self.g, self.score_fn, self.filtered = g, score_fn, filtered
        self.calls = self.scored = 0
        self.events = {"hop1_break": 0, "hop2_break_mid_list": 0, "hop2_then_hop1": 0}

    def ok(self, p):                                  # ScorerFilters::check_vector
        return self.filtered is None or not self.filtered[p]

    def score(self, ids):
        if not ids:
            return []
        self.calls += 1
        self.scored += len(ids)
        return [np.float32(s) for s in self.score_fn(np.asarray(ids, np.uint32))]

    def entry(self, entry, top_level):                # search_entry / search_entry_on_level, graph_layers.rs:247-316
        cur = None
        for level in range(top_level, 0, -1):
            limit = self.g.m
            best, best_s = entry, self.score([entry])[0]
            changed = True
            while changed:
                changed = False
                ids = [l for l in self.g.links(best, level) if self.ok(l)][:limit]
                for i, s in zip(ids, self.score(ids)):
                    if s > best_s:
                        best, best_s, changed = i, s, True
            entry, cur = best, (best, best_s)
        return cur if cur is not None else (entry, self.score([entry])[0])

    def acorn(self, level_entry, ef):                 # search_on_level_acorn, graph_layers.rs:154-243
        hop1, hop2 = {level_entry[0]}, set()
        nearest, candidates = [], []                  # FixedLengthPriorityQueue (min-heap on score), BinaryHeap (max)

        def process(idx, s):                          # SearchContext::process_candidate
            if len(nearest) < ef:
                heapq.heappush(nearest, (s, idx))
            elif nearest[0][0] < s:
                heapq.heapreplace(nearest, (s, idx))
            else:
                return
            heapq.heappush(candidates, (-s, idx))

        process(level_entry[0], level_entry[1])
        limit = self.g.m0
        while candidates:
            neg, cand = heapq.heappop(candidates)
            if -neg < nearest[0][0]:                  # candidate.score < lower_bound()
                break
            to_score, to_explore = [], []
            links = self.g.links(cand, 0)
            for k, l in enumerate(links):
                if l in hop1:
                    continue
                hop1.add(l)
                if self.ok(l):
                    to_score.append(l)
                    if len(to_score) >= limit:
                        self.events["hop1_break"] += k + 1 < len(links)
                        break
                else:
                    if l in hop2:
                        self.events["hop2_then_hop1"] += 1
                    to_explore.append(l)
            for h in to_explore:
                total = len(to_score) + limit
                links2 = self.g.links(h, 0)
                for k, l in enumerate(links2):
                    if l in hop1:
                        continue
                    if l in hop2:
                        continue
                    hop2.add(l)
                    if self.ok(l):
                        hop1.add(l)
                        to_score.append(l)
                        if len(to_score) >= total:
                            self.events["hop2_break_mid_list"] += k + 1 < len(links2)
                            break
            for i, s in zip(to_score, self.score(to_score)):
                process(i, s)
        return sorted(nearest, key=lambda t: (-t[0], t[1]))

    def search(self, entry, entry_level, top, ef):
        e = self.entry(entry, entry_level)
        res = self.acorn(e, max(ef, top))[:top]
        out = np.zeros(len(res), dtype=ar.SCORED)
        out["idx"] = [i for _, i in res]
        out["score"] = [s for s, _ in res]
        return out


# ------------------------------------------------------------------------------------------------ helpers
def _built(oracle, n, dim, m, seed, dist=None, clusters=0):
    rng = np.random.default_rng(seed)
    dist = oracle.COSINE if dist is None else dist
    if clusters:
        centres = rng.standard_normal((clusters, dim)).astype(np.float32) * 3
        label = rng.integers(0, clusters, n)
        base = (centres[label] + rng.standard_normal((n, dim))).astype(np.float32)
    else:
        label = None
        base = rng.standard_normal((n, dim)).astype(np.float32)
    base = oracle.preprocess_rows_f32(dist, base) if dist == oracle.COSINE else base
    g = oracle.HNSW(base, dist, m=m, ef_construct=64, seed=seed, threads=1)
    return g, base, label, rng


def _queries(oracle, rng, nq, dim, dist):
    q = rng.standard_normal((nq, dim)).astype(np.float32)
    return np.stack([oracle.preprocess_f32(dist, x) for x in q])


def _py_vs_c(oracle, blob, m, m0, base, dist, qp, entry, lvl, filtered, top, ef):
    pyg = PyGraph(blob, m, m0)
    cg = ar.Graph(blob, m, m0, base.shape[0])
    want = cg.search_batch(oracle, base, dist, qp, top, ef, entry, lvl, ar.ACORN, filtered)
    calls, scored = cg.stats()[:2]
    events = {}
    pc = ps = 0
    for q, w in zip(qp, want):
        s = PySearch(pyg, lambda ids, q=q: oracle.score_points_f32(dist, base, q, ids), filtered)
        got = s.search(entry, lvl, top, ef)
        assert_topk_equal(got, w, what="python restatement vs C")
        assert np.array_equal(got["idx"], w["idx"])
        pc += s.calls; ps += s.scored
        for k, v in s.events.items():
            events[k] = events.get(k, 0) + v
    assert (pc, ps) == (calls, scored)
    cg.close()
    return events


# ------------------------------------------------------------------------------------------------ (a)
@pytest.mark.parametrize("m", [4, 16, 32])
@pytest.mark.parametrize("sel", [0.02, 0.1, 0.5])
def test_python_restatement_equals_c_on_built_graphs(oracle, m, sel):
    n, dim = 1500, 16
    g, base, _, rng = _built(oracle, n, dim, m, seed=m)
    entry, lvl, gm, gm0 = g.entry()
    qp = _queries(oracle, rng, 6, dim, oracle.COSINE)
    filtered = rng.random(n) >= sel
    filtered[entry] = False
    for top, ef in ((10, 32), (5, 100)):
        _py_vs_c(oracle, g.export_plain(), gm, gm0, base, oracle.COSINE, qp, entry, lvl, filtered, top, ef)
    g.close()


@pytest.mark.parametrize("m0,sel", [(8, 0.7), (8, 0.9), (16, 0.5), (32, 0.05)])
def test_python_restatement_equals_c_on_wide_lists(oracle, m0, sel):
    """random graphs whose lists hold up to 2 x m0 links with repeats: the breaks cut lists short"""
    n, dim = 1200, 8
    rng = np.random.default_rng(m0 * 7 + int(sel * 100))
    m = m0 // 2
    edges = gl.random_links(rng, n, 3, m, m0)
    edges = [[links if lvl == 0 else [x for x in links if len(edges[x]) > lvl] for lvl, links in enumerate(e)] for e in edges]   # upper links stay on their level
    lo, reindex, nb, off = gl.edges_to_plain_arrays(edges)
    blob = np.frombuffer(gl.serialize_plain(n, lo, reindex, nb, off), np.uint8)
    top_level = max(len(e) for e in edges) - 1
    entry = next(p for p, e in enumerate(edges) if len(e) - 1 == top_level)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    qp = rng.standard_normal((8, dim)).astype(np.float32)
    filtered = rng.random(n) >= sel
    filtered[entry] = False
    events = _py_vs_c(oracle, blob, m, m0, base, oracle.DOT, qp, entry, top_level, filtered, 10, 64)
    assert events["hop2_then_hop1"] > 0, events
    if sel >= 0.5:
        assert events["hop1_break"] > 0 and events["hop2_break_mid_list"] > 0, events


# ------------------------------------------------------------------------------------------------ (b)
@pytest.mark.parametrize("m", [4, 16, 32])
def test_unfiltered_acorn_equals_hnsw_and_oracle(oracle, m):
    n, dim = 3000, 24
    g, base, _, rng = _built(oracle, n, dim, m, seed=100 + m, dist=oracle.EUCLID)
    entry, lvl, gm, gm0 = g.entry()
    qp = _queries(oracle, rng, 40, dim, oracle.EUCLID)
    cg = ar.Graph(g.export_plain(), gm, gm0, n)
    for top, ef in ((10, 64), (30, 16)):
        g.stats(reset=True)
        want = g.search_batch(qp, top, ef, threads=2)
        want_stats = g.stats(reset=True)
        h = cg.search_batch(oracle, base, oracle.EUCLID, qp, top, ef, entry, lvl, ar.HNSW, threads=2)
        h_stats = cg.stats()
        a = cg.search_batch(oracle, base, oracle.EUCLID, qp, top, ef, entry, lvl, ar.ACORN, threads=2)
        a_stats = cg.stats()
        assert h_stats[:2] == want_stats and a_stats[:2] == want_stats
        assert a_stats[2] == h_stats[2] and a_stats[3] == 0          # the same hop1 marks, no 2-hop exploration
        for x, y, z in zip(want, h, a):
            assert np.array_equal(x, y) and np.array_equal(x, z)
    cg.close(); g.close()


def test_filtered_hnsw_equals_oracle(oracle):
    """the C traversal's search_entry and HNSW level 0 under a filter are the oracle's (so its ACORN starts from the same entry)"""
    n, dim = 4000, 32
    g, base, _, rng = _built(oracle, n, dim, 16, seed=5)
    entry, lvl, gm, gm0 = g.entry()
    qp = _queries(oracle, rng, 40, dim, oracle.COSINE)
    filtered = rng.random(n) >= 0.2
    filtered[entry] = False
    cg = ar.Graph(g.export_plain(), gm, gm0, n)
    g.stats(reset=True)
    want = g.search_batch(qp, 10, 64, deleted=pack_bitmap(filtered), threads=2)
    got = cg.search_batch(oracle, base, oracle.COSINE, qp, 10, 64, entry, lvl, ar.HNSW, filtered, threads=2)
    assert cg.stats()[:2] == g.stats(reset=True)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    # the callback path (used for quantized scorers) takes the filter too and gives the same lists
    for q, w in zip(qp[:5], got[:5]):
        r = cg.search(lambda ids, q=q: oracle.score_points_f32(oracle.COSINE, base, q, ids), 10, 64, entry, lvl, ar.HNSW, pack_bitmap(filtered))
        assert np.array_equal(r, w)
    cg.close(); g.close()


# ------------------------------------------------------------------------------------------------ (c)
def test_acorn_recall_above_hnsw_under_restrictive_filter(oracle):
    n, dim, k = 20_000, 32, 10
    g, base, label, rng = _built(oracle, n, dim, 16, seed=21, clusters=50)
    entry, lvl, gm, gm0 = g.entry()
    qp = _queries(oracle, rng, 200, dim, oracle.COSINE)
    filtered = rng.random(n) >= 0.02
    filtered[entry] = False
    exact = oracle.scan_f32(oracle.COSINE, base, qp, k, deleted=pack_bitmap(filtered))
    cg = ar.Graph(g.export_plain(), gm, gm0, n)
    recall = {}
    for name, algo in (("hnsw", ar.HNSW), ("acorn", ar.ACORN)):
        got = cg.search_batch(oracle, base, oracle.COSINE, qp, k, 64, entry, lvl, algo, filtered, threads=4)
        recall[name] = np.mean([len(set(a["idx"].tolist()) & set(e["idx"].tolist())) / max(len(e), 1) for a, e in zip(got, exact)])
    print(f"recall@10, 2 % random filter, 20k x 32 clustered cosine, m 16, ef 64: {recall}")
    assert recall["acorn"] >= recall["hnsw"] + 0.2, recall
    cg.close(); g.close()
