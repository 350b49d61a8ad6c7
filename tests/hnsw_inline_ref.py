"""CPU restatement of GraphLayers::search_with_vectors (lib/segment/src/index/hnsw_index/graph_layers.rs:336-452, 564-596) over the
reader of tests/graph_links_with_vectors.py, for tests (never imported by the product).

    search_entry_with_vectors            the entry point scored by the quantized storage, then per level a greedy move to a
                                         strictly better link (links filtered, truncated to m, scored from their inline vectors)
    search_on_level_with_vectors         level 0 with two SearchContexts: `links` (the beam, on link scores) and `base` (exact
                                         scores of every popped candidate, including the one whose pop ends the loop)
    SearchContext / FixedLengthPriorityQueue   search_context.rs:8-41, fixed_length_priority_queue.rs

keyed=True orders every level-0 comparison (both heaps, the lower bound, the candidate test) by (score desc, id asc), the tie
contract the device search keeps; keyed=False compares scores only, like the reference (heap order among equal scores is the
first-come order here).  Scores come from the callers: link_score(bytes) for an inline SQ8 link vector, base_score(bytes) for an
inline f32 base vector, entry_score(id) for the entry point's storage row.
"""
from __future__ import annotations

import ctypes as C
import heapq

import numpy as np


class _Ctx:
    """SearchContext over FixedLengthPriorityQueue(ef): nearest keeps the ef best; candidates = every point that entered nearest."""

    def __init__(self, ef: int, keyed: bool):
        self.ef, self.keyed = ef, keyed
        self.nearest = []       # min-heap of (key, seq, id, score)
        self.candidates = []    # max-heap as negated keys
        self.seq = 0

    def key(self, idx: int, score: float):
        return (score, -idx) if self.keyed else (score,)

    def lower_bound(self):
        return self.nearest[0][0] if len(self.nearest) == self.ef else None

    def process(self, idx: int, score: float):
        k = self.key(idx, score)
        self.seq += 1
        entry = (k, self.seq, idx, score)
        if len(self.nearest) < self.ef:
            heapq.heappush(self.nearest, entry)
        elif self.nearest[0][0] < k:
            heapq.heapreplace(self.nearest, entry)
        else:
            return False
        heapq.heappush(self.candidates, (tuple(-x for x in k), self.seq, idx, score))
        return True

    def pop(self):
        if not self.candidates:
            return None
        nk, _, idx, score = heapq.heappop(self.candidates)
        return idx, score, tuple(-x for x in nk)

    def sorted(self):
        return [(i, s) for k, _, i, s in sorted(self.nearest, key=lambda e: (e[0], -e[1]), reverse=True)]


def search_with_vectors(view, entry_score, link_score, base_score, top: int, ef: int, entry: int, entry_level: int, filtered=None, keyed: bool = True):
    """-> (result [(id, score)], stats: hops, link_scored, base_scored, break_id / break_evicted (the pop that ended the search
    below the lower bound, and whether it had left `nearest`), expanded (level-0 candidates in pop order), hop_ids (the ids each
    level-0 hop scored), links_nearest (the links context's final list))"""
    ok = (lambda i: True) if filtered is None else (lambda i: not filtered[i])
    st = {"hops": 1, "link_scored": 1, "base_scored": 0, "break_id": None, "break_evicted": False, "expanded": [], "hop_ids": []}
    cur, cur_s = entry, np.float32(entry_score(entry))
    for level in range(entry_level, 0, -1):
        changed = True
        while changed:
            changed = False
            _, links, vecs = view.links_with_vectors(cur, level)
            pts = [(l, v) for l, v in zip(links, vecs) if ok(l)][: view.m]
            if pts:
                st["hops"] += 1
                st["link_scored"] += len(pts)
            for l, v in pts:
                s = np.float32(link_score(v))
                if s > cur_s:
                    changed, cur, cur_s = True, l, s
    ef = max(top, ef)
    links_ctx, base_ctx = _Ctx(ef, keyed), _Ctx(ef, keyed)
    visited = {cur}
    links_ctx.process(cur, float(cur_s))
    in_nearest = lambda i: any(e[2] == i for e in links_ctx.nearest)
    while True:
        c = links_ctx.pop()
        if c is None:
            break
        idx, score, k = c
        lb = links_ctx.lower_bound()
        if lb is not None and (k < lb if keyed else score < lb[0]):
            base, _, _ = view.links_with_vectors(idx, 0)
            base_ctx.process(idx, float(base_score(base)))
            st["base_scored"] += 1
            st["break_id"], st["break_evicted"] = idx, not in_nearest(idx)
            break
        base, links, vecs = view.links_with_vectors(idx, 0)
        pts = [(l, v) for l, v in zip(links, vecs) if l not in visited]
        base_ctx.process(idx, float(base_score(base)))
        st["base_scored"] += 1
        st["expanded"].append(idx)
        pts = [(l, v) for l, v in pts if ok(l)][: view.m0]
        if pts:
            st["hops"] += 1
            st["link_scored"] += len(pts)
            st["hop_ids"].append([l for l, _ in pts])
        for l, v in pts:
            links_ctx.process(l, float(np.float32(link_score(v))))
            visited.add(l)
    st["links_nearest"] = links_ctx.sorted()
    return base_ctx.sorted()[:top], st


# ------------------------------------------------------------------------------------------------ scorers from the oracle
def sq8_bytes_scorer(oracle, sq, q_pre):
    """EncodedVectorsU8::score_bytes of an inline link vector (the oracle's SQ8 score of those bytes) for one query"""
    code, off = sq.encode_query(q_pre)
    code = np.ascontiguousarray(code)
    lib = oracle.lib()
    cache = {}

    def score(v: bytes) -> np.float32:
        s = cache.get(v)
        if s is None:
            row = np.frombuffer(v, np.uint8).copy()
            s = cache[v] = np.float32(lib.qo_sq8_score(C.byref(sq.meta), code.ctypes.data_as(C.POINTER(C.c_uint8)), C.c_float(float(off)),
                                                       row.ctypes.data_as(C.POINTER(C.c_uint8))))
        return s

    return score


def f32_bytes_scorer(oracle, distance: int, q_pre):
    """MetricQueryScorer::score_bytes of an inline f32 base vector for one (preprocessed) query"""
    cache = {}

    def score(v: bytes) -> np.float32:
        s = cache.get(v)
        if s is None:
            row = np.frombuffer(v, np.float32)[None, :]
            s = cache[v] = np.float32(oracle.score_points_f32(distance, row, q_pre, [0])[0])
        return s

    return score


def run(oracle, view, sq, distance: int, queries, top: int, ef: int, entry: int, entry_level: int, filtered=None, keyed: bool = True):
    """the checker over a batch of raw queries: (lists as [(id, score)], summed stats, per-query stats)"""
    out, per = [], []
    tot = {"hops": 0, "link_scored": 0, "base_scored": 0}
    for q in np.atleast_2d(queries):
        q_pre = oracle.preprocess_f32(distance, q)
        ls = sq8_bytes_scorer(oracle, sq, q_pre)
        code, off = sq.encode_query(q_pre)
        res, st = search_with_vectors(view, lambda i: sq.score(code, off, i), ls, f32_bytes_scorer(oracle, distance, q_pre), top, ef, entry, entry_level,
                                      filtered, keyed)
        out.append(res)
        per.append(st)
        for k in tot:
            tot[k] += st[k]
    return out, tot, per
