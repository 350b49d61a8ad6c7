"""The CompressedWithVectors writer and reader (tests/graph_links_with_vectors.py), and the search_with_vectors checker
(tests/hnsw_inline_ref.py), on the CPU.

Re-types graph_links/tests.rs::test_save_load (1000 points, 10 levels, m = 8, lists up to 2 x level_m, vector layouts
(base align, link align) = (1, 16), (4, 1), (4, 16)) and test_graph_links_construction's literal graphs: links and vectors
round-trip byte for byte."""
import numpy as np
import pytest

from tests import graph_links_compressed as gl
from tests import graph_links_with_vectors as gv
from tests import hnsw_inline_ref as ref
from tests.test_graph_links_compressed import LITERAL_GRAPHS


def _vectors(rng, n, size):
    return [bytes(rng.integers(0, 256, size, dtype=np.uint8)) for _ in range(n)]


def _round_trip(edges, m, m0, base_layout, link_layout, seed=0):
    rng = np.random.default_rng(seed)
    ids = 1 + max([len(edges)] + [x for levels in edges for lst in levels for x in lst])   # literal graphs link ids >= point_count
    base, link = _vectors(rng, len(edges), base_layout[0]), _vectors(rng, ids, link_layout[0])
    blob = gv.serialize_with_vectors(edges, m, m0, base.__getitem__, link.__getitem__, base_layout, link_layout)
    r = gv.WithVectorsLinks(blob)
    assert (r.point_count, r.m, r.m0) == (len(edges), m, m0)
    assert r.records_at % max(base_layout[1], link_layout[1]) == 0
    for p, levels in enumerate(edges):
        assert r.point_level(p) == len(levels) - 1
        for lvl, raw in enumerate(levels):
            b, links, vecs, lv_at = r.record(p, lvl)
            assert links == gl.normalize_links(m0 if lvl == 0 else m, raw)
            assert b == (base[p] if lvl == 0 else b"")
            assert vecs == [link[x] for x in links]
            assert lv_at % link_layout[1] == 0
    return blob


@pytest.mark.parametrize("layouts", [((8, 1), (16, 16)), ((12, 4), (5, 1)), ((16, 4), (32, 16))])
def test_save_load(layouts):
    rng = np.random.default_rng(42)
    edges = gl.random_links(rng, 1000, 10, 8, 16)
    edges = [[sorted(set(lst)) if i % 3 else lst for i, lst in enumerate(levels)] for levels in edges]
    _round_trip(edges, 8, 16, *layouts)


@pytest.mark.parametrize("graph", range(len(LITERAL_GRAPHS)))
def test_literal_graphs(graph):
    for layouts in (((4, 4), (5, 1)), ((8, 4), (16, 16))):
        _round_trip(LITERAL_GRAPHS[graph], 8, 16, *layouts)


def test_varint():
    for v in (0, 1, 127, 128, 300, 2 ** 35, 2 ** 64 - 1):
        b = gv.write_varint(v)
        assert gv.decode_varint(b, 0, len(b)) == (v, len(b))
    assert gv.decode_varint(b"\x80\x80", 0, 2) is None


# ------------------------------------------------------------------------------------------------ the checker
class _View:
    """a small in-memory graph with inline vectors: links[point][level], base / link scores as ids' own values"""

    def __init__(self, links, m, m0):
        self.l, self.m, self.m0 = links, m, m0

    def links_with_vectors(self, p, level):
        return bytes([p]), self.l[p][level], [bytes([x]) for x in self.l[p][level]]


def _scores(view, link_s, base_s, top, ef, keyed=True, filtered=None):
    return ref.search_with_vectors(view, lambda i: link_s[i], lambda v: link_s[v[0]], lambda v: base_s[v[0]], top, ef, 0, 0, filtered, keyed)


def _independent(view, link_s, base_s, top, ef, filtered=None):
    """a second restatement with sorted lists instead of heaps (tie-free input)"""
    ef = max(top, ef)
    nearest, cands, expanded, visited = [(link_s[0], 0)], [(link_s[0], 0)], set(), {0}
    base, hops, scored = [], 1, 1
    while cands:
        cands.sort()
        s, c = cands.pop()
        if len(nearest) == ef and s < min(nearest)[0]:
            base.append((base_s[c], c))
            break
        pts = [x for x in view.l[c][0] if x not in visited]
        base.append((base_s[c], c))
        pts = [x for x in pts if filtered is None or not filtered[x]][: view.m0]
        if pts:
            hops += 1; scored += len(pts)
        for x in pts:
            k = (link_s[x], x)
            if len(nearest) < ef:
                nearest.append(k); cands.append(k)
            elif k > min(nearest):
                nearest.remove(min(nearest)); nearest.append(k); cands.append(k)
            visited.add(x)
    return [(i, s) for s, i in sorted(base, reverse=True)[:top]], hops, scored, len(base)


@pytest.mark.parametrize("seed", range(12))
def test_checker_equals_independent_restatement(seed):
    rng = np.random.default_rng(seed)
    n = 60
    links = [[[int(x) for x in rng.choice(n, int(rng.integers(1, 12)), replace=False) if x != p]] for p in range(n)]
    link_s = rng.permutation(n).astype(np.float32) / 7
    base_s = rng.permutation(n).astype(np.float32) / 5
    view = _View(links, 4, 6)
    filtered = rng.random(n) < 0.2 if seed % 2 else None
    for top, ef in ((3, 3), (1, 2), (5, 10), (10, 4)):
        got, st = _scores(view, link_s, base_s, top, ef, filtered=filtered)
        want, hops, scored, based = _independent(view, link_s, base_s, top, ef, filtered)
        assert [(i, float(s)) for i, s in got] == [(i, float(s)) for i, s in want]
        assert (st["hops"], st["link_scored"], st["base_scored"]) == (hops, scored, based)
        unkeyed, st2 = _scores(view, link_s, base_s, top, ef, keyed=False, filtered=filtered)   # tie-free: keyed == unkeyed
        assert unkeyed == got and st2 == st


def test_checker_break_candidate_is_an_evicted_point():
    # entry 0 -> links 1, 2, 3 (link scores 3, 2, 1) with ef 2: 3 enters then is evicted by 1 and 2 while unexpanded; after both are
    # expanded (no new links) the heap top is 3, below the lower bound: it is base-scored and, with the best base score, returned first
    links = [[[1, 2, 3]], [[0]], [[0]], [[0]]]
    link_s = np.array([0.5, 3, 2, 1], np.float32)
    base_s = np.array([0.0, 0.1, 0.2, 9.0], np.float32)
    got, st = _scores(_View(links, 2, 4), link_s, base_s, 2, 2)
    assert st["break_id"] is None and [i for i, _ in got] == [2, 1]    # in this order 3 never enters the links context
    links[0][0] = [3, 1, 2]       # stored order: 3 enters first, then is evicted
    got, st = _scores(_View(links, 2, 4), link_s, base_s, 2, 2)
    assert st["break_id"] == 3 and st["break_evicted"]
    assert got[0] == (3, np.float32(9.0))


def test_batched_writer_equals_writer():
    # serialize_plain_with_vectors (the probe's writer for millions of points) == serialize_with_vectors, byte for byte
    rng = np.random.default_rng(5)
    n = 3000
    edges = [[sorted(set(lst)) for lst in levels] for levels in gl.random_links(rng, n, 6, 8, 16)]
    edges[7][0] = list(range(200))   # a two-byte varint
    base = rng.integers(0, 256, (n, 40), dtype=np.uint8)
    link = rng.integers(0, 256, (n, 21), dtype=np.uint8)
    plain = np.frombuffer(gl.serialize_plain(n, *gl.edges_to_plain_arrays(edges)), np.uint8)
    want = gv.serialize_with_vectors(edges, 8, 16, lambda i: base[i].tobytes(), lambda i: link[i].tobytes(), (40, 4), (21, 1))
    assert gv.serialize_plain_with_vectors(plain, 8, 16, base, link).tobytes() == want


@pytest.mark.parametrize("seed,ef", [(0, 4), (1, 8), (2, 16), (3, 3), (4, 32)])
def test_checker_links_context_equals_the_regular_traversal(seed, ef):
    """The links context is the regular HNSW beam over the link scores: its hops score the same ids in the same order as the ACORN
    checker's HNSW traversal (tests/hnsw_acorn_ref.c) with that scorer, on the same graph, and its final list is that traversal's
    result.  The result is the best `top` base scores of the expanded candidates plus the break candidate."""
    from tests import hnsw_acorn_ref as ar

    rng = np.random.default_rng(seed)
    n, m0 = 400, 16
    edges = [[gl.normalize_links(m0, [int(x) for x in rng.choice(n, int(rng.integers(1, m0 + 1)), replace=False) if x != p])] for p in range(n)]
    link_s = (rng.permutation(n).astype(np.float32) + 1) / 3          # distinct: no tie order involved
    base_s = (rng.permutation(n).astype(np.float32) + 1) / 7
    ids4 = lambda i: np.uint32(i).tobytes()
    blob = gv.serialize_with_vectors(edges, 8, m0, ids4, ids4, (4, 4), (4, 1))
    view = gv.WithVectorsLinks(blob)
    as_id = lambda v: int(np.frombuffer(v, np.uint32)[0])
    top = 5
    got, st = ref.search_with_vectors(view, lambda i: link_s[i], lambda v: link_s[as_id(v)], lambda v: base_s[as_id(v)], top, ef, 0, 0)

    plain = np.frombuffer(gl.serialize_plain(n, *gl.edges_to_plain_arrays(edges)), np.uint8)
    g = ar.Graph(plain, 8, m0, n)
    calls = []

    def score(ids):
        calls.append([int(x) for x in ids])
        return link_s[ids]

    want = g.search(score, max(top, ef), max(top, ef), 0, 0, algo=ar.HNSW)
    g.close()
    assert calls[0] == [0] and calls[1:] == st["hop_ids"]
    assert [int(i) for i in want["idx"]] == [i for i, _ in st["links_nearest"]]
    pool = st["expanded"] + ([st["break_id"]] if st["break_id"] is not None else [])
    assert [i for i, _ in got] == sorted(pool, key=lambda i: -base_s[i])[:top]
