"""CPU checks of the restatement of the incremental device graph build (tests/hnsw_build_incr_ref.c), the checker
qb_hnsw_build_incremental is held to.

(a) One heal item: the two phases are the serial heal, so the healed graph equals a line-by-line Python transliteration of
    heal_point_on_level / search_shortcuts_on_level (graph_layers_healer.rs:82-207) over the oracle's scores.
(b) No unmapped point: nothing is healed; with no new point either the result is the old graph renamed, and the old graph itself under
    the identity mapping.
(c) One point per batch is serial link_new_point of the new points, in the order, on top of the healed graph, levels above the old top
    included.
(d) The fixture of the reference's quirk: an unmapped point is healed too, and its backlink displaces a live link that the renumbering
    then drops."""
import heapq

import numpy as np
import pytest

from tests.hnsw_build_incr_ref import GONE, IncrGraph, build_incremental
from tests.hnsw_build_ref import PlainGraph, RefGraph

COSINE, EUCLID, DOT, MANHATTAN = 0, 1, 2, 3


def _levels(n, m, seed):
    u = 1.0 - np.random.default_rng(seed).random(n)
    return np.minimum(np.round(-np.log(u) / np.log(m)), 30).astype(np.uint8)


def _data(n, dim, dist, seed, oracle):
    base = np.random.default_rng(seed).standard_normal((n, dim)).astype(np.float32)
    return oracle.preprocess_rows_f32(dist, base) if dist == COSINE else base


def _old(oracle, dist, n=600, dim=16, m=8, m0=16, ef=32, seed=1):
    base = _data(n, dim, dist, seed, oracle)
    lv = _levels(n, m, seed + 1)
    g = RefGraph.batched(base, dist, m, m0, ef, lv, batch=16, serial_points=32)
    blob = g.export_plain()
    g.close()
    return base, lv, blob


def _lists(blob):
    pg = PlainGraph(blob)
    return pg, {(p, l): [int(x) for x in pg.links(l, p)] for p in range(pg.n) for l in range(int(pg.point_level[p]) + 1)}


def _heal_one(oracle, dist, base, lists, m, m0, o2n, ef, p, l):
    """heal_point_on_level(p, l) with the reference's code shape, then its backlinks; `lists` is changed in place"""
    lm = m0 if l == 0 else m
    sim = lambda a, b: float(oracle.similarity_f32(dist, base[a], base[b]))
    gone = lambda x: o2n[x] == GONE
    valid = [x for x in lists[(p, l)] if not gone(x)]
    # search_shortcuts_on_level
    visited = {p}
    nearest = []   # FixedLengthPriorityQueue: a min-heap of (score, id)
    pending = []
    for x in lists[(p, l)]:
        if not gone(x):
            visited.add(x)
        else:
            pending.append((x, sim(p, x)))
    while pending:
        idx, score = pending.pop()
        if len(nearest) == ef and score < nearest[0][0]:
            continue
        if idx in visited:
            continue
        visited.add(idx)
        neighbours = [x for x in lists[(idx, l)] if x not in visited]
        for x in neighbours:
            s = sim(p, x)
            if not gone(x):
                if len(nearest) < ef:
                    heapq.heappush(nearest, (s, x))
                elif nearest[0][0] < s:
                    heapq.heapreplace(nearest, (s, x))
            else:
                pending.append((x, s))
    shortcuts = sorted(nearest, key=lambda e: (-e[0], e[1]))
    # fill_from_sorted_with_heuristic, then the valid links
    container = []
    for s, c in shortcuts:
        if len(container) >= lm - len(valid):
            break
        if all(sim(c, k) <= s for k in container):
            container.append(c)
    container += valid
    lists[(p, l)] = container
    for other in container:
        ol = lists[(other, l)]
        if p in ol:
            continue
        if len(ol) < lm:
            ol.append(p)
            continue
        cand = sorted([(sim(other, x), x) for x in ol + [p]], key=lambda e: (-e[0], e[1]))
        kept = []
        for s, c in cand:
            if len(kept) >= lm:
                break
            if all(sim(c, k) <= s for k in kept):
                kept.append(c)
        lists[(other, l)] = kept


@pytest.mark.parametrize("dist,item", [(COSINE, 0), (EUCLID, 3), (DOT, 1), (MANHATTAN, 5)])
def test_one_item_is_heal_point_on_level(oracle, dist, item):
    m, m0, ef = 8, 16, 24
    base, lv, blob = _old(oracle, dist, m=m, m0=m0)
    n = lv.size
    o2n = np.arange(n, dtype=np.uint32)
    o2n[np.random.default_rng(5).choice(n, 40, replace=False)] = GONE
    g = IncrGraph.from_plain(base, dist, m, m0, blob)
    _, lists = _lists(blob)
    items = [(p, l) for (p, l), ls in sorted(lists.items()) if any(o2n[x] == GONE for x in ls)]
    assert g.heal(o2n, ef, only_item=item) == len(items) > item
    _heal_one(oracle, dist, base, lists, m, m0, o2n, ef, *items[item])
    _, got = _lists(g.export_plain())
    assert got == lists
    g.close()


@pytest.mark.parametrize("dist", [COSINE, EUCLID])
def test_no_gone_points_heal_nothing(oracle, dist):
    m, m0 = 8, 16
    base, lv, blob = _old(oracle, dist, m=m, m0=m0)
    n = lv.size
    # identity: the old graph itself
    g, entry = build_incremental(base, blob, dist, m, m0, base, np.arange(n, dtype=np.uint32), lv, ef_construct=32)
    assert np.array_equal(g.export_plain(), blob)
    old = RefGraph.batched(base, dist, m, m0, 32, lv, batch=16, serial_points=32)
    assert entry == old.entry()
    old.close(); g.close()
    # a permutation: the old graph renamed
    perm = np.random.default_rng(9).permutation(n).astype(np.uint32)
    nb = np.empty_like(base)
    nb[perm] = base
    nlv = np.empty_like(lv)
    nlv[perm] = lv
    h = IncrGraph.from_plain(base, dist, m, m0, blob)
    assert h.heal(perm, 32) == 0
    h.close()
    g, _ = build_incremental(base, blob, dist, m, m0, nb, perm, nlv, ef_construct=32)
    _, want = _lists(blob)
    _, got = _lists(g.export_plain())
    assert got == {(int(perm[p]), l): [int(perm[x]) for x in ls] for (p, l), ls in want.items()}
    g.close()


@pytest.mark.parametrize("dist,serial,high", [(COSINE, 1, False), (EUCLID, 5, True), (DOT, 256, True), (MANHATTAN, 3, False)])
def test_batch_of_one_is_serial_insertion(oracle, dist, serial, high):
    m, m0, ef = 8, 16, 24
    base, lv, blob = _old(oracle, dist, m=m, m0=m0)
    n = lv.size
    rng = np.random.default_rng(7)
    keep = rng.random(n) >= 0.1
    n_new = int(keep.sum()) + 150
    o2n = np.full(n, GONE, dtype=np.uint32)
    o2n[keep] = np.arange(int(keep.sum()), dtype=np.uint32)
    nb = np.concatenate([base[keep], _data(150, base.shape[1], dist, 8, oracle)])
    nlv = np.concatenate([lv[keep], _levels(150, m, 9)])
    if high:
        nlv[-3:] = int(lv.max()) + np.array([2, 1, 2])
    deleted = np.zeros(n_new, dtype=bool)
    deleted[-10:-5] = True
    a, ea = build_incremental(base, blob, dist, m, m0, nb, o2n, nlv, ef_construct=ef, deleted=deleted, batch=1, serial_points=serial)
    b, eb = build_incremental(base, blob, dist, m, m0, nb, o2n, nlv, ef_construct=ef, deleted=deleted, serial=True)
    assert ea == eb
    if high:
        assert ea == (n_new - 3, int(lv.max()) + 2)
    assert np.array_equal(a.export_plain(), b.export_plain())
    pg = PlainGraph(a.export_plain())
    for p in np.flatnonzero(deleted):
        for l in range(int(nlv[p]) + 1):
            assert pg.links(l, int(p)).size == 0
    a.close(); b.close()


def test_gone_point_backlink_displaces_a_live_link(oracle):
    """The reference heals lists of points that are going away too; such a list's backlinks go into live lists, where they can evict a
    live link by the heuristic.  The renumbering drops the gone point, so the live list ends shorter than it was."""
    m, m0 = 4, 8
    base, lv, blob = _old(oracle, EUCLID, n=800, dim=8, m=m, m0=m0, ef=16, seed=3)
    n = lv.size
    o2n = np.arange(n, dtype=np.uint32)
    o2n[np.random.default_rng(11).choice(n, 240, replace=False)] = GONE
    _, before = _lists(blob)
    g = IncrGraph.from_plain(base, EUCLID, m, m0, blob)
    g.heal(o2n, 16)
    _, after = _lists(g.export_plain())
    g.close()
    displaced = [(p, l) for (p, l), ls in after.items() if o2n[p] != GONE and any(o2n[x] == GONE and x not in before[(p, l)] for x in ls)
                 and any(o2n[x] != GONE and x not in ls for x in before[(p, l)])]
    assert displaced, "the fixture no longer shows a gone point's backlink displacing a live link"
