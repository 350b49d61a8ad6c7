"""HNSW graphs with inline vectors (GraphLinksFormat::CompressedWithVectors): qb_hnsw_create_with_vectors and
qb_hnsw_search_with_vectors_batch against the CPU reader and checker (tests/graph_links_with_vectors.py, tests/hnsw_inline_ref.py).

1. Links: qb_hnsw_links on the handle equals the reader for every point and level (lists wider than level_m, link vectors at odd
   byte offsets).
2. Errors: malformed files return QB_ERR_INVALID and the device stays usable; unsupported storages / layouts QB_ERR_UNSUPPORTED.
3. Search: the device equals the checker in keyed mode (lists, score bits, hops, scored points, counters) across metrics, dims
   (both base chains, both SQ8 chains), m0, ef, top > ef, filters, lists wider than m0, batches; the host and device-resident
   entries agree; the break candidate (a point evicted from the beam while unexpanded) reaches the results.
4. The regular searches (HNSW, ACORN, custom) on the handle equal those on a Compressed handle of the same edges."""
import numpy as np
import pytest

from tests import graph_links_compressed as gl
from tests import graph_links_with_vectors as gv
from tests import hnsw_inline_ref as ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _sq8(qb, oracle, base, d):
    dt, inv = qb.construct_vector_parameters(d)
    sq = oracle.SQ8.encode(base, int(dt), bool(inv))
    st = qb.ScalarQuantizedVectors(sq.rows, base.shape[1], sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, d)
    return sq, st


def _file(edges, base, sq, m, m0, base_align=4):
    return gv.serialize_with_vectors(edges, m, m0, lambda i: base[i].tobytes(), lambda i: sq.rows[i].tobytes(), (base.shape[1] * 4, base_align),
                                     (sq.row_bytes, 1))


class _Case:
    """an oracle-built graph over `base` written with inline SQ8 vectors"""

    def __init__(self, qb, oracle, dist, dim, n, m=16, m0=None, seed=3, widen=0):
        self.d = getattr(qb.Distance, dist)
        rng = np.random.default_rng(seed)
        base = rng.standard_normal((n, dim)).astype(np.float32)
        if self.d == qb.Distance.Cosine:
            base = oracle.preprocess_rows_f32(oracle.COSINE, base)
        self.base, self.rng = base, rng
        g = oracle.HNSW(base, int(self.d), m=m, ef_construct=64, seed=11, threads=4)
        self.entry, self.level, self.m, gm0 = g.entry()
        self.m0 = gm0 if m0 is None else m0
        edges = gv.edges_of_plain(g.export_plain())
        g.close()
        if widen:   # lists longer than m0: extra distinct links appended to level 0
            for p, lv in enumerate(edges):
                extra = [int(x) for x in rng.choice(n, widen, replace=False) if x != p and x not in lv[0]]
                lv[0] = lv[0] + extra
        self.edges = edges
        self.sq, self.st = _sq8(qb, oracle, base, self.d)
        self.blob = _file(edges, base, self.sq, self.m, self.m0)
        self.view = gv.WithVectorsLinks(self.blob)
        self.h = qb.HnswGraph.from_compressed_with_vectors(self.st, self.blob)

    def close(self):
        self.h.close(); self.st.close()


def _assert_lists(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for a, b in zip(got, want):
        assert [int(x) for x in a["idx"]] == [i for i, _ in b], what
        assert np.array_equal(a["score"].view(np.uint32), np.array([s for _, s in b], np.float32).view(np.uint32)), what


def _check_search(qb, oracle, c, queries, top, ef, filtered=None, resident=None):
    if resident is not None:
        c.st.set_deleted(resident)
    both = None
    if filtered is not None or resident is not None:
        both = np.zeros(c.base.shape[0], bool)
        for f in (filtered, resident):
            if f is not None:
                both |= f
    want, tot, per = ref.run(oracle, c.view, c.sq, int(c.d), queries, top, ef, c.entry, c.level, both)
    c.h.stats(reset=True)
    cnt = qb.HwCounters()
    got = c.h.search_with_vectors(queries, top, ef, c.entry, c.level, point_deleted=filtered, counters=cnt)
    _assert_lists(got, want, f"top {top} ef {ef}")
    assert c.h.stats(reset=True) == (tot["hops"], tot["link_scored"])
    dim = c.base.shape[1]
    assert cnt.cpu == tot["link_scored"] * dim + tot["base_scored"] * dim * 4
    assert cnt.vector_io_read == 0
    if resident is not None:
        c.st.set_deleted(np.zeros(c.base.shape[0], bool))
    return per


# ------------------------------------------------------------------------------------------------ 1. links
@pytest.mark.parametrize("graph", [1, 2, 3, 4])
def test_links_literal_graphs(qb, oracle, graph):
    from tests.test_graph_links_compressed import LITERAL_GRAPHS

    edges = LITERAL_GRAPHS[graph]
    n = len(edges)
    base = np.random.default_rng(n).standard_normal((n, 13)).astype(np.float32)
    sq, st = _sq8(qb, oracle, base, qb.Distance.Dot)
    blob = _file(edges, base, sq, 8, 16)
    r = gv.WithVectorsLinks(blob)
    h = qb.HnswGraph.from_compressed_with_vectors(st, blob)
    for lvl in range(r.levels_count):
        ids = np.array([p for p in range(n) if r.point_level(p) >= lvl], dtype=np.uint32)
        for p, g in zip(ids, h.links(lvl, ids)):
            assert g.tolist() == r.links(int(p), lvl), (int(p), lvl)
    h.close(); st.close()


def test_links_wide_lists_odd_offsets(qb, oracle):
    rng = np.random.default_rng(7)
    n = 1000
    edges = gl.random_links(rng, n, 10, 8, 16)          # up to 2 x level_m links per list
    base = rng.standard_normal((n, 21)).astype(np.float32)
    sq, st = _sq8(qb, oracle, base, qb.Distance.Euclid)  # link vectors of 4 + 32 bytes at any byte offset
    blob = _file(edges, base, sq, 8, 16)
    r = gv.WithVectorsLinks(blob)
    assert any(r.record(p, 0)[3] % 4 for p in range(n))
    h = qb.HnswGraph.from_compressed_with_vectors(st, blob)
    hc = qb.HnswGraph.from_compressed(st, gl.serialize_compressed(edges, 8, 16))
    for lvl in range(r.levels_count):
        ids = np.array([p for p in range(n) if r.point_level(p) >= lvl], dtype=np.uint32)
        got = h.links(lvl, ids)
        for p, g in zip(ids, got):
            assert g.tolist() == r.links(int(p), lvl), (int(p), lvl)
        for a, b in zip(got, hc.links(lvl, ids)):
            assert np.array_equal(a, b)
    assert h.info()[2] > hc.info()[2] + len(r.neighbors)
    assert np.array_equal(h.export_plain(), hc.export_plain())
    h.close(); hc.close(); st.close()


# ------------------------------------------------------------------------------------------------ 2. errors
def _rebuild(blob, *, boff=None, reindex=None, records=None):
    """the same file with its record byte offsets / reindex / records replaced"""
    r = gv.WithVectorsLinks(blob)
    b = bytearray(blob)
    if boff is None:
        boff = [gl.read_pair(r.offsets, r.params, i)[0] for i in range(r.params.length - 1)] + [r.total_neighbors_bytes]
    recs = bytes(r.neighbors) if records is None else records
    reindex = r.reindex if reindex is None else np.asarray(reindex, np.uint32)
    coff, p = gl.compress(boff, 7)
    b[24:32] = len(recs).to_bytes(8, "little")
    b[32:40] = p.length.to_bytes(8, "little")
    b[40], b[41], b[42] = p.base_bits, p.delta_bits, p.chunk_len_log2
    head = 80 + 8 * r.levels_count
    return bytes(b[:head]) + reindex.tobytes() + bytes(b[head + 4 * r.point_count:r.records_at]) + recs + coff


def test_malformed_and_unsupported(qb, oracle):
    import torch

    n, dim = 400, 24
    rng = np.random.default_rng(1)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    g = oracle.HNSW(base, oracle.DOT, m=8, ef_construct=32, seed=11, threads=1)
    entry, lvl, m, m0 = g.entry()
    edges = gv.edges_of_plain(g.export_plain())
    g.close()
    sq, st = _sq8(qb, oracle, base, qb.Distance.Dot)
    blob = _file(edges, base, sq, m, m0)
    r = gv.WithVectorsLinks(blob)
    boff = [gl.read_pair(r.offsets, r.params, i)[0] for i in range(r.params.length - 1)] + [r.total_neighbors_bytes]

    def patched(offset, data):
        b = bytearray(blob); b[offset:offset + len(data)] = data; return bytes(b)

    recs = bytearray(r.neighbors)
    bad_varint = bytearray(recs); bad_varint[boff[0] + dim * 4:boff[1]] = b"\xff" * (boff[1] - boff[0] - dim * 4)
    big_count = bytearray(recs); big_count[boff[0] + dim * 4] = len(edges[0][0]) + 1   # link vectors run past the record
    base_cut = list(boff)
    base_cut[1] = boff[0] + dim * 4 - 4                                                 # record 0 ends inside its base vector
    up = min((e for e in range(n, len(boff) - 1) if recs[boff[e]]), key=lambda e: boff[e + 1] - boff[e])   # the shortest upper-level list
    long_links = bytearray(recs); long_links[boff[up]] = 127; long_links[boff[up] + 1] |= 31   # 127 links of 39 bits: past its end
    plain = np.frombuffer(gl.serialize_plain(n, *gl.edges_to_plain_arrays(edges)), np.uint8)
    bad = {
        "truncated header": blob[:60],
        "truncated body": blob[:200],
        "truncated tail": blob[:-1],
        "plain file": bytes(plain),
        "compressed file": gl.serialize_compressed(edges, m, m0),
        "wrong point count": patched(0, (n - 1).to_bytes(8, "little")),
        "delta_bits 0": patched(41, b"\x00"),
        "link size": patched(68, (sq.row_bytes + 1).to_bytes(8, "little")),
        "base size": patched(59, (dim * 4 + 4).to_bytes(8, "little")),
        "alignment 3": patched(76, b"\x03"),
        "varint past the record": _rebuild(blob, records=bytes(bad_varint)),
        "link vectors past the record": _rebuild(blob, records=bytes(big_count)),
        "base vector past the record": _rebuild(blob, boff=base_cut),
        "packed links past the record": _rebuild(blob, records=bytes(long_links)),
        "offsets decrease": _rebuild(blob, boff=boff[:3] + [boff[4], boff[3]] + boff[5:]),
        "offset past the end": _rebuild(blob, boff=boff[:-1] + [boff[-1] + 9]),
        "reindex out of range": _rebuild(blob, reindex=np.r_[np.uint32(n + 5), r.reindex[1:]]),
    }
    # the full message of each refusal
    message = {
        "truncated header": "hnsw_create_with_vectors: 60 bytes is smaller than HeaderCompressedWithVectors",
        "truncated body": "hnsw_create_with_vectors: 200 bytes, header describes 260096 before the offsets",
        "truncated tail": "hnsw_create_with_vectors: 550 offsets do not fit the 972 bytes after the records",
        "plain file": "hnsw_create_with_vectors: version word 0000000000000005 is not HEADER_VERSION_COMPRESSED_WITH_VECTORS (a Compressed or plain links.bin?)",
        "compressed file": "hnsw_create_with_vectors: version word ffffffffffffff01 is not HEADER_VERSION_COMPRESSED_WITH_VECTORS (a Compressed or plain links.bin?)",
        "wrong point count": "hnsw_create_with_vectors: graph has 399 points, storage 400",
        "delta_bits 0": "hnsw_create_with_vectors: offsets parameters base_bits 18 delta_bits 0 chunk_len_log2 2",
        'link size': "hnsw_create_with_vectors: link vectors of 37 bytes, the storage's rows have 36",
        "base size": "hnsw_create_with_vectors: base vectors of 100 bytes, dim 24",
        "alignment 3": "hnsw_create_with_vectors: vector alignments 4 / 3 are not powers of two",
        'varint past the record': "hnsw_create_with_vectors: a record's count, links or link vectors run past its end",
        'link vectors past the record': "hnsw_create_with_vectors: a record's count, links or link vectors run past its end",
        'base vector past the record': "hnsw_create_with_vectors: a record's count, links or link vectors run past its end",
        'packed links past the record': "hnsw_create_with_vectors: a record's count, links or link vectors run past its end",
        "offsets decrease": "hnsw_create_with_vectors: record offsets decrease",
        "offset past the end": "hnsw_create_with_vectors: a record offset lies past total_neighbors_bytes",
        "reindex out of range": "hnsw_create_with_vectors: a reindex entry is >= point_count",
        "f16 base": "hnsw_create_with_vectors: base vectors of 48 bytes at dim 24 are f16 or u8; only f32 base vectors are supported",
        "u8 base": "hnsw_create_with_vectors: base vectors of 24 bytes at dim 24 are f16 or u8; only f32 base vectors are supported",
        "list of 129 links": "hnsw_create_with_vectors: a list has more than 128 links",
    }
    for what, b in bad.items():
        with pytest.raises(qb.QbError) as ei:
            qb.HnswGraph.from_compressed_with_vectors(st, b)
        assert ei.value.status == -1, (what, str(ei.value))
        assert str(ei.value) == f"qb_status -1: {message[what]}", what
    wide = [[list(lv[0]) + [x for x in range(n) if x not in lv[0]][:129 - len(lv[0])]] + lv[1:] if p == 5 else lv for p, lv in enumerate(edges)]
    unsupported = {
        "f16 base": patched(59, (dim * 2).to_bytes(8, "little")),
        "u8 base": patched(59, dim.to_bytes(8, "little")[:8] + b"\x01"),
        "list of 129 links": _file(wide, base, sq, m, m0),
    }
    for what, b in unsupported.items():
        with pytest.raises(qb.QbError) as ei:
            qb.HnswGraph.from_compressed_with_vectors(st, b)
        assert ei.value.status == -3, (what, str(ei.value))
        assert str(ei.value) == f"qb_status -3: {message[what]}", what
    dense = qb.DenseVectorStorage(base, qb.Distance.Dot)
    pq = oracle.PQ.encode(base, 4, rng.standard_normal((256, dim)).astype(np.float32), oracle.QD_DOT, False)
    pqs = qb.ProductQuantizedVectors(pq.codes, rng.standard_normal((256, dim)).astype(np.float32), 4, dim, qb.Distance.Dot)
    bq = oracle.BQ.encode(base, oracle.BQ_ONE, 0, oracle.QD_DOT, False, None)
    bqs = qb.BinaryQuantizedVectors(bq.rows, dim, qb.Distance.Dot, qb.BQEncoding.OneBit, qb.BQQueryEncoding(0), None)
    for other in (dense, pqs, bqs):                          # link vectors are SQ8 rows only
        with pytest.raises(qb.QbError) as ei:
            qb.HnswGraph.from_compressed_with_vectors(other, blob)
        assert ei.value.status == -3
        assert str(ei.value) == 'qb_status -3: hnsw_create_with_vectors: the link vectors are read as rows of the bound storage, which must be scalar-quantized (SQ8)'
    pqs.close(); bqs.close()
    hc = qb.HnswGraph.from_compressed(st, gl.serialize_compressed(edges, m, m0))
    with pytest.raises(qb.QbError) as ei:
        hc.search_with_vectors(base[:2], 10, 32, entry, lvl)
    assert ei.value.status == -3
    torch.cuda.synchronize()
    # the rebuilt file itself is valid, and searches
    h = qb.HnswGraph.from_compressed_with_vectors(st, _rebuild(blob))
    want, _, _ = ref.run(oracle, r, sq, oracle.DOT, base[:8], 10, 32, entry, lvl)
    _assert_lists(h.search_with_vectors(base[:8], 10, 32, entry, lvl), want, "after refusals")
    with pytest.raises(qb.QbError) as ei:
        h.search_with_vectors(base[:2], 10, 32, entry, lvl, is_stopped=True)
    assert ei.value.status == -5
    h.close(); hc.close(); dense.close(); st.close()


# ------------------------------------------------------------------------------------------------ 3. search against the checker
@pytest.mark.parametrize("dist,dim,n,m", [("Cosine", 96, 6000, 16), ("Euclid", 100, 3000, 4), ("Dot", 8, 3000, 16), ("Manhattan", 40, 3000, 16),
                                          ("Cosine", 768, 3000, 16), ("Dot", 1056, 1500, 32)])
def test_search_equals_checker(qb, oracle, dist, dim, n, m):
    c = _Case(qb, oracle, dist, dim, n, m=m)
    queries = c.rng.standard_normal((24, dim)).astype(np.float32)
    in_result = 0   # queries whose last pop was a point evicted from the beam while unexpanded, and whose result holds it
    for top, ef in ((10, 64), (5, 16), (40, 20), (2, 1)):
        got = c.h.search_with_vectors(queries, top, ef, c.entry, c.level)
        per = _check_search(qb, oracle, c, queries, top, ef)
        in_result += sum(1 for s, g in zip(per, got) if s["break_evicted"] and s["break_id"] in g["idx"].tolist())
    assert in_result > 0
    c.close()


def test_search_filters_and_wide_lists(qb, oracle):
    c = _Case(qb, oracle, "Cosine", 64, 4000, m=8, widen=20)          # m0 = 16, level-0 lists up to ~36: truncation after the filter
    assert max(len(lv[0]) for lv in c.edges) > c.m0
    queries = c.rng.standard_normal((16, 64)).astype(np.float32)
    for sel in (0.01, 0.3, 1.0):
        keep = c.rng.random(4000) < sel
        keep[c.entry] = True
        f = ~keep
        _check_search(qb, oracle, c, queries, 10, 32, filtered=f)
        _check_search(qb, oracle, c, queries, 10, 32, resident=f)
        half = c.rng.random(4000) < 0.5
        half[c.entry] = False
        _check_search(qb, oracle, c, queries, 10, 32, filtered=f & half, resident=f & ~half)
    c.close()


def test_search_large_ef_and_batch(qb, oracle):
    c = _Case(qb, oracle, "Euclid", 32, 1500, m=32)                  # m0 = 64
    assert c.m0 == 64
    _check_search(qb, oracle, c, c.rng.standard_normal((3, 32)).astype(np.float32), 50, 4096)
    _check_search(qb, oracle, c, c.rng.standard_normal((3, 32)).astype(np.float32), 300, 100)
    # more queries than resident CTAs, and the device-resident entry
    import torch

    from qdrant_b200._capi import check, lib, vp

    queries = c.rng.standard_normal((2500, 32)).astype(np.float32)
    got = c.h.search_with_vectors(queries, 10, 32, c.entry, c.level)
    want, _, _ = ref.run(oracle, c.view, c.sq, int(c.d), queries[::97], 10, 32, c.entry, c.level)
    _assert_lists(got[::97], want, "batch")
    dq = torch.from_numpy(queries).cuda()
    out = torch.zeros((2500, 10, 2), dtype=torch.int32, device="cuda")
    cnt = torch.zeros(2500, dtype=torch.int32, device="cuda")
    check(lib().qb_hnsw_search_with_vectors_batch_device(c.h._h, vp(dq.data_ptr()), 2500, 10, 32, c.entry, c.level, vp(out.data_ptr()),
                                                         vp(cnt.data_ptr())))
    torch.cuda.synchronize()
    rec = out.cpu().numpy().view(qb.SCORED_POINT_OFFSET).reshape(2500, 10)
    for i in range(2500):
        assert np.array_equal(rec[i, : cnt[i]], got[i])
    c.close()


# ------------------------------------------------------------------------------------------------ 4. regular searches on the same handle
def test_regular_searches_equal_compressed_handle(qb, oracle):
    c = _Case(qb, oracle, "Cosine", 48, 3000, m=8)
    hc = qb.HnswGraph.from_compressed(c.st, gl.serialize_compressed(c.edges, c.m, c.m0))
    queries = c.rng.standard_normal((20, 48)).astype(np.float32)
    f = c.rng.random(3000) < 0.7
    f[c.entry] = False
    for algo in ("hnsw", "acorn"):
        for a, b in zip(c.h.search(queries, 10, 32, c.entry, c.level, point_deleted=f, algorithm=algo),
                        hc.search(queries, 10, 32, c.entry, c.level, point_deleted=f, algorithm=algo)):
            assert np.array_equal(a, b)
    ex = c.rng.standard_normal((20, 3, 48)).astype(np.float32)
    for a, b in zip(c.h.search_custom(qb.QueryKind.RecommendBestScore, ex, 2, 1, top=10, ef=32, entry_point=c.entry, entry_level=c.level),
                    hc.search_custom(qb.QueryKind.RecommendBestScore, ex, 2, 1, top=10, ef=32, entry_point=c.entry, entry_level=c.level)):
        assert np.array_equal(a, b)
    hc.close(); c.close()


def test_recall_against_exact_scan(qb, oracle):
    c = _Case(qb, oracle, "Cosine", 128, 20000)
    queries = c.rng.standard_normal((50, 128)).astype(np.float32)
    qp = np.stack([oracle.preprocess_f32(oracle.COSINE, q) for q in queries])
    exact = oracle.scan_f32(oracle.COSINE, c.base, qp, 10)
    got = c.h.search_with_vectors(queries, 10, 64, c.entry, c.level)
    want, _, _ = ref.run(oracle, c.view, c.sq, int(c.d), queries[:10], 10, 64, c.entry, c.level)
    _assert_lists(got[:10], want, "oracle graph")
    recall = lambda lists: np.mean([len(set(a["idx"].tolist()) & set(b["idx"].tolist())) / 10 for a, b in zip(lists, exact)])
    dense = qb.DenseVectorStorage(c.base, c.d)
    hf = qb.HnswGraph.from_compressed(dense, gl.serialize_compressed(c.edges, c.m, c.m0))
    r_vec, r_sq8, r_f32 = recall(got), recall(c.h.search(queries, 10, 64, c.entry, c.level)), recall(hf.search(queries, 10, 64, c.entry, c.level))
    # Gaussian rows at 128-d are a hard case for any graph; the numbers are reported, the lists are what the test holds to the checker
    print(f"recall@10 at ef 64, 20000 x 128 Gaussian cosine: with-vectors {r_vec:.3f}, SQ8 traversal {r_sq8:.3f}, f32 traversal {r_f32:.3f}")
    assert r_vec > 0.25
    hf.close(); dense.close(); c.close()
