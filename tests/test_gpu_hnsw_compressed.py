"""HNSW graphs loaded from the reference's compressed links.bin (qb_hnsw_create_compressed), decoded on the device.

1. qb_hnsw_links on the decoded graph equals the independent CPU reader (tests/graph_links_compressed.py) for every point on every
   level, and equals the plain-loaded graph of the same (normalised) edges.
2. The traversal over a compressed graph equals the CPU traversal of the same graph (tie-aware lists, score bits, hops and scored
   points) and the plain-loaded graph's lists.  Within one (node, level) the compressed file stores the first level_m links sorted,
   the CPU graph in build order; a hop scores the same set either way, so the traversals agree whenever scores are distinct.
3. Malformed files return QB_ERR_INVALID (or QB_ERR_UNSUPPORTED) from validation alone, and the device stays usable."""
import numpy as np
import pytest

from tests import graph_links_compressed as gl
from tests.util import assert_topk_equal, pack_bitmap

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def _storage(qb, n, dim=8):
    return qb.DenseVectorStorage(np.random.default_rng(n).standard_normal((n, dim)).astype(np.float32), qb.Distance.Dot)


def _check_links_exact(qb, st, blob, plain=None):
    r = gl.CompressedLinks(blob)
    hg = qb.HnswGraph.from_compressed(st, blob)
    hp = qb.HnswGraph(st, plain, r.m, r.m0) if plain is not None else None
    assert hg.info()[:2] == (r.point_count, r.levels_count)
    for lvl in range(r.levels_count):
        ids = np.array([p for p in range(r.point_count) if r.point_level(p) >= lvl], dtype=np.uint32)
        got = hg.links(lvl, ids)
        for p, g in zip(ids, got):
            assert g.tolist() == r.links(int(p), lvl), (int(p), lvl)
        if hp is not None:
            for a, b in zip(got, hp.links(lvl, ids)):
                assert np.array_equal(a, b)
        # truncation to cap keeps the full count
        if ids.size:
            assert [x.tolist() for x in hg.links(lvl, ids[:50], cap=3)] == [x[:3].tolist() for x in got[:50]]
        absent = [p for p in range(r.point_count) if r.point_level(p) < lvl]
        if absent:
            with pytest.raises(qb.QbError) as ei:
                hg.links(lvl, absent[:1])
            assert ei.value.status == -1
    hg.close()
    if hp is not None:
        hp.close()


def _normalised_plain(edges, m, m0):
    norm = [[gl.normalize_links(m0 if lvl == 0 else m, links) for lvl, links in enumerate(levels)] for levels in edges]
    lo, reindex, nb, off = gl.edges_to_plain_arrays(norm)
    return np.frombuffer(gl.serialize_plain(len(edges), lo, reindex, nb, off), np.uint8)


@pytest.mark.parametrize("graph", [1, 2, 3, 4, 5])
def test_links_literal_graphs(qb, graph):
    from tests.test_graph_links_compressed import LITERAL_GRAPHS

    edges = LITERAL_GRAPHS[graph]
    st = _storage(qb, len(edges))
    for log2 in (None, 0, 3, 7):
        _check_links_exact(qb, st, gl.serialize_compressed(edges, 8, 16, log2), _normalised_plain(edges, 8, 16))
    st.close()


@pytest.mark.parametrize("log2", [None, 0, 1, 2, 3, 4, 5, 6, 7])
def test_links_random_links(qb, log2):
    rng = np.random.default_rng(11 + (log2 or 0))
    edges = gl.random_links(rng, 1000, 10, 16, 32)
    st = _storage(qb, 1000)
    blob = gl.serialize_compressed(edges, 16, 32, log2)
    _check_links_exact(qb, st, blob, _normalised_plain(edges, 16, 32) if log2 is not None else None)
    st.close()


def test_links_18_bit_unsorted_ids(qb):
    n = (1 << 17) + 3
    rng = np.random.default_rng(17)
    lo, reindex, nb, off = gl.synthetic_graph(rng, n, 16, 32, full=False)
    blob = gl.compress_plain_csr(n, lo, reindex, nb, off, 16, 32)
    r = gl.CompressedLinks(blob)
    assert r.bits_per_unsorted == 18
    st = _storage(qb, n, 4)
    _check_links_exact(qb, st, blob)
    st.close()


def test_links_10m_points_sample(qb):
    n = 10_000_000
    rng = np.random.default_rng(10)
    lo, reindex, nb, off = gl.synthetic_graph(rng, n, 16, 32)
    blob = gl.compress_plain_csr(n, lo, reindex, nb, off, 16, 32)
    del nb
    r = gl.CompressedLinks(blob)
    st = qb.DenseVectorStorage(np.zeros((n, 1), np.float32), qb.Distance.Dot)
    hg = qb.HnswGraph.from_compressed(st, blob)
    sample = np.random.default_rng(1)
    for lvl in range(r.levels_count):
        on = int(r.level_offsets[lvl + 1] - r.level_offsets[lvl])            # back_index order: reindex < count <=> on the level
        ids = sample.choice(n, 100_000, replace=False).astype(np.uint32) if lvl == 0 else \
            np.flatnonzero(r.reindex < on)[sample.permutation(on)[:100_000]].astype(np.uint32)
        for p, g in zip(ids, hg.links(lvl, ids)):
            assert g.tolist() == r.links(int(p), lvl), (int(p), lvl)
    hg.close(); st.close()


# ------------------------------------------------------------------------------------------------ traversal parity
def _graph(oracle, base, dist, threads=4, m=16):
    g = oracle.HNSW(base, dist, m=m, ef_construct=64, seed=11, threads=threads)
    entry, entry_level, gm, gm0 = g.entry()
    plain = g.export_plain()
    return g, plain, gl.plain_to_compressed(plain, gm, gm0), entry, entry_level, gm, gm0


@pytest.mark.parametrize("dist,dim,n", [("Cosine", 96, 20_000), ("Euclid", 100, 6_000), ("Dot", 8, 3_000), ("Manhattan", 40, 3_000), ("Cosine", 768, 4_000)])
def test_compressed_traversal_equals_cpu_and_plain_f32(qb, oracle, dist, dim, n):
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(3)
    base = rng.standard_normal((n, dim)).astype(np.float32)
    if d == qb.Distance.Cosine:
        base = oracle.preprocess_rows_f32(oracle.COSINE, base)
    queries = rng.standard_normal((70, dim)).astype(np.float32)
    qp = np.stack([oracle.preprocess_f32(int(d), q) for q in queries])
    g, plain, comp, entry, lvl, m, m0 = _graph(oracle, base, int(d))
    st = qb.DenseVectorStorage(base, d)
    hc = qb.HnswGraph.from_compressed(st, comp)
    hp = qb.HnswGraph(st, plain, m, m0)
    for top, ef in ((10, 128), (5, 16), (40, 20)):
        g.stats(reset=True); hc.stats(reset=True)
        want = g.search_batch(qp, top, ef, threads=2)
        cnt = qb.HwCounters()
        got = hc.search(queries, top, ef, entry, lvl, counters=cnt)
        for i, (a, b) in enumerate(zip(got, want)):
            assert_topk_equal(a, b, what=f"{dist} dim {dim} top {top} ef {ef} query {i}")
        calls, scored = g.stats(reset=True)
        assert cnt.cpu == scored * dim * 4
        assert hc.stats(reset=True) == (calls, scored)
        for a, b in zip(got, hp.search(queries, top, ef, entry, lvl)):
            assert np.array_equal(a, b)
    hc.close(); hp.close(); st.close(); g.close()


def test_compressed_traversal_sq8(qb, oracle):
    n, dim = 6_000, 96
    d = qb.Distance.Cosine
    rng = np.random.default_rng(9)
    base = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((n, dim)).astype(np.float32))
    queries = rng.standard_normal((24, dim)).astype(np.float32)
    g, plain, comp, entry, lvl, m, m0 = _graph(oracle, base, int(d))
    dt, inv = qb.construct_vector_parameters(d)
    sq = oracle.SQ8.encode(base, int(dt), bool(inv))
    qst = qb.ScalarQuantizedVectors(sq.rows, dim, sq.meta.alpha, sq.meta.offset, sq.meta.multiplier, d)
    hc = qb.HnswGraph.from_compressed(qst, comp)
    hp = qb.HnswGraph(qst, plain, m, m0)
    got = hc.search(queries, 10, 64, entry, lvl)
    for q, a, b in zip(queries, got, hp.search(queries, 10, 64, entry, lvl)):
        qpre = oracle.preprocess_f32(int(d), q)
        code, off = sq.encode_query(qpre)
        want = g.search(qpre, 10, 64, score_points=lambda ids, code=code, off=off: np.array([sq.score(code, off, int(i)) for i in ids], np.float32))
        assert_topk_equal(a, want, what="sq8 traversal")
        assert np.array_equal(a, b)
    hc.close(); hp.close(); qst.close(); g.close()


def test_compressed_traversal_with_deletions(qb, oracle):
    n, dim = 8_000, 64
    rng = np.random.default_rng(5)
    base = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((n, dim)).astype(np.float32))
    queries = rng.standard_normal((40, dim)).astype(np.float32)
    qp = np.stack([oracle.preprocess_f32(oracle.COSINE, q) for q in queries])
    g, plain, comp, entry, lvl, m, m0 = _graph(oracle, base, oracle.COSINE)
    deleted = rng.random(n) < 0.3
    deleted[entry] = False
    st = qb.DenseVectorStorage(base, qb.Distance.Cosine)
    hc = qb.HnswGraph.from_compressed(st, comp)
    hp = qb.HnswGraph(st, plain, m, m0)
    want = g.search_batch(qp, 10, 64, deleted=pack_bitmap(deleted))
    got = hc.search(queries, 10, 64, entry, lvl, point_deleted=deleted)
    for a, b, c in zip(got, want, hp.search(queries, 10, 64, entry, lvl, point_deleted=deleted)):
        assert_topk_equal(a, b, what="per-call deletions")
        assert np.array_equal(a, c)
    st.set_deleted(deleted)
    for a, b in zip(hc.search(queries, 10, 64, entry, lvl), want):
        assert_topk_equal(a, b, what="resident deletions")
    hc.close(); hp.close(); st.close(); g.close()


# ------------------------------------------------------------------------------------------------ malformed files
def _rebuild(blob, *, boff=None, lo=None, reindex=None):
    """the same file with its decoded byte offsets / level offsets / reindex replaced (offsets re-compressed, header updated)"""
    r = gl.CompressedLinks(blob)
    b = bytearray(blob)
    if boff is None:
        boff = [gl.read_pair(r.offsets, r.params, i)[0] for i in range(r.params.length - 1)] + [r.total_neighbors_bytes]
    lo = list(r.level_offsets[:-1]) if lo is None else lo
    reindex = r.reindex if reindex is None else np.asarray(reindex, np.uint32)
    coff, p = gl.compress(boff, 7)      # one base per 128 offsets: any planted value below the total fits the deltas
    b[16:24] = len(lo).to_bytes(8, "little")
    b[32:40] = p.length.to_bytes(8, "little")
    b[40], b[41], b[42] = p.base_bits, p.delta_bits, p.chunk_len_log2
    links_at = 64 + 8 * r.levels_count + 4 * r.point_count
    return bytes(b[:64]) + np.asarray(lo, np.uint64).tobytes() + reindex.tobytes() + bytes(b[links_at:links_at + r.total_neighbors_bytes]) + coff


def test_malformed_files_are_refused_and_the_device_stays_usable(qb, oracle):
    import torch

    n, dim = 500, 32
    base = np.random.default_rng(1).standard_normal((n, dim)).astype(np.float32)
    g, plain, comp, entry, lvl, m, m0 = _graph(oracle, base, oracle.DOT, threads=1)
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    r = gl.CompressedLinks(comp)
    assert r.levels_count > 1
    boff = [gl.read_pair(r.offsets, r.params, i)[0] for i in range(r.params.length - 1)] + [r.total_neighbors_bytes]

    def patched(offset, data):
        b = bytearray(comp); b[offset:offset + len(data)] = data; return bytes(b)

    bad = {
        "truncated header": comp[:40],
        "truncated body": comp[:100],
        "truncated tail": comp[:-1],
        "plain file": bytes(plain),
        "wrong point count": patched(0, (n - 1).to_bytes(8, "little")),
        "delta_bits 0": patched(41, b"\x00"),
        "delta_bits 57": patched(41, b"\x39"),
        "chunk_len_log2 8": patched(42, b"\x08"),
        "base_bits 0": patched(40, b"\x00"),
        "m 0": patched(43, (0).to_bytes(8, "little")),
        "offsets decrease": _rebuild(comp, boff=boff[:3] + [boff[4], boff[3]] + boff[5:]),
        "offset past total_neighbors_bytes": _rebuild(comp, boff=boff[:-1] + [boff[-1] + 9]),
        "level offset >= length": _rebuild(comp, lo=list(r.level_offsets[:-2]) + [r.params.length + 3]),
        "level 0 not the first n entries": _rebuild(comp, lo=[1] + list(r.level_offsets[1:-1])),
        "reindex out of range": _rebuild(comp, reindex=np.r_[np.uint32(n + 5), r.reindex[1:]]),
    }
    # the full message of each refusal
    message = {
        "truncated header": "hnsw_create_compressed: 40 bytes is smaller than HeaderCompressed",
        "truncated body": "hnsw_create_compressed: 100 bytes, header describes 13537 before the offsets",
        "truncated tail": "hnsw_create_compressed: 617 offsets do not fit the 708 bytes after the links",
        "plain file": "hnsw_create_compressed: version word 0000000000000004 is not HEADER_VERSION_COMPRESSED (a plain links.bin?)",
        "wrong point count": "hnsw_create_compressed: graph has 499 points, storage 500",
        "delta_bits 0": "hnsw_create_compressed: offsets parameters base_bits 14 delta_bits 0 chunk_len_log2 3",
        "delta_bits 57": "hnsw_create_compressed: offsets parameters base_bits 14 delta_bits 57 chunk_len_log2 3",
        "chunk_len_log2 8": "hnsw_create_compressed: offsets parameters base_bits 14 delta_bits 8 chunk_len_log2 8",
        "base_bits 0": "hnsw_create_compressed: offsets parameters base_bits 0 delta_bits 8 chunk_len_log2 3",
        "m 0": "hnsw_create_compressed: m 0 / m0 32",
        "offsets decrease": "hnsw_create_compressed: links offsets decrease",
        "offset past total_neighbors_bytes": "hnsw_create_compressed: a links offset lies past total_neighbors_bytes",
        "level offset >= length": "hnsw_create_compressed: level offset 3 (620) out of range",
        "level 0 not the first n entries": "hnsw_create_compressed: level offset 0 (1) out of range",
        "reindex out of range": "hnsw_create_compressed: a reindex entry is >= point_count",
        "CompressedWithVectors": "hnsw_create_compressed: CompressedWithVectors (inline storage) graphs are searched from the quantized vectors stored with the links (graph_layers.rs:336-388), a different algorithm; this loader takes GraphLinksFormat::Compressed",
        "m0 65": "hnsw_create_compressed: m 16 / m0 65 outside [1,64]",
    }
    for what, blob in bad.items():
        with pytest.raises(qb.QbError) as ei:
            qb.HnswGraph.from_compressed(st, blob)
        assert ei.value.status == -1, (what, str(ei.value))
        assert str(ei.value) == f"qb_status -1: {message[what]}", what
    with_vectors = patched(8, gl.VERSION_COMPRESSED_WITH_VECTORS.to_bytes(8, "little"))
    for what, blob in {"CompressedWithVectors": with_vectors, "m0 65": patched(51, (65).to_bytes(8, "little"))}.items():
        with pytest.raises(qb.QbError) as ei:
            qb.HnswGraph.from_compressed(st, blob)
        assert ei.value.status == -3, (what, str(ei.value))
        assert what != "CompressedWithVectors" or "CompressedWithVectors" in str(ei.value)
        assert str(ei.value) == f"qb_status -3: {message[what]}", what
    torch.cuda.synchronize()
    # the rebuilt file itself is valid: only the planted values were wrong
    hc = qb.HnswGraph.from_compressed(st, _rebuild(comp))
    hp = qb.HnswGraph(st, plain, m, m0)
    for a, b in zip(hc.search(base[:8], 10, 32, entry, lvl), hp.search(base[:8], 10, 32, entry, lvl)):
        assert np.array_equal(a, b)
    with pytest.raises(qb.QbError):
        hc.links(r.levels_count, [0])                              # no such level
    with pytest.raises(qb.QbError):
        hc.links(0, [n])                                           # no such point
    hc.close(); hp.close(); st.close(); g.close()
