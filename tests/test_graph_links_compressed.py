"""The compressed HNSW links format as the tests restate it (tests/graph_links_compressed.py): re-typed reference tests pin
the bit I/O, the links packer and the ordered offsets codec; writer -> independent reader round trips pin the file."""
import numpy as np
import pytest

from tests import graph_links_compressed as gl


def test_bit_io_known_answer():
    """bitpacking.rs:214-240 (test_simple)"""
    out = bytearray()
    w = gl.BitWriter(out)
    vals = [(0b01010, 5), (0b10110, 5), (0b10100, 5), (0b010110010, 9), (0b101100001, 9), (0b001001101, 9), (0x12345678, 32)]
    for v, b in vals:
        w.write(v, b)
    w.finish()
    assert len(out) == 10
    r = gl.BitReader(bytes(out))
    for v, b in vals:
        r.set_bits(b)
        assert r.read() == v


@pytest.mark.parametrize("case", ["only_unsorted", "only_sorted", "only_sorted_exact", "empty", "both"])
def test_pack_iterate_round_trip(case):
    """bitpacking_links.rs:234-302 (test_random): pack, iterate, and packed_links_size unchanged by trailing garbage"""
    rng = np.random.default_rng(42 + ["only_unsorted", "only_sorted", "only_sorted_exact", "empty", "both"].index(case))
    for _ in range(300):
        if case == "only_unsorted":
            sorted_count, total = 0, int(rng.integers(1, 100))
        elif case == "only_sorted":
            sorted_count = int(rng.integers(2, 100)); total = int(rng.integers(1, sorted_count))
        elif case == "only_sorted_exact":
            sorted_count = int(rng.integers(1, 100)); total = sorted_count
        elif case == "empty":
            sorted_count, total = int(rng.integers(0, 100)), 0
        else:
            sorted_count = int(rng.integers(0, 100)); total = int(rng.integers(sorted_count, sorted_count + 100))
        bpu = int(rng.integers(8, 33))
        raw = [int(x) for x in rng.choice(1 << min(bpu, 20), size=total, replace=False)] if total else []
        raw = [x << (bpu - min(bpu, 20)) for x in raw]               # unique values spread over [0, 2^bpu)
        packed, stored = gl.pack_links(raw, bpu, sorted_count)
        want = sorted(raw[:min(sorted_count, total)]) + raw[min(sorted_count, total):]
        assert stored == want
        assert gl.iterate_packed_links(packed, bpu, sorted_count) == want
        data = bytearray(packed)
        for _ in range(10):
            assert gl.packed_links_size(bytes(data), bpu, sorted_count, total) == len(packed)
            data.append(int(rng.integers(0, 256)))


def _sequences():
    rng = np.random.default_rng(42)
    out = [[], [0], [1], [gl.M64], [gl.M64, gl.M64], [0, gl.M64]]
    for max_delta, length in ((10, 1000), (20, 10_000), (10_000_000, 10_000), (0x123456789AB, 1000)):
        out.append([int(x) for x in np.cumsum(rng.integers(0, max_delta + 1, length, dtype=np.uint64), dtype=np.uint64)])
    out.append(sorted(int(x) for x in rng.integers(0, 2**63, 1000, dtype=np.uint64) * 2 + rng.integers(0, 2, 1000, dtype=np.uint64)))
    for k in range(1, 9):                                            # lengths 2^k +- 1 around every chunk length
        for length in ((1 << k) - 1, 1 << k, (1 << k) + 1):
            out.append([int(x) for x in np.cumsum(rng.integers(0, 300, length))])
    return out


@pytest.mark.parametrize("seq", range(len(_sequences())))
def test_offsets_compress_decompress_every_parameter_set(seq):
    """bitpacking_ordered.rs:343-407 (test_compress_decompress) over every chunk_len_log2 that try_all offers"""
    values = _sequences()[seq]
    params = gl.try_all(values)
    assert params and {p.chunk_len_log2 for p in params} <= set(range(8))
    for p in params:
        data = gl.compress_with_parameters(values, p)
        assert len(data) == p.compressed_size_bytes() and data.endswith(b"\xff" * 7)
        for i in range(len(values) - 1):
            assert gl.read_pair(data, p, i) == (values[i], values[i + 1])
        assert gl.read_pair(data, p, max(len(values) - 1, 0)) is None
    best = gl.find_best(values)
    assert best.compressed_size_bytes() == min(p.compressed_size_bytes() for p in params)


def test_offsets_every_chunk_length_is_reachable():
    values = [int(x) for x in np.cumsum(np.random.default_rng(1).integers(0, 90, 777))]
    assert sorted(p.chunk_len_log2 for p in gl.try_all(values)) == list(range(8))


LITERAL_GRAPHS = [
    [],
    [[[]], [[]]],
    [[[1]], [[0]]],
    [[[1, 2]], [[0, 2], [], [2]], [[0, 1], [], [1]]],
    [[[1, 2], [2], []], [[0, 2], [1], []], [[0, 1]]],
    [[[1, 2, 5, 6]], [[0, 2, 7, 8], [], [34, 45, 10]], [[0, 1, 1, 2], [3, 5, 9], [9, 8], [9], []], [[0, 1, 5, 6], [1, 5, 0]],
     [[0, 1, 9, 18], [1, 5, 6], [5], [9]]],
]


def _normalized(edges, m, m0):
    return [[gl.normalize_links(m0 if lvl == 0 else m, links) for lvl, links in enumerate(levels)] for levels in edges]


def _check_round_trip(edges, m, m0, log2=None):
    blob = gl.serialize_compressed(edges, m, m0, chunk_len_log2=log2)
    r = gl.CompressedLinks(blob)
    assert (r.point_count, r.m, r.m0) == (len(edges), m, m0)
    if log2 is not None:
        assert r.params.chunk_len_log2 == log2
    assert r.to_edges() == _normalized(edges, m, m0)
    return blob


@pytest.mark.parametrize("graph", range(len(LITERAL_GRAPHS)))
@pytest.mark.parametrize("m,m0", [(8, 8), (8, 16), (16, 8), (1, 1), (2, 3)])
def test_writer_reader_literal_graphs(graph, m, m0):
    """graph_links/tests.rs:181-211 for the compressed format"""
    _check_round_trip(LITERAL_GRAPHS[graph], m, m0)


@pytest.mark.parametrize("log2", [None, 0, 1, 2, 3, 4, 5, 6, 7])
def test_writer_reader_random_links(log2):
    """random_links-shaped graphs (tests.rs:59-80): 1000 points, up to 10 levels, up to 2 x level_m links, repeats"""
    rng = np.random.default_rng(7 + (log2 or 0))
    edges = gl.random_links(rng, 1000, 10, 8, 16)
    _check_round_trip(edges, 8, 16, log2)


def test_writer_reader_ids_beyond_point_count():
    rng = np.random.default_rng(3)
    edges = gl.random_links(rng, 200, 6, 4, 8)
    for levels in edges[::7]:
        levels[0] += [255, 201, 200]                                 # bits_per_unsorted is 8 at 200 points
    _check_round_trip(edges, 4, 8)


def test_plain_and_compressed_exports_describe_the_same_edges(oracle):
    rng = np.random.default_rng(5)
    base = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((3000, 24)).astype(np.float32))
    g = oracle.HNSW(base, oracle.COSINE, m=6, ef_construct=32, seed=2, threads=1)
    _, _, m, m0 = g.entry()
    plain = g.export_plain()
    n, lo, reindex, nb, off = gl.parse_plain(plain)
    r = gl.CompressedLinks(gl.plain_to_compressed(plain, m, m0))
    assert np.array_equal(r.reindex, reindex) and r.level_offsets[:-1] == [int(x) for x in lo] and r.level_offsets[-1] == off.size - 1
    for p in range(n):
        for lvl in range(r.point_level(p) + 1):
            idx = p if lvl == 0 else int(lo[lvl]) + int(reindex[p])
            want = [int(x) for x in nb[int(off[idx]):int(off[idx + 1])]]
            assert r.links(p, lvl) == gl.normalize_links(r.level_m(lvl), want)
    g.close()
