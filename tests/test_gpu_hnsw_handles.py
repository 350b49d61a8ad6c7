"""What every HNSW loader and device build makes of one input, pinned exactly:

1. The plain loader (qb_hnsw_create_plain) refuses malformed files with these statuses and messages, and the multivector loaders refuse a
   graph whose point count is not the collection's.
2. One seeded graph through each loader and build gives these info() triples (points, levels, HBM bytes) and launches this many kernels.

Every case ends with the device usable."""
import numpy as np
import pytest

from tests import graph_links_compressed as gl
from tests import graph_links_with_vectors as gv

pytestmark = pytest.mark.gpu

N, DIM, M, M0 = 300, 16, 8, 16


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


class _Fixture:
    """a graph over N points built by the oracle, its plain / compressed / inline-vector files, the storages and a multivector view"""

    def __init__(self, qb, oracle):
        rng = np.random.default_rng(7)
        self.base = rng.standard_normal((N, DIM)).astype(np.float32)
        g = oracle.HNSW(self.base, oracle.DOT, m=M, ef_construct=32, seed=5, threads=1)
        self.entry, self.level, m, m0 = g.entry()
        assert (m, m0) == (M, M0)
        self.plain = np.asarray(g.export_plain(), np.uint8)
        g.close()
        self.comp = gl.plain_to_compressed(self.plain, M, M0)
        self.st = qb.DenseVectorStorage(self.base, qb.Distance.Dot)
        dt, inv = qb.construct_vector_parameters(qb.Distance.Dot)
        self.sq = oracle.SQ8.encode(self.base, int(dt), bool(inv))
        self.sqst = qb.ScalarQuantizedVectors(self.sq.rows, DIM, self.sq.meta.alpha, self.sq.meta.offset, self.sq.meta.multiplier, qb.Distance.Dot)
        self.inline = gv.serialize_with_vectors(gv.edges_of_plain(self.plain), M, M0, lambda i: self.base[i].tobytes(),
                                                lambda i: self.sq.rows[i].tobytes(), (DIM * 4, 4), (self.sq.row_bytes, 1))
        # N points of 1-4 tokens each over a token storage
        runs = rng.integers(1, 5, N)
        self.off = np.concatenate([[0], np.cumsum(runs)]).astype(np.uint32)
        self.tokens = qb.DenseVectorStorage(rng.standard_normal((int(self.off[-1]), DIM)).astype(np.float32), qb.Distance.Dot)
        self.view = qb.MultiVectorView(self.tokens, self.off)
        self.old = qb.HnswGraph(self.st, self.plain, M, M0)   # the old graph of the incremental build

    def close(self):
        self.old.close(); self.st.close(); self.sqst.close(); self.tokens.close()


@pytest.fixture(scope="module")
def fx(qb, oracle):
    f = _Fixture(qb, oracle)
    yield f
    f.close()


def _patched(blob, offset, value):
    b = bytearray(blob)
    b[offset:offset + 8] = int(value).to_bytes(8, "little")
    return np.frombuffer(bytes(b), np.uint8)


def refusal_cases(qb, fx):
    """name -> a call that must raise"""
    p = fx.plain
    levels, n_off = int(p[8:16].view(np.uint64)[0]), int(p[24:32].view(np.uint64)[0])
    assert levels > 1
    short_view = qb.MultiVectorView(fx.tokens, fx.off[:-1])
    return {
        "shorter than 64 bytes": lambda: qb.HnswGraph(fx.st, p[:40], M, M0),
        "header describes more bytes": lambda: qb.HnswGraph(fx.st, p[:-1], M, M0),
        "padding 8": lambda: qb.HnswGraph(fx.st, _patched(p, 32, 8), M, M0),
        "65 levels": lambda: qb.HnswGraph(fx.st, _patched(p, 8, 65), M, M0),
        "offsets count <= n": lambda: qb.HnswGraph(fx.st, _patched(p, 24, N), M, M0),
        "level offset >= offsets count": lambda: qb.HnswGraph(fx.st, _patched(p, 64 + 8 * (levels - 1), n_off), M, M0),
        "wrong point count": lambda: qb.HnswGraph(fx.st, _patched(p, 0, N - 1), M, M0),
        "m 0": lambda: qb.HnswGraph(fx.st, p, 0, M0),
        "m0 65": lambda: qb.HnswGraph(fx.st, p, M, 65),
        "plain multivector, other point count": lambda: qb.HnswGraph.multivector(short_view, p, M, M0),
        "compressed multivector, other point count": lambda: qb.HnswGraph.from_compressed_multivector(short_view, fx.comp),
    }


REFUSALS = {
    "shorter than 64 bytes": (-1, "qb_status -1: hnsw_create_plain: 40 bytes is smaller than HeaderPlain"),
    "header describes more bytes": (-1, "qb_status -1: hnsw_create_plain: 20063 bytes, header describes 20064"),
    "padding 8": (-1, "qb_status -1: hnsw_create_plain: offsets padding 8"),
    "65 levels": (-1, "qb_status -1: hnsw_create_plain: bad header (levels 65, offsets 407)"),
    "offsets count <= n": (-1, "qb_status -1: hnsw_create_plain: bad header (levels 5, offsets 300)"),
    "level offset >= offsets count": (-1, "qb_status -1: hnsw_create_plain: level offset 4 out of range"),
    "wrong point count": (-1, "qb_status -1: hnsw_create_plain: graph has 299 points, storage 300"),
    "m 0": (-3, "qb_status -3: hnsw_create_plain: m 0 / m0 16 outside [1,64]"),
    "m0 65": (-3, "qb_status -3: hnsw_create_plain: m 8 / m0 65 outside [1,64]"),
    "plain multivector, other point count": (-1, "qb_status -1: hnsw_create_plain: graph has 300 points, collection 299"),
    "compressed multivector, other point count": (-1, "qb_status -1: hnsw_create_compressed: graph has 300 points, collection 299"),
}


def handle_cases(qb, fx):
    """name -> a call that returns a handle"""
    o2n = np.where(np.arange(N) % 10 == 3, -1, np.arange(N))   # every tenth point gone, the others kept in place
    return {
        "plain": lambda: qb.HnswGraph(fx.st, fx.plain, M, M0),
        "compressed": lambda: qb.HnswGraph.from_compressed(fx.st, fx.comp),
        "with vectors": lambda: qb.HnswGraph.from_compressed_with_vectors(fx.sqst, fx.inline),
        "plain multivector": lambda: qb.HnswGraph.multivector(fx.view, fx.plain, M, M0),
        "compressed multivector": lambda: qb.HnswGraph.from_compressed_multivector(fx.view, fx.comp),
        "build": lambda: qb.HnswGraph.build(fx.st, m=M, ef_construct=32, seed=3, batch=64, serial_points=16),
        "build multivector": lambda: qb.HnswGraph.build_multivector(fx.view, m=M, ef_construct=32, seed=3, batch=64, serial_points=16),
        "build incremental": lambda: qb.HnswGraph.build_incremental(fx.st, fx.old, o2n, ef_construct=32, seed=3, batch=64, serial_points=16),
    }


# name -> (info(), kernels launched by the call)
HANDLES = {
    "plain": ((300, 5, 39196), 1),
    "compressed": ((300, 5, 41596), 6),
    "with vectors": ((300, 5, 151513), 6),
    "plain multivector": ((300, 5, 40400), 1),
    "compressed multivector": ((300, 5, 42800), 6),
    "build": ((300, 5, 38992), 149),
    "build multivector": ((300, 5, 40376), 149),
    "build incremental": ((300, 4, 39904), 123),
}


def _launches(qb):
    from qdrant_b200._capi import lib

    return int(lib().qb_kernel_launch_count())


def _device_usable(qb, fx):
    import torch

    torch.cuda.synchronize()
    h = qb.HnswGraph(fx.st, fx.plain, M, M0)
    assert h.search(fx.base[:4], 5, 16, fx.entry, fx.level)[0].size == 5
    h.close()


@pytest.mark.parametrize("what", sorted(REFUSALS))
def test_refusals_keep_their_status_and_message(qb, fx, what):
    with pytest.raises(qb.QbError) as ei:
        refusal_cases(qb, fx)[what]()
    assert (ei.value.status, str(ei.value)) == REFUSALS[what]
    _device_usable(qb, fx)


@pytest.mark.parametrize("what", sorted(HANDLES))
def test_handles_keep_their_info_and_launches(qb, fx, what):
    make = handle_cases(qb, fx)[what]
    before = _launches(qb)
    h = make()
    launched = _launches(qb) - before
    assert (h.info(), launched) == HANDLES[what]
    h.close()
    _device_usable(qb, fx)
