"""ctypes driver of tests/hnsw_custom_ref.c, the checker of qb_hnsw_search_custom_batch / qb_hnsw_search_discover_batch: the CPU
traversal of a plain links.bin with a custom scorer (E similarities through the oracle's qo_similarity_f32, folded by its
qo_custom_score / qo_feedback_score), custom entry points, and the keyed tie order; plus discover restated in Python as the reference's
two stages (discover_search_with_graph, hnsw/read_view/search.rs:314-349).  The library is compiled on first use into a per-user
temporary directory keyed by the source's hash, so a read-only checkout works too."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tests.hnsw_acorn_ref import ACORN, HNSW, SCORE_CB, SCORED, _bitmap

FEEDBACK = 5                      # QB_QUERY_FEEDBACK_NAIVE
DISCOVERY_ENTRY_POINT_COUNT = 10  # search.rs:325

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hnsw_custom_ref.c")
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        src = open(_SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), f"qb_custom_ref_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libcustomref_{hashlib.sha256(src).hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            # the oracle's flags (oracle/Makefile): no contraction, so the folds are the oracle's own
            subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-fvisibility=hidden", "-o", tmp, _SRC, "-lm", "-lpthread"],
                           check=True, capture_output=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32p, u64p, f32p = C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_float)
        L.qc_graph_load.restype, L.qc_graph_load.argtypes = vp, [vp, C.c_uint64, C.c_uint32, C.c_uint32]
        L.qc_graph_free.restype, L.qc_graph_free.argtypes = None, [vp]
        L.qc_get_entry_point.restype, L.qc_get_entry_point.argtypes = C.c_int, [vp, vp, u32p, C.c_uint32, C.c_uint32, C.c_uint32, u32p]
        L.qc_search_cb.restype = C.c_uint32
        L.qc_search_cb.argtypes = [vp, C.c_int, C.c_int, C.c_uint32, C.c_uint32, u32p, C.c_uint32, vp, vp, vp, C.c_uint32, C.c_uint32, vp, u64p]
        L.qc_search_custom_batch.restype = None
        L.qc_search_custom_batch.argtypes = [vp, C.c_int, C.c_int, C.c_uint32, C.c_uint32, f32p, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32,
                                             vp, vp, vp, vp, vp, C.c_uint32, f32p, C.c_uint32, C.c_int, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32,
                                             vp, u32p, u64p]
        _LIB = L
    return _LIB


class Graph:
    """A plain links.bin held on the host.  stats() = (scorer calls with n > 0, scored points, max hop1 / hop2 visited-list entries of
    one search), summed since the last reset."""

    def __init__(self, links_bin, m: int, m0: int, n_points: int):
        blob = np.ascontiguousarray(links_bin, dtype=np.uint8)
        self.n = n_points
        self._g = lib().qc_graph_load(blob.ctypes.data_as(C.c_void_p), blob.size, m, m0)
        assert self._g, "malformed links.bin"
        self._stats = np.zeros(4, np.uint64)

    def stats(self, reset: bool = True):
        s = tuple(int(x) for x in self._stats)
        if reset:
            self._stats[:] = 0
        return s

    def close(self):
        if self._g:
            lib().qc_graph_free(self._g)
            self._g = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def n_examples(kind: int, n_a: int, n_b: int) -> int:
    return {1: n_a + n_b, 2: n_a + n_b, 3: 1 + 2 * n_a, 4: 2 * n_a, FEEDBACK: 1 + 2 * n_a}[kind]


def _cep(cep, nq):
    """list (one array of ids per query) -> ([nq, width] u32, counts u32, width), or Nones"""
    if cep is None:
        return None, None, 0
    width = max(1, max((len(c) for c in cep), default=1))
    arr = np.zeros((nq, width), np.uint32)
    counts = np.zeros(nq, np.uint32)
    for i, c in enumerate(cep):
        arr[i, : len(c)] = c
        counts[i] = len(c)
    return arr, counts, width


def get_entry_point(graph: Graph, cep, entry: int, entry_level: int, filtered=None):
    """GraphLayers::get_entry_point: (entry, level, taken from the custom list)"""
    ids = np.ascontiguousarray(cep, dtype=np.uint32)
    out = np.zeros(2, np.uint32)
    bm = _bitmap(filtered, graph.n)
    r = lib().qc_get_entry_point(graph._g, None if bm is None else bm.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.POINTER(C.c_uint32)), ids.size,
                                 entry, entry_level, out.ctypes.data_as(C.POINTER(C.c_uint32)))
    return int(out[0]), int(out[1]), bool(r)


def search_custom_batch(graph: Graph, oracle, base, distance: int, examples_pre, kind: int, n_a: int, n_b: int, top: int, ef: int, entry: int,
                        entry_level: int, algo: int = HNSW, filtered=None, coef=None, cep=None, keyed: bool = True, threads: int = 4):
    """examples_pre: [nq, E, dim] preprocessed examples in the qb_scorer_create_custom layout; coef: [nq, 1 + n_a] for feedback;
    cep: one array of custom entry points per query, or None"""
    base = np.ascontiguousarray(base, dtype=np.float32)
    ex = np.ascontiguousarray(examples_pre, dtype=np.float32)
    nq, ne, dim = ex.shape
    assert ne == n_examples(kind, n_a, n_b) and dim == base.shape[1]
    cf = None if coef is None else np.ascontiguousarray(coef, dtype=np.float32).reshape(nq, 1 + n_a)
    arr, counts, width = _cep(cep, nq)
    out = np.zeros((nq, max(top, 1)), dtype=SCORED)
    cnt = np.zeros(nq, dtype=np.uint32)
    bm = _bitmap(filtered, graph.n)
    ol = oracle.lib()
    vp = C.c_void_p
    lib().qc_search_custom_batch(graph._g, algo, 1 if keyed else 0, entry, entry_level, ex.ctypes.data_as(C.POINTER(C.c_float)), ne, nq, kind, n_a, n_b,
                                 None if cf is None else cf.ctypes.data_as(vp), C.cast(ol.qo_custom_score, vp), C.cast(ol.qo_feedback_score, vp),
                                 None if arr is None else arr.ctypes.data_as(vp), None if counts is None else counts.ctypes.data_as(vp), width,
                                 base.ctypes.data_as(C.POINTER(C.c_float)), dim, distance, C.cast(ol.qo_similarity_f32, vp),
                                 None if bm is None else bm.ctypes.data_as(vp), top, ef, threads, out.ctypes.data_as(vp),
                                 cnt.ctypes.data_as(C.POINTER(C.c_uint32)), graph._stats.ctypes.data_as(C.POINTER(C.c_uint64)))
    return [out[i, : cnt[i]].copy() for i in range(nq)]


def search_cb(graph: Graph, score_points, top: int, ef: int, entry: int, entry_level: int, algo: int = HNSW, filtered=None, cep=None,
              keyed: bool = True):
    """one search scored through a callable ids -> scores (e.g. qb_score_points on a custom scorer)"""
    def _cb(user, ids, n, scores):
        np.ctypeslib.as_array(scores, shape=(n,))[:] = score_points(np.ctypeslib.as_array(ids, shape=(n,)).copy())

    cb = SCORE_CB(_cb)
    ids = None if cep is None else np.ascontiguousarray(cep, dtype=np.uint32)
    out = np.zeros(max(top, 1), dtype=SCORED)
    bm = _bitmap(filtered, graph.n)
    n = lib().qc_search_cb(graph._g, algo, 1 if keyed else 0, entry, entry_level, None if ids is None else ids.ctypes.data_as(C.POINTER(C.c_uint32)),
                              0 if ids is None else ids.size, C.cast(cb, C.c_void_p), None, None if bm is None else bm.ctypes.data_as(C.c_void_p),
                              top, ef, out.ctypes.data_as(C.c_void_p), graph._stats.ctypes.data_as(C.POINTER(C.c_uint64)))
    return out[:n].copy()


def discover(graph: Graph, oracle, base, distance: int, examples_pre, n_pairs: int, top: int, ef: int, entry: int, entry_level: int,
             algo: int = HNSW, filtered=None, keyed: bool = True, threads: int = 4):
    """discover_search_with_graph (search.rs:314-349): a context search over the pairs for the 10 best points, then the discover
    search from them as custom entry points.  examples_pre: [nq, 1 + 2 n_pairs, dim] (target, then the pairs)."""
    ex = np.ascontiguousarray(examples_pre, dtype=np.float32)
    stage1 = search_custom_batch(graph, oracle, base, distance, ex[:, 1:], 4, n_pairs, 0, DISCOVERY_ENTRY_POINT_COUNT, ef, entry, entry_level, algo,
                                 filtered, keyed=keyed, threads=threads)
    return search_custom_batch(graph, oracle, base, distance, ex, 3, n_pairs, 0, top, ef, entry, entry_level, algo, filtered,
                               cep=[s["idx"].copy() for s in stage1], keyed=keyed, threads=threads)
