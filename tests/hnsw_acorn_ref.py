"""ctypes driver of tests/hnsw_acorn_ref.c: the CPU traversal of a plain links.bin with either level-0 algorithm of
GraphLayers::search (HNSW = 0, ACORN-1 = 1).  The library is compiled on first use into a per-user temporary directory
keyed by the source's hash, so a read-only checkout works too."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HNSW, ACORN = 0, 1
SCORED = np.dtype([("idx", np.uint32), ("score", np.float32)])
SCORE_CB = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(C.c_float))

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hnsw_acorn_ref.c")
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        src = open(_SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), f"qb_acorn_ref_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libacornref_{hashlib.sha256(src).hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            # the oracle's flags (oracle/Makefile): no contraction, so scores through the callback path are the scorer's own
            subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-fvisibility=hidden", "-o", tmp, _SRC, "-lm", "-lpthread"],
                           check=True, capture_output=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32p, u64p, f32p = C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_float)
        L.qa_graph_load.restype, L.qa_graph_load.argtypes = vp, [vp, C.c_uint64, C.c_uint32, C.c_uint32]
        L.qa_graph_free.restype, L.qa_graph_free.argtypes = None, [vp]
        L.qa_search_cb.restype = C.c_uint32
        L.qa_search_cb.argtypes = [vp, C.c_int, C.c_uint32, C.c_uint32, vp, vp, vp, C.c_uint32, C.c_uint32, vp, u64p]
        L.qa_search_batch.restype = None
        L.qa_search_batch.argtypes = [vp, C.c_int, C.c_uint32, C.c_uint32, f32p, C.c_uint32, f32p, C.c_uint32, C.c_int, vp, vp,
                                      C.c_uint32, C.c_uint32, C.c_uint32, vp, u32p, u64p]
        _LIB = L
    return _LIB


def _bitmap(filtered, n):
    """bool[n] (True = fails the filter) or a packed u64 bitmap -> contiguous u64 words, or None"""
    if filtered is None:
        return None
    f = np.asarray(filtered)
    if f.dtype == np.bool_:
        words = np.zeros((n + 63) // 64, np.uint64)
        idx = np.flatnonzero(f).astype(np.uint64)
        np.bitwise_or.at(words, (idx >> np.uint64(6)).astype(np.int64), np.uint64(1) << (idx & np.uint64(63)))
        return words
    return np.ascontiguousarray(f, dtype=np.uint64)


class Graph:
    """A plain links.bin held on the host; search_batch() scores with the oracle's f32 similarity, search() with a callable
    ids -> scores.  stats() = (scorer calls with n > 0, scored points, max hop1 / hop2 visited-list entries of one search)."""

    def __init__(self, links_bin, m: int, m0: int, n_points: int):
        blob = np.ascontiguousarray(links_bin, dtype=np.uint8)
        self.n = n_points
        self._g = lib().qa_graph_load(blob.ctypes.data_as(C.c_void_p), blob.size, m, m0)
        assert self._g, "malformed links.bin"
        self._stats = np.zeros(4, np.uint64)

    def search_batch(self, oracle, base, distance: int, queries_pre, top: int, ef: int, entry: int, entry_level: int, algo: int = ACORN,
                     filtered=None, threads: int = 1):
        base = np.ascontiguousarray(base, dtype=np.float32)
        q = np.ascontiguousarray(np.atleast_2d(queries_pre), dtype=np.float32)
        nq = q.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED)
        counts = np.zeros(nq, dtype=np.uint32)
        bm = _bitmap(filtered, self.n)
        sim = C.cast(oracle.lib().qo_similarity_f32, C.c_void_p)
        lib().qa_search_batch(self._g, algo, entry, entry_level, q.ctypes.data_as(C.POINTER(C.c_float)), nq,
                              base.ctypes.data_as(C.POINTER(C.c_float)), base.shape[1], distance, sim,
                              None if bm is None else bm.ctypes.data_as(C.c_void_p), top, ef, threads, out.ctypes.data_as(C.c_void_p),
                              counts.ctypes.data_as(C.POINTER(C.c_uint32)), self._stats.ctypes.data_as(C.POINTER(C.c_uint64)))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def search(self, score_points, top: int, ef: int, entry: int, entry_level: int, algo: int = ACORN, filtered=None):
        def _cb(user, ids, n, scores):
            np.ctypeslib.as_array(scores, shape=(n,))[:] = score_points(np.ctypeslib.as_array(ids, shape=(n,)).copy())

        cb = SCORE_CB(_cb)
        out = np.zeros(max(top, 1), dtype=SCORED)
        bm = _bitmap(filtered, self.n)
        n = lib().qa_search_cb(self._g, algo, entry, entry_level, C.cast(cb, C.c_void_p), None, None if bm is None else bm.ctypes.data_as(C.c_void_p),
                               top, ef, out.ctypes.data_as(C.c_void_p), self._stats.ctypes.data_as(C.POINTER(C.c_uint64)))
        return out[:n].copy()

    def stats(self, reset: bool = True):
        s = tuple(int(x) for x in self._stats)
        if reset:
            self._stats[:] = 0
        return s

    def close(self):
        if self._g:
            lib().qa_graph_free(self._g)
            self._g = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
