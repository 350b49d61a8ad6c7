"""ctypes driver of tests/sparse_custom_ref.c, the checker of the device's custom queries over a sparse vector storage: score_vectors,
the points peek_top_iter scores, the (score desc, id asc) top-k and the counters restated in C; the per-example similarities are folded by
the oracle's Query::score_by (custom_combine / feedback_score).  The library is compiled on first use into a per-user temporary directory
keyed by the source's hash, so a read-only checkout works too."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

SCORED = np.dtype([("idx", np.uint32), ("score", np.float32)])
FEEDBACK = 5

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sparse_custom_ref.c")
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        src = open(_SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), f"qb_sparse_custom_ref_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libsparsecustomref_{hashlib.sha256(src).hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            # no contraction: every product and sum of score_vectors rounds as in the reference
            subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-fvisibility=hidden", "-o", tmp, _SRC], check=True, capture_output=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u64p = C.c_void_p, C.POINTER(C.c_uint64)
        L.scr_storage_new.restype = vp
        L.scr_storage_new.argtypes = [C.c_uint32, vp, vp, vp, C.c_int]
        L.scr_storage_free.argtypes = [vp]
        L.scr_score.restype = C.c_float
        L.scr_score.argtypes = [vp, vp, C.c_uint32, vp, vp, C.c_uint32, C.POINTER(C.c_int)]
        L.scr_sims.argtypes = [vp, C.c_uint32, vp, vp, vp, vp, C.c_uint64, vp]
        L.scr_points.restype = C.c_uint64
        L.scr_points.argtypes = [vp, vp, vp, C.c_uint64, vp]
        L.scr_counters.argtypes = [vp, vp, C.c_uint64, C.c_uint32, vp, u64p, u64p]
        L.scr_topk.restype = C.c_uint64
        L.scr_topk.argtypes = [vp, vp, C.c_uint64, C.c_uint32, vp, vp]
        _LIB = L
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def score(a, b):
    """score_vectors(a, b) for two (dims, weights) pairs -> the score, or None when no dim is shared (the reference's Option)"""
    ad, aw = np.ascontiguousarray(a[0], np.uint32), np.ascontiguousarray(a[1], np.float32)
    bd, bw = np.ascontiguousarray(b[0], np.uint32), np.ascontiguousarray(b[1], np.float32)
    ov = C.c_int(0)
    s = lib().scr_score(_p(ad), _p(aw), ad.size, _p(bd), _p(bw), bd.size, C.byref(ov))
    return float(np.float32(s)) if ov.value else None


def examples_csr(examples):
    """a list of (dims, weights) pairs -> (offsets u64, dims u32, weights f32)"""
    ptr = np.zeros(len(examples) + 1, np.uint64)
    ptr[1:] = np.cumsum([len(d) for d, _ in examples])
    dims = np.ascontiguousarray(np.concatenate([np.asarray(d, np.uint32) for d, _ in examples]) if examples else np.zeros(0, np.uint32), np.uint32)
    w = np.ascontiguousarray(np.concatenate([np.asarray(x, np.float32) for _, x in examples]) if examples else np.zeros(0, np.float32), np.float32)
    return ptr, dims, w


def fold(o, kind: int, n_a: int, n_b: int, sims, coef=None) -> np.ndarray:
    """Query::score_by of every column of the E x N similarity matrix, by the oracle"""
    if sims.shape[1] == 0:
        return np.zeros(0, np.float32)
    if kind == FEEDBACK:
        c = np.asarray(coef, np.float32).reshape(-1)
        return o.feedback_score(float(c[0]), c[1:], sims)
    return o.custom_combine(kind, n_a, n_b, sims)


class Storage:
    """The reference's sparse vector storage over CSR rows (point r = dims / weights [indptr[r], indptr[r + 1]), user dims)"""

    def __init__(self, indptr, dims, weights, on_disk: bool = False):
        self.indptr = np.ascontiguousarray(indptr, np.uint64)
        self.dims = np.ascontiguousarray(dims, np.uint32)
        self.weights = np.ascontiguousarray(weights, np.float32)
        self.n_points = self.indptr.size - 1
        self.h = lib().scr_storage_new(self.n_points, _p(self.indptr), _p(self.dims), _p(self.weights), int(bool(on_disk)))

    def close(self):
        if self.h:
            lib().scr_storage_free(self.h)
            self.h = None

    def points(self, deleted=None, id_list=None) -> np.ndarray:
        """the ids peek_top_iter scores; deleted = 64-bit words (bit = 1 deleted)"""
        dl = None if deleted is None else np.ascontiguousarray(deleted, np.uint64)
        il = None if id_list is None else np.ascontiguousarray(id_list, np.uint32)
        out = np.zeros(max(self.n_points if il is None else il.size, 1), np.uint32)
        n = lib().scr_points(self.h, _p(dl), _p(il), 0 if il is None else il.size, _p(out))
        return out[:n].copy()

    def sims(self, examples, ids) -> np.ndarray:
        """E x N: similarity of each listed point to each example (a list of (dims, weights) pairs)"""
        ptr, d, w = examples_csr(examples)
        ids = np.ascontiguousarray(ids, np.uint32)
        out = np.zeros((len(examples), ids.size), np.float32)
        lib().scr_sims(self.h, len(examples), _p(ptr), _p(d), _p(w), _p(ids), ids.size, _p(out))
        return out

    def counters(self, examples, ids) -> tuple[int, int]:
        ptr, _, _ = examples_csr(examples)
        ids = np.ascontiguousarray(ids, np.uint32)
        cpu, io = C.c_uint64(0), C.c_uint64(0)
        lib().scr_counters(self.h, _p(ids), ids.size, len(examples), _p(ptr), C.byref(cpu), C.byref(io))
        return int(cpu.value), int(io.value)

    def scores(self, o, kind: int, n_a: int, n_b: int, examples, ids, coef=None) -> np.ndarray:
        """score_stored_batch of one query over ids"""
        return fold(o, kind, n_a, n_b, self.sims(examples, ids), coef)

    def search(self, o, kind: int, n_a: int, n_b: int, examples, top: int, coef=None, deleted=None, id_list=None):
        """search_scored of one query -> (SCORED array in (score desc, id asc) order, cpu, vector_io_read)"""
        ids = self.points(deleted, id_list)
        sc = np.ascontiguousarray(self.scores(o, kind, n_a, n_b, examples, ids, coef), np.float32)
        oi, os_ = np.zeros(max(top, 1), np.uint32), np.zeros(max(top, 1), np.float32)
        n = lib().scr_topk(_p(ids), _p(sc), ids.size, top, _p(oi), _p(os_))
        out = np.zeros(n, SCORED)
        out["idx"], out["score"] = oi[:n], os_[:n]
        cpu, io = self.counters(examples, ids)
        return out, cpu, io


def random_rows(rng, n_points: int, mean_nnz: float, dim_pool, negative: float = 0.0, empty: float = 0.0):
    """CSR rows over user dims drawn from dim_pool (u32, any values): about mean_nnz distinct dims per row in shuffled order, weights in
    [0.01, 1.01) with a `negative` share negated; an `empty` share of rows has no element"""
    pool = np.asarray(dim_pool, np.uint32)
    counts = np.minimum(rng.poisson(mean_nnz, n_points), pool.size)
    counts[rng.random(n_points) < empty] = 0
    dims = np.concatenate([rng.choice(pool, size=c, replace=False) for c in counts]).astype(np.uint32) if counts.sum() else np.zeros(0, np.uint32)
    indptr = np.zeros(n_points + 1, np.uint64)
    indptr[1:] = np.cumsum(counts)
    w = rng.random(dims.size).astype(np.float32) + np.float32(0.01)
    if negative:
        w[rng.random(dims.size) < negative] *= -1
    return indptr, dims, w
