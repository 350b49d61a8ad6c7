"""ctypes driver of tests/sparse_ref.c, the checker of the device sparse index: the reference's PostingBuilder, TopK and SearchContext
(search with its pruning, plain_search) restated in C.  The library is compiled on first use into a per-user temporary directory keyed by
the source's hash, so a read-only checkout works too."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

SCORED = np.dtype([("idx", np.uint32), ("score", np.float32)])

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sparse_ref.c")
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        src = open(_SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), f"qb_sparse_ref_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libsparseref_{hashlib.sha256(src).hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            # no contraction: weight * query_weight and every sum round as in the reference
            subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-fvisibility=hidden", "-o", tmp, _SRC], check=True, capture_output=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32p, f32p, u64p = C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_uint64)
        L.sr_index_new.restype = vp
        L.sr_index_new.argtypes = [C.c_uint32, C.c_uint32, vp, vp, vp]
        L.sr_index_free.argtypes = [vp]
        L.sr_ctx_new.restype = vp
        L.sr_ctx_new.argtypes = [vp, vp, vp, C.c_uint32, C.c_uint32, C.c_int, C.c_int]
        L.sr_ctx_free.argtypes = [vp]
        L.sr_ctx_list_len.restype = C.c_uint32
        L.sr_ctx_list_len.argtypes = [vp, C.c_uint32]
        L.sr_ctx_list_dim.restype = C.c_uint32
        L.sr_ctx_list_dim.argtypes = [vp, C.c_uint32]
        L.sr_ctx_promote.argtypes = [vp]
        L.sr_ctx_prune.restype = C.c_int
        L.sr_ctx_prune.argtypes = [vp, C.c_float]
        L.sr_ctx_search.restype = C.c_uint32
        L.sr_ctx_search.argtypes = [vp, vp, vp, vp, u64p]
        L.sr_ctx_plain.restype = C.c_uint32
        L.sr_ctx_plain.argtypes = [vp, vp, vp, vp, C.c_uint32, vp, vp, u64p]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def remap(dims, weights, n_dims: int):
    """RemappedSparseVector of a query: the dims the index knows (< n_dims), sorted by dim"""
    d = np.asarray(dims, np.uint32)
    w = np.asarray(weights, np.float32)
    keep = d < n_dims
    o = np.argsort(d[keep], kind="stable")
    return np.ascontiguousarray(d[keep][o]), np.ascontiguousarray(w[keep][o])


class Index:
    """The reference's inverted index over CSR rows (point r = dims / weights [indptr[r], indptr[r + 1]))"""

    def __init__(self, indptr, dims, weights, n_dims: int):
        self.indptr = np.ascontiguousarray(indptr, np.uint64)
        self.dims = np.ascontiguousarray(dims, np.uint32)
        self.weights = np.ascontiguousarray(weights, np.float32)
        self.n_points, self.n_dims = self.indptr.size - 1, n_dims
        self.h = lib().sr_index_new(self.n_points, n_dims, _p(self.indptr), _p(self.dims), _p(self.weights))

    def close(self):
        if self.h:
            lib().sr_index_free(self.h)
            self.h = None

    def context(self, dims, weights, top: int, reliable: bool = True, keyed: bool = True):
        """SearchContext::new over an already remapped query"""
        return Context(self, np.ascontiguousarray(dims, np.uint32), np.ascontiguousarray(weights, np.float32), top, reliable, keyed)

    def search(self, dims, weights, top: int, reliable: bool = True, deleted=None, keyed: bool = True):
        """one query (user dims: remapped here) -> (SCORED array, cpu units)"""
        c = self.context(*remap(dims, weights, self.n_dims), top, reliable, keyed)
        try:
            return c.search(deleted)
        finally:
            c.close()

    def plain(self, dims, weights, ids, top: int, keyed: bool = True):
        c = self.context(*remap(dims, weights, self.n_dims), top, True, keyed)
        try:
            return c.plain(ids)
        finally:
            c.close()


class Context:
    def __init__(self, index: Index, d, w, top, reliable, keyed):
        self.d, self.w, self.top = d, w, top
        self.h = lib().sr_ctx_new(index.h, _p(d), _p(w), d.size, top, int(reliable), int(keyed))

    def close(self):
        if self.h:
            lib().sr_ctx_free(self.h)
            self.h = None

    def list_len(self, i: int) -> int:
        return lib().sr_ctx_list_len(self.h, i)

    def list_dim(self, i: int) -> int:
        return lib().sr_ctx_list_dim(self.h, i)

    def promote(self):
        lib().sr_ctx_promote(self.h)

    def prune(self, min_score: float) -> bool:
        return bool(lib().sr_ctx_prune(self.h, C.c_float(min_score)))

    def _out(self, n, ids, sc):
        o = np.zeros(n, SCORED)
        o["idx"], o["score"] = ids[:n], sc[:n]
        return o

    def search(self, deleted=None):
        ids, sc, cpu = np.zeros(max(self.top, 1), np.uint32), np.zeros(max(self.top, 1), np.float32), C.c_uint64(0)
        dl = None if deleted is None else np.ascontiguousarray(deleted, np.uint64)
        n = lib().sr_ctx_search(self.h, None if dl is None else _p(dl), _p(ids), _p(sc), C.byref(cpu))
        return self._out(n, ids, sc), int(cpu.value)

    def plain(self, point_ids):
        pid = np.ascontiguousarray(point_ids, np.uint32)
        ids, sc, cpu = np.zeros(max(self.top, 1), np.uint32), np.zeros(max(self.top, 1), np.float32), C.c_uint64(0)
        n = lib().sr_ctx_plain(self.h, _p(self.d), _p(self.w), _p(pid), pid.size, _p(ids), _p(sc), C.byref(cpu))
        return self._out(n, ids, sc), int(cpu.value)


def deleted_bitmap(deleted_mask):
    """bool mask (True = deleted) -> the 64-bit words the library and the checker take"""
    m = np.asarray(deleted_mask, bool)
    bits = np.zeros(((m.size + 63) // 64) * 64, np.uint8)
    bits[: m.size] = m
    return np.packbits(bits, bitorder="little").view(np.uint64).copy()


def random_csr(rng, n_points: int, n_dims: int, mean_nnz: float, zipf: float = 1.1, negative: float = 0.0, id_gap: int = 1):
    """Random sparse rows: about mean_nnz dims per row drawn Zipf-like over n_dims (hot dims have long lists; a dim drawn twice in a row
    is kept once), weights in [0.01, 1.01) with a `negative` share of them negated, each row's dims shuffled.  id_gap > 1 leaves all rows
    but every id_gap-th empty, so the ids span more batches."""
    p = 1.0 / np.arange(1, n_dims + 1) ** zipf
    p /= p.sum()
    counts = rng.poisson(mean_nnz, n_points)
    counts[np.arange(n_points) % id_gap != 0] = 0
    rows = np.repeat(np.arange(n_points, dtype=np.uint64), counts)
    keys = np.unique(rows * np.uint64(n_dims) + rng.choice(n_dims, size=rows.size, p=p).astype(np.uint64))
    rows, dims = keys // np.uint64(n_dims), (keys % np.uint64(n_dims)).astype(np.uint32)
    order = np.lexsort((rng.random(dims.size), rows))
    dims = dims[order]
    indptr = np.zeros(n_points + 1, np.uint64)
    indptr[1:] = np.cumsum(np.bincount(rows.astype(np.int64), minlength=n_points))
    w = rng.random(dims.size).astype(np.float32) + np.float32(0.01)
    if negative:
        w[rng.random(dims.size) < negative] *= -1
    return indptr, dims, w
