"""ctypes driver of tests/mmr_sparse_ref.c, the checker of qb_mmr_sparse_batch: maximal marginal relevance over sparse vector candidates,
restated with score_vectors, a lazily filled pair matrix, an explicit swap-remove position array and last-wins OrderedFloat comparisons.
The library is compiled on first use into a per-user temporary directory keyed by the source's hash, so a read-only checkout works too."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

SCORED = np.dtype([("idx", np.uint32), ("score", np.float32)])

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mmr_sparse_ref.c")
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        src = open(_SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), f"qb_mmr_ref_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libmmrsparseref_{hashlib.sha256(src).hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            # no contraction: every product and sum of score_vectors, and the four mmr operations, round as in the reference
            subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-fvisibility=hidden", "-o", tmp, _SRC], check=True, capture_output=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u64p = C.c_void_p, C.POINTER(C.c_uint64)
        L.qms_score.restype = C.c_float
        L.qms_score.argtypes = [vp, vp, C.c_uint64, vp, vp, C.c_uint64]
        L.qms_mmr.restype = C.c_uint32
        L.qms_mmr.argtypes = [vp, vp, vp, vp, vp, C.c_uint64, C.c_float, vp, C.c_uint32, C.c_uint32, vp, u64p, u64p]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def score(a, b) -> np.float32:
    """score_vectors(a, b) for two (dims, weights) pairs in any order; +0.0 when no dim is shared"""
    ad, aw = np.ascontiguousarray(a[0], np.uint32), np.ascontiguousarray(a[1], np.float32)
    bd, bw = np.ascontiguousarray(b[0], np.uint32), np.ascontiguousarray(b[1], np.float32)
    return np.float32(lib().qms_score(_p(ad), _p(aw), ad.size, _p(bd), _p(bw), bd.size))


def mmr(csr, query, lam: float, candidates, limit: int):
    """One query -> (selected candidates as a SCORED array with their input scores, cpu units, vector_io_read units).
    csr: the storage's (indptr, dims, weights); query: (dims, weights); candidates: SCORED array, ids < n_points."""
    ip, dims, w = (np.ascontiguousarray(csr[0], np.uint64), np.ascontiguousarray(csr[1], np.uint32), np.ascontiguousarray(csr[2], np.float32))
    qd, qw = np.ascontiguousarray(query[0], np.uint32), np.ascontiguousarray(query[1], np.float32)
    cand = np.ascontiguousarray(np.asarray(candidates, dtype=SCORED))
    out = np.zeros(max(cand.size, 1), dtype=SCORED)
    cpu, io = C.c_uint64(0), C.c_uint64(0)
    n = lib().qms_mmr(_p(ip), _p(dims), _p(w), _p(qd), _p(qw), qd.size, C.c_float(lam), _p(cand), cand.size, limit, _p(out), C.byref(cpu), C.byref(io))
    return out[:n].copy(), int(cpu.value), int(io.value)


def mmr_batch(csr, queries, lambdas, candidates, limit: int):
    """mmr over a batch: queries = one (dims, weights) pair per query, candidates = one SCORED array per query -> (list of SCORED arrays,
    summed cpu, summed vector_io_read)"""
    res, cpu, io = [], 0, 0
    for q, lam, c in zip(queries, lambdas, candidates):
        o, a, b = mmr(csr, q, float(lam), c, limit)
        res.append(o)
        cpu += a
        io += b
    return res, cpu, io
