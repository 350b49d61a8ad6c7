"""ctypes driver of tests/mmr_maxsim_ref.c, the checker of qb_mmr_maxsim_batch: maximal marginal relevance over multivector candidates,
restated over the oracle's qo_maxsim_f32 / qo_preprocess_f32 with a lazily filled MaxSim matrix, an explicit swap-remove position array
and last-wins OrderedFloat comparisons.  The library is compiled on first use into a per-user temporary directory keyed by the source's
hash, so a read-only checkout works too."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

SCORED = np.dtype([("idx", np.uint32), ("score", np.float32)])

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mmr_maxsim_ref.c")
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        src = open(_SRC, "rb").read()
        d = os.path.join(tempfile.gettempdir(), f"qb_mmr_ref_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libmmrmaxsimref_{hashlib.sha256(src).hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            # the oracle's flags (oracle/Makefile): no contraction, so mmr = lambda * rel - (1 - lambda) * maxsim rounds each operation
            subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-fvisibility=hidden", "-o", tmp, _SRC], check=True, capture_output=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u64p = C.c_void_p, C.POINTER(C.c_uint64)
        L.qmm_mmr.restype = C.c_uint32
        L.qmm_mmr.argtypes = [vp, vp, C.c_int, vp, vp, C.c_uint32, vp, C.c_uint32, C.c_float, vp, C.c_uint32, C.c_uint32, vp, u64p, u64p]
        _LIB = L
    return _LIB


def mmr(oracle, rows, offsets, distance: int, query, lam: float, candidates, limit: int):
    """One query -> (selected candidates as a SCORED array with their input scores, cpu units, vector_io_read units).
    rows: the token storage (n_rows x dim f32, as stored); offsets: point p = rows [offsets[p], offsets[p+1]); query: [T_q, dim] raw;
    candidates: SCORED array (or (idx, score) pairs), ids = point offsets with token rows."""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    off = np.ascontiguousarray(offsets, dtype=np.uint32)
    q = np.ascontiguousarray(np.atleast_2d(np.asarray(query, dtype=np.float32)))
    cand = np.ascontiguousarray(np.asarray(candidates, dtype=SCORED))
    assert q.shape[1] == rows.shape[1]
    out = np.zeros(max(cand.size, 1), dtype=SCORED)
    cpu, io = C.c_uint64(0), C.c_uint64(0)
    ol = oracle.lib()
    n = lib().qmm_mmr(C.cast(ol.qo_maxsim_f32, C.c_void_p), C.cast(ol.qo_preprocess_f32, C.c_void_p), distance, rows.ctypes.data_as(C.c_void_p),
                      off.ctypes.data_as(C.c_void_p), rows.shape[1], q.ctypes.data_as(C.c_void_p), q.shape[0], C.c_float(lam),
                      cand.ctypes.data_as(C.c_void_p), cand.size, limit, out.ctypes.data_as(C.c_void_p), C.byref(cpu), C.byref(io))
    return out[:n].copy(), int(cpu.value), int(io.value)


def mmr_batch(oracle, rows, offsets, distance: int, queries, lambdas, candidates, limit: int):
    """mmr over a batch: queries = one [T_q, dim] array per query, candidates = one SCORED array per query -> (list of SCORED arrays,
    summed cpu, summed vector_io_read)"""
    res, cpu, io = [], 0, 0
    for q, lam, c in zip(queries, lambdas, candidates):
        o, a, b = mmr(oracle, rows, offsets, distance, q, float(lam), c, limit)
        res.append(o)
        cpu += a
        io += b
    return res, cpu, io
