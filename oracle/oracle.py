"""ctypes/numpy front-end of the CPU oracle (oracle/oracle.c + oracle/_ref/libsimd_utils.so).

TEST INFRASTRUCTURE ONLY.  Importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs — never from qdrant_b200/ (the product).

`ensure_built()` compiles liboracle.so with gcc when it is missing.  The reference's own C kernels
(`_ref/libsimd_utils.so`, `make -C oracle ref REF=<qdrant source tree>`) are only needed to regenerate the golden
vectors under tests/golden/; the tests compare with those.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_REF = None

COSINE, EUCLID, DOT, MANHATTAN = 0, 1, 2, 3          # lib/segment/src/types.rs:313-322
QD_COSINE, QD_DOT, QD_L1, QD_L2 = 0, 1, 2, 3          # lib/quantization/src/encoded_vectors.rs:13
BQ_ONE, BQ_TWO, BQ_ONE_AND_HALF = 0, 1, 2             # encoded_vectors_binary.rs:34-39
BQQ_SAME, BQQ_SCALAR4, BQQ_SCALAR8 = 0, 1, 2          # encoded_vectors_binary.rs:48-54

SCORED = np.dtype([("idx", np.uint32), ("score", np.float32)])  # #[repr(C)] ScoredPointOffset


def ensure_built() -> None:
    so = os.path.join(_HERE, "liboracle.so")
    need = not os.path.exists(so) or any(os.path.getmtime(so) < os.path.getmtime(os.path.join(_HERE, f)) for f in ("oracle.c", "hnsw.c", "mt.c", "train.c"))
    if need:
        subprocess.run(["make", "-C", _HERE, "liboracle.so"], check=True, capture_output=True)


class SQ8Meta(C.Structure):
    _fields_ = [
        ("dim", C.c_uint32),
        ("actual_dim", C.c_uint32),
        ("alpha", C.c_float),
        ("offset", C.c_float),
        ("multiplier", C.c_float),
        ("distance_type", C.c_int32),
        ("invert", C.c_int32),
    ]


def _p(a: np.ndarray, t):
    return a.ctypes.data_as(C.POINTER(t))


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        ensure_built()
        L = C.CDLL(os.path.join(_HERE, "liboracle.so"))
        f32p, u8p, u32p, u64p = (C.POINTER(C.c_float), C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64))
        for name in ("dot", "euclid", "manhattan"):
            for tier in ("avx", "sse", "scalar"):
                fn = getattr(L, f"qo_{name}_{tier}")
                fn.restype, fn.argtypes = C.c_float, [f32p, f32p, C.c_size_t]
        for tier in ("avx", "sse", "scalar"):
            fn = getattr(L, f"qo_cosine_preprocess_{tier}")
            fn.restype, fn.argtypes = None, [f32p, f32p, C.c_size_t]
        L.qo_similarity_f32.restype, L.qo_similarity_f32.argtypes = C.c_float, [C.c_int, f32p, f32p, C.c_size_t]
        L.qo_maxsim_f32.restype, L.qo_maxsim_f32.argtypes = C.c_float, [C.c_int, f32p, C.c_uint32, f32p, C.c_uint32, C.c_uint32]
        L.qo_maxsim_fold.restype, L.qo_maxsim_fold.argtypes = None, [f32p, C.c_uint64, C.c_uint32, u32p, C.c_uint64, f32p]
        L.qo_fast_sigmoid.restype, L.qo_fast_sigmoid.argtypes = C.c_float, [C.c_float]
        L.qo_scaled_fast_sigmoid.restype, L.qo_scaled_fast_sigmoid.argtypes = C.c_float, [C.c_float]
        L.qo_custom_score.restype, L.qo_custom_score.argtypes = C.c_float, [C.c_int, C.c_uint32, C.c_uint32, f32p, C.c_uint64]
        L.qo_custom_combine.restype, L.qo_custom_combine.argtypes = None, [C.c_int, C.c_uint32, C.c_uint32, f32p, C.c_uint64, C.c_uint64, f32p]
        L.qo_feedback_score.restype, L.qo_feedback_score.argtypes = C.c_float, [C.c_uint32, C.c_float, f32p, f32p, C.c_uint64]
        L.qo_feedback_pairs.restype, L.qo_feedback_pairs.argtypes = C.c_uint32, [f32p, C.c_uint32, C.c_float, C.c_float, u32p, u32p, f32p]
        L.qo_preprocess_f32.restype, L.qo_preprocess_f32.argtypes = None, [C.c_int, f32p, f32p, C.c_size_t]
        L.qo_postprocess_f32.restype, L.qo_postprocess_f32.argtypes = C.c_float, [C.c_int, C.c_float]
        for name in ("dot", "cosine", "euclid", "manhattan"):
            for tier in ("avx", "scalar"):
                fn = getattr(L, f"qo_u8_{name}_{tier}")
                fn.restype, fn.argtypes = C.c_float, [u8p, u8p, C.c_size_t]
        u16p = C.POINTER(C.c_uint16)
        for n in ("qo_f16_dot_avx", "qo_f16_euclid_avx", "qo_f16_manhattan_avx", "qo_f16_dot_scalar"):
            fn = getattr(L, n)
            fn.restype, fn.argtypes = C.c_float, [u16p, u16p, C.c_size_t]
        L.qo_similarity_f16.restype, L.qo_similarity_f16.argtypes = C.c_float, [C.c_int, u16p, u16p, C.c_size_t]
        L.qo_score_rows_f16.restype = None
        L.qo_score_rows_f16.argtypes = [C.c_int, u16p, C.c_uint64, C.c_uint32, u16p, u32p, f32p]
        L.qo_score_rows_u8.restype = None
        L.qo_score_rows_u8.argtypes = [C.c_int, u8p, C.c_uint64, C.c_uint32, u8p, u32p, f32p]
        L.qo_f32_to_f16.restype, L.qo_f32_to_f16.argtypes = None, [f32p, C.c_uint64, u16p]
        L.qo_f32_to_u8.restype, L.qo_f32_to_u8.argtypes = None, [f32p, C.c_uint64, u8p]
        L.qo_sq8_dot_avx.restype, L.qo_sq8_dot_avx.argtypes = C.c_float, [u8p, u8p, C.c_uint32]
        L.qo_sq8_l1_avx.restype, L.qo_sq8_l1_avx.argtypes = C.c_float, [u8p, u8p, C.c_uint32]
        mp = C.POINTER(SQ8Meta)
        L.qo_sq8_get_shift.restype, L.qo_sq8_get_shift.argtypes = C.c_float, [mp]
        L.qo_sq8_make_meta.restype, L.qo_sq8_make_meta.argtypes = None, [f32p, C.c_uint64, C.c_uint32, C.c_int, C.c_int, mp]
        L.qo_sq8_encode.restype, L.qo_sq8_encode.argtypes = None, [mp, f32p, C.c_uint64, u8p]
        L.qo_sq8_encode_query.restype, L.qo_sq8_encode_query.argtypes = C.c_float, [mp, f32p, u8p]
        L.qo_sq8_score.restype, L.qo_sq8_score.argtypes = C.c_float, [mp, u8p, C.c_float, u8p]
        L.qo_sq8_score_internal.restype, L.qo_sq8_score_internal.argtypes = C.c_float, [mp, u8p, u8p]
        L.qo_pq_encode.restype, L.qo_pq_encode.argtypes = None, [f32p, C.c_uint64, C.c_uint32, C.c_uint32, f32p, C.c_uint32, u8p]
        L.qo_pq_encode_query.restype, L.qo_pq_encode_query.argtypes = None, [f32p, C.c_uint32, C.c_uint32, f32p, C.c_uint32, C.c_int, C.c_int, f32p]
        L.qo_pq_score.restype, L.qo_pq_score.argtypes = C.c_float, [f32p, C.c_uint32, u8p, C.c_uint32]
        L.qo_pq_score_internal.restype, L.qo_pq_score_internal.argtypes = C.c_float, [u8p, u8p, C.c_uint32, C.c_uint32, f32p, C.c_int, C.c_int]
        L.qo_bq_row_bytes.restype, L.qo_bq_row_bytes.argtypes = C.c_uint32, [C.c_uint32, C.c_int]
        L.qo_bq_encode.restype, L.qo_bq_encode.argtypes = None, [f32p, C.c_uint32, C.c_int, f32p, u8p]
        L.qo_bq_encode_scalar_query.restype, L.qo_bq_encode_scalar_query.argtypes = C.c_uint32, [f32p, C.c_uint32, C.c_int, C.c_uint32, u8p]
        L.qo_bq_score.restype, L.qo_bq_score.argtypes = C.c_float, [u8p, u8p, C.c_uint32, C.c_int, C.c_uint32, C.c_int, C.c_int]
        L.qo_topk.restype, L.qo_topk.argtypes = C.c_uint32, [u32p, f32p, C.c_uint64, C.c_uint32, C.c_void_p]
        L.qo_scan_f32.restype = None
        L.qo_scan_f32.argtypes = [C.c_int, f32p, C.c_uint64, C.c_uint64, C.c_uint32, f32p, C.c_uint32, C.c_uint32, u64p, C.c_void_p, u32p]
        L.qo_scan_sq8.restype = None
        L.qo_scan_sq8.argtypes = [mp, u8p, C.c_uint64, C.c_uint64, u8p, f32p, C.c_uint32, C.c_uint32, u64p, C.c_void_p, u32p]
        L.qo_scan_pq.restype = None
        L.qo_scan_pq.argtypes = [u8p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, f32p, C.c_uint32, C.c_uint32, u64p, C.c_void_p, u32p]
        L.qo_scan_bq.restype = None
        L.qo_scan_bq.argtypes = [u8p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_int, C.c_uint32, C.c_int, C.c_int, u8p, C.c_uint32, C.c_uint32, C.c_uint32, u64p, C.c_void_p, u32p]
        L.qo_score_rows_sq8.restype = None
        L.qo_score_rows_sq8.argtypes = [mp, u8p, C.c_uint64, u8p, C.c_float, u32p, f32p]
        L.qo_score_rows_pq.restype = None
        L.qo_score_rows_pq.argtypes = [u8p, C.c_uint64, C.c_uint32, C.c_uint32, f32p, u32p, f32p]
        L.qo_score_rows_bq.restype = None
        L.qo_score_rows_bq.argtypes = [u8p, C.c_uint64, C.c_uint32, C.c_int, C.c_uint32, C.c_int, C.c_int, u8p, u32p, f32p]
        L.qo_score_points_f32.restype = None
        L.qo_score_points_f32.argtypes = [C.c_int, f32p, C.c_uint32, f32p, u32p, C.c_uint64, f32p]
        L.qo_score_rows_f32.restype = None
        L.qo_score_rows_f32.argtypes = [C.c_int, f32p, C.c_uint64, C.c_uint32, f32p, f32p]
        L.qo_preprocess_rows_f32.restype = None
        L.qo_preprocess_rows_f32.argtypes = [C.c_int, f32p, f32p, C.c_uint64, C.c_uint32]
        L.qo_hnsw_build.restype = C.c_void_p
        L.qo_hnsw_build.argtypes = [f32p, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32, C.c_uint64]
        L.qo_hnsw_search.restype = C.c_uint32
        L.qo_hnsw_search.argtypes = [C.c_void_p, f32p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        L.qo_hnsw_stats.restype, L.qo_hnsw_stats.argtypes = None, [C.c_void_p, u64p, u64p, C.c_int]
        L.qo_hnsw_free.restype, L.qo_hnsw_free.argtypes = None, [C.c_void_p]
        L.qo_hnsw_build_mt.restype = C.c_void_p
        L.qo_hnsw_build_mt.argtypes = [f32p, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32]
        L.qo_hnsw_search_batch.restype = None
        L.qo_hnsw_search_batch.argtypes = [C.c_void_p, f32p, C.c_uint32, C.c_uint32, C.c_uint32, u64p, C.c_uint32, C.c_void_p, u32p]
        L.qo_hnsw_entry.restype, L.qo_hnsw_entry.argtypes = None, [C.c_void_p, u32p, u32p, u32p, u32p]
        L.qo_hnsw_export_plain.restype, L.qo_hnsw_export_plain.argtypes = C.c_uint64, [C.c_void_p, C.c_void_p]
        L.qo_bq_vector_stats.restype, L.qo_bq_vector_stats.argtypes = None, [f32p, C.c_uint64, C.c_uint32, f32p, f32p]
        L.qo_sq8_quantile_interval.restype, L.qo_sq8_quantile_interval.argtypes = C.c_int, [f32p, C.c_uint64, C.c_uint32, C.c_float, f32p, f32p]
        L.qo_kmeans_pq.restype = C.c_uint32
        L.qo_kmeans_pq.argtypes = [f32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_uint32, C.c_uint64, f32p]
        L.qo_pool_create.restype, L.qo_pool_create.argtypes = C.c_void_p, [C.c_uint32]
        L.qo_pool_destroy.restype, L.qo_pool_destroy.argtypes = None, [C.c_void_p]
        L.qo_pool_threads.restype, L.qo_pool_threads.argtypes = C.c_uint32, [C.c_void_p]
        L.qo_pool_load_f32.restype, L.qo_pool_load_f32.argtypes = C.c_int, [C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_uint64, f32p]
        L.qo_pool_scan_f32.restype, L.qo_pool_scan_f32.argtypes = None, [C.c_void_p, f32p, C.c_uint32, C.c_uint32, C.c_void_p, u32p]
        L.qo_pool_scan_sq8.restype = None
        L.qo_pool_scan_sq8.argtypes = [C.c_void_p, mp, u8p, C.c_uint64, u8p, f32p, C.c_uint32, C.c_uint32, C.c_void_p, u32p]
        L.qo_pool_scan_pq.restype = None
        L.qo_pool_scan_pq.argtypes = [C.c_void_p, u8p, C.c_uint64, C.c_uint32, C.c_uint32, f32p, C.c_uint32, C.c_uint32, C.c_void_p, u32p]
        _LIB = L
    return _LIB


def ref():
    """The reference's own C kernels compiled verbatim (None when the prebuilt .so is absent)."""
    global _REF
    if _REF is None:
        ensure_built()
        path = os.path.join(_HERE, "_ref", "libsimd_utils.so")
        if not os.path.exists(path):
            return None
        R = C.CDLL(path)
        u8p = C.POINTER(C.c_uint8)
        for n in ("impl_score_dot_avx", "impl_score_l1_avx", "impl_score_dot_sse", "impl_score_l1_sse"):
            fn = getattr(R, n)
            fn.restype, fn.argtypes = C.c_float, [u8p, u8p, C.c_uint32]
        for n in ("impl_xor_popcnt_scalar8_avx_uint128", "impl_xor_popcnt_scalar4_avx_uint128",
                  "impl_xor_popcnt_sse_uint128", "impl_xor_popcnt_scalar8_sse_uint128",
                  "impl_xor_popcnt_scalar4_sse_uint128"):
            fn = getattr(R, n)
            fn.restype, fn.argtypes = C.c_uint32, [u8p, u8p, C.c_uint32]
        _REF = R
    return _REF


# ------------------------------------------------------------------ f32 metrics
def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _u8(a):
    return np.ascontiguousarray(a, dtype=np.uint8)


def similarity_f32(distance: int, q, v) -> np.float32:
    q, v = _f32(q), _f32(v)
    return np.float32(lib().qo_similarity_f32(distance, _p(q, C.c_float), _p(v, C.c_float), q.size))


def preprocess_f32(distance: int, v) -> np.ndarray:
    v = _f32(v)
    out = np.empty_like(v)
    lib().qo_preprocess_f32(distance, _p(v, C.c_float), _p(out, C.c_float), v.size)
    return out


def preprocess_rows_f32(distance: int, rows) -> np.ndarray:
    rows = _f32(rows)
    out = np.empty_like(rows)
    lib().qo_preprocess_rows_f32(distance, _p(rows, C.c_float), _p(out, C.c_float), rows.shape[0], rows.shape[1])
    return out


def postprocess_f32(distance: int, s) -> np.float32:
    return np.float32(lib().qo_postprocess_f32(distance, float(s)))


def raw_f32(name: str, tier: str, a, b) -> np.float32:
    a, b = _f32(a), _f32(b)
    return np.float32(getattr(lib(), f"qo_{name}_{tier}")(_p(a, C.c_float), _p(b, C.c_float), a.size))


def raw_cosine_preprocess(tier: str, v) -> np.ndarray:
    v = _f32(v)
    out = np.empty_like(v)
    getattr(lib(), f"qo_cosine_preprocess_{tier}")(_p(v, C.c_float), _p(out, C.c_float), v.size)
    return out


def raw_u8(name: str, tier: str, a, b) -> np.float32:
    a, b = _u8(a), _u8(b)
    return np.float32(getattr(lib(), f"qo_u8_{name}_{tier}")(_p(a, C.c_uint8), _p(b, C.c_uint8), a.size))


def similarity_u8(distance: int, q, v) -> np.float32:
    """Metric<u8>::similarity dispatch (metric_uint/simple_*.rs): avx2 for dim>=32, else integer-exact tiers."""
    name = {COSINE: "cosine", EUCLID: "euclid", DOT: "dot", MANHATTAN: "manhattan"}[distance]
    q = _u8(q)
    return raw_u8(name, "avx" if q.size >= 32 else "scalar", q, v)


def similarity_f16(distance: int, q, v) -> np.float32:
    """Metric<f16>::similarity; q, v are numpy float16 arrays (cosine == dot on pre-normalised vectors)."""
    q = np.ascontiguousarray(q, dtype=np.float16).view(np.uint16)
    v = np.ascontiguousarray(v, dtype=np.float16).view(np.uint16)
    return np.float32(lib().qo_similarity_f16(distance, _p(q, C.c_uint16), _p(v, C.c_uint16), q.size))


def raw_f16(name: str, a, b) -> np.float32:
    a = np.ascontiguousarray(a, dtype=np.float16).view(np.uint16)
    b = np.ascontiguousarray(b, dtype=np.float16).view(np.uint16)
    return np.float32(getattr(lib(), f"qo_f16_{name}")(_p(a, C.c_uint16), _p(b, C.c_uint16), a.size))


def to_f16_query(distance: int, q) -> np.ndarray:
    """The query of an f16 storage: Metric::preprocess in f32, then f16::from_f32 (round to nearest even, overflow to inf)."""
    pre = preprocess_f32(distance, q)
    out = np.empty(pre.size, dtype=np.uint16)
    lib().qo_f32_to_f16(_p(pre, C.c_float), pre.size, _p(out, C.c_uint16))
    return out.view(np.float16)


def to_u8_query(q) -> np.ndarray:
    """The query of a u8 storage: `x as u8` on the raw f32 values (no preprocess, not even for Cosine): NaN -> 0, truncate, saturate."""
    q = _f32(q)
    out = np.empty(q.size, dtype=np.uint8)
    lib().qo_f32_to_u8(_p(q, C.c_float), q.size, _p(out, C.c_uint8))
    return out


def _score_rows_x(fn, ct, distance: int, rows, q, ids):
    rows, q = np.ascontiguousarray(rows), np.ascontiguousarray(q)
    assert rows.ndim == 2 and q.shape == (rows.shape[1],)
    if ids is not None:
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        assert ids.size == 0 or int(ids.max()) < rows.shape[0]
    out = np.empty(rows.shape[0] if ids is None else ids.size, dtype=np.float32)
    fn(distance, _p(rows, ct), out.size, rows.shape[1], _p(q, ct), None if ids is None else _p(ids, C.c_uint32), _p(out, C.c_float))
    return out


def score_rows_f16(distance: int, rows, q_f16, ids=None) -> np.ndarray:
    """Metric<f16>::similarity(q, row) for every row (or every row listed in ids); q_f16 already converted (to_f16_query)."""
    rows = np.ascontiguousarray(rows, dtype=np.float16).view(np.uint16)
    q = np.ascontiguousarray(q_f16, dtype=np.float16).view(np.uint16)
    return _score_rows_x(lib().qo_score_rows_f16, C.c_uint16, distance, rows, q, ids)


def score_rows_u8(distance: int, rows, q_u8, ids=None) -> np.ndarray:
    """Metric<u8>::similarity(q, row) for every row (or every row listed in ids); q_u8 already converted (to_u8_query)."""
    return _score_rows_x(lib().qo_score_rows_u8, C.c_uint8, distance, _u8(rows), _u8(q_u8), ids)


def _scan_x(score_rows, distance: int, base, queries, top: int, deleted):
    """peek_top_iter over all rows like scan_f32: rows in order, deleted ones skipped, one heap per query."""
    live = None
    if deleted is not None:
        bits = np.unpackbits(np.ascontiguousarray(deleted, dtype=np.uint64).view(np.uint8), bitorder="little")[: base.shape[0]]
        live = np.flatnonzero(bits == 0).astype(np.uint32)
    return [topk(score_rows(distance, base, q, live), top, live) for q in queries]


def scan_f16(distance: int, base, queries_f16, top: int, deleted=None):
    """Top-k of an f16 storage for converted queries ([nq, dim] f16) -> list of SCORED arrays (one per query, descending)."""
    return _scan_x(score_rows_f16, distance, base, np.atleast_2d(np.asarray(queries_f16, dtype=np.float16)), top, deleted)


def scan_u8(distance: int, base, queries_u8, top: int, deleted=None):
    """Top-k of a u8 storage for converted queries ([nq, dim] u8) -> list of SCORED arrays (one per query, descending)."""
    return _scan_x(score_rows_u8, distance, base, np.atleast_2d(_u8(queries_u8)), top, deleted)


def score_rows_f32(distance: int, rows, q_pre) -> np.ndarray:
    rows, q_pre = _f32(rows), _f32(q_pre)
    out = np.empty(rows.shape[0], dtype=np.float32)
    lib().qo_score_rows_f32(distance, _p(rows, C.c_float), rows.shape[0], rows.shape[1], _p(q_pre, C.c_float), _p(out, C.c_float))
    return out


def score_points_f32(distance: int, base, q_pre, ids) -> np.ndarray:
    base, q_pre = _f32(base), _f32(q_pre)
    ids = np.ascontiguousarray(ids, dtype=np.uint32)
    out = np.empty(ids.size, dtype=np.float32)
    lib().qo_score_points_f32(distance, _p(base, C.c_float), base.shape[1], _p(q_pre, C.c_float), _p(ids, C.c_uint32), ids.size, _p(out, C.c_float))
    return out


def _bitmap_ptr(deleted):
    if deleted is None:
        return None, None
    d = np.ascontiguousarray(deleted, dtype=np.uint64)
    return d, _p(d, C.c_uint64)


def scan_f32(distance: int, base, queries_pre, top: int, deleted=None, row_begin=0, row_end=None):
    """peek_top_iter over rows [row_begin,row_end) -> list of SCORED arrays (one per query, descending)."""
    base, queries_pre = _f32(base), np.atleast_2d(_f32(queries_pre))
    nq = queries_pre.shape[0]
    row_end = base.shape[0] if row_end is None else row_end
    out = np.zeros((nq, max(top, 1)), dtype=SCORED)
    counts = np.zeros(nq, dtype=np.uint32)
    keep, dp = _bitmap_ptr(deleted)
    lib().qo_scan_f32(distance, _p(base, C.c_float), row_begin, row_end, base.shape[1], _p(queries_pre, C.c_float), nq, top,
                      dp, out.ctypes.data_as(C.c_void_p), _p(counts, C.c_uint32))
    return [out[i, : counts[i]].copy() for i in range(nq)]


def topk(scores, top: int, ids=None) -> np.ndarray:
    scores = _f32(scores)
    out = np.zeros(max(top, 1), dtype=SCORED)
    idp = None
    if ids is not None:
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        idp = _p(ids, C.c_uint32)
    n = lib().qo_topk(idp, _p(scores, C.c_float), scores.size, top, out.ctypes.data_as(C.c_void_p))
    return out[:n].copy()


def _row_ids(ids, count: int):
    """(kept array, pointer or None, number of scores) for the optional id list of the quantized score_rows"""
    if ids is None:
        return None, None, count
    ids = np.ascontiguousarray(ids, dtype=np.uint32)
    assert ids.size == 0 or int(ids.max()) < count
    return ids, _p(ids, C.c_uint32), ids.size


# ------------------------------------------------------------------ SQ8
@dataclass
class SQ8:
    meta: SQ8Meta
    rows: np.ndarray  # [count, 4 + actual_dim] u8

    @property
    def row_bytes(self) -> int:
        return 4 + self.meta.actual_dim

    @staticmethod
    def encode(data, distance_type: int, invert: bool, alpha=None, offset=None) -> "SQ8":
        """EncodedVectorsU8::encode with quantile=None (encoded_vectors_u8.rs:143-316).  alpha/offset override the min/max
        metadata (what a quantile-clipped range does, :194-208): values outside the range exercise the clamp."""
        data = _f32(data)
        m = SQ8Meta()
        lib().qo_sq8_make_meta(_p(data, C.c_float), data.shape[0], data.shape[1], distance_type, int(invert), C.byref(m))
        if alpha is not None:
            a = np.float32(alpha)
            m.alpha, m.offset = a, np.float32(offset)
            mult = a * a if distance_type in (QD_DOT, QD_COSINE) else (a if distance_type == QD_L1 else np.float32(-2.0) * a * a)   # :210-225
            m.multiplier = np.float32(-mult if invert else mult)
        rows = np.zeros((data.shape[0], 4 + m.actual_dim), dtype=np.uint8)
        lib().qo_sq8_encode(C.byref(m), _p(data, C.c_float), data.shape[0], _p(rows, C.c_uint8))
        return SQ8(m, rows)

    def encode_query(self, q):
        q = _f32(q)
        code = np.zeros(self.meta.actual_dim, dtype=np.uint8)
        off = lib().qo_sq8_encode_query(C.byref(self.meta), _p(q, C.c_float), _p(code, C.c_uint8))
        return code, np.float32(off)

    def score(self, q_code, q_off, row_id: int) -> np.float32:
        row = np.ascontiguousarray(self.rows[row_id])
        return np.float32(lib().qo_sq8_score(C.byref(self.meta), _p(_u8(q_code), C.c_uint8), C.c_float(float(q_off)), _p(row, C.c_uint8)))

    def score_internal(self, i: int, j: int) -> np.float32:
        ri, rj = np.ascontiguousarray(self.rows[i]), np.ascontiguousarray(self.rows[j])
        return np.float32(lib().qo_sq8_score_internal(C.byref(self.meta), _p(ri, C.c_uint8), _p(rj, C.c_uint8)))

    def score_rows(self, q_code, q_off, ids=None) -> np.ndarray:
        """score(q_code, q_off, row) for every row (or every row listed in ids)."""
        rows, q_code = np.ascontiguousarray(self.rows), _u8(q_code)
        assert q_code.size == self.meta.actual_dim
        ids, idp, n = _row_ids(ids, rows.shape[0])
        out = np.empty(n, dtype=np.float32)
        lib().qo_score_rows_sq8(C.byref(self.meta), _p(rows, C.c_uint8), n, _p(q_code, C.c_uint8), C.c_float(float(q_off)), idp, _p(out, C.c_float))
        return out

    def score_all(self, q_code, q_off) -> np.ndarray:
        return self.score_rows(q_code, q_off)

    def scan(self, q_codes, q_offs, top: int, deleted=None):
        q_codes = np.atleast_2d(_u8(q_codes))
        q_offs = np.atleast_1d(_f32(q_offs))
        nq = q_codes.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED)
        counts = np.zeros(nq, dtype=np.uint32)
        keep, dp = _bitmap_ptr(deleted)
        rows = np.ascontiguousarray(self.rows)
        lib().qo_scan_sq8(C.byref(self.meta), _p(rows, C.c_uint8), 0, rows.shape[0], _p(q_codes, C.c_uint8), _p(q_offs, C.c_float),
                          nq, top, dp, out.ctypes.data_as(C.c_void_p), _p(counts, C.c_uint32))
        return [out[i, : counts[i]].copy() for i in range(nq)]


# ------------------------------------------------------------------ PQ
def kmeans_pq_centroids(data, chunk: int, n_centroids: int = 256, iters: int = 8, seed: int = 7, sample: int = 10_000) -> np.ndarray:
    """OUR k-means (the reference's training is RNG-dependent and unpinned, SURVEY §8c): per-chunk Lloyd
    on a seeded sample; returns centroids as n_centroids full-dim vectors (Metadata.centroids layout,
    encoded_vectors_pq.rs:47-51)."""
    data = _f32(data)
    rng = np.random.default_rng(seed)
    n, dim = data.shape
    samp = data[rng.choice(n, size=min(sample, n), replace=False)]
    cents = np.zeros((n_centroids, dim), dtype=np.float32)
    for s in range(0, dim, chunk):
        e = min(s + chunk, dim)
        x = samp[:, s:e]
        c = x[rng.choice(x.shape[0], size=n_centroids, replace=x.shape[0] < n_centroids)].copy()
        for _ in range(iters):
            d = (x * x).sum(1)[:, None] - 2.0 * x @ c.T + (c * c).sum(1)[None, :]
            a = d.argmin(1)
            for k in range(n_centroids):
                sel = x[a == k]
                if len(sel):
                    c[k] = sel.mean(0)
        cents[:, s:e] = c
    return cents


@dataclass
class PQ:
    dim: int
    chunk: int
    centroids: np.ndarray  # [n_centroids, dim] f32
    codes: np.ndarray      # [count, m] u8
    distance_type: int
    invert: bool

    @property
    def m(self) -> int:
        return (self.dim + self.chunk - 1) // self.chunk

    @staticmethod
    def encode(data, chunk: int, centroids, distance_type: int, invert: bool) -> "PQ":
        data, centroids = _f32(data), _f32(centroids)
        dim = data.shape[1]
        m = (dim + chunk - 1) // chunk
        codes = np.zeros((data.shape[0], m), dtype=np.uint8)
        lib().qo_pq_encode(_p(data, C.c_float), data.shape[0], dim, chunk, _p(centroids, C.c_float), centroids.shape[0], _p(codes, C.c_uint8))
        return PQ(dim, chunk, centroids, codes, distance_type, invert)

    def encode_query(self, q) -> np.ndarray:
        q = _f32(q)
        lut = np.zeros((self.m, self.centroids.shape[0]), dtype=np.float32)
        lib().qo_pq_encode_query(_p(q, C.c_float), self.dim, self.chunk, _p(self.centroids, C.c_float), self.centroids.shape[0],
                                 self.distance_type, int(self.invert), _p(lut, C.c_float))
        return lut

    def score(self, lut, row_id: int) -> np.float32:
        code = np.ascontiguousarray(self.codes[row_id])
        lut = _f32(lut)
        return np.float32(lib().qo_pq_score(_p(lut, C.c_float), self.centroids.shape[0], _p(code, C.c_uint8), self.m))

    def score_rows(self, lut, ids=None) -> np.ndarray:
        """score(lut, row) for every row (or every row listed in ids)."""
        codes, lut = np.ascontiguousarray(self.codes), _f32(lut)
        assert lut.shape == (self.m, self.centroids.shape[0])
        ids, idp, n = _row_ids(ids, codes.shape[0])
        out = np.empty(n, dtype=np.float32)
        lib().qo_score_rows_pq(_p(codes, C.c_uint8), n, self.m, self.centroids.shape[0], _p(lut, C.c_float), idp, _p(out, C.c_float))
        return out

    def score_internal(self, i: int, j: int) -> np.float32:
        ci, cj = np.ascontiguousarray(self.codes[i]), np.ascontiguousarray(self.codes[j])
        return np.float32(lib().qo_pq_score_internal(_p(ci, C.c_uint8), _p(cj, C.c_uint8), self.dim, self.chunk,
                                                     _p(self.centroids, C.c_float), self.distance_type, int(self.invert)))

    def scan(self, luts, top: int, deleted=None):
        luts = _f32(luts)
        if luts.ndim == 2:
            luts = luts[None]
        nq = luts.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED)
        counts = np.zeros(nq, dtype=np.uint32)
        keep, dp = _bitmap_ptr(deleted)
        codes = np.ascontiguousarray(self.codes)
        lib().qo_scan_pq(_p(codes, C.c_uint8), 0, codes.shape[0], self.m, self.centroids.shape[0], _p(luts, C.c_float), nq, top, dp,
                         out.ctypes.data_as(C.c_void_p), _p(counts, C.c_uint32))
        return [out[i, : counts[i]].copy() for i in range(nq)]


# ------------------------------------------------------------------ BQ
def bq_row_bytes(dim: int, encoding: int) -> int:
    return int(lib().qo_bq_row_bytes(dim, encoding))


def bq_mean_std(data) -> np.ndarray:
    """Per-coordinate (mean, stddev) for the 2-bit / 1.5-bit encodings.  The reference computes them with a
    streaming estimator (vector_stats.rs); training parity is unpinned, so tests feed the SAME stats to both sides."""
    data = _f32(data)
    return np.stack([data.mean(0), data.std(0)], axis=1).astype(np.float32)


@dataclass
class BQ:
    dim: int
    encoding: int
    query_encoding: int
    rows: np.ndarray  # [count, row_bytes] u8
    distance_type: int
    invert: bool
    mean_std: np.ndarray | None = None

    @property
    def query_bits(self) -> int:
        return {BQQ_SAME: 1, BQQ_SCALAR4: 4, BQQ_SCALAR8: 8}[self.query_encoding]

    @staticmethod
    def encode(data, encoding: int, query_encoding: int, distance_type: int, invert: bool, mean_std=None) -> "BQ":
        data = _f32(data)
        dim = data.shape[1]
        rb = bq_row_bytes(dim, encoding)
        rows = np.zeros((data.shape[0], rb), dtype=np.uint8)
        ms = None if mean_std is None else _f32(mean_std)
        for i in range(data.shape[0]):
            lib().qo_bq_encode(_p(data[i], C.c_float), dim, encoding, None if ms is None else _p(ms, C.c_float),
                               rows[i].ctypes.data_as(C.POINTER(C.c_uint8)))
        return BQ(dim, encoding, query_encoding, rows, distance_type, invert, ms)

    @property
    def query_bytes(self) -> int:
        return self.rows.shape[1] * self.query_bits

    def encode_query(self, q) -> np.ndarray:
        q = _f32(q)
        if self.query_encoding == BQQ_SAME:
            out = np.zeros(self.rows.shape[1], dtype=np.uint8)
            lib().qo_bq_encode(_p(q, C.c_float), self.dim, self.encoding, None if self.mean_std is None else _p(self.mean_std, C.c_float),
                               _p(out, C.c_uint8))
            return out
        out = np.zeros(self.query_bytes, dtype=np.uint8)
        n = lib().qo_bq_encode_scalar_query(_p(q, C.c_float), self.dim, self.encoding, self.query_bits, _p(out, C.c_uint8))
        assert n == out.size, (n, out.size)
        return out

    def score(self, q_enc, row_id: int) -> np.float32:
        row = np.ascontiguousarray(self.rows[row_id])
        q_enc = _u8(q_enc)
        return np.float32(lib().qo_bq_score(_p(row, C.c_uint8), _p(q_enc, C.c_uint8), self.dim, self.encoding, self.query_bits,
                                            self.distance_type, int(self.invert)))

    def score_rows(self, q_enc, ids=None) -> np.ndarray:
        """score(q_enc, row) for every row (or every row listed in ids)."""
        rows, q_enc = np.ascontiguousarray(self.rows), _u8(q_enc)
        assert q_enc.size == (self.rows.shape[1] if self.query_encoding == BQQ_SAME else self.query_bytes)
        ids, idp, n = _row_ids(ids, rows.shape[0])
        out = np.empty(n, dtype=np.float32)
        lib().qo_score_rows_bq(_p(rows, C.c_uint8), n, self.dim, self.encoding, self.query_bits, self.distance_type, int(self.invert),
                               _p(q_enc, C.c_uint8), idp, _p(out, C.c_float))
        return out

    def scan(self, q_encs, top: int, deleted=None):
        q_encs = np.atleast_2d(_u8(q_encs))
        nq = q_encs.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED)
        counts = np.zeros(nq, dtype=np.uint32)
        keep, dp = _bitmap_ptr(deleted)
        rows = np.ascontiguousarray(self.rows)
        lib().qo_scan_bq(_p(rows, C.c_uint8), 0, rows.shape[0], self.dim, self.encoding, self.query_bits, self.distance_type, int(self.invert),
                         _p(q_encs, C.c_uint8), q_encs.shape[1], nq, top, dp, out.ctypes.data_as(C.c_void_p), _p(counts, C.c_uint32))
        return [out[i, : counts[i]].copy() for i in range(nq)]


# ------------------------------------------------------------------ HNSW traversal driver (config #5 harness)
HNSW_SCORE_CB = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(C.c_float))


class HNSW:
    """From-spec CPU HNSW (oracle/hnsw.c): graph built with CPU scoring; search() drives the traversal either with the
    CPU oracle scorer (score_points=None) or with any callable ids -> scores (e.g. a GPU RawScorer.score_points)."""

    def __init__(self, base, distance: int, m: int = 16, ef_construct: int = 100, seed: int = 42, threads: int = 1):
        """threads > 1: the first 256 points serially, the rest on `threads` workers with per-point link locks (like the
        reference's builder, hnsw/build.rs:285-355); such graphs are not deterministic."""
        self.base = _f32(base)
        self.distance = distance
        self._h = lib().qo_hnsw_build_mt(_p(self.base, C.c_float), self.base.shape[0], self.base.shape[1], distance, m, ef_construct, seed, threads)

    def entry(self):
        """(entry point, its level, m, m0)"""
        a, b, c, d = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        lib().qo_hnsw_entry(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d))
        return int(a.value), int(b.value), int(c.value), int(d.value)

    def export_plain(self) -> np.ndarray:
        """bytes of the reference's plain `links.bin` (graph_links/serializer.rs, GraphLinksFormat::Plain)"""
        n = int(lib().qo_hnsw_export_plain(self._h, None))
        out = np.zeros(n, dtype=np.uint8)
        lib().qo_hnsw_export_plain(self._h, out.ctypes.data_as(C.c_void_p))
        return out

    def search_batch(self, queries_pre, top: int, ef: int, deleted=None, threads: int = 1):
        """CPU-scored searches, one per thread at a time; returns a list of SCORED arrays."""
        q = np.ascontiguousarray(np.atleast_2d(_f32(queries_pre)))
        nq = q.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED)
        counts = np.zeros(nq, dtype=np.uint32)
        keep, dp = _bitmap_ptr(deleted)
        lib().qo_hnsw_search_batch(self._h, _p(q, C.c_float), nq, top, ef, dp, threads, out.ctypes.data_as(C.c_void_p), _p(counts, C.c_uint32))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def search(self, query_pre, top: int, ef: int, score_points=None) -> np.ndarray:
        q = _f32(query_pre)
        out = np.zeros(max(top, 1), dtype=SCORED)
        cb = None
        if score_points is not None:
            def _cb(user, ids, n, scores):
                a = np.ctypeslib.as_array(ids, shape=(n,))
                res = score_points(a)
                np.ctypeslib.as_array(scores, shape=(n,))[:] = res
            cb = HNSW_SCORE_CB(_cb)
        n = lib().qo_hnsw_search(self._h, _p(q, C.c_float), C.cast(cb, C.c_void_p) if cb else None, None, top, ef, out.ctypes.data_as(C.c_void_p))
        return out[:n].copy()

    def stats(self, reset=True):
        a, b = C.c_uint64(), C.c_uint64()
        lib().qo_hnsw_stats(self._h, C.byref(a), C.byref(b), int(reset))
        return int(a.value), int(b.value)

    def close(self):
        if self._h:
            lib().qo_hnsw_free(self._h)
            self._h = None


# ------------------------------------------------------------------------------------------------ custom queries
RECO_BEST_SCORE, RECO_SUM_SCORES, DISCOVER, CONTEXT = 1, 2, 3, 4   # include/qb200.h qb_query_kind


def fast_sigmoid(x) -> np.float32:
    return np.float32(lib().qo_fast_sigmoid(np.float32(x)))


def scaled_fast_sigmoid(x) -> np.float32:
    return np.float32(lib().qo_scaled_fast_sigmoid(np.float32(x)))


def custom_examples(kind: int, n_a: int, n_b: int) -> int:
    return {RECO_BEST_SCORE: n_a + n_b, RECO_SUM_SCORES: n_a + n_b, DISCOVER: 1 + 2 * n_a, CONTEXT: 2 * n_a}[kind]


def custom_score(kind: int, n_a: int, n_b: int, sims) -> np.float32:
    """Query::score_by for ONE candidate; sims = its similarities to the examples, in the layout of qb_scorer_create_custom."""
    sims = _f32(sims).reshape(-1)
    assert sims.size == custom_examples(kind, n_a, n_b)
    return np.float32(lib().qo_custom_score(kind, n_a, n_b, _p(sims, C.c_float), 1))


def custom_combine(kind: int, n_a: int, n_b: int, sims) -> np.ndarray:
    """sims: [examples, candidates] -> [candidates] scores."""
    sims = np.ascontiguousarray(_f32(sims))
    assert sims.ndim == 2 and sims.shape[0] == custom_examples(kind, n_a, n_b)
    out = np.empty(sims.shape[1], dtype=np.float32)
    lib().qo_custom_combine(kind, n_a, n_b, _p(sims, C.c_float), sims.shape[1], sims.shape[1], _p(out, C.c_float))
    return out


def feedback_pairs(scores, b: float, c: float):
    """extract_context_pairs with margin 0 (feedback_query.rs:114-146): (positive index, negative index, partial_computation) per pair."""
    sc = _f32(scores).reshape(-1)
    n = sc.size
    cap = max(n * (n - 1), 1)
    pos, neg, part = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32), np.zeros(cap, np.float32)
    k = lib().qo_feedback_pairs(_p(sc, C.c_float), n, np.float32(b), np.float32(c), _p(pos, C.c_uint32), _p(neg, C.c_uint32), _p(part, C.c_float))
    return pos[:k].copy(), neg[:k].copy(), part[:k].copy()


def feedback_score(a: float, partial, sims) -> np.ndarray:
    """FeedbackQuery::score_by per candidate; sims: [1 + 2 * pairs, candidates] (target, pos0, neg0, ...)."""
    sims = np.ascontiguousarray(np.atleast_2d(_f32(sims)))
    part = _f32(partial).reshape(-1)
    assert sims.shape[0] == 1 + 2 * part.size
    return np.array([lib().qo_feedback_score(part.size, np.float32(a), _p(part, C.c_float) if part.size else None, _p(sims[:, i].copy(), C.c_float), 1)
                     for i in range(sims.shape[1])], dtype=np.float32)


# ------------------------------------------------------------------------------------------------ multivector MaxSim
def maxsim_f32(distance: int, a_pre, b_pre) -> np.float32:
    """score_max_similarity(query vectors a, stored vectors b), both [n, dim] and already preprocessed."""
    a, b = np.atleast_2d(_f32(a_pre)), np.atleast_2d(_f32(b_pre))
    assert a.shape[1] == b.shape[1]
    return np.float32(lib().qo_maxsim_f32(distance, _p(a, C.c_float), a.shape[0], _p(b, C.c_float), b.shape[0], a.shape[1]))


def maxsim_fold(sims, offsets) -> np.ndarray:
    """sims: [query vectors, rows]; offsets: n_points + 1 row offsets -> per-point MaxSim scores."""
    sims = np.ascontiguousarray(_f32(sims))
    off = np.ascontiguousarray(offsets, dtype=np.uint32)
    out = np.empty(off.size - 1, dtype=np.float32)
    lib().qo_maxsim_fold(_p(sims, C.c_float), sims.shape[1], sims.shape[0], _p(off, C.c_uint32), off.size - 1, _p(out, C.c_float))
    return out


# ------------------------------------------------------------------------------------------------ many-core CPU arm (oracle/mt.c)
class CpuPool:
    """T pinned threads; each owns (allocates, first-touches, scans) one contiguous segment — one blocking task per segment
    like the reference's SegmentsSearcher — with a T-way host merge.  bench.py's cpu_baseline / --impl reference legs."""

    def __init__(self, threads: int | None = None):
        self.threads = threads or (os.cpu_count() or 1)
        self._p = lib().qo_pool_create(self.threads)

    def load_f32(self, rows: int, dim: int, distance: int, seed: int = 42, src=None):
        """src = None: seeded standard-normal rows, Metric::preprocess applied, generated by the owning threads."""
        if src is not None:
            src = np.ascontiguousarray(_f32(src)); assert src.shape == (rows, dim)
        rc = lib().qo_pool_load_f32(self._p, rows, dim, distance, seed, None if src is None else _p(src, C.c_float))
        if rc != 0:
            raise MemoryError("CpuPool.load_f32: mmap failed")
        self.rows, self.dim = rows, dim

    def scan_f32(self, queries_pre, top: int):
        q = np.ascontiguousarray(np.atleast_2d(_f32(queries_pre)))
        nq = q.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED); counts = np.zeros(nq, dtype=np.uint32)
        lib().qo_pool_scan_f32(self._p, _p(q, C.c_float), nq, top, out.ctypes.data_as(C.c_void_p), _p(counts, C.c_uint32))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def scan_sq8(self, meta: SQ8Meta, rows: np.ndarray, q_codes: np.ndarray, q_offs: np.ndarray, top: int):
        nq = q_codes.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED); counts = np.zeros(nq, dtype=np.uint32)
        lib().qo_pool_scan_sq8(self._p, C.byref(meta), _p(rows, C.c_uint8), rows.shape[0], _p(q_codes, C.c_uint8), _p(q_offs, C.c_float), nq, top,
                               out.ctypes.data_as(C.c_void_p), _p(counts, C.c_uint32))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def scan_pq(self, codes: np.ndarray, n_centroids: int, luts: np.ndarray, top: int):
        nq = luts.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED); counts = np.zeros(nq, dtype=np.uint32)
        lib().qo_pool_scan_pq(self._p, _p(codes, C.c_uint8), codes.shape[0], codes.shape[1], n_centroids, _p(luts, C.c_float), nq, top,
                              out.ctypes.data_as(C.c_void_p), _p(counts, C.c_uint32))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def close(self):
        if self._p:
            lib().qo_pool_destroy(self._p)
            self._p = None


# ------------------------------------------------------------------------------------------------ quantizer training (oracle/train.c)
def bq_vector_stats(data):
    """VectorStats::build (vector_stats.rs:48-117): (mean_std [dim, 2], min_max [dim, 2]) from sequential f64 Welford updates."""
    data = np.ascontiguousarray(_f32(data))
    ms, mm = np.zeros((data.shape[1], 2), np.float32), np.zeros((data.shape[1], 2), np.float32)
    lib().qo_bq_vector_stats(_p(data, C.c_float), data.shape[0], data.shape[1], _p(ms, C.c_float), _p(mm, C.c_float))
    return ms, mm


def sq8_quantile_interval(sample, quantile: float):
    """find_quantile_interval on the sampled vectors (quantile.rs:35-88) -> (alpha, offset) or None."""
    sample = np.ascontiguousarray(_f32(sample))
    a, o = C.c_float(), C.c_float()
    ok = lib().qo_sq8_quantile_interval(_p(sample, C.c_float), sample.shape[0], sample.shape[1], np.float32(quantile), C.byref(a), C.byref(o))
    return (np.float32(a.value), np.float32(o.value)) if ok else None


def kmeans_pq(sample, chunk: int, n_centroids: int = 256, max_iter: int = 100, accuracy: float = 1e-5, groups: int = 1, seed: int = 0):
    """find_centroids / kmeans (encoded_vectors_pq.rs:342-407, kmeans.rs:9-167) on the sampled vectors -> (centroids [K, dim], iterations)."""
    sample = np.ascontiguousarray(_f32(sample))
    out = np.zeros((n_centroids, sample.shape[1]), np.float32)
    it = lib().qo_kmeans_pq(_p(sample, C.c_float), sample.shape[0], sample.shape[1], chunk, n_centroids, max_iter, np.float32(accuracy), groups, seed, _p(out, C.c_float))
    return out, int(it)
