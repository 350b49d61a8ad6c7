"""ctypes binding of libqdrant_b200.so (include/qb200.h).  No torch, no numpy arithmetic: this module only
marshals pointers.  Importing it on a box where the library has not been built raises loudly — there is no
Python or CPU fallback for any scoring call."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("QB_LIB_PATH") or os.path.join(_HERE, "lib", "libqdrant_b200.so")   # QB_LIB_PATH: experiment builds (build.py --variant)

QB_OK, QB_ERR_INVALID, QB_ERR_CUDA, QB_ERR_UNSUPPORTED, QB_ERR_OOM, QB_ERR_CANCELLED, QB_ERR_NO_DEVICE = 0, -1, -2, -3, -4, -5, -6

f32p = C.POINTER(C.c_float)
u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
i32p = C.POINTER(C.c_int32)
vp = C.c_void_p


class ScoredPoint(C.Structure):
    _fields_ = [("idx", C.c_uint32), ("score", C.c_float)]


class HwCounters(C.Structure):
    _fields_ = [("cpu", C.c_uint64), ("vector_io_read", C.c_uint64)]


# name -> (restype, argtypes): every symbol include/qb200.h declares
SIGNATURES = {
    "qb_last_error": (C.c_char_p, []),
    "qb_abi_version": (C.c_int32, []),
    "qb_device_count": (C.c_int32, [i32p]),
    "qb_kernel_launch_count": (C.c_uint64, []),
    "qb_storage_create_dense": (C.c_int32, [C.c_int32, C.c_int, C.c_int, C.c_uint32, C.c_uint64, vp, C.c_uint64, C.POINTER(vp)]),
    "qb_storage_write_rows": (C.c_int32, [vp, C.c_uint64, C.c_uint64, vp, C.c_uint64]),
    "qb_storage_write_rows_device": (C.c_int32, [vp, C.c_uint64, C.c_uint64, vp, C.c_uint64]),
    "qb_storage_read_rows": (C.c_int32, [vp, u32p, C.c_uint64, vp]),
    "qb_storage_create_sq8": (C.c_int32, [C.c_int32, C.c_uint32, C.c_uint64, u8p, C.c_uint32, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int32, C.c_int, C.POINTER(vp)]),
    "qb_storage_create_pq": (C.c_int32, [C.c_int32, C.c_uint32, C.c_uint32, u32p, f32p, C.c_uint32, u8p, C.c_uint64, C.c_int, C.c_int32, C.c_int, C.POINTER(vp)]),
    "qb_storage_create_bq": (C.c_int32, [C.c_int32, C.c_uint32, C.c_int, C.c_int, u8p, C.c_uint32, C.c_uint64, C.c_int, C.c_int32, f32p, C.c_int, C.POINTER(vp)]),
    "qb_storage_load_dense_file": (C.c_int32, [C.c_int32, C.c_int, C.c_int, C.c_uint32, u8p, C.c_uint64, C.POINTER(vp)]),
    "qb_storage_load_quantized": (C.c_int32, [C.c_int32, C.c_int, C.c_char_p, C.c_uint64, u8p, C.c_uint64, C.c_uint64, C.POINTER(vp)]),
    "qb_storage_destroy": (None, [vp]),
    "qb_storage_info": (C.c_int32, [vp, u32p, u64p, u64p]),
    "qb_storage_set_deleted": (C.c_int32, [vp, u64p, C.c_uint64]),
    "qb_storage_stream": (vp, [vp]),
    "qb_metric_preprocess": (C.c_int32, [C.c_int32, C.c_int, C.c_uint32, C.c_uint64, f32p, f32p]),
    "qb_metric_preprocess_device": (C.c_int32, [C.c_int32, C.c_int, C.c_uint32, C.c_uint64, vp, C.c_uint64]),
    "qb_metric_postprocess": (C.c_float, [C.c_int, C.c_float]),
    "qb_scorer_create": (C.c_int32, [vp, f32p, C.POINTER(vp)]),
    "qb_scorer_create_internal": (C.c_int32, [vp, C.c_uint32, C.POINTER(vp)]),
    "qb_scorer_destroy": (None, [vp]),
    "qb_score_points": (C.c_int32, [vp, u32p, C.c_size_t, f32p]),
    "qb_score_point": (C.c_int32, [vp, C.c_uint32, f32p]),
    "qb_score_internal": (C.c_int32, [vp, C.c_uint32, C.c_uint32, f32p]),
    "qb_scorer_take_counters": (C.c_int32, [vp, C.POINTER(HwCounters)]),
    "qb_search_batch": (C.c_int32, [vp, f32p, C.c_uint32, C.c_uint32, u64p, u32p, C.c_uint64, i32p, C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters)]),
    "qb_search_batch_device": (C.c_int32, [vp, vp, C.c_uint32, C.c_uint32, vp, vp]),
    "qb_scorer_create_custom": (C.c_int32, [vp, C.c_int, f32p, C.c_uint32, C.c_uint32, C.POINTER(vp)]),
    "qb_search_custom": (C.c_int32, [vp, C.c_int, f32p, C.c_uint32, C.c_uint32, C.c_uint32, u64p, u32p, C.c_uint64, i32p, C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters)]),
    "qb_scorer_create_feedback": (C.c_int32, [vp, f32p, C.c_uint32, C.c_float, f32p, C.POINTER(vp)]),
    "qb_search_feedback": (C.c_int32, [vp, f32p, C.c_uint32, C.c_float, f32p, C.c_uint32, u64p, u32p, C.c_uint64, i32p, C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters)]),
    "qb_sq8_find_alpha_offset_device": (C.c_int32, [C.c_int32, C.c_uint32, C.c_uint64, vp, C.c_uint64, f32p, f32p]),
    "qb_sq8_encode_rows_device": (C.c_int32, [C.c_int32, C.c_uint32, C.c_uint64, vp, C.c_uint64, C.c_float, C.c_float, C.c_int, C.c_int, vp, vp]),
    "qb_bq_row_bytes": (C.c_uint32, [C.c_uint32, C.c_int]),
    "qb_bq_encode_rows_device": (C.c_int32, [C.c_int32, C.c_uint32, C.c_uint64, vp, C.c_uint64, C.c_int, f32p, vp, vp]),
    "qb_pq_encode_rows_device": (C.c_int32, [C.c_int32, C.c_uint32, C.c_uint32, C.c_uint32, f32p, C.c_uint64, vp, C.c_uint64, vp, vp]),
    "qb_search_maxsim": (C.c_int32, [vp, u32p, C.c_uint32, f32p, C.c_uint32, C.c_uint32, u64p, C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters)]),
    "qb_score_maxsim": (C.c_int32, [vp, u32p, C.c_uint32, f32p, C.c_uint32, u32p, C.c_size_t, f32p]),
    "qb_bq_vector_stats_device": (C.c_int32, [C.c_int32, C.c_uint32, C.c_uint64, vp, C.c_uint64, f32p, f32p]),
    "qb_sq8_quantile_interval_device": (C.c_int32, [C.c_int32, C.c_uint32, C.c_uint64, vp, C.c_uint64, C.c_float, f32p, f32p, i32p]),
    "qb_pq_train_device": (C.c_int32, [C.c_int32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, vp, C.c_uint64, C.c_uint32, C.c_float, C.c_uint32, C.c_uint64, f32p, u32p]),
    "qb_search_maxsim_custom": (C.c_int32, [vp, u32p, C.c_uint32, C.c_int, f32p, u32p, C.c_uint32, C.c_uint32, f32p, C.c_uint32, u64p, C.POINTER(ScoredPoint), u32p,
                                            C.POINTER(HwCounters)]),
    "qb_score_maxsim_custom": (C.c_int32, [vp, u32p, C.c_uint32, C.c_int, f32p, u32p, C.c_uint32, C.c_uint32, f32p, u32p, C.c_size_t, f32p]),
    "qb_rescore": (C.c_int32, [vp, u32p, C.c_size_t, C.c_uint32, C.POINTER(ScoredPoint), u32p]),
    "qb_storage_set_id_base": (C.c_int32, [vp, C.c_uint32]),
    "qb_topk_merge_device": (C.c_int32, [C.c_int32, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, vp, C.c_uint64, vp]),
    "qb_set_option": (C.c_int32, [C.c_char_p, C.c_int64]),
    "qb_storage_set_on_disk": (C.c_int32, [vp, C.c_int32]),
    "qb_search_stats": (C.c_int32, [vp, u64p, u64p, C.c_int32]),
    "qb_comm_create": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_uint32, C.c_uint32, C.POINTER(vp)]),
    "qb_comm_local_handle": (C.c_int32, [vp, u8p]),
    "qb_comm_connect": (C.c_int32, [vp, u8p]),
    "qb_comm_connect_local": (C.c_int32, [C.POINTER(vp), C.c_int32]),
    "qb_comm_destroy": (None, [vp]),
    "qb_comm_stream": (vp, [vp]),
    "qb_comm_check": (C.c_int32, [vp]),
    "qb_multi_search_batch": (C.c_int32, [vp, vp, f32p, C.c_uint32, C.c_uint32, u64p, i32p, C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters)]),
    "qb_multi_search_batch_device": (C.c_int32, [vp, vp, vp, C.c_uint32, C.c_uint32, vp, vp, vp, vp]),
    "qb_hnsw_create_plain": (C.c_int32, [vp, u8p, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(vp)]),
    "qb_hnsw_create_compressed": (C.c_int32, [vp, u8p, C.c_uint64, C.POINTER(vp)]),
    "qb_hnsw_create_with_vectors": (C.c_int32, [vp, u8p, C.c_uint64, C.POINTER(vp)]),
    "qb_hnsw_links": (C.c_int32, [vp, C.c_uint32, u32p, C.c_uint32, C.c_uint32, u32p, u32p]),
    "qb_hnsw_destroy": (None, [vp]),
    "qb_hnsw_info": (C.c_int32, [vp, u32p, u32p, u64p]),
    "qb_hnsw_build": (C.c_int32, [vp, C.c_uint32, C.c_uint32, C.c_uint32, u8p, C.c_uint32, C.c_uint32, C.POINTER(vp), u32p, u32p]),
    "qb_hnsw_build_incremental": (C.c_int32, [vp, vp, u32p, C.c_uint32, u8p, C.c_uint32, C.c_uint32, C.POINTER(vp), u32p, u32p]),
    "qb_hnsw_export_plain": (C.c_int32, [vp, u8p, C.c_uint64, u64p]),
    "qb_hnsw_search_batch": (C.c_int32, [vp, f32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, u64p, i32p, C.POINTER(ScoredPoint), u32p,
                                         C.POINTER(HwCounters)]),
    "qb_hnsw_search_batch_device": (C.c_int32, [vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp]),
    "qb_hnsw_search_batch_algo": (C.c_int32, [vp, f32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, u64p, i32p, C.POINTER(ScoredPoint),
                                              u32p, C.POINTER(HwCounters), C.c_int32]),
    "qb_hnsw_search_batch_device_algo": (C.c_int32, [vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, C.c_int32]),
    "qb_hnsw_search_with_vectors_batch": (C.c_int32, [vp, f32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, u64p, i32p,
                                                      C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters)]),
    "qb_hnsw_search_with_vectors_batch_device": (C.c_int32, [vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp]),
    "qb_hnsw_build_multivector": (C.c_int32, [vp, u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, u8p, u64p, C.c_uint32, C.c_uint32, C.POINTER(vp), u32p, u32p]),
    "qb_hnsw_create_plain_multivector": (C.c_int32, [vp, u32p, C.c_uint32, u8p, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(vp)]),
    "qb_hnsw_create_compressed_multivector": (C.c_int32, [vp, u32p, C.c_uint32, u8p, C.c_uint64, C.POINTER(vp)]),
    "qb_hnsw_search_maxsim_batch": (C.c_int32, [vp, f32p, u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, u64p, i32p,
                                                C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters), C.c_int32]),
    "qb_hnsw_search_maxsim_batch_device": (C.c_int32, [vp, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                       vp, vp, C.c_int32]),
    "qb_hnsw_search_maxsim_custom_batch": (C.c_int32, [vp, C.c_int, f32p, u32p, C.c_uint32, C.c_uint32, f32p, C.c_uint32, C.c_uint32, C.c_uint32,
                                                       C.c_uint32, C.c_uint32, u32p, u32p, C.c_uint32, u64p, i32p, C.POINTER(ScoredPoint), u32p,
                                                       C.POINTER(HwCounters), C.c_int32]),
    "qb_hnsw_search_maxsim_discover_batch": (C.c_int32, [vp, f32p, u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, u64p,
                                                         i32p, C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters), C.c_int32]),
    "qb_hnsw_stats": (C.c_int32, [vp, u64p, u64p, C.c_int32]),
    "qb_hnsw_search_custom_batch": (C.c_int32, [vp, C.c_int, f32p, C.c_uint32, C.c_uint32, f32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                u32p, u32p, C.c_uint32, u64p, i32p, C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters), C.c_int32]),
    "qb_hnsw_search_discover_batch": (C.c_int32, [vp, f32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, u64p, i32p,
                                                  C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters), C.c_int32]),
    "qb_mmr_batch": (C.c_int32, [vp, f32p, C.c_uint32, f32p, C.POINTER(ScoredPoint), u32p, C.c_uint32, C.c_uint32, C.POINTER(ScoredPoint), u32p,
                                 C.POINTER(HwCounters)]),
    "qb_mmr_batch_device": (C.c_int32, [vp, vp, C.c_uint32, vp, vp, vp, C.c_uint32, C.c_uint32, vp, vp]),
    "qb_mmr_maxsim_batch": (C.c_int32, [vp, u32p, C.c_uint32, f32p, u32p, C.c_uint32, f32p, C.POINTER(ScoredPoint), u32p, C.c_uint32, C.c_uint32,
                                        C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters)]),
    "qb_mmr_maxsim_batch_device": (C.c_int32, [vp, u32p, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, vp, vp, vp, C.c_uint32, C.c_uint32, vp,
                                               vp]),
    "qb_mmr_sparse_batch": (C.c_int32, [vp, u64p, u32p, f32p, C.c_uint32, f32p, C.POINTER(ScoredPoint), u32p, C.c_uint32, C.c_uint32,
                                        C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters)]),
    "qb_sparse_index_create": (C.c_int32, [C.c_int32, C.c_int, C.c_uint32, C.c_uint32, u64p, u32p, f32p, C.POINTER(vp)]),
    "qb_sparse_index_destroy": (None, [vp]),
    "qb_sparse_index_info": (C.c_int32, [vp, u32p, u32p, u64p, u64p]),
    "qb_sparse_index_stream": (vp, [vp]),
    "qb_sparse_search_batch": (C.c_int32, [vp, u64p, u32p, f32p, C.c_uint32, C.c_uint32, u64p, i32p, C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters)]),
    "qb_sparse_search_batch_device": (C.c_int32, [vp, vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, vp]),
    "qb_sparse_search_plain_batch": (C.c_int32, [vp, u64p, u32p, f32p, C.c_uint32, u64p, u32p, C.c_uint32, i32p, C.POINTER(ScoredPoint), u32p,
                                                 C.POINTER(HwCounters)]),
    "qb_sparse_storage_create": (C.c_int32, [C.c_int32, C.c_uint32, u64p, u32p, f32p, C.c_int32, C.POINTER(vp)]),
    "qb_sparse_storage_destroy": (None, [vp]),
    "qb_sparse_storage_info": (C.c_int32, [vp, u32p, u64p, u64p]),
    "qb_sparse_search_custom_batch": (C.c_int32, [vp, C.c_int, C.c_uint32, C.c_uint32, u64p, u32p, f32p, f32p, C.c_uint32, C.c_uint32, u64p, u32p,
                                                  C.c_uint64, i32p, C.POINTER(ScoredPoint), u32p, C.POINTER(HwCounters)]),
    "qb_sparse_score_custom": (C.c_int32, [vp, C.c_int, C.c_uint32, C.c_uint32, u64p, u32p, f32p, f32p, u32p, C.c_uint64, f32p, C.POINTER(HwCounters)]),
    "qb_profile_enable": (C.c_int32, [vp, C.c_int32]),
    "qb_profile_read": (C.c_int32, [vp, u64p, C.POINTER(C.c_double), C.c_int32]),
}

_lib = None


class QbError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"qb_status {status}: {message}")
        self.status = status


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -m qdrant_b200.build` (nvcc, sm_90a). "
                "qdrant_b200 has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the symbol is not exported
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(status: int) -> None:
    if status != QB_OK:
        raise QbError(status, lib().qb_last_error().decode("utf-8", "replace"))
