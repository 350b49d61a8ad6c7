"""Host-side mirror of the reference's scorer interface, over the C ABI (include/qb200.h).

Same names, argument meaning and error behaviour as lib/segment:
    Distance                         lib/segment/src/types.rs:313-370
    RawScorer                        lib/segment/src/vector_storage/raw_scorer.rs:39-54
    RawScorerBuilder.build_raw_scorer                               raw_scorer.rs:122-128
    QuantizedVectorsRead.raw_scorer / raw_internal_scorer           quantized/quantized_vectors/read_access.rs:26-34
    FilteredScorer                   lib/segment/src/index/hnsw_index/point_scorer.rs:53-58,160-304
    BatchFilteredSearcher            point_scorer.rs:312-472
    get_oversampled_top / postprocess_search_result                 index/vector_index_search_common.rs:27-91
All scoring happens in libqdrant_b200.so on the GPU; this file holds no arithmetic (numpy is used for buffers).
"""
from __future__ import annotations

import ctypes as C
import enum
import sys
from typing import Iterable, Optional, Sequence

import numpy as np

from . import _capi
from ._capi import HwCounters, QbError, ScoredPoint, check, f32p, i32p, lib, u8p, u32p, u64p, vp

SCORED_POINT_OFFSET = np.dtype([("idx", np.uint32), ("score", np.float32)])  # #[repr(C)] ScoredPointOffset
VECTOR_READ_BATCH_SIZE = 64  # lib/segment/src/vector_storage/common.rs:20


class Distance(enum.IntEnum):
    Cosine = 0
    Euclid = 1
    Dot = 2
    Manhattan = 3

    def postprocess_score(self, score: float) -> float:
        """Distance::postprocess_score (types.rs:349-358) — applied at shard level for Nearest queries."""
        return float(lib().qb_metric_postprocess(int(self), C.c_float(score)))


class VectorStorageDatatype(enum.IntEnum):
    Float32 = 0
    Float16 = 1
    Uint8 = 2


class DistanceType(enum.IntEnum):  # quantization::DistanceType
    Cosine = 0
    Dot = 1
    L1 = 2
    L2 = 3


class BQEncoding(enum.IntEnum):
    OneBit = 0
    TwoBits = 1
    OneAndHalfBits = 2


class BQQueryEncoding(enum.IntEnum):
    SameAsStorage = 0
    Scalar4bits = 1
    Scalar8bits = 2


def construct_vector_parameters(distance: Distance) -> tuple[DistanceType, bool]:
    """construct_vector_parameters (quantized_vectors.rs:205-234): Cosine -> Dot; invert = Euclid | Manhattan."""
    dt = {Distance.Cosine: DistanceType.Dot, Distance.Dot: DistanceType.Dot, Distance.Euclid: DistanceType.L2,
          Distance.Manhattan: DistanceType.L1}[distance]
    return dt, distance in (Distance.Euclid, Distance.Manhattan)


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


def _ids(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.uint32)


def _bitmap(point_deleted, count: int) -> Optional[np.ndarray]:
    """bool mask / BitSlice -> u64 words, bit i set = point i deleted."""
    if point_deleted is None:
        return None
    m = np.asarray(point_deleted)
    if m.dtype == np.uint64:
        if m.size < (count + 63) // 64:   # the library reads ceil(count / 64) words
            raise ValueError(f"deleted bitmap has {m.size} words, need {(count + 63) // 64}")
        return np.ascontiguousarray(m)
    bits = np.zeros(((count + 63) // 64) * 64, dtype=bool)
    bits[: m.size] = m.astype(bool)
    return np.packbits(bits, bitorder="little").view(np.uint64).copy()


def metric_preprocess(distance: Distance, vectors, device: int = 0) -> np.ndarray:
    """Metric::preprocess for a batch (cosine normalisation at insert time, types.rs:334-347)."""
    v = np.atleast_2d(_f32(vectors))
    out = np.empty_like(v)
    check(lib().qb_metric_preprocess(device, int(distance), v.shape[1], v.shape[0], v.ctypes.data_as(f32p), out.ctypes.data_as(f32p)))
    return out.reshape(np.shape(vectors))


class QueryKind(enum.IntEnum):  # QueryVector variants beyond Nearest (data_types/vectors.rs)
    RecommendBestScore = 1
    RecommendSumScores = 2
    Discover = 3
    Context = 4
    FeedbackNaive = 5


class RecoQuery:
    """vector_storage/query/reco_query.rs:12-29 — positives and negatives; wrap in RecoBestScoreQuery / RecoSumScoresQuery."""

    def __init__(self, positives, negatives):
        self.positives = [np.asarray(v, dtype=np.float32) for v in positives]
        self.negatives = [np.asarray(v, dtype=np.float32) for v in negatives]


class RecoBestScoreQuery:
    kind = QueryKind.RecommendBestScore

    def __init__(self, query: RecoQuery):
        self.query = query

    def flat(self):
        return self.query.positives + self.query.negatives, len(self.query.positives), len(self.query.negatives)


class RecoSumScoresQuery(RecoBestScoreQuery):
    kind = QueryKind.RecommendSumScores


class ContextPair:
    """vector_storage/query/context_query.rs:13-17"""

    def __init__(self, positive, negative):
        self.positive = np.asarray(positive, dtype=np.float32)
        self.negative = np.asarray(negative, dtype=np.float32)


class DiscoverQuery:
    """vector_storage/query/discover_query.rs:27-36 — a target and context pairs."""
    kind = QueryKind.Discover

    def __init__(self, target, pairs: Sequence[ContextPair]):
        self.target = np.asarray(target, dtype=np.float32)
        self.pairs = list(pairs)

    def flat(self):
        return [self.target] + [v for p in self.pairs for v in (p.positive, p.negative)], len(self.pairs), 0


class ContextQuery:
    """vector_storage/query/context_query.rs:87-99"""
    kind = QueryKind.Context

    def __init__(self, pairs: Sequence[ContextPair]):
        self.pairs = list(pairs)

    def flat(self):
        return [v for p in self.pairs for v in (p.positive, p.negative)], len(self.pairs), 0


class FeedbackQuery:
    """vector_storage/query/feedback_query.rs:150-226 — the scoring form of NaiveFeedbackQuery: a target, context pairs with their
    partial_computation (confidence^b * c, derived from the feedback scores by the host exactly as FeedbackQuery::new does) and the
    coefficient `a`."""
    kind = QueryKind.FeedbackNaive

    def __init__(self, target, pairs: Sequence[ContextPair], partial_computations, a: float):
        self.target = np.asarray(target, dtype=np.float32)
        self.pairs = list(pairs)
        self.partial = np.ascontiguousarray(partial_computations, dtype=np.float32).reshape(-1)
        self.a = float(a)
        assert self.partial.size == len(self.pairs)

    def flat(self):
        return [self.target] + [v for p in self.pairs for v in (p.positive, p.negative)], len(self.pairs), 0


class RawScorer:
    """Box<dyn RawScorer>.  Scoring calls are infallible in the reference; here a CUDA failure raises QbError."""

    def __init__(self, storage: "_Storage", handle: int):
        self._storage = storage  # keeps the borrow alive ('a)
        self._h = vp(handle)

    def score_points(self, points: Sequence[int], scores: Optional[np.ndarray] = None) -> np.ndarray:
        ids = _ids(points)
        if scores is None:
            scores = np.empty(ids.size, dtype=np.float32)
        assert scores.size == ids.size  # raw_scorer.rs:562
        check(lib().qb_score_points(self._h, ids.ctypes.data_as(u32p), ids.size, scores.ctypes.data_as(f32p)))
        return scores

    def score_point(self, point: int) -> float:
        s = C.c_float()
        check(lib().qb_score_point(self._h, int(point), C.byref(s)))
        return np.float32(s.value)

    def score_internal(self, point_a: int, point_b: int) -> float:
        s = C.c_float()
        st = lib().qb_score_internal(self._h, int(point_a), int(point_b), C.byref(s))
        if st == _capi.QB_ERR_INVALID:
            raise IndexError(lib().qb_last_error().decode())  # "Panics if any id is out of range"
        check(st)
        return np.float32(s.value)

    def scorer_bytes(self):
        return None  # a GPU scorer has no QueryScorerBytes view

    def take_hardware_counters(self) -> tuple[int, int]:
        hc = HwCounters()
        check(lib().qb_scorer_take_counters(self._h, C.byref(hc)))
        return int(hc.cpu), int(hc.vector_io_read)

    def close(self):
        if self._h:
            lib().qb_scorer_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            if sys is None or sys.is_finalizing():  # the CUDA runtime / library may already be torn down at interpreter exit
                return
            self.close()
        except Exception:
            pass


class _Storage:
    def __init__(self):
        self._h = vp()
        self.count = 0
        self.dim = 0
        self.device = 0

    def _raw_scorer(self, query) -> RawScorer:
        q = _f32(query)
        if q.size != self.dim:
            raise ValueError(f"query has dim {q.size}, storage has {self.dim}")  # OperationError at construction
        h = vp()
        check(lib().qb_scorer_create(self._h, q.ctypes.data_as(f32p), C.byref(h)))
        return RawScorer(self, h.value)

    def _flat_custom(self, query):
        vecs, n_a, n_b = query.flat()
        if not vecs:
            raise ValueError("custom query without example vectors")
        m = np.ascontiguousarray(np.stack([_f32(v).reshape(-1) for v in vecs]))
        if m.shape[1] != self.dim:
            raise ValueError(f"query vectors have dim {m.shape[1]}, storage has {self.dim}")
        return m, n_a, n_b

    def raw_scorer_custom(self, query) -> RawScorer:
        """new_raw_scorer for QueryVector::{RecommendBestScore, RecommendSumScores, Discover, Context} (raw_scorer.rs:228-333)."""
        m, n_a, n_b = self._flat_custom(query)
        h = vp()
        if query.kind == QueryKind.FeedbackNaive:
            check(lib().qb_scorer_create_feedback(self._h, m.ctypes.data_as(f32p), n_a, C.c_float(query.a),
                                                  query.partial.ctypes.data_as(f32p) if n_a else None, C.byref(h)))
        else:
            check(lib().qb_scorer_create_custom(self._h, int(query.kind), m.ctypes.data_as(f32p), n_a, n_b, C.byref(h)))
        return RawScorer(self, h.value)

    def search_custom(self, query, top: int, point_deleted=None, id_list=None, counters: Optional[HwCounters] = None):
        """peek_top_iter driven by a custom-query scorer -> SCORED_POINT_OFFSET array, descending."""
        m, n_a, n_b = self._flat_custom(query)
        out = np.zeros(max(top, 1), dtype=SCORED_POINT_OFFSET)
        count = C.c_uint32()
        bm = _bitmap(point_deleted, self.count)
        ids = None if id_list is None else _ids(id_list)
        tail = (None if bm is None else bm.ctypes.data_as(u64p), None if ids is None else ids.ctypes.data_as(u32p), 0 if ids is None else ids.size, None,
                out.ctypes.data_as(C.POINTER(ScoredPoint)), C.byref(count), None if counters is None else C.byref(counters))
        if query.kind == QueryKind.FeedbackNaive:
            check(lib().qb_search_feedback(self._h, m.ctypes.data_as(f32p), n_a, C.c_float(query.a), query.partial.ctypes.data_as(f32p) if n_a else None,
                                           int(top), *tail))
        else:
            check(lib().qb_search_custom(self._h, int(query.kind), m.ctypes.data_as(f32p), n_a, n_b, int(top), *tail))
        return out[: count.value].copy()

    def _raw_internal_scorer(self, point_id: int) -> RawScorer:
        h = vp()
        check(lib().qb_scorer_create_internal(self._h, int(point_id), C.byref(h)))
        return RawScorer(self, h.value)

    def set_deleted(self, point_deleted) -> None:
        bm = _bitmap(point_deleted, self.count)
        if bm is None:
            check(lib().qb_storage_set_deleted(self._h, None, 0))
        else:
            check(lib().qb_storage_set_deleted(self._h, bm.ctypes.data_as(u64p), bm.size))

    def hbm_bytes(self) -> int:
        b = C.c_uint64()
        check(lib().qb_storage_info(self._h, None, None, C.byref(b)))
        return int(b.value)

    def stream_ptr(self) -> int:
        return int(lib().qb_storage_stream(self._h) or 0)

    def set_on_disk(self, on_disk: bool) -> None:
        """VectorStorage::is_on_disk of the storage this copy caches (decides vector_io_read metering)."""
        check(lib().qb_storage_set_on_disk(self._h, 1 if on_disk else 0))

    def search_stats(self, reset: bool = False) -> tuple[int, int]:
        """(fused searches, reruns after a broken fast-path assumption)"""
        a, b = C.c_uint64(), C.c_uint64()
        check(lib().qb_search_stats(self._h, C.byref(a), C.byref(b), 1 if reset else 0))
        return int(a.value), int(b.value)

    def profile(self, on: bool) -> None:
        check(lib().qb_profile_enable(self._h, 1 if on else 0))

    def profile_read(self, reset: bool = True) -> tuple[int, float]:
        n, ms = C.c_uint64(), C.c_double()
        check(lib().qb_profile_read(self._h, C.byref(n), C.byref(ms), 1 if reset else 0))
        return int(n.value), float(ms.value)

    def search_batch(self, queries, top: int, point_deleted=None, id_list=None, is_stopped=None, counters: Optional[HwCounters] = None):
        """Fused BatchFilteredSearcher scan -> list (one per query) of SCORED_POINT_OFFSET arrays, descending."""
        q = np.atleast_2d(_f32(queries))
        if q.shape[1] != self.dim:
            raise ValueError(f"queries have dim {q.shape[1]}, storage has {self.dim}")
        nq = q.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(nq, dtype=np.uint32)
        bm = _bitmap(point_deleted, self.count)
        ids = None if id_list is None else _ids(id_list)
        stop = None
        if is_stopped is not None:
            stop = is_stopped if isinstance(is_stopped, C.c_int32) else C.c_int32(int(bool(is_stopped)))
        check(lib().qb_search_batch(
            self._h, q.ctypes.data_as(f32p), nq, int(top),
            None if bm is None else bm.ctypes.data_as(u64p),
            None if ids is None else ids.ctypes.data_as(u32p), 0 if ids is None else ids.size,
            None if stop is None else C.byref(stop),
            out.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p),
            None if counters is None else C.byref(counters)))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def close(self):
        if self._h:
            lib().qb_storage_destroy(self._h)
            self._h = vp()

    def __del__(self):
        try:
            if sys is None or sys.is_finalizing():     # interpreter shutdown: module globals may already be gone
                return
            self.close()
        except Exception:
            pass


class DenseVectorStorage(_Storage):
    """A segment's dense vectors resident in HBM (the GPU copy is a cache of VectorStorageEnum's rows)."""

    def __init__(self, vectors, distance: Distance, datatype: VectorStorageDatatype = VectorStorageDatatype.Float32, device: int = 0,
                 count: Optional[int] = None, dim: Optional[int] = None):
        super().__init__()
        self.distance, self.datatype, self.device = Distance(distance), VectorStorageDatatype(datatype), device
        np_dt = {VectorStorageDatatype.Float32: np.float32, VectorStorageDatatype.Float16: np.float16, VectorStorageDatatype.Uint8: np.uint8}[self.datatype]
        if vectors is None:
            self.count, self.dim = int(count), int(dim)
            ptr, stride = None, 0
        else:
            v = np.ascontiguousarray(vectors, dtype=np_dt)
            assert v.ndim == 2
            self.count, self.dim = v.shape
            ptr, stride = v.ctypes.data_as(vp), v.strides[0]
        check(lib().qb_storage_create_dense(device, int(self.datatype), int(self.distance), self.dim, self.count, ptr, stride, C.byref(self._h)))

    # RawScorerBuilder
    def build_raw_scorer(self, query) -> RawScorer:
        return self._raw_scorer(query)

    def raw_internal_scorer(self, point_id: int) -> RawScorer:
        return self._raw_internal_scorer(point_id)

    def write_rows_device(self, first_row: int, n_rows: int, dev_ptr: int, row_stride_bytes: int = 0) -> None:
        check(lib().qb_storage_write_rows_device(self._h, first_row, n_rows, vp(dev_ptr), row_stride_bytes))

    def write_rows(self, first_row: int, rows) -> None:
        r = np.ascontiguousarray(rows)
        check(lib().qb_storage_write_rows(self._h, first_row, r.shape[0], r.ctypes.data_as(vp), r.strides[0]))

    def mmr(self, queries, candidates, lambdas, limit: int, counters: Optional[HwCounters] = None):
        """Maximal marginal relevance (mmr_from_points_with_vector, shard/src/query/mmr/mod.rs:42-279) over candidates whose vectors are
        this storage's rows: queries [nq, dim] raw f32; candidates = one SCORED_POINT_OFFSET array per query (what the searches return);
        lambdas = one per query (1 - diversity) or one for all -> list (one per query) of the selected candidates with their input scores."""
        q = np.atleast_2d(_f32(queries))
        if q.shape[1] != self.dim:
            raise ValueError(f"queries have dim {q.shape[1]}, storage has {self.dim}")
        nq = q.shape[0]
        if len(candidates) != nq:
            raise ValueError(f"{len(candidates)} candidate lists for {nq} queries")
        lam = np.ascontiguousarray(np.broadcast_to(np.asarray(lambdas, np.float32), (nq,)))
        max_c = max((len(c) for c in candidates), default=0)
        cand = np.zeros((nq, max(max_c, 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(nq, dtype=np.uint32)
        for i, c in enumerate(candidates):
            c = np.asarray(c, dtype=SCORED_POINT_OFFSET)
            cand[i, : c.size] = c
            counts[i] = c.size
        out = np.zeros((nq, max(int(limit), 1)), dtype=SCORED_POINT_OFFSET)
        out_counts = np.zeros(nq, dtype=np.uint32)
        check(lib().qb_mmr_batch(self._h, q.ctypes.data_as(f32p), nq, lam.ctypes.data_as(f32p), cand.ctypes.data_as(C.POINTER(ScoredPoint)),
                                 counts.ctypes.data_as(u32p), cand.shape[1] if max_c else 0, int(limit), out.ctypes.data_as(C.POINTER(ScoredPoint)),
                                 out_counts.ctypes.data_as(u32p), None if counters is None else C.byref(counters)))
        return [out[i, : out_counts[i]].copy() for i in range(nq)]

    def get_dense(self, ids) -> np.ndarray:
        ids = _ids(ids)
        np_dt = {VectorStorageDatatype.Float32: np.float32, VectorStorageDatatype.Float16: np.float16, VectorStorageDatatype.Uint8: np.uint8}[self.datatype]
        out = np.empty((ids.size, self.dim), dtype=np_dt)
        check(lib().qb_storage_read_rows(self._h, ids.ctypes.data_as(u32p), ids.size, out.ctypes.data_as(vp)))
        return out


class ScalarQuantizedVectors(_Storage):
    """QuantizedVectors backed by EncodedVectorsU8: `rows` is quantized.data ([f32 v_off][actual_dim u8] per row)."""

    def __init__(self, rows, dim: int, alpha: float, offset: float, multiplier: float, distance: Distance, device: int = 0,
                 rows_ptr: Optional[int] = None, count: Optional[int] = None):
        """`rows`: numpy [count, 4 + actual_dim] u8, or None with `rows_ptr` = address (host or device) of such rows."""
        super().__init__()
        self.dim, self.device, self.distance = int(dim), device, Distance(distance)
        actual_dim = self.dim + (16 - self.dim % 16) % 16
        if rows is not None:
            r = np.ascontiguousarray(rows, dtype=np.uint8)
            self.count, ptr, row_bytes = r.shape[0], r.ctypes.data_as(u8p), (r.shape[1] if r.ndim == 2 else 0)
        else:
            self.count, ptr, row_bytes = int(count), C.cast(vp(int(rows_ptr)), u8p), 4 + actual_dim
        dt, invert = construct_vector_parameters(self.distance)
        check(lib().qb_storage_create_sq8(device, self.dim, self.count, ptr, row_bytes, C.c_float(alpha),
                                          C.c_float(offset), C.c_float(multiplier), int(dt), int(invert), int(self.distance), C.byref(self._h)))

    def raw_scorer(self, query) -> RawScorer:
        return self._raw_scorer(query)

    def raw_internal_scorer(self, point_id: int) -> RawScorer:
        return self._raw_internal_scorer(point_id)


class ProductQuantizedVectors(_Storage):
    def __init__(self, codes, centroids, chunk: int, dim: int, distance: Distance, device: int = 0):
        super().__init__()
        c = np.ascontiguousarray(codes, dtype=np.uint8)
        cent = _f32(centroids)
        self.count, self.dim, self.device, self.distance = c.shape[0], int(dim), device, Distance(distance)
        starts = np.arange(0, dim, chunk, dtype=np.uint32)  # get_vector_division, encoded_vectors_pq.rs:164-169
        div = np.stack([starts, np.minimum(starts + chunk, dim).astype(np.uint32)], axis=1).astype(np.uint32).copy()
        self.m = div.shape[0]
        assert c.shape[1] == self.m
        dt, invert = construct_vector_parameters(self.distance)
        check(lib().qb_storage_create_pq(device, self.dim, self.m, div.ctypes.data_as(u32p), cent.ctypes.data_as(f32p), cent.shape[0],
                                         c.ctypes.data_as(u8p), self.count, int(dt), int(invert), int(self.distance), C.byref(self._h)))

    def raw_scorer(self, query) -> RawScorer:
        return self._raw_scorer(query)

    def raw_internal_scorer(self, point_id: int) -> RawScorer:
        """InternalScorerUnsupported for PQ (quantized_query_scorer.rs:60-66): raises QbError(QB_ERR_UNSUPPORTED)."""
        return self._raw_internal_scorer(point_id)


class BinaryQuantizedVectors(_Storage):
    def __init__(self, rows, dim: int, distance: Distance, encoding: BQEncoding = BQEncoding.OneBit,
                 query_encoding: BQQueryEncoding = BQQueryEncoding.SameAsStorage, mean_std=None, device: int = 0):
        super().__init__()
        r = np.ascontiguousarray(rows, dtype=np.uint8)
        self.count, self.dim, self.device, self.distance = r.shape[0], int(dim), device, Distance(distance)
        dt, invert = construct_vector_parameters(self.distance)
        ms = None if mean_std is None else _f32(mean_std)
        check(lib().qb_storage_create_bq(device, self.dim, int(encoding), int(query_encoding), r.ctypes.data_as(u8p), r.shape[1], self.count, int(dt),
                                         int(invert), None if ms is None else ms.ctypes.data_as(f32p), int(self.distance), C.byref(self._h)))

    def raw_scorer(self, query) -> RawScorer:
        return self._raw_scorer(query)

    def raw_internal_scorer(self, point_id: int) -> RawScorer:
        return self._raw_internal_scorer(point_id)


class FilteredScorer:
    """point_scorer.rs:53-58: a RawScorer plus the deleted-points filter; score_points clobbers and truncates `ids`."""

    def __init__(self, raw_scorer: RawScorer, point_deleted=None, filter_fn=None):
        self.raw_scorer = raw_scorer
        self.point_deleted = None if point_deleted is None else np.asarray(point_deleted, dtype=bool)
        self.filter_fn = filter_fn

    @classmethod
    def new(cls, query, vectors: _Storage, quantized_vectors: Optional[_Storage] = None, point_deleted=None, filter_fn=None):
        # point_scorer.rs:172-175
        rs = quantized_vectors.raw_scorer(query) if quantized_vectors is not None else vectors.build_raw_scorer(query)
        return cls(rs, point_deleted, filter_fn)

    @classmethod
    def new_internal(cls, point_id: int, vectors: _Storage, quantized_vectors: Optional[_Storage] = None, point_deleted=None):
        # point_scorer.rs:183-218: fall back to the original vectors when the quantizer cannot build an internal scorer (PQ)
        rs = None
        if quantized_vectors is not None:
            try:
                rs = quantized_vectors.raw_internal_scorer(point_id)
            except QbError as e:
                if e.status != _capi.QB_ERR_UNSUPPORTED:
                    raise
        if rs is None:
            rs = vectors.raw_internal_scorer(point_id)
        return cls(rs, point_deleted)

    def check_vector(self, point_id: int) -> bool:
        if self.point_deleted is not None and point_id < self.point_deleted.size and self.point_deleted[point_id]:
            return False
        return self.filter_fn is None or bool(self.filter_fn(point_id))

    def score_points(self, point_ids: list, limit: int = 0) -> np.ndarray:
        """point_scorer.rs:265-295 -> array of ScoredPointOffset for the ids that passed the filters."""
        kept = [p for p in point_ids if self.check_vector(p)]
        if limit:
            kept = kept[:limit]
        point_ids[:] = kept
        out = np.zeros(len(kept), dtype=SCORED_POINT_OFFSET)
        if kept:
            out["idx"] = kept
            out["score"] = self.raw_scorer.score_points(kept)
        return out

    def score_point(self, point_id: int) -> float:
        return self.raw_scorer.score_point(point_id)

    def score_internal(self, a: int, b: int) -> float:
        return self.raw_scorer.score_internal(a, b)


class BatchFilteredSearcher:
    """point_scorer.rs:312-472.  The reference keeps one RawScorer + one heap per query and walks 64-id chunks;
    here the whole scan + top-k is ONE fused call into the library (qb_search_batch)."""

    def __init__(self, queries, storage: _Storage, top: int, point_deleted=None):
        self.queries = np.atleast_2d(_f32(queries))
        self.storage = storage
        self.top = int(top)
        self.point_deleted = point_deleted
        if self.top == 0:
            raise ValueError("length must be greater than zero")  # FixedLengthPriorityQueue::new expect()

    @classmethod
    def new(cls, queries, vectors: _Storage, quantized_vectors: Optional[_Storage], top: int, point_deleted=None):
        return cls(queries, quantized_vectors if quantized_vectors is not None else vectors, top, point_deleted)

    def peek_top_all(self, is_stopped=None):
        return self.storage.search_batch(self.queries, self.top, point_deleted=self.point_deleted, is_stopped=is_stopped)

    def peek_top_iter(self, points: Iterable[int], is_stopped=None):
        ids = _ids(list(points))
        return self.storage.search_batch(self.queries, self.top, point_deleted=self.point_deleted, id_list=ids, is_stopped=is_stopped)


def rescore(original_scorer: RawScorer, ids, top: int) -> np.ndarray:
    """The rescoring step of postprocess_search_result (vector_index_search_common.rs:74-91) for a scorer that already exists:
    score `ids` with the original-vector scorer, sort descending, truncate to `top`."""
    ids = _ids(ids)
    out = np.zeros(max(int(top), 1), dtype=SCORED_POINT_OFFSET)
    n = C.c_uint32()
    check(lib().qb_rescore(original_scorer._h, ids.ctypes.data_as(u32p), ids.size, int(top), out.ctypes.data_as(C.POINTER(ScoredPoint)), C.byref(n)))
    return out[: n.value].copy()


def get_oversampled_top(top: int, quantized: bool, oversampling: Optional[float]) -> int:
    """vector_index_search_common.rs:27-45."""
    if quantized and oversampling is not None and oversampling > 1.0:
        return int(oversampling * top)
    return top


def postprocess_search_result(search_result: np.ndarray, original: DenseVectorStorage, query, top: int, rescore: bool) -> np.ndarray:
    """vector_index_search_common.rs:48-91: optionally rescore the candidates with the original vectors, sort desc, truncate."""
    if not rescore:
        return search_result[:top].copy()
    sc = original.build_raw_scorer(query)
    ids = _ids(search_result["idx"])
    out = np.zeros(max(top, 1), dtype=SCORED_POINT_OFFSET)
    n = C.c_uint32()
    check(lib().qb_rescore(sc._h, ids.ctypes.data_as(u32p), ids.size, int(top), out.ctypes.data_as(C.POINTER(ScoredPoint)), C.byref(n)))
    sc.close()
    return out[: n.value].copy()


# ------------------------------------------------------------------------------------------------ multivectors
def _multi_rows(vectors, dim: int) -> np.ndarray:
    q = np.atleast_2d(_f32(vectors))
    if q.shape[1] != dim:
        raise ValueError(f"query vectors have dim {q.shape[1]}, storage has {dim}")
    return np.ascontiguousarray(q)


def _flat_multi(query, dim: int):
    """a custom query whose examples are 2-D arrays (vectors x dim) -> (example vectors, example offsets, n_a, n_b, coef or None), the
    examples in the qb_scorer_create_custom order"""
    examples, n_a, n_b = query.flat()
    mats = [_multi_rows(e, dim) for e in examples]
    off = np.concatenate([[0], np.cumsum([m.shape[0] for m in mats])]).astype(np.uint32)
    coef = None
    if query.kind == QueryKind.FeedbackNaive:
        coef = np.concatenate([[np.float32(query.a)], query.partial]).astype(np.float32)
    return np.ascontiguousarray(np.concatenate(mats)), off, n_a, n_b, coef


class MultiVectorView:
    """A multivector collection over a token-level storage: point p = rows [offsets[p], offsets[p+1]) (the flattened layout of
    vector_storage/multi_dense).  Scores are ColBERT MaxSim (score_max_similarity, query_scorer/mod.rs:77-98)."""

    def __init__(self, storage: _Storage, offsets):
        self.storage = storage
        self.offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
        assert self.offsets.ndim == 1 and self.offsets.size >= 1
        self.n_points = self.offsets.size - 1

    def _query(self, query_vectors) -> np.ndarray:
        return _multi_rows(query_vectors, self.storage.dim)

    def search(self, query_vectors, top: int, point_deleted=None, counters: Optional[HwCounters] = None) -> np.ndarray:
        q = self._query(query_vectors)
        out = np.zeros(max(top, 1), dtype=SCORED_POINT_OFFSET)
        count = C.c_uint32()
        bm = _bitmap(point_deleted, self.n_points)
        check(lib().qb_search_maxsim(self.storage._h, self.offsets.ctypes.data_as(u32p), self.n_points, q.ctypes.data_as(f32p), q.shape[0], int(top),
                                     None if bm is None else bm.ctypes.data_as(u64p), out.ctypes.data_as(C.POINTER(ScoredPoint)), C.byref(count),
                                     None if counters is None else C.byref(counters)))
        return out[: count.value].copy()

    def score_points(self, query_vectors, points: Sequence[int]) -> np.ndarray:
        q = self._query(query_vectors)
        ids = _ids(points)
        scores = np.empty(ids.size, dtype=np.float32)
        check(lib().qb_score_maxsim(self.storage._h, self.offsets.ctypes.data_as(u32p), self.n_points, q.ctypes.data_as(f32p), q.shape[0],
                                    ids.ctypes.data_as(u32p), ids.size, scores.ctypes.data_as(f32p)))
        return scores

    def mmr(self, queries, candidates, lambdas, limit: int, counters: Optional[HwCounters] = None):
        """Maximal marginal relevance over multivector candidates (mmr_from_points_with_vector, shard/src/query/mmr/mod.rs:42-125, with
        MaxSim pair scores): queries = one [T_q, dim] array per query (raw f32); candidates = one SCORED_POINT_OFFSET array per query, ids
        are point offsets (what the MaxSim searches return); lambdas = one per query (1 - diversity) or one for all -> list (one per
        query) of the selected candidates with their input scores."""
        qs = [self._query(q) for q in queries]
        nq = len(qs)
        if len(candidates) != nq:
            raise ValueError(f"{len(candidates)} candidate lists for {nq} queries")
        q_off = np.concatenate([[0], np.cumsum([q.shape[0] for q in qs], dtype=np.int64)]).astype(np.uint32)
        qv = np.ascontiguousarray(np.concatenate(qs)) if nq else np.zeros((1, self.storage.dim), np.float32)
        lam = np.ascontiguousarray(np.broadcast_to(np.asarray(lambdas, np.float32), (nq,)))
        max_c = max((len(c) for c in candidates), default=0)
        cand = np.zeros((nq, max(max_c, 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(nq, dtype=np.uint32)
        for i, c in enumerate(candidates):
            c = np.asarray(c, dtype=SCORED_POINT_OFFSET)
            cand[i, : c.size] = c
            counts[i] = c.size
        out = np.zeros((nq, max(int(limit), 1)), dtype=SCORED_POINT_OFFSET)
        out_counts = np.zeros(nq, dtype=np.uint32)
        check(lib().qb_mmr_maxsim_batch(self.storage._h, self.offsets.ctypes.data_as(u32p), self.n_points, qv.ctypes.data_as(f32p), q_off.ctypes.data_as(u32p),
                                        nq, lam.ctypes.data_as(f32p), cand.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p),
                                        cand.shape[1] if max_c else 0, int(limit), out.ctypes.data_as(C.POINTER(ScoredPoint)), out_counts.ctypes.data_as(u32p),
                                        None if counters is None else C.byref(counters)))
        return [out[i, : out_counts[i]].copy() for i in range(nq)]

    # ---- custom queries whose examples are multivectors (MultiCustomQueryScorer, multi_custom_query_scorer.rs:88-104).  `query` is one of the
    # query classes above with 2-D arrays (vectors x dim) in place of vectors.
    def _flat_multi(self, query):
        return _flat_multi(query, self.storage.dim)

    def search_custom(self, query, top: int, point_deleted=None) -> np.ndarray:
        vecs, off, n_a, n_b, coef = self._flat_multi(query)
        out = np.zeros(max(top, 1), dtype=SCORED_POINT_OFFSET)
        count = C.c_uint32()
        bm = _bitmap(point_deleted, self.n_points)
        check(lib().qb_search_maxsim_custom(self.storage._h, self.offsets.ctypes.data_as(u32p), self.n_points, int(query.kind), vecs.ctypes.data_as(f32p),
                                            off.ctypes.data_as(u32p), n_a, n_b, None if coef is None else coef.ctypes.data_as(f32p), int(top),
                                            None if bm is None else bm.ctypes.data_as(u64p), out.ctypes.data_as(C.POINTER(ScoredPoint)), C.byref(count), None))
        return out[: count.value].copy()

    def score_points_custom(self, query, points: Sequence[int]) -> np.ndarray:
        vecs, off, n_a, n_b, coef = self._flat_multi(query)
        ids = _ids(points)
        scores = np.empty(ids.size, dtype=np.float32)
        check(lib().qb_score_maxsim_custom(self.storage._h, self.offsets.ctypes.data_as(u32p), self.n_points, int(query.kind), vecs.ctypes.data_as(f32p),
                                           off.ctypes.data_as(u32p), n_a, n_b, None if coef is None else coef.ctypes.data_as(f32p), ids.ctypes.data_as(u32p), ids.size,
                                           scores.ctypes.data_as(f32p)))
        return scores


# ------------------------------------------------------------------------------------------------ quantizer encode on the device
# Thin wrappers over the C ABI (include/qb200.h, "quantizer encode on the device"): every pointer is a raw device address.
def sq8_multiplier(alpha: float, distance: Distance) -> np.float32:
    """EncodedVectorsU8::encode, encoded_vectors_u8.rs:210-225: Dot a^2, L1 a, L2 -2a^2; negated when `invert`."""
    dt, inv = construct_vector_parameters(distance)
    a = np.float32(alpha)
    m = {DistanceType.Dot: a * a, DistanceType.L1: a, DistanceType.L2: np.float32(-2.0) * a * a}[dt]
    return np.float32(-m if inv else m)


def sq8_find_alpha_offset(rows_ptr: int, count: int, dim: int, row_stride_bytes: int = 0, device: int = 0) -> tuple[np.float32, np.float32]:
    a, o = C.c_float(), C.c_float()
    check(lib().qb_sq8_find_alpha_offset_device(device, dim, count, vp(rows_ptr), row_stride_bytes, C.byref(a), C.byref(o)))
    return np.float32(a.value), np.float32(o.value)


def sq8_encode_rows(rows_ptr: int, count: int, dim: int, alpha: float, offset: float, distance: Distance, out_ptr: int, row_stride_bytes: int = 0,
                    device: int = 0, stream: int = 0) -> None:
    """out_ptr: count x (4 + actual_dim) bytes, the row format qb_storage_create_sq8 / ScalarQuantizedVectors(rows_ptr=...) takes."""
    dt, inv = construct_vector_parameters(distance)
    check(lib().qb_sq8_encode_rows_device(device, dim, count, vp(rows_ptr), row_stride_bytes, np.float32(alpha), np.float32(offset), int(dt), int(inv), vp(out_ptr),
                                          vp(stream)))


def bq_row_bytes(dim: int, encoding: BQEncoding) -> int:
    return int(lib().qb_bq_row_bytes(dim, int(encoding)))


def bq_encode_rows(rows_ptr: int, count: int, dim: int, encoding: BQEncoding, out_ptr: int, mean_std=None, row_stride_bytes: int = 0, device: int = 0,
                   stream: int = 0) -> None:
    ms = None if mean_std is None else _f32(mean_std)
    check(lib().qb_bq_encode_rows_device(device, dim, count, vp(rows_ptr), row_stride_bytes, int(encoding), None if ms is None else ms.ctypes.data_as(f32p),
                                         vp(out_ptr), vp(stream)))


def pq_encode_rows(rows_ptr: int, count: int, dim: int, chunk: int, centroids, out_ptr: int, row_stride_bytes: int = 0, device: int = 0, stream: int = 0) -> None:
    c = _f32(centroids)
    assert c.ndim == 2 and c.shape[1] == dim
    check(lib().qb_pq_encode_rows_device(device, dim, chunk, c.shape[0], c.ctypes.data_as(f32p), count, vp(rows_ptr), row_stride_bytes, vp(out_ptr), vp(stream)))


class _LoadedStorage(_Storage):
    def __init__(self, handle, device: int, distance: Distance):
        super().__init__()
        self._h, self.device, self.distance = handle, device, Distance(distance)
        d, n = C.c_uint32(), C.c_uint64()
        check(lib().qb_storage_info(self._h, C.byref(d), C.byref(n), None))
        self.dim, self.count = int(d.value), int(n.value)

    def raw_scorer(self, query) -> RawScorer:
        return self._raw_scorer(query)

    def raw_internal_scorer(self, point_id: int) -> RawScorer:
        return self._raw_internal_scorer(point_id)


def load_dense_file(file_bytes, distance: Distance, dim: int, datatype: VectorStorageDatatype = VectorStorageDatatype.Float32, device: int = 0) -> _Storage:
    """A segment's `matrix.dat` (b"data" header + rows, dense/immutable_dense_vectors.rs:100-113) as it lies on disk."""
    blob = np.frombuffer(bytes(file_bytes), dtype=np.uint8) if not isinstance(file_bytes, np.ndarray) else np.ascontiguousarray(file_bytes, dtype=np.uint8)
    h = vp()
    check(lib().qb_storage_load_dense_file(device, int(datatype), int(distance), int(dim), blob.ctypes.data_as(u8p), blob.size, C.byref(h)))
    return _LoadedStorage(h, device, distance)


def load_quantized(meta_json, data, metric: Distance, count: int = 0, device: int = 0) -> _Storage:
    """`quantized.meta.json` + `quantized.data` of a segment, unchanged (quantized/quantized_storage.rs:63-69)."""
    meta = meta_json.encode() if isinstance(meta_json, str) else bytes(meta_json)
    blob = np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
    h = vp()
    check(lib().qb_storage_load_quantized(device, int(metric), meta, len(meta), blob.ctypes.data_as(u8p), blob.size, int(count), C.byref(h)))
    return _LoadedStorage(h, device, metric)


class SparseIndexKind(enum.IntEnum):  # qb_sparse_kind
    Ram = 0           # InvertedIndexRam: search may prune
    Compressed = 1    # the immutable / mmap compressed indexes with f32 weights: never prunes
    CompressedF16 = 2
    CompressedU8 = 3


def _csr(vectors):
    """(indptr, dims, weights) as given, or a list of (dims, weights) pairs -> u64 offsets, u32 dims, f32 weights"""
    if isinstance(vectors, tuple) and len(vectors) == 3:
        indptr, dims, weights = vectors
    else:
        vectors = list(vectors)
        indptr = np.zeros(len(vectors) + 1, np.uint64)
        indptr[1:] = np.cumsum([len(d) for d, _ in vectors])
        dims = np.concatenate([np.asarray(d, np.uint32) for d, _ in vectors]) if vectors else np.zeros(0, np.uint32)
        weights = np.concatenate([np.asarray(w, np.float32) for _, w in vectors]) if vectors else np.zeros(0, np.float32)
    indptr = np.ascontiguousarray(indptr, np.uint64)
    dims = np.ascontiguousarray(dims, np.uint32)
    weights = np.ascontiguousarray(weights, np.float32)
    if dims.size != weights.size or indptr.size == 0:
        raise ValueError("sparse vectors: dims and weights differ in length, or no offsets")
    return indptr, dims, weights


class SparseVectorIndex:
    """An inverted index over sparse vectors in HBM and the reference's SearchContext over it (qb_sparse_*).  Points and queries are
    CSR triples (indptr, dims, weights) or lists of (dims, weights) pairs, with internal dims (the caller's IndicesTracker remapping)."""

    def __init__(self, vectors, n_dims: int, kind: SparseIndexKind = SparseIndexKind.Ram, device: int = 0):
        indptr, dims, weights = _csr(vectors)
        self._h = vp()
        h = vp()
        check(lib().qb_sparse_index_create(int(device), int(kind), indptr.size - 1, int(n_dims), indptr.ctypes.data_as(u64p), dims.ctypes.data_as(u32p),
                                           weights.ctypes.data_as(f32p), C.byref(h)))
        self._h = h
        self.count, self.n_dims = indptr.size - 1, int(n_dims)

    def info(self) -> tuple[int, int, int, int]:
        """(points, dims, posting elements, HBM bytes)"""
        n, d, e, b = C.c_uint32(), C.c_uint32(), C.c_uint64(), C.c_uint64()
        check(lib().qb_sparse_index_info(self._h, C.byref(n), C.byref(d), C.byref(e), C.byref(b)))
        return n.value, d.value, e.value, b.value

    @staticmethod
    def _stop(is_stopped):
        if is_stopped is None:
            return None
        return is_stopped if isinstance(is_stopped, C.c_int32) else C.c_int32(int(bool(is_stopped)))

    def search(self, queries, top: int, point_deleted=None, is_stopped=None, counters: Optional[HwCounters] = None):
        """SearchContext::search per query -> list of SCORED_POINT_OFFSET arrays, (score desc, id asc)"""
        qp, qd, qw = _csr(queries)
        nq = qp.size - 1
        out = np.zeros((nq, max(int(top), 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(nq, dtype=np.uint32)
        bm = _bitmap(point_deleted, self.count)
        stop = self._stop(is_stopped)
        check(lib().qb_sparse_search_batch(self._h, qp.ctypes.data_as(u64p), qd.ctypes.data_as(u32p), qw.ctypes.data_as(f32p), nq, int(top),
                                           None if bm is None else bm.ctypes.data_as(u64p), None if stop is None else C.byref(stop),
                                           out.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p),
                                           None if counters is None else C.byref(counters)))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def search_plain(self, queries, id_lists, top: int, is_stopped=None, counters: Optional[HwCounters] = None):
        """SearchContext::plain_search per query over its own (already filtered) ids -> list of SCORED_POINT_OFFSET arrays"""
        qp, qd, qw = _csr(queries)
        nq = qp.size - 1
        lists = [np.asarray(x, np.uint32) for x in id_lists]
        if len(lists) != nq:
            raise ValueError(f"{len(lists)} id lists for {nq} queries")
        ip = np.zeros(nq + 1, np.uint64)
        ip[1:] = np.cumsum([x.size for x in lists])
        ids = np.ascontiguousarray(np.concatenate(lists) if lists else np.zeros(0, np.uint32), np.uint32)
        out = np.zeros((nq, max(int(top), 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(nq, dtype=np.uint32)
        stop = self._stop(is_stopped)
        check(lib().qb_sparse_search_plain_batch(self._h, qp.ctypes.data_as(u64p), qd.ctypes.data_as(u32p), qw.ctypes.data_as(f32p), nq,
                                                 ip.ctypes.data_as(u64p), ids.ctypes.data_as(u32p), int(top), None if stop is None else C.byref(stop),
                                                 out.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p),
                                                 None if counters is None else C.byref(counters)))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def close(self):
        if self._h:
            lib().qb_sparse_index_destroy(self._h)
            self._h = vp()

    def __del__(self):
        try:
            if sys is None or sys.is_finalizing():
                return
            self.close()
        except Exception:
            pass


class SparseVectorStorage:
    """The sparse vector storage of a named vector in HBM, in user dims, and search_scored over it (qb_sparse_storage_*): the
    recommend / discover / context / feedback queries, which skip the inverted index.  Points are a CSR triple (indptr, dims, weights) or
    a list of (dims, weights) pairs; on_disk=True counts vector_io_read as an mmap storage does."""

    def __init__(self, vectors, on_disk: bool = False, device: int = 0):
        indptr, dims, weights = _csr(vectors)
        self._h = vp()
        h = vp()
        check(lib().qb_sparse_storage_create(int(device), indptr.size - 1, indptr.ctypes.data_as(u64p), dims.ctypes.data_as(u32p),
                                             weights.ctypes.data_as(f32p), int(bool(on_disk)), C.byref(h)))
        self._h = h
        self.count = indptr.size - 1

    def info(self) -> tuple[int, int, int]:
        """(points, elements, HBM bytes)"""
        n, e, b = C.c_uint32(), C.c_uint64(), C.c_uint64()
        check(lib().qb_sparse_storage_info(self._h, C.byref(n), C.byref(e), C.byref(b)))
        return n.value, e.value, b.value

    @staticmethod
    def _examples(examples, kind: int, n_a: int, n_b: int):
        """a CSR triple over queries x E examples, or one list of E (dims, weights) pairs per query -> (CSR, queries)"""
        n_ex = {1: n_a + n_b, 2: n_a + n_b, 3: 1 + 2 * n_a, 4: 2 * n_a, 5: 1 + 2 * n_a}.get(kind, 0)
        if isinstance(examples, tuple) and len(examples) == 3:
            csr = _csr(examples)
        else:
            flat = [e for q in examples for e in q]
            if any(len(q) != n_ex for q in examples):
                raise ValueError(f"every query needs {n_ex} examples")
            csr = _csr(flat) if flat else (np.zeros(1, np.uint64), np.zeros(0, np.uint32), np.zeros(0, np.float32))
        return csr, ((csr[0].size - 1) // n_ex if n_ex else 0)

    def search_custom(self, kind: QueryKind, examples, n_a: int, n_b: int = 0, coef=None, top: int = 10, point_deleted=None, id_list=None,
                      is_stopped=None, counters: Optional[HwCounters] = None):
        """search_scored per query (qb_sparse_search_custom_batch), one kind and shape per call: examples = one list of E (dims, weights)
        pairs per query in the qb_scorer_create_custom order, or a CSR triple over queries x E; coef: [queries, 1 + n_a] for feedback;
        id_list: the ids to score, shared by the batch -> list of SCORED_POINT_OFFSET arrays, (score desc, id asc)"""
        (ep, ed, ew), nq = self._examples(examples, int(kind), n_a, n_b)
        cf = None if coef is None else np.ascontiguousarray(_f32(coef).reshape(-1))
        ids = None if id_list is None else _ids(id_list)
        out = np.zeros((max(nq, 1), max(int(top), 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(max(nq, 1), dtype=np.uint32)
        bm = _bitmap(point_deleted, self.count)
        stop = SparseVectorIndex._stop(is_stopped)
        check(lib().qb_sparse_search_custom_batch(self._h, int(kind), int(n_a), int(n_b), ep.ctypes.data_as(u64p), ed.ctypes.data_as(u32p),
                                                  ew.ctypes.data_as(f32p), None if cf is None else cf.ctypes.data_as(f32p), nq, int(top),
                                                  None if bm is None else bm.ctypes.data_as(u64p), None if ids is None else ids.ctypes.data_as(u32p),
                                                  0 if ids is None else ids.size, None if stop is None else C.byref(stop),
                                                  out.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p),
                                                  None if counters is None else C.byref(counters)))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def score_points_custom(self, kind: QueryKind, examples, n_a: int, n_b: int, ids, coef=None, counters: Optional[HwCounters] = None) -> np.ndarray:
        """score_stored_batch of ONE query (examples: its E (dims, weights) pairs) over ids (qb_sparse_score_custom) -> f32 scores"""
        (ep, ed, ew), _ = self._examples([list(examples)] if not (isinstance(examples, tuple) and len(examples) == 3) else examples, int(kind), n_a, n_b)
        cf = None if coef is None else np.ascontiguousarray(_f32(coef).reshape(-1))
        ids = _ids(ids)
        scores = np.zeros(ids.size, np.float32)
        check(lib().qb_sparse_score_custom(self._h, int(kind), int(n_a), int(n_b), ep.ctypes.data_as(u64p), ed.ctypes.data_as(u32p), ew.ctypes.data_as(f32p),
                                           None if cf is None else cf.ctypes.data_as(f32p), ids.ctypes.data_as(u32p), ids.size, scores.ctypes.data_as(f32p),
                                           None if counters is None else C.byref(counters)))
        return scores

    def mmr(self, queries, candidates, lambdas, limit: int, counters: Optional[HwCounters] = None):
        """Maximal marginal relevance (mmr_from_points_with_vector, shard/src/query/mmr/mod.rs:42-279) over candidates whose sparse vectors
        are this storage's points (qb_mmr_sparse_batch): queries = a CSR triple or one (dims, weights) pair per query, user dims in any
        order; candidates = one SCORED_POINT_OFFSET array per query; lambdas = one per query (1 - diversity) or one for all -> list (one
        per query) of the selected candidates with their input scores."""
        qp, qd, qw = _csr(queries)
        nq = qp.size - 1
        if len(candidates) != nq:
            raise ValueError(f"{len(candidates)} candidate lists for {nq} queries")
        lam = np.ascontiguousarray(np.broadcast_to(np.asarray(lambdas, np.float32), (nq,)))
        max_c = max((len(c) for c in candidates), default=0)
        cand = np.zeros((max(nq, 1), max(max_c, 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(max(nq, 1), dtype=np.uint32)
        for i, c in enumerate(candidates):
            c = np.asarray(c, dtype=SCORED_POINT_OFFSET)
            cand[i, : c.size] = c
            counts[i] = c.size
        out = np.zeros((max(nq, 1), max(int(limit), 1)), dtype=SCORED_POINT_OFFSET)
        out_counts = np.zeros(max(nq, 1), dtype=np.uint32)
        check(lib().qb_mmr_sparse_batch(self._h, qp.ctypes.data_as(u64p), qd.ctypes.data_as(u32p), qw.ctypes.data_as(f32p), nq, lam.ctypes.data_as(f32p),
                                        cand.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p), cand.shape[1] if max_c else 0, int(limit),
                                        out.ctypes.data_as(C.POINTER(ScoredPoint)), out_counts.ctypes.data_as(u32p),
                                        None if counters is None else C.byref(counters)))
        return [out[i, : out_counts[i]].copy() for i in range(nq)]

    def close(self):
        if self._h:
            lib().qb_sparse_storage_destroy(self._h)
            self._h = vp()

    def __del__(self):
        try:
            if sys is None or sys.is_finalizing():
                return
            self.close()
        except Exception:
            pass


def set_option(name: str, value: int) -> None:
    """Debugging / experiment switches of the library (qb_set_option)."""
    check(lib().qb_set_option(name.encode(), int(value)))


class HnswGraph:
    """GraphLayers::search with the traversal on the device (qb_hnsw_*): a graph in the reference's plain links.bin layout
    bound to a storage (dense f32, dense Uint8 or SQ8); search() answers a batch of queries in one call.  from_compressed() takes the
    compressed links.bin the reference writes for every index it builds."""

    def __init__(self, storage: _Storage, links_bin, m: int, m0: int):
        self._storage = storage
        self._h = vp()
        blob = np.ascontiguousarray(links_bin, dtype=np.uint8)
        h = vp()
        check(lib().qb_hnsw_create_plain(storage._h, blob.ctypes.data_as(u8p), blob.size, int(m), int(m0), C.byref(h)))
        self._h = h
        self._m = int(m)

    @classmethod
    def from_compressed(cls, storage: _Storage, links_bin) -> "HnswGraph":
        """A graph from `links.bin` in GraphLinksFormat::Compressed (m and m0 are in its header), decoded on the device."""
        self = cls.__new__(cls)
        self._storage = storage
        self._h = vp()
        blob = np.ascontiguousarray(np.frombuffer(links_bin, dtype=np.uint8) if isinstance(links_bin, (bytes, bytearray)) else links_bin,
                                    dtype=np.uint8).reshape(-1)
        h = vp()
        check(lib().qb_hnsw_create_compressed(storage._h, blob.ctypes.data_as(u8p), blob.size, C.byref(h)))
        self._h = h
        return self

    @classmethod
    def from_compressed_with_vectors(cls, storage: _Storage, links_bin) -> "HnswGraph":
        """A graph from `links.bin` in GraphLinksFormat::CompressedWithVectors (inline storage), bound to the segment's SQ8 storage
        (qb_hnsw_create_with_vectors).  search_with_vectors() runs the reference's search over the inline vectors; search() and the
        custom searches run the regular traversal on the same handle."""
        self = cls.__new__(cls)
        self._storage = storage
        self._h = vp()
        blob = np.ascontiguousarray(np.frombuffer(links_bin, dtype=np.uint8) if isinstance(links_bin, (bytes, bytearray)) else links_bin,
                                    dtype=np.uint8).reshape(-1)
        h = vp()
        check(lib().qb_hnsw_create_with_vectors(storage._h, blob.ctypes.data_as(u8p), blob.size, C.byref(h)))
        self._h = h
        return self

    @classmethod
    def multivector(cls, view: "MultiVectorView", links_bin, m: int, m0: int) -> "HnswGraph":
        """A plain links.bin over the POINTS of a multivector collection (qb_hnsw_create_plain_multivector); search it with search_maxsim()."""
        return cls._multivector(view, links_bin, lambda h, blob: lib().qb_hnsw_create_plain_multivector(
            view.storage._h, view.offsets.ctypes.data_as(u32p), view.n_points, blob.ctypes.data_as(u8p), blob.size, int(m), int(m0), C.byref(h)))

    @classmethod
    def from_compressed_multivector(cls, view: "MultiVectorView", links_bin) -> "HnswGraph":
        """A compressed links.bin over the points of a multivector collection (qb_hnsw_create_compressed_multivector)."""
        return cls._multivector(view, links_bin, lambda h, blob: lib().qb_hnsw_create_compressed_multivector(
            view.storage._h, view.offsets.ctypes.data_as(u32p), view.n_points, blob.ctypes.data_as(u8p), blob.size, C.byref(h)))

    @classmethod
    def _multivector(cls, view: "MultiVectorView", links_bin, create) -> "HnswGraph":
        self = cls.__new__(cls)
        self._storage = view.storage
        self._view = view
        self._h = vp()
        blob = np.ascontiguousarray(np.frombuffer(links_bin, dtype=np.uint8) if isinstance(links_bin, (bytes, bytearray)) else links_bin,
                                    dtype=np.uint8).reshape(-1)
        h = vp()
        check(create(h, blob))
        self._h = h
        return self

    def search_maxsim(self, queries, top: int, ef: int, entry_point: int, entry_level: int, point_deleted=None, counters: Optional[HwCounters] = None,
                      algorithm: str = "hnsw"):
        """GraphLayers::search with a MaxSim scorer on a multivector() graph (qb_hnsw_search_maxsim_batch).  queries: a list of
        [Q_i, dim] arrays (1..4096 vectors each); point_deleted: over points.  Returns one list of point offsets per query; a score
        equals MultiVectorView.score_points on that point, bit for bit."""
        if algorithm not in self.ALGORITHMS:
            raise ValueError(f"algorithm {algorithm!r} is not one of {sorted(self.ALGORITHMS)}")
        view = getattr(self, "_view", None)
        mats = [np.atleast_2d(_f32(q)) for q in queries]
        for m in mats:
            if m.shape[1] != self._storage.dim:
                raise ValueError(f"query vectors have dim {m.shape[1]}, storage has {self._storage.dim}")
        nq = len(mats)
        vecs = np.ascontiguousarray(np.concatenate(mats) if nq else np.zeros((0, self._storage.dim), np.float32))
        off = np.concatenate([[0], np.cumsum([m.shape[0] for m in mats])]).astype(np.uint32)
        out = np.zeros((max(nq, 1), max(top, 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(max(nq, 1), dtype=np.uint32)
        bm = _bitmap(point_deleted, view.n_points if view is not None else self.info()[0])
        check(lib().qb_hnsw_search_maxsim_batch(self._h, vecs.ctypes.data_as(f32p), off.ctypes.data_as(u32p), nq, int(top), int(ef), int(entry_point),
                                                int(entry_level), None if bm is None else bm.ctypes.data_as(u64p), None,
                                                out.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p),
                                                None if counters is None else C.byref(counters), self.ALGORITHMS[algorithm]))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    @classmethod
    def build(cls, storage: _Storage, m: int = 16, ef_construct: int = 100, levels=None, seed: int = 0, batch: int = 0, serial_points: int = 0,
              m0: Optional[int] = None) -> "HnswGraph":
        """Builds the graph of a dense f32 or Uint8 storage on the device (qb_hnsw_build; m0 defaults to 2m).  levels: one per point (<= 30);
        by default round(-ln(U) / ln(m)) with U uniform in (0, 1] from numpy's generator seeded with `seed` (get_random_layer,
        graph_layers_builder.rs:388-396).  batch / serial_points 0 = 512 / 256.  The entry point is in .entry_point / .entry_level."""
        m0 = 2 * m if m0 is None else m0
        lv = cls._build_levels(levels, storage.count, m, seed)
        self = cls.__new__(cls)
        self._storage = storage
        self._h = vp()
        h, e, el = vp(), C.c_uint32(), C.c_uint32()
        check(lib().qb_hnsw_build(storage._h, int(m), int(m0), int(ef_construct), lv.ctypes.data_as(u8p), int(batch), int(serial_points), C.byref(h),
                                  C.byref(e), C.byref(el)))
        self._h = h
        self._m = int(m)
        self.entry_point, self.entry_level, self.levels = int(e.value), int(el.value), lv
        return self

    @classmethod
    def build_multivector(cls, view: "MultiVectorView", m: int = 16, ef_construct: int = 100, levels=None, seed: int = 0, batch: int = 0,
                          serial_points: int = 0, m0: Optional[int] = None, point_deleted=None) -> "HnswGraph":
        """Builds the graph over the POINTS of a multivector collection on the device (qb_hnsw_build_multivector): build()'s schedule
        with MaxSim between stored points.  The view's storage must be dense f32; levels / seed / batch / serial_points / m0 as in
        build(), one level per point; point_deleted: bool per point (such points are not inserted).  Search it with search_maxsim();
        the entry point is in .entry_point / .entry_level."""
        m0 = 2 * m if m0 is None else m0
        lv = cls._build_levels(levels, view.n_points, m, seed)
        bm = _bitmap(point_deleted, view.n_points)
        self = cls.__new__(cls)
        self._storage = view.storage
        self._view = view
        self._h = vp()
        h, e, el = vp(), C.c_uint32(), C.c_uint32()
        check(lib().qb_hnsw_build_multivector(view.storage._h, view.offsets.ctypes.data_as(u32p), view.n_points, int(m), int(m0), int(ef_construct),
                                              lv.ctypes.data_as(u8p), None if bm is None else bm.ctypes.data_as(u64p), int(batch), int(serial_points),
                                              C.byref(h), C.byref(e), C.byref(el)))
        self._h = h
        self.entry_point, self.entry_level, self.levels = int(e.value), int(el.value), lv
        return self

    @classmethod
    def build_incremental(cls, storage: _Storage, old: "HnswGraph", old_to_new, ef_construct: int = 100, levels=None, seed: int = 0, batch: int = 0,
                          serial_points: int = 0) -> "HnswGraph":
        """Builds the graph of a dense f32 or Uint8 storage from an old segment's graph over the same datatype (qb_hnsw_build_incremental): the old graph's lists are
        healed where points have gone, renumbered, and only the points it did not have are inserted.  old_to_new: one per old point,
        its id in `storage` or -1 (not carried over).  m / m0 are old's.  levels: one per point; by default a mapped point keeps its old
        level and the others are drawn as build() draws them (`seed`).  The entry point is in .entry_point / .entry_level."""
        n_old = old.info()[0]
        o2n = np.asarray(old_to_new, dtype=np.int64)
        if o2n.shape != (n_old,):
            raise ValueError(f"old_to_new has shape {o2n.shape}, the old graph has {n_old} points")
        o2n = np.ascontiguousarray(np.where(o2n < 0, 0xFFFFFFFF, o2n), dtype=np.uint32)
        m = getattr(old, "_m", None)
        if levels is None:
            if m is None:
                raise ValueError("the old graph's m is not known here (a compressed links.bin): pass levels")
            lv = cls._build_levels(None, storage.count, m, seed).copy()
            keep = (o2n != 0xFFFFFFFF) & (o2n < storage.count)
            lv[o2n[keep]] = old.point_levels()[keep]
        else:
            lv = cls._build_levels(levels, storage.count, m or 2, seed)
        self = cls.__new__(cls)
        self._storage = storage
        self._h = vp()
        h, e, el = vp(), C.c_uint32(), C.c_uint32()
        check(lib().qb_hnsw_build_incremental(storage._h, old._h, o2n.ctypes.data_as(u32p), int(ef_construct), lv.ctypes.data_as(u8p), int(batch),
                                              int(serial_points), C.byref(h), C.byref(e), C.byref(el)))
        self._h = h
        self._m = m
        self.entry_point, self.entry_level, self.levels = int(e.value), int(el.value), lv
        return self

    def point_levels(self) -> np.ndarray:
        """Each point's top level (point_level, view.rs:354-369), from the graph's plain links.bin."""
        b = self.export_plain()
        n, levels = (int(x) for x in b[:16].view(np.uint64))
        n_off = int(b[24:32].view(np.uint64)[0])
        lo = np.append(b[64:64 + 8 * levels].view(np.uint64).astype(np.int64), n_off - 1)
        reindex = b[64 + 8 * levels:64 + 8 * levels + 4 * n].view(np.uint32).astype(np.int64)
        out = np.zeros(n, dtype=np.uint8)
        for lvl in range(1, levels):
            out[reindex < lo[lvl + 1] - lo[lvl]] = lvl
        return out

    @staticmethod
    def _build_levels(levels, n: int, m: int, seed: int) -> np.ndarray:
        """levels as u8, one per point; by default round(-ln(U) / ln(m)) with U uniform in (0, 1] from numpy's generator seeded with
        `seed` (get_random_layer, graph_layers_builder.rs:388-396)"""
        if levels is None:
            u = 1.0 - np.random.default_rng(seed).random(n)
            levels = np.minimum(np.round(-np.log(u) / np.log(max(m, 2))), 30)
        lv = np.ascontiguousarray(levels, dtype=np.int64)
        if lv.shape != (n,):
            raise ValueError(f"levels has shape {lv.shape}, the graph has {n} points")
        return np.ascontiguousarray(np.clip(lv, 0, 255), dtype=np.uint8)   # a level > 30 is rejected by the library

    def export_plain(self) -> np.ndarray:
        """The graph as a plain links.bin (qb_hnsw_export_plain), for any handle."""
        n = C.c_uint64()
        check(lib().qb_hnsw_export_plain(self._h, None, 0, C.byref(n)))
        out = np.zeros(n.value, dtype=np.uint8)
        check(lib().qb_hnsw_export_plain(self._h, out.ctypes.data_as(u8p), n.value, C.byref(n)))
        return out

    def links(self, level: int, ids, cap: int = 0):
        """GraphLinks::links for each of `ids` on `level`, in the graph's stored order: a list of uint32 arrays.  cap = 0 returns every
        link (two calls: counts first); cap > 0 truncates each list to cap links."""
        ids = np.ascontiguousarray(np.atleast_1d(ids), dtype=np.uint32)
        n = ids.size
        counts = np.zeros(n, dtype=np.uint32)
        if cap <= 0:
            check(lib().qb_hnsw_links(self._h, int(level), ids.ctypes.data_as(u32p), n, 0, None, counts.ctypes.data_as(u32p)))
            cap = int(counts.max()) if n else 0
        out = np.zeros((n, max(cap, 1)), dtype=np.uint32)
        check(lib().qb_hnsw_links(self._h, int(level), ids.ctypes.data_as(u32p), n, int(cap), out.ctypes.data_as(u32p), counts.ctypes.data_as(u32p)))
        return [out[i, : min(int(counts[i]), cap)].copy() for i in range(n)]

    def info(self) -> tuple[int, int, int]:
        """(points, levels, bytes of HBM the graph holds)"""
        a, b, c = C.c_uint32(), C.c_uint32(), C.c_uint64()
        check(lib().qb_hnsw_info(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return int(a.value), int(b.value), int(c.value)

    ALGORITHMS = {"hnsw": 0, "acorn": 1}   # qb_hnsw_algorithm (SearchAlgorithm, graph_layers.rs:80-84)

    def search(self, queries, top: int, ef: int, entry_point: int, entry_level: int, point_deleted=None, counters: Optional[HwCounters] = None,
               algorithm: str = "hnsw"):
        """algorithm: "hnsw" (search_on_level) or "acorn" (ACORN-1, search_on_level_acorn) on level 0; which one a filtered request
        takes is the caller's decision (include/qb200.h, qb_hnsw_algorithm)."""
        if algorithm not in self.ALGORITHMS:
            raise ValueError(f"algorithm {algorithm!r} is not one of {sorted(self.ALGORITHMS)}")
        q = np.atleast_2d(_f32(queries))
        if q.shape[1] != self._storage.dim:
            raise ValueError(f"queries have dim {q.shape[1]}, storage has {self._storage.dim}")
        nq = q.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(nq, dtype=np.uint32)
        bm = _bitmap(point_deleted, self._storage.count)
        check(lib().qb_hnsw_search_batch_algo(self._h, q.ctypes.data_as(f32p), nq, int(top), int(ef), int(entry_point), int(entry_level),
                                              None if bm is None else bm.ctypes.data_as(u64p), None, out.ctypes.data_as(C.POINTER(ScoredPoint)),
                                              counts.ctypes.data_as(u32p), None if counters is None else C.byref(counters), self.ALGORITHMS[algorithm]))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def search_with_vectors(self, queries, top: int, ef: int, entry_point: int, entry_level: int, point_deleted=None,
                            counters: Optional[HwCounters] = None, is_stopped: bool = False):
        """GraphLayers::search_with_vectors on a from_compressed_with_vectors() graph (qb_hnsw_search_with_vectors_batch): the beam on
        the inline SQ8 link vectors, every popped candidate scored exactly from its inline f32 vector; the best `top` exact scores.
        Pass ef = max(ef, oversampled top), as the reference does."""
        q = np.atleast_2d(_f32(queries))
        if q.shape[1] != self._storage.dim:
            raise ValueError(f"queries have dim {q.shape[1]}, storage has {self._storage.dim}")
        nq = q.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(nq, dtype=np.uint32)
        bm = _bitmap(point_deleted, self._storage.count)
        stop = C.c_int32(1) if is_stopped else None
        check(lib().qb_hnsw_search_with_vectors_batch(self._h, q.ctypes.data_as(f32p), nq, int(top), int(ef), int(entry_point), int(entry_level),
                                                      None if bm is None else bm.ctypes.data_as(u64p), None if stop is None else C.byref(stop),
                                                      out.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p),
                                                      None if counters is None else C.byref(counters)))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def _examples(self, examples, n_ex: int):
        ex = _f32(examples)
        if ex.ndim == 2:
            ex = ex[None]
        if ex.ndim != 3 or ex.shape[1] != n_ex or ex.shape[2] != self._storage.dim:
            raise ValueError(f"examples must be [queries, {n_ex}, {self._storage.dim}], got {ex.shape}")
        return np.ascontiguousarray(ex)

    def search_custom(self, kind: QueryKind, examples, n_a: int, n_b: int = 0, coef=None, top: int = 10, ef: int = 64, entry_point: int = 0,
                      entry_level: int = 0, point_deleted=None, counters: Optional[HwCounters] = None, custom_entry_points=None,
                      algorithm: str = "hnsw"):
        """Custom queries through the device traversal (qb_hnsw_search_custom_batch).  examples: [queries, E, dim] raw f32 in the
        qb_scorer_create_custom layout (one kind and shape per call); coef: [queries, 1 + n_a] [a, partial...] for feedback queries;
        custom_entry_points: one sequence of point offsets per query (GraphLayers::search's custom_entry_points), or None."""
        if algorithm not in self.ALGORITHMS:
            raise ValueError(f"algorithm {algorithm!r} is not one of {sorted(self.ALGORITHMS)}")
        kind = int(kind)
        n_ex = {1: n_a + n_b, 2: n_a + n_b, 3: 1 + 2 * n_a, 4: 2 * n_a, 5: 1 + 2 * n_a}.get(kind, 0)
        ex = self._examples(examples, n_ex) if n_ex else _f32(examples)
        nq = ex.shape[0] if n_ex else 0
        cf = None if coef is None else np.ascontiguousarray(_f32(coef).reshape(nq, -1))
        cep_arr, cep_cnt, width = self._entry_lists(custom_entry_points, nq)
        out = np.zeros((max(nq, 1), max(top, 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(max(nq, 1), dtype=np.uint32)
        bm = _bitmap(point_deleted, self._storage.count)
        check(lib().qb_hnsw_search_custom_batch(self._h, kind, ex.ctypes.data_as(f32p), int(n_a), int(n_b), None if cf is None else cf.ctypes.data_as(f32p),
                                                nq, int(top), int(ef), int(entry_point), int(entry_level),
                                                None if cep_arr is None else cep_arr.ctypes.data_as(u32p), None if cep_cnt is None else cep_cnt.ctypes.data_as(u32p),
                                                width, None if bm is None else bm.ctypes.data_as(u64p), None, out.ctypes.data_as(C.POINTER(ScoredPoint)),
                                                counts.ctypes.data_as(u32p), None if counters is None else C.byref(counters), self.ALGORITHMS[algorithm]))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    @staticmethod
    def _entry_lists(custom_entry_points, nq: int):
        """one sequence of point offsets per query -> ([nq, width] u32, counts u32, width), or (None, None, 0)"""
        if custom_entry_points is None:
            return None, None, 0
        if len(custom_entry_points) != nq:
            raise ValueError(f"custom_entry_points has {len(custom_entry_points)} lists for {nq} queries")
        width = max(1, max((len(c) for c in custom_entry_points), default=1))
        cep_arr = np.zeros((nq, width), np.uint32)
        cep_cnt = np.zeros(nq, np.uint32)
        for i, c in enumerate(custom_entry_points):
            cep_arr[i, : len(c)] = np.asarray(c, dtype=np.uint32)
            cep_cnt[i] = len(c)
        return cep_arr, cep_cnt, width

    def _multi_batch(self, queries):
        """custom queries with multivector examples -> (kind, n_a, n_b, example vectors, example offsets, coef [nq, 1 + n_a] or None);
        one kind and one shape per batch"""
        flat = [_flat_multi(q, self._storage.dim) for q in queries]
        if not flat:
            return int(QueryKind.RecommendBestScore), 1, 0, np.zeros((0, self._storage.dim), np.float32), np.zeros(1, np.uint32), None
        kind, n_a, n_b = int(queries[0].kind), flat[0][2], flat[0][3]
        for q, f in zip(queries, flat):
            if int(q.kind) != kind or (f[2], f[3]) != (n_a, n_b):
                raise ValueError("one query kind and one shape (n_a, n_b) per call")
        base = np.cumsum([0] + [f[0].shape[0] for f in flat[:-1]])
        off = np.concatenate([f[1][:-1] + b for f, b in zip(flat, base)] + [[base[-1] + flat[-1][1][-1]]]).astype(np.uint32)
        coef = np.stack([f[4] for f in flat]) if kind == QueryKind.FeedbackNaive else None
        return kind, n_a, n_b, np.ascontiguousarray(np.concatenate([f[0] for f in flat])), off, coef

    def search_maxsim_custom(self, queries, top: int, ef: int, entry_point: int, entry_level: int, point_deleted=None,
                             counters: Optional[HwCounters] = None, custom_entry_points=None, algorithm: str = "hnsw"):
        """Custom queries whose examples are multivectors, on a multivector() graph (qb_hnsw_search_maxsim_custom_batch).  queries: a list of
        RecoBestScoreQuery / RecoSumScoresQuery / ContextQuery / FeedbackQuery / DiscoverQuery (one discover search) whose vectors are
        [vectors, dim] arrays, all of one kind and shape; custom_entry_points: one sequence of point offsets per query, or None;
        point_deleted: over points.  Returns one list of point offsets per query; a score equals MultiVectorView.score_points_custom."""
        if algorithm not in self.ALGORITHMS:
            raise ValueError(f"algorithm {algorithm!r} is not one of {sorted(self.ALGORITHMS)}")
        kind, n_a, n_b, vecs, off, coef = self._multi_batch(queries)
        nq = len(queries)
        cep_arr, cep_cnt, width = self._entry_lists(custom_entry_points, nq)
        out = np.zeros((max(nq, 1), max(top, 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(max(nq, 1), dtype=np.uint32)
        bm = _bitmap(point_deleted, self.info()[0])
        check(lib().qb_hnsw_search_maxsim_custom_batch(self._h, kind, vecs.ctypes.data_as(f32p), off.ctypes.data_as(u32p), int(n_a), int(n_b),
                                                       None if coef is None else coef.ctypes.data_as(f32p), nq, int(top), int(ef), int(entry_point),
                                                       int(entry_level), None if cep_arr is None else cep_arr.ctypes.data_as(u32p),
                                                       None if cep_cnt is None else cep_cnt.ctypes.data_as(u32p), width,
                                                       None if bm is None else bm.ctypes.data_as(u64p), None, out.ctypes.data_as(C.POINTER(ScoredPoint)),
                                                       counts.ctypes.data_as(u32p), None if counters is None else C.byref(counters),
                                                       self.ALGORITHMS[algorithm]))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def search_maxsim_discover(self, queries, top: int, ef: int, entry_point: int, entry_level: int, point_deleted=None,
                               counters: Optional[HwCounters] = None, algorithm: str = "hnsw"):
        """Discover with multivector examples as the reference runs it on an indexed segment (qb_hnsw_search_maxsim_discover_batch): a
        context search over the pairs for 10 entry points, then the discover search from them, in one call.  queries: DiscoverQuery
        objects with [vectors, dim] arrays, all with the same number of pairs."""
        if algorithm not in self.ALGORITHMS:
            raise ValueError(f"algorithm {algorithm!r} is not one of {sorted(self.ALGORITHMS)}")
        if any(int(q.kind) != QueryKind.Discover for q in queries):
            raise ValueError("search_maxsim_discover takes DiscoverQuery objects")
        _, n_pairs, _, vecs, off, _ = self._multi_batch(queries)
        nq = len(queries)
        out = np.zeros((max(nq, 1), max(top, 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(max(nq, 1), dtype=np.uint32)
        bm = _bitmap(point_deleted, self.info()[0])
        check(lib().qb_hnsw_search_maxsim_discover_batch(self._h, vecs.ctypes.data_as(f32p), off.ctypes.data_as(u32p), int(n_pairs), nq, int(top), int(ef),
                                                         int(entry_point), int(entry_level), None if bm is None else bm.ctypes.data_as(u64p), None,
                                                         out.ctypes.data_as(C.POINTER(ScoredPoint)), counts.ctypes.data_as(u32p),
                                                         None if counters is None else C.byref(counters), self.ALGORITHMS[algorithm]))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def search_discover(self, examples, n_pairs: int, top: int = 10, ef: int = 64, entry_point: int = 0, entry_level: int = 0, point_deleted=None,
                        counters: Optional[HwCounters] = None, algorithm: str = "hnsw"):
        """Discover as the reference runs it on an indexed segment (qb_hnsw_search_discover_batch): a context search over the pairs for
        10 entry points, then the discover search from them, in one call.  examples: [queries, 1 + 2 n_pairs, dim] (target, then pairs)."""
        if algorithm not in self.ALGORITHMS:
            raise ValueError(f"algorithm {algorithm!r} is not one of {sorted(self.ALGORITHMS)}")
        ex = self._examples(examples, 1 + 2 * int(n_pairs))
        nq = ex.shape[0]
        out = np.zeros((nq, max(top, 1)), dtype=SCORED_POINT_OFFSET)
        counts = np.zeros(nq, dtype=np.uint32)
        bm = _bitmap(point_deleted, self._storage.count)
        check(lib().qb_hnsw_search_discover_batch(self._h, ex.ctypes.data_as(f32p), int(n_pairs), nq, int(top), int(ef), int(entry_point), int(entry_level),
                                                  None if bm is None else bm.ctypes.data_as(u64p), None, out.ctypes.data_as(C.POINTER(ScoredPoint)),
                                                  counts.ctypes.data_as(u32p), None if counters is None else C.byref(counters), self.ALGORITHMS[algorithm]))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def stats(self, reset: bool = True) -> tuple[int, int]:
        a, b = C.c_uint64(), C.c_uint64()
        check(lib().qb_hnsw_stats(self._h, C.byref(a), C.byref(b), 1 if reset else 0))
        return int(a.value), int(b.value)

    def close(self):
        if self._h:
            lib().qb_hnsw_destroy(self._h)
            self._h = vp()

    def __del__(self):
        try:
            if sys is None or sys.is_finalizing():     # interpreter shutdown: module globals may already be gone
                return
            self.close()
        except Exception:
            pass
