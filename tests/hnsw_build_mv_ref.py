"""ctypes driver of tests/hnsw_build_mv_ref.c, the CPU restatement of the device graph build over multivector points
(qb_hnsw_build_multivector): the oracle's serial builder and the batched two-phase schedule of tests/hnsw_build_ref.c, every pair score
being the oracle's MaxSim (qo_maxsim_f32) with the first point's token rows as the query.  Compiled on first use like
tests/hnsw_build_ref.py, into a per-user temporary directory keyed by the sources' hash."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tests import hnsw_build_ref as br

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_SRCS = [os.path.join(_HERE, "hnsw_build_mv_ref.c")] + [os.path.join(_ORACLE, f) for f in ("oracle.c", "mt.c", "train.c")]
_DEPS = _SRCS + [os.path.join(_HERE, "hnsw_build_ref.c"), os.path.join(_ORACLE, "hnsw.c")]
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        h = hashlib.sha256(b"".join(open(f, "rb").read() for f in _DEPS)).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"qb_build_ref_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libbuildmvref_{h}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["gcc", "-O3", "-march=haswell", "-mpopcnt", "-ffp-contract=off", "-fPIC", "-shared", "-fvisibility=hidden", "-o", tmp, *_SRCS,
                            "-lm", "-lpthread"], check=True, capture_output=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u8p, u32p, u64p, f32p = C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_float)
        u32 = C.c_uint32
        L.qo_mv_bind.restype, L.qo_mv_bind.argtypes = None, [f32p, f32p, u32p, u32]
        L.qo_hnsw_build_levels.restype, L.qo_hnsw_build_levels.argtypes = vp, [f32p, u32, u32, C.c_int, u32, u32, u32, u8p, u32p]
        L.qo_hnsw_build_batched.restype = vp
        L.qo_hnsw_build_batched.argtypes = [f32p, u32, u32, C.c_int, u32, u32, u32, u8p, u64p, u32, u32, C.c_uint64]
        L.qo_hnsw_entry.restype, L.qo_hnsw_entry.argtypes = None, [vp, u32p, u32p, u32p, u32p]
        L.qo_hnsw_export_plain.restype, L.qo_hnsw_export_plain.argtypes = C.c_uint64, [vp, vp]
        L.qo_hnsw_free.restype, L.qo_hnsw_free.argtypes = None, [vp]
        _LIB = L
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class MvRefGraph:
    """A graph over multivector points built on the CPU.  tokens: the stored (preprocessed) token rows [rows, dim]; offsets: n + 1 row
    offsets (point p = rows offsets[p] .. offsets[p + 1))."""

    def __init__(self, h, keep):
        self._h, self._keep = h, keep

    @staticmethod
    def _bind(tokens, offsets):
        tokens = np.ascontiguousarray(tokens, dtype=np.float32)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint32)
        base = np.zeros(offsets.size - 1, dtype=np.float32)
        lib().qo_mv_bind(_p(base, C.c_float), _p(tokens, C.c_float), _p(offsets, C.c_uint32), tokens.shape[1])
        return base, tokens, offsets

    @classmethod
    def serial(cls, tokens, offsets, distance: int, m: int, m0: int, ef_construct: int, levels, order=None) -> "MvRefGraph":
        """link_new_point for every point of `order` (default: id order) with the given levels."""
        base, tokens, offsets = cls._bind(tokens, offsets)
        levels = np.ascontiguousarray(levels, dtype=np.uint8)
        o = None if order is None else np.ascontiguousarray(order, dtype=np.uint32)
        h = lib().qo_hnsw_build_levels(_p(base, C.c_float), base.size, 1, distance, m, m0, ef_construct, _p(levels, C.c_uint8),
                                       None if o is None else _p(o, C.c_uint32))
        return cls(h, (base, tokens, offsets, levels, o))

    @classmethod
    def batched(cls, tokens, offsets, distance: int, m: int, m0: int, ef_construct: int, levels, deleted=None, batch: int = 512,
                serial_points: int = 256, shuffle: int = 0) -> "MvRefGraph":
        """qb_hnsw_build_multivector's schedule, single-threaded; deleted = bool per point (not inserted)."""
        base, tokens, offsets = cls._bind(tokens, offsets)
        levels = np.ascontiguousarray(levels, dtype=np.uint8)
        bm = None if deleted is None else bitmap(deleted)
        h = lib().qo_hnsw_build_batched(_p(base, C.c_float), base.size, 1, distance, m, m0, ef_construct, _p(levels, C.c_uint8),
                                        None if bm is None else _p(bm, C.c_uint64), batch, serial_points, shuffle)
        return cls(h, (base, tokens, offsets, levels, bm))

    def entry(self):
        a, b, c, d = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        lib().qo_hnsw_entry(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d))
        return int(a.value), int(b.value)

    def export_plain(self) -> np.ndarray:
        n = int(lib().qo_hnsw_export_plain(self._h, None))
        out = np.zeros(n, dtype=np.uint8)
        lib().qo_hnsw_export_plain(self._h, out.ctypes.data_as(C.c_void_p))
        return out

    def close(self):
        if self._h:
            lib().qo_hnsw_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def bitmap(deleted) -> np.ndarray:
    """bool per point -> the u64 bitmap the builds take"""
    bits = np.packbits(np.asarray(deleted, dtype=bool), bitorder="little")
    bm = np.zeros((bits.size + 7) // 8 * 8, dtype=np.uint8)
    bm[: bits.size] = bits
    return bm.view(np.uint64)


PlainGraph = br.PlainGraph


def clustered_tokens(oracle, distance: int, n_points: int, dim: int, lens=(1, 12), seed: int = 1, empty: float = 0.0):
    """A seeded multivector collection like the one tests/test_gpu_hnsw_multivector.py searches: token runs of lens[0] .. lens[1] rows
    (a share `empty` of the points with none), each point's tokens around one of n_points / 8 centres.  Returns the stored
    (preprocessed) rows and the n_points + 1 offsets."""
    rng = np.random.default_rng(seed)
    runs = rng.integers(lens[0], lens[1] + 1, n_points)
    runs[rng.random(n_points) < empty] = 0
    off = np.concatenate([[0], np.cumsum(runs)]).astype(np.uint32)
    centers = rng.standard_normal((max(n_points // 8, 1), dim)).astype(np.float32)
    raw = (centers[np.repeat(rng.integers(0, centers.shape[0], n_points), runs)] + 0.5 * rng.standard_normal((int(off[-1]), dim))).astype(np.float32)
    return oracle.preprocess_rows_f32(distance, raw), off
