"""ctypes driver of tests/hnsw_build_ref.c, the CPU restatement of the device graph build (qb_hnsw_build): the oracle's serial builder
with given levels and order, the batched two-phase schedule, and the levels the oracle's own builder drew.  The library is compiled on
first use, from the oracle's sources with the oracle's flags (oracle/Makefile), into a per-user temporary directory keyed by the
sources' hash, so a read-only checkout works too."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_SRCS = [os.path.join(_HERE, "hnsw_build_ref.c")] + [os.path.join(_ORACLE, f) for f in ("oracle.c", "mt.c", "train.c")]
_DEPS = _SRCS + [os.path.join(_ORACLE, "hnsw.c")]
_LIB = None
SCORED = np.dtype([("idx", np.uint32), ("score", np.float32)])   # #[repr(C)] ScoredPointOffset


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        h = hashlib.sha256(b"".join(open(f, "rb").read() for f in _DEPS)).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"qb_build_ref_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libbuildref_{h}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["gcc", "-O3", "-march=haswell", "-mpopcnt", "-ffp-contract=off", "-fPIC", "-shared", "-fvisibility=hidden", "-o", tmp, *_SRCS,
                            "-lm", "-lpthread"], check=True, capture_output=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u8p, u32p, u64p, f32p = C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_float)
        u32 = C.c_uint32
        L.qo_hnsw_build_levels.restype, L.qo_hnsw_build_levels.argtypes = vp, [f32p, u32, u32, C.c_int, u32, u32, u32, u8p, u32p]
        L.qo_hnsw_build_batched.restype = vp
        L.qo_hnsw_build_batched.argtypes = [f32p, u32, u32, C.c_int, u32, u32, u32, u8p, u64p, u32, u32, C.c_uint64]
        L.qo_hnsw_build.restype, L.qo_hnsw_build.argtypes = vp, [f32p, u32, u32, C.c_int, u32, u32, C.c_uint64]
        L.qo_hnsw_levels.restype, L.qo_hnsw_levels.argtypes = None, [vp, u8p]
        L.qo_hnsw_entry.restype, L.qo_hnsw_entry.argtypes = None, [vp, u32p, u32p, u32p, u32p]
        L.qo_hnsw_export_plain.restype, L.qo_hnsw_export_plain.argtypes = C.c_uint64, [vp, vp]
        L.qo_hnsw_free.restype, L.qo_hnsw_free.argtypes = None, [vp]
        L.qo_hnsw_search_batch.restype = None
        L.qo_hnsw_search_batch.argtypes = [vp, f32p, u32, u32, u32, u64p, u32, vp, u32p]
        _LIB = L
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class RefGraph:
    """A graph built on the CPU by the oracle's HNSW code.  `base` = the stored (preprocessed) rows."""

    def __init__(self, h, base, levels):
        self._h, self._base, self._levels = h, base, levels

    @classmethod
    def serial(cls, base, distance: int, m: int, m0: int, ef_construct: int, levels, order=None) -> "RefGraph":
        """link_new_point for every point of `order` (default: id order) with the given levels."""
        base = np.ascontiguousarray(base, dtype=np.float32)
        levels = np.ascontiguousarray(levels, dtype=np.uint8)
        o = None if order is None else np.ascontiguousarray(order, dtype=np.uint32)
        h = lib().qo_hnsw_build_levels(_p(base, C.c_float), base.shape[0], base.shape[1], distance, m, m0, ef_construct, _p(levels, C.c_uint8),
                                       None if o is None else _p(o, C.c_uint32))
        return cls(h, base, (levels, o))

    @classmethod
    def batched(cls, base, distance: int, m: int, m0: int, ef_construct: int, levels, deleted=None, batch: int = 512, serial_points: int = 256,
                shuffle: int = 0) -> "RefGraph":
        """The device build's schedule (qb_hnsw_build), single-threaded; deleted = bool per point (not inserted)."""
        base = np.ascontiguousarray(base, dtype=np.float32)
        levels = np.ascontiguousarray(levels, dtype=np.uint8)
        bm = None
        if deleted is not None:
            bits = np.packbits(np.asarray(deleted, dtype=bool), bitorder="little")
            bm = np.zeros((bits.size + 7) // 8 * 8, dtype=np.uint8)
            bm[: bits.size] = bits
            bm = bm.view(np.uint64)
        h = lib().qo_hnsw_build_batched(_p(base, C.c_float), base.shape[0], base.shape[1], distance, m, m0, ef_construct, _p(levels, C.c_uint8),
                                        None if bm is None else _p(bm, C.c_uint64), batch, serial_points, shuffle)
        return cls(h, base, (levels, bm))

    @classmethod
    def oracle_build(cls, base, distance: int, m: int, ef_construct: int, seed: int) -> "RefGraph":
        """The oracle's own builder (qo_hnsw_build, one thread, m0 = 2m, its own level draw)."""
        base = np.ascontiguousarray(base, dtype=np.float32)
        h = lib().qo_hnsw_build(_p(base, C.c_float), base.shape[0], base.shape[1], distance, m, ef_construct, seed)
        return cls(h, base, None)

    def levels(self) -> np.ndarray:
        out = np.zeros(self._base.shape[0], dtype=np.uint8)
        lib().qo_hnsw_levels(self._h, _p(out, C.c_uint8))
        return out

    def entry(self):
        a, b, c, d = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        lib().qo_hnsw_entry(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d))
        return int(a.value), int(b.value)

    def export_plain(self) -> np.ndarray:
        n = int(lib().qo_hnsw_export_plain(self._h, None))
        out = np.zeros(n, dtype=np.uint8)
        lib().qo_hnsw_export_plain(self._h, out.ctypes.data_as(C.c_void_p))
        return out

    def search_batch(self, queries_pre, top: int, ef: int, threads: int = 4):
        """GraphLayers::search on this graph with the oracle's traversal and CPU scorer (queries already preprocessed)."""
        q = np.ascontiguousarray(np.atleast_2d(queries_pre), dtype=np.float32)
        nq = q.shape[0]
        out = np.zeros((nq, top), dtype=SCORED)
        counts = np.zeros(nq, dtype=np.uint32)
        lib().qo_hnsw_search_batch(self._h, _p(q, C.c_float), nq, top, ef, None, threads, out.ctypes.data_as(C.c_void_p), _p(counts, C.c_uint32))
        return [out[i, : counts[i]].copy() for i in range(nq)]

    def close(self):
        if self._h:
            lib().qo_hnsw_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PlainGraph:
    """A plain links.bin parsed on the host: links(level, p) = GraphLinks::links (view.rs:203-215)."""

    def __init__(self, blob):
        b = np.ascontiguousarray(blob, dtype=np.uint8)
        n, levels, n_nb, n_off, pad = (int(x) for x in b[:40].view(np.uint64))
        o = 64
        self.n, self.levels = n, levels
        self.level_offsets = b[o:o + 8 * levels].view(np.uint64); o += 8 * levels
        self.reindex = b[o:o + 4 * n].view(np.uint32); o += 4 * n
        self.neighbors = b[o:o + 4 * n_nb].view(np.uint32); o += 4 * n_nb + pad
        self.offsets = b[o:o + 8 * n_off].view(np.uint64)
        # a point's level: the last level whose row count its reindex is below (point_level, view.rs:354-369)
        counts = [int(self.level_offsets[l + 1] - self.level_offsets[l]) if l + 1 < levels else n_off - 1 - int(self.level_offsets[l]) for l in range(levels)]
        self.point_level = np.zeros(n, dtype=np.int64)
        for l in range(1, levels):
            self.point_level[self.reindex < counts[l]] = l

    def links(self, level: int, p: int) -> np.ndarray:
        idx = p if level == 0 else int(self.level_offsets[level]) + int(self.reindex[p])
        return self.neighbors[int(self.offsets[idx]):int(self.offsets[idx + 1])]
