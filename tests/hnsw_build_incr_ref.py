"""ctypes driver of tests/hnsw_build_incr_ref.c, the CPU restatement of the incremental device graph build (qb_hnsw_build_incremental):
a graph from a plain links.bin, the two-phase heal, the renumbering and the insertion of the new points, every step the oracle's own
arithmetic.  Compiled on first use like tests/hnsw_build_ref.py, into a per-user temporary directory keyed by the sources' hash."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from tests.hnsw_build_ref import SCORED

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_SRCS = [os.path.join(_HERE, "hnsw_build_incr_ref.c")] + [os.path.join(_ORACLE, f) for f in ("oracle.c", "mt.c", "train.c")]
_DEPS = _SRCS + [os.path.join(_HERE, "hnsw_build_ref.c"), os.path.join(_ORACLE, "hnsw.c")]
_LIB = None
GONE = 0xFFFFFFFF


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        h = hashlib.sha256(b"".join(open(f, "rb").read() for f in _DEPS)).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"qb_build_ref_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, f"libbuildincrref_{h}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.run(["gcc", "-O3", "-march=haswell", "-mpopcnt", "-ffp-contract=off", "-fPIC", "-shared", "-fvisibility=hidden", "-o", tmp, *_SRCS,
                            "-lm", "-lpthread"], check=True, capture_output=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u8p, u32p, f32p = C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_float)
        u32 = C.c_uint32
        L.qo_hnsw_from_plain.restype, L.qo_hnsw_from_plain.argtypes = vp, [f32p, u32, C.c_int, u32, u32, u32, u8p]
        L.qo_hnsw_heal.restype, L.qo_hnsw_heal.argtypes = u32, [vp, u32p, u32, C.c_int64]
        L.qo_hnsw_renumber.restype, L.qo_hnsw_renumber.argtypes = vp, [vp, u32p, f32p, u32, u8p, u32]
        L.qo_hnsw_insert_new.restype, L.qo_hnsw_insert_new.argtypes = None, [vp, u8p, u32, u32, C.c_int]
        L.qo_hnsw_entry.restype, L.qo_hnsw_entry.argtypes = None, [vp, u32p, u32p, u32p, u32p]
        L.qo_hnsw_export_plain.restype, L.qo_hnsw_export_plain.argtypes = C.c_uint64, [vp, vp]
        L.qo_hnsw_free.restype, L.qo_hnsw_free.argtypes = None, [vp]
        L.qo_hnsw_search_batch.restype = None
        L.qo_hnsw_search_batch.argtypes = [vp, f32p, u32, u32, u32, C.POINTER(C.c_uint64), u32, vp, u32p]
        _LIB = L
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class IncrGraph:
    """A graph of the restatement: the old graph (healed or not) over the old rows, or the new graph over the new rows."""

    def __init__(self, h, base):
        self._h, self._base = h, base

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

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

    @classmethod
    def from_plain(cls, base, distance: int, m: int, m0: int, blob) -> "IncrGraph":
        """A plain links.bin over `base` (the stored rows), each list cut to its first level_m links."""
        base = np.ascontiguousarray(base, dtype=np.float32)
        b = np.ascontiguousarray(blob, dtype=np.uint8)
        return cls(lib().qo_hnsw_from_plain(_p(base, C.c_float), base.shape[1], distance, m, m0, 1, _p(b, C.c_uint8)), base)

    def heal(self, old_to_new, ef_construct: int, only_item: int = -1) -> int:
        """The two-phase heal in place; returns the number of to-heal items.  only_item >= 0 heals that item alone."""
        self._o2n = np.ascontiguousarray(old_to_new, dtype=np.uint32)
        return int(lib().qo_hnsw_heal(self._h, _p(self._o2n, C.c_uint32), ef_construct, only_item))

    def renumber(self, old_to_new, new_base, levels, ef: int) -> "IncrGraph":
        o2n = np.ascontiguousarray(old_to_new, dtype=np.uint32)
        nb = np.ascontiguousarray(new_base, dtype=np.float32)
        lv = np.ascontiguousarray(levels, dtype=np.uint8)
        return IncrGraph(lib().qo_hnsw_renumber(self._h, _p(o2n, C.c_uint32), _p(nb, C.c_float), nb.shape[0], _p(lv, C.c_uint8), ef), nb)

    def insert_new(self, is_new, batch: int, serial_points: int, serial: bool = False) -> None:
        m = np.ascontiguousarray(is_new, dtype=np.uint8)
        lib().qo_hnsw_insert_new(self._h, _p(m, C.c_uint8), batch, serial_points, 1 if serial else 0)

    def entry(self):
        a, b, c, d = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        lib().qo_hnsw_entry(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d))
        return int(a.value), int(b.value)

    def export_plain(self) -> np.ndarray:
        n = int(lib().qo_hnsw_export_plain(self._h, None))
        out = np.zeros(n, dtype=np.uint8)
        lib().qo_hnsw_export_plain(self._h, out.ctypes.data_as(C.c_void_p))
        return out


def build_incremental(old_base, old_blob, distance: int, m: int, m0: int, new_base, old_to_new, levels, ef_construct: int = 100, deleted=None,
                      batch: int = 512, serial_points: int = 256, serial: bool = False):
    """The whole of qb_hnsw_build_incremental on the CPU: returns (new graph, (entry, entry level)).  deleted: bool per new point (the
    storage's resident flags); batch / serial_points as given to the device (0 = 512 / 256)."""
    batch = batch or 512
    serial_points = serial_points or 256
    o2n = np.ascontiguousarray(old_to_new, dtype=np.uint32)
    n_new = np.asarray(new_base).shape[0]
    old = IncrGraph.from_plain(old_base, distance, m, m0, old_blob)
    old.heal(o2n, ef_construct)
    g = old.renumber(o2n, new_base, levels, max(ef_construct, m0))
    old.close()
    is_new = np.ones(n_new, dtype=bool)
    is_new[o2n[o2n != GONE]] = False
    if deleted is not None:
        is_new &= ~np.asarray(deleted, dtype=bool)
    g.insert_new(is_new, batch, serial_points, serial)
    return g, g.entry()
