"""ctypes driver of the build restatements in the device's tie order, the checkers of the device builds over Uint8 storages.

One library per (datatype, keyed): the incremental restatement (tests/hnsw_build_incr_ref.c, which compiles tests/hnsw_build_ref.c and
the oracle's HNSW into itself) for f32 rows, or its u8 form (tests/hnsw_build_u8_ref.c, Metric<u8>::similarity of two stored rows as
the pair score).  keyed=False compiles the sources as they are: the reference's score-only heaps.  keyed=True compiles copies of them in
a directory of their own whose oracle/hnsw.c is tests/hnsw_keyed_oracle.c, so every level-0 comparison of an insert's search and of the
heal's `nearest` is made on (score desc, id asc) keys, as on the device; the restatements' own code is the same.  Built on first use with
the oracle's flags into a per-user temporary directory keyed by the sources' hash, so a read-only checkout works too."""
import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

from tests.hnsw_build_incr_ref import GONE

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_REST = [os.path.join(_ORACLE, f) for f in ("oracle.c", "mt.c", "train.c")]
_MAIN = {"f32": "hnsw_build_incr_ref.c", "u8": "hnsw_build_u8_ref.c"}
_INCLUDED = ["hnsw_build_incr_ref.c", "hnsw_build_ref.c", "hnsw_build_u8_ref.c", "hnsw_keyed_oracle.c"]
_LIBS = {}


def lib(dtype: str = "u8", keyed: bool = True) -> C.CDLL:
    if (dtype, keyed) in _LIBS:
        return _LIBS[(dtype, keyed)]
    deps = [os.path.join(_HERE, f) for f in _INCLUDED] + [os.path.join(_ORACLE, "hnsw.c")] + _REST
    h = hashlib.sha256(b"".join(open(f, "rb").read() for f in deps) + f"{dtype} {keyed}".encode()).hexdigest()[:16]
    d = os.path.join(tempfile.gettempdir(), f"qb_build_ref_{os.getuid()}")
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, f"libbuildkeyed_{dtype}_{int(keyed)}_{h}.so")
    if not os.path.exists(so):
        main, defines = os.path.join(_HERE, _MAIN[dtype]), []
        tree = None
        if keyed:
            # <tree>/tests: the restatements, <tree>/oracle/hnsw.c: the keyed oracle, which includes the real one
            tree = tempfile.mkdtemp(dir=d)
            os.makedirs(os.path.join(tree, "tests")); os.makedirs(os.path.join(tree, "oracle"))
            for f in ("hnsw_build_incr_ref.c", "hnsw_build_ref.c", "hnsw_build_u8_ref.c"):
                shutil.copy(os.path.join(_HERE, f), os.path.join(tree, "tests", f))
            shutil.copy(os.path.join(_HERE, "hnsw_keyed_oracle.c"), os.path.join(tree, "oracle", "hnsw.c"))
            main = os.path.join(tree, "tests", _MAIN[dtype])
            defines = [f'-DQB_ORACLE_HNSW="{os.path.join(_ORACLE, "hnsw.c")}"']
        tmp = f"{so}.{os.getpid()}.tmp"
        try:
            subprocess.run(["gcc", "-O3", "-march=haswell", "-mpopcnt", "-ffp-contract=off", "-fPIC", "-shared", "-fvisibility=hidden", *defines, "-o", tmp,
                            main, *_REST, "-lm", "-lpthread"], check=True, capture_output=True)
        finally:
            if tree:
                shutil.rmtree(tree, ignore_errors=True)
        os.replace(tmp, so)
    L = C.CDLL(so)
    vp, u8p, u32p, u64p, f32p, u32 = C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_float), C.c_uint32
    L.qo_hnsw_build_batched.restype = vp
    L.qo_hnsw_build_batched.argtypes = [f32p, u32, u32, C.c_int, u32, u32, u32, u8p, u64p, u32, u32, C.c_uint64]
    L.qo_hnsw_build_levels.restype, L.qo_hnsw_build_levels.argtypes = vp, [f32p, u32, u32, C.c_int, u32, u32, u32, u8p, u32p]
    L.qo_hnsw_from_plain.restype, L.qo_hnsw_from_plain.argtypes = vp, [f32p, u32, C.c_int, u32, u32, u32, u8p]
    L.qo_hnsw_heal.restype, L.qo_hnsw_heal.argtypes = u32, [vp, u32p, u32, C.c_int64]
    L.qo_hnsw_renumber.restype, L.qo_hnsw_renumber.argtypes = vp, [vp, u32p, f32p, u32, u8p, u32]
    L.qo_hnsw_insert_new.restype, L.qo_hnsw_insert_new.argtypes = None, [vp, u8p, u32, u32, C.c_int]
    L.qo_hnsw_entry.restype, L.qo_hnsw_entry.argtypes = None, [vp, u32p, u32p, u32p, u32p]
    L.qo_hnsw_export_plain.restype, L.qo_hnsw_export_plain.argtypes = C.c_uint64, [vp, vp]
    L.qo_hnsw_free.restype, L.qo_hnsw_free.argtypes = None, [vp]
    if dtype == "u8":
        L.qo_u8_bind.restype, L.qo_u8_bind.argtypes = None, [f32p, u8p, u32]
    _LIBS[(dtype, keyed)] = L
    return L


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


class Graph:
    """A graph of one of the libraries; keeps alive the arrays it was built over"""

    def __init__(self, L, h, keep):
        self._L, self._h, self._keep = L, h, keep

    def entry(self):
        a, b, c, d = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        self._L.qo_hnsw_entry(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d))
        return int(a.value), int(b.value)

    def export_plain(self) -> np.ndarray:
        n = int(self._L.qo_hnsw_export_plain(self._h, None))
        out = np.zeros(n, dtype=np.uint8)
        self._L.qo_hnsw_export_plain(self._h, out.ctypes.data_as(C.c_void_p))
        return out

    def close(self):
        if self._h:
            self._L.qo_hnsw_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _base(L, dtype, rows):
    """f32: the rows themselves; u8: one float per point naming it, the rows bound to the library"""
    if dtype == "f32":
        return np.ascontiguousarray(rows, dtype=np.float32), None
    r = np.ascontiguousarray(rows, dtype=np.uint8)
    base = np.zeros((r.shape[0], 1), dtype=np.float32)
    L.qo_u8_bind(_p(base, C.c_float), _p(r, C.c_uint8), r.shape[1])
    return base, r


def _bitmap(deleted):
    if deleted is None:
        return None
    bits = np.packbits(np.asarray(deleted, dtype=bool), bitorder="little")
    bm = np.zeros((bits.size + 7) // 8 * 8, dtype=np.uint8)
    bm[: bits.size] = bits
    return bm.view(np.uint64)


def batched(rows, distance: int, m: int, m0: int, ef_construct: int, levels, deleted=None, batch: int = 512, serial_points: int = 256,
            dtype: str = "u8", keyed: bool = True) -> Graph:
    """qb_hnsw_build's schedule over the rows (the oracle's distance codes), single-threaded; deleted = bool per point (not inserted)"""
    L = lib(dtype, keyed)
    base, r = _base(L, dtype, rows)
    lv = np.ascontiguousarray(levels, dtype=np.uint8)
    bm = _bitmap(deleted)
    h = L.qo_hnsw_build_batched(_p(base, C.c_float), base.shape[0], base.shape[1], distance, m, m0, ef_construct, _p(lv, C.c_uint8),
                                None if bm is None else _p(bm, C.c_uint64), batch, serial_points, 0)
    return Graph(L, h, (base, r, lv, bm))


def serial(rows, distance: int, m: int, m0: int, ef_construct: int, levels, dtype: str = "u8", keyed: bool = True) -> Graph:
    """link_new_point for every point in id order with the given levels"""
    L = lib(dtype, keyed)
    base, r = _base(L, dtype, rows)
    lv = np.ascontiguousarray(levels, dtype=np.uint8)
    h = L.qo_hnsw_build_levels(_p(base, C.c_float), base.shape[0], base.shape[1], distance, m, m0, ef_construct, _p(lv, C.c_uint8), None)
    return Graph(L, h, (base, r, lv))


def build_incremental(old_rows, old_blob, distance: int, m: int, m0: int, new_rows, old_to_new, levels, ef_construct: int = 100, deleted=None,
                      batch: int = 512, serial_points: int = 256, dtype: str = "u8", keyed: bool = True):
    """qb_hnsw_build_incremental on the CPU (tests/hnsw_build_incr_ref.py's steps): returns (new graph, (entry, entry level)).  The old and
    the new rows are bound as one array, the old graph's points first, so one binding serves the heal and the inserts."""
    L = lib(dtype, keyed)
    n_old = np.asarray(old_rows).shape[0]
    base, r = _base(L, dtype, np.concatenate([np.asarray(old_rows), np.asarray(new_rows)]))
    ob, nb = base[:n_old], base[n_old:]
    blob = np.ascontiguousarray(old_blob, dtype=np.uint8)
    old = L.qo_hnsw_from_plain(_p(ob, C.c_float), base.shape[1], distance, m, m0, 1, _p(blob, C.c_uint8))
    o2n = np.ascontiguousarray(old_to_new, dtype=np.uint32)
    L.qo_hnsw_heal(old, _p(o2n, C.c_uint32), ef_construct, -1)
    lv = np.ascontiguousarray(levels, dtype=np.uint8)
    g = Graph(L, L.qo_hnsw_renumber(old, _p(o2n, C.c_uint32), _p(nb, C.c_float), nb.shape[0], _p(lv, C.c_uint8), max(ef_construct, m0)),
              (base, r, lv))
    L.qo_hnsw_free(old)
    is_new = np.ones(nb.shape[0], dtype=bool)
    is_new[o2n[o2n != GONE]] = False
    if deleted is not None:
        is_new &= ~np.asarray(deleted, dtype=bool)
    mask = np.ascontiguousarray(is_new, dtype=np.uint8)
    L.qo_hnsw_insert_new(g._h, _p(mask, C.c_uint8), batch or 512, serial_points or 256, 0)
    return g, g.entry()
