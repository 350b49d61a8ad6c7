"""The checker of the sparse custom queries (tests/sparse_custom_ref.c) needs no GPU: it reproduces the reference's own score_vectors
cases (kept as data in tests/golden/sparse_score_reference_cases.json), agrees with a NumPy restatement on random data, and shows on a
crafted point why the storage keeps user dims.  The kernels of qb_sparse.o that predate the custom scan compile to the machine code
recorded in tests/golden/sparse_kernels_sass.json (needs cuobjdump and a built library, no GPU)."""
import json
import os
import shutil
import sys

import numpy as np
import pytest

sys.dont_write_bytecode = True
from tests import sparse_custom_ref as scr  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def o():
    from oracle import oracle

    oracle.ensure_built()
    return oracle


def test_reference_score_cases():
    with open(os.path.join(ROOT, "tests", "golden", "sparse_score_reference_cases.json")) as f:
        cases = json.load(f)["cases"]
    assert len(cases) == 5
    for c in cases:
        assert scr.score(c["a"], c["b"]) == c["score"], c["name"]


def _numpy_sim(row, example) -> np.float32:
    """score_vectors as an ordered loop: both sides sorted by dim, 0 + products of the shared dims in ascending order, f32 throughout"""
    rd, rw = row
    ed, ew = example
    ro, eo = np.argsort(rd, kind="stable"), np.argsort(ed, kind="stable")
    rd, rw, ed, ew = rd[ro], rw[ro], ed[eo], ew[eo]
    s = np.float32(0.0)
    i = j = 0
    while i < rd.size and j < ed.size:
        if rd[i] < ed[j]:
            i += 1
        elif rd[i] > ed[j]:
            j += 1
        else:
            s = np.float32(s + np.float32(ew[j] * rw[i]))
            i += 1
            j += 1
    return s


def _examples(rng, E, pool, empty_at=None):
    ex = []
    for j in range(E):
        k = 0 if j == empty_at else int(rng.integers(1, 12))
        d = rng.choice(pool, size=k, replace=False).astype(np.uint32)
        w = (rng.standard_normal(k) * 0.7).astype(np.float32)
        ex.append((d, w))
    return ex


def _orderable(x) -> int:
    """the (score desc) half of the project's keys: -0.0 below +0.0, NaN above +inf"""
    u = int(np.float32(x).view(np.uint32))
    if (u & 0x7FFFFFFF) > 0x7F800000:
        return 0xFFC00000
    return (~u & 0xFFFFFFFF) if u & 0x80000000 else (u | 0x80000000)


SHAPES = [(1, 1, 0), (1, 3, 2), (2, 0, 1), (2, 2, 2), (3, 0, 0), (3, 2, 0), (4, 1, 0), (4, 3, 0), (5, 2, 0)]


@pytest.mark.parametrize("kind,n_a,n_b", SHAPES)
def test_checker_equals_numpy_restatement(o, kind, n_a, n_b):
    rng = np.random.default_rng(kind * 10 + n_a)
    pool = np.concatenate([[0, 0xFFFFFFFF], rng.choice(1 << 31, 60, replace=False) * 2 + 1]).astype(np.uint32)
    indptr, dims, w = scr.random_rows(rng, 300, 8, pool, negative=0.3, empty=0.05)
    st = scr.Storage(indptr, dims, w)
    E = {1: n_a + n_b, 2: n_a + n_b, 3: 1 + 2 * n_a, 4: 2 * n_a, 5: 1 + 2 * n_a}[kind]
    ex = _examples(rng, E, pool, empty_at=E - 1 if E > 1 else None)
    coef = None
    if kind == scr.FEEDBACK:
        _, _, part = o.feedback_pairs(rng.random(4).astype(np.float32), 1.5, 0.4)
        coef = np.concatenate([[0.9], part[:n_a], np.zeros(max(0, n_a - part.size))]).astype(np.float32)
    deleted = rng.random(300) < 0.2
    bm = np.packbits(np.concatenate([deleted, np.zeros(20, bool)]), bitorder="little").view(np.uint64)[: (300 + 63) // 64].copy()
    id_list = rng.choice(300, 90, replace=False).astype(np.uint32)
    for dl, il in ((None, None), (bm, None), (bm, id_list), (None, id_list)):
        ids = st.points(dl, il)
        want_ids = [i for i in (range(300) if il is None else il) if dl is None or not deleted[i]]
        assert ids.tolist() == want_ids
        rows = [(dims[indptr[i]:indptr[i + 1]], w[indptr[i]:indptr[i + 1]]) for i in ids]
        sims = np.array([[_numpy_sim(r, e) for r in rows] for e in ex], np.float32).reshape(E, len(rows))
        got_sims = st.sims(ex, ids)
        assert np.array_equal(got_sims.view(np.uint32), sims.view(np.uint32))
        scores = scr.fold(o, kind, n_a, n_b, sims, coef)
        for top in (1, 10, 400):
            got, cpu, io = st.search(o, kind, n_a, n_b, ex, top, coef, dl, il)
            order = sorted(range(len(ids)), key=lambda k: (-_orderable(scores[k]), int(ids[k])))[:top]
            assert got["idx"].tolist() == [int(ids[k]) for k in order]
            assert np.array_equal(got["score"].view(np.uint32), scores[order].view(np.uint32))
            lens = np.array([len(r[0]) for r in rows], np.int64)
            assert cpu == sum(4 * (int(lens.sum()) + len(ids) * len(d)) for d, _ in ex) and io == 0
    st.close()


def test_on_disk_counts_vector_io_read():
    rng = np.random.default_rng(3)
    indptr, dims, w = scr.random_rows(rng, 50, 6, np.arange(40, dtype=np.uint32))
    ex = _examples(rng, 3, np.arange(40, dtype=np.uint32))
    ids = np.arange(50, dtype=np.uint32)
    for on_disk, mult in ((False, 0), (True, 4)):
        st = scr.Storage(indptr, dims, w, on_disk=on_disk)
        cpu, io = st.counters(ex, ids)
        assert io == 2 * int(indptr[-1]) * mult
        assert cpu == sum(4 * (int(indptr[-1]) + 50 * len(d)) for d, _ in ex)
        st.close()


def test_user_dim_order_differs_from_internal_order():
    """Products 1, 1e8 and -1e8 at user dims 5, 7 and 9.  Summed in user-dim order: 0 + 1 + 1e8 - 1e8 = 0.0 (the 1 is lost in 1e8).  An
    IndicesTracker that met dim 9 first and dim 5 last numbers them 0, 1, 2, and the internal order sums -1e8 + 1e8 + 1 = 1.0.  The
    custom scorer merges in user dims, so the storage keeps them."""
    stored = (np.array([5, 7, 9], np.uint32), np.array([1.0, 1e4, 1e4], np.float32))
    example = (np.array([9, 5, 7], np.uint32), np.array([-1e4, 1.0, 1e4], np.float32))
    assert scr.score(example, stored) == 0.0
    tracker = {9: 0, 7: 1, 5: 2}
    remap = lambda v: (np.array([tracker[int(d)] for d in v[0]], np.uint32), v[1])   # noqa: E731
    assert scr.score(remap(example), remap(stored)) == 1.0
    st = scr.Storage(np.array([0, 3], np.uint64), *stored)
    assert st.sims([example], [0])[0, 0] == 0.0
    st.close()


def test_pre_existing_sparse_kernels_compile_to_the_same_code():
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    if not os.path.exists(cuobjdump) and not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not installed")
    from tests.test_kernels_unchanged import kernels

    with open(os.path.join(ROOT, "tests", "golden", "sparse_kernels_sass.json")) as f:
        golden = json.load(f)
    for obj, funcs in golden.items():
        path = os.path.join(ROOT, "qdrant_b200", "lib", obj)
        if not os.path.exists(path):
            pytest.skip(f"{path} not built (build() compiles the library)")
        got = kernels(path)
        assert len(funcs) == 6
        for name, want in funcs.items():
            assert name in got, f"{obj}: {name} is gone"
            assert got[name] == want, f"{obj}: {name} changed: {got[name]} != {want}"
