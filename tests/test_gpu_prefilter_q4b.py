"""The first stage of the 6-bit plane's scan on the block-scaled 4-bit plane (dense_q4b_filter_kernel, the default) and on the 6-bit plane's own
5-bit codes (option prefilter_stage1 = 5).  Either way results must equal the exact f32 scan bit for bit, and overflowing lists fall back on
the device."""
import numpy as np
import pytest

from tests.test_gpu_prefilter_planes import search_both_ways
from tests.test_gpu_prefilter_sample import set_id_base

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def with_stage1(qb, stage1, fn):
    qb.set_option("prefilter_stage1", stage1)
    try:
        return fn()
    finally:
        qb.set_option("prefilter_stage1", 0)


@pytest.mark.parametrize("dist,n,dim,top", [("Dot", 540_001, 40, 5), ("Dot", 524_289, 200, 16), ("Cosine", 530_000, 768, 10), ("Cosine", 524_300, 1000, 1)])
def test_block_scaled_stage_is_exact(qb, oracle, dist, n, dim, top):
    """Dims that are not a multiple of the 16-dimension blocks, odd row counts, rows with one large block and the rest near zero, zero and
    denormal rows, deletions and id_base != 0: bit-identical to the exact scan and to the 5-bit stage, no fallback."""
    d = getattr(qb.Distance, dist)
    rng = np.random.default_rng(dim * 5 + top)
    base = rng.standard_normal((n, dim), dtype=np.float32)
    base[500:600, 16:] *= np.float32(1e-3)                  # one block far above the rest of the row
    base[700:710, : dim // 2] = 0.0                          # all-zero blocks
    if d == qb.Distance.Cosine:
        base = oracle.preprocess_rows_f32(oracle.COSINE, base)
    else:
        base *= rng.uniform(0.2, 3.0, (n, 1)).astype(np.float32)
        base[1000:1010] = 0.0
        base[2000:2010] *= np.float32(1e-38)
    queries = [rng.standard_normal(dim).astype(np.float32) for _ in range(2)] + [base[n - 1] * 2.0, base[550] * 3.0]
    deleted = rng.random(n) < 0.02
    deleted[[n - 1, 550]] = False
    st = qb.DenseVectorStorage(base, d)
    set_id_base(st, 7)
    got4, (s4, r4) = search_both_ways(qb, st, queries, top, 0, deleted)
    got5, (s5, r5) = with_stage1(qb, 5, lambda: search_both_ways(qb, st, queries, top, 0, deleted))
    assert (s4, r4, s5, r5) == (4, 0, 4, 0)
    for a, b in zip(got4, got5):
        np.testing.assert_array_equal(a["idx"], b["idx"])
        np.testing.assert_array_equal(a["score"].view(np.uint32), b["score"].view(np.uint32))
    st.close()


@pytest.mark.parametrize("stage1", [0, 5])
def test_first_stage_overflow_falls_back_on_either_stage(qb, stage1):
    """2 200 000 copies of a row whose quantised codes are poor but whose exact score lies just below the sample threshold overflow the
    first-stage list (2^21 rows) on both stages: the search falls back.  With 200 000 of them deleted the list holds the rest and the 6-bit
    test drops them."""
    rng = np.random.default_rng(21)
    n, dim = 2_400_000, 32
    z = rng.integers(-30, 31, dim).astype(np.float32)
    z[0] = 31.0
    q = (z / 18.0 + rng.standard_normal(dim) * 0.05).astype(np.float32)
    base = rng.standard_normal((n, dim), dtype=np.float32)
    base[:16] = z + np.float32(2.0 / float(q @ q)) * q
    base[100_000:2_300_000] = z
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    deleted = np.zeros(n, bool); deleted[2_100_000:2_300_000] = True
    for dl, expect in [(None, 1), (deleted, 0)]:
        got, (s, r) = with_stage1(qb, stage1, lambda: search_both_ways(qb, st, [q], 10, 0, dl))
        assert (s, r) == (1, expect)
        assert list(got[0]["idx"]) == list(range(10))
    st.close()


def test_rows_rewritten_after_the_first_search(qb):
    """write_rows after a search rebuilds the block-scaled plane: the next search sees the new rows."""
    rng = np.random.default_rng(5)
    n, dim = 1 << 19, 64
    base = rng.standard_normal((n, dim), dtype=np.float32)
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    q = rng.standard_normal(dim).astype(np.float32)
    search_both_ways(qb, st, [q], 10, 0)
    new = np.tile(q * 5.0, (3, 1)).astype(np.float32)
    st.write_rows(400_000, new)
    got, (s, r) = search_both_ways(qb, st, [q], 10, 0)
    assert (s, r) == (1, 0)
    assert list(got[0]["idx"][:3]) == [400_000, 400_001, 400_002]
    st.close()
