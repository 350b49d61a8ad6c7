"""The 6-bit plane's two stages (qb_prefilter.cu): the 5-bit first stage appends to its own list, the second stage completes the 6-bit test
from the side plane.  An overflowing first-stage list must fall back to the exact scan on the device, like an overflowing candidate list."""
import numpy as np
import pytest

from tests.test_gpu_prefilter_planes import search_both_ways

pytestmark = pytest.mark.gpu

N, DIM = 600_000, 96            # candidate list: n / 32 = 18 750 rows; the first-stage list holds every row up to 2^21


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def test_first_stage_overflow_falls_back_on_the_device(qb):
    """2 200 000 copies of an integer-valued row z (its 6-bit codes are exact, its 5-bit codes are off by 1/2 everywhere) score just below the
    sample threshold: the 5-bit bound lets them all through, the 6-bit bound none.  They overflow the first-stage list (2^21 rows), and the
    search falls back; with 200 000 of them deleted the list holds the rest, the second stage drops them, and no fallback is needed."""
    rng = np.random.default_rng(21)
    n, dim = 2_400_000, 32
    z = rng.integers(-30, 31, dim).astype(np.float32)
    z[0] = 31.0                                                   # max |z| = 31: scale 1, codes = z
    q = (z / 18.0 + rng.standard_normal(dim) * 0.05).astype(np.float32)
    base = rng.standard_normal((n, dim), dtype=np.float32)
    base[:16] = z + np.float32(2.0 / float(q @ q)) * q           # the sample's best rows: q . z + 2 (the 5-bit bound of z is ~17, its 6-bit one < 0.1)
    base[100_000:2_300_000] = z
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    deleted = np.zeros(n, bool); deleted[2_100_000:2_300_000] = True
    for dl, expect in [(None, 1), (deleted, 0)]:
        got, (s, r) = search_both_ways(qb, st, [q], 10, 0, dl)
        assert (s, r) == (1, expect)
        assert list(got[0]["idx"]) == list(range(10))
    st.close()


def test_undecidable_queries_fall_back_on_the_device(qb):
    """Mass ties beyond n / 32 candidates (that fit in the first stage), a NaN query, a sample without `top` live rows: the exact scan answers."""
    rng = np.random.default_rng(9)
    base = rng.standard_normal((N, DIM), dtype=np.float32)
    base[100_000:140_000] = base[99_999]
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    q_nan = rng.standard_normal(DIM).astype(np.float32); q_nan[5] = np.nan
    q_plain = rng.standard_normal(DIM).astype(np.float32)
    del_prefix = np.zeros(N, bool); del_prefix[:200_000] = True; del_prefix[:4] = False
    for q, dl, expect in [(base[99_999] * 4.0, None, 1), (q_nan, None, 1), (q_plain, del_prefix, 1), (q_plain, None, 0)]:
        _, (s, r) = search_both_ways(qb, st, [q], 10, 0, dl)
        assert (s, r) == (1, expect)
    st.close()
