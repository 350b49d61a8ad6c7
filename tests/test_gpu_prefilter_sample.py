"""The threshold sample of the 6-bit plane (qb_prefilter.cu): the first stage ranks the rows of a prefix (n / 8 rows) by their approximate
score, re-scores each CTA's best `top` exactly, and the k-th best of those exact scores is the threshold.  Whatever rows the approximation
picks, results must equal the exact f32 scan bit for bit."""
import numpy as np
import pytest

from tests.test_gpu_prefilter_planes import search_both_ways

pytestmark = pytest.mark.gpu

N = (1 << 19) + 1               # just above the prefilter's minimum; the sample prefix is n / 8 = 65 536 rows (rounded up to a tile)


@pytest.fixture(scope="module")
def qb():
    from qdrant_b200 import scorer

    return scorer


def set_id_base(st, base):
    from qdrant_b200._capi import check, lib

    check(lib().qb_storage_set_id_base(st._h, base))


@pytest.mark.parametrize("dim,top", [(40, 1), (96, 10), (768, 16), (1000, 10)])
def test_best_rows_inside_or_after_the_prefix(qb, dim, top):
    """Best matches only after the prefix, only inside it, and a plain query; per-call deletions and id_base != 0."""
    rng = np.random.default_rng(dim * 3 + top)
    base = rng.standard_normal((N, dim), dtype=np.float32)
    best = [N - 7, N // 8 - 40, 3]
    queries = [base[r].copy() for r in best] + [rng.standard_normal(dim).astype(np.float32)]
    base[best] *= 3.0
    deleted = rng.random(N) < 0.02
    deleted[best] = False
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    set_id_base(st, 1000)
    got, (searches, reruns) = search_both_ways(qb, st, queries, top, 0, deleted)
    assert (searches, reruns) == (4, 0)
    assert [int(g["idx"][0]) for g in got[:3]] == [r + 1000 for r in best]
    st.close()


def test_ties_at_the_kth_score_straddle_the_prefix_boundary(qb):
    """Twelve identical best rows on both sides of row n / 8: the top 10 are the ten with the lowest ids."""
    rng = np.random.default_rng(5)
    dim = 96
    base = rng.standard_normal((N, dim), dtype=np.float32)
    v = base[7].copy()
    pos = [N // 8 - 4200 + 700 * k for k in range(12)]
    base[pos] = v * 3.0
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    got, (searches, reruns) = search_both_ways(qb, st, [v], 10, 0)
    assert (searches, reruns) == (1, 0)
    assert list(got[0]["idx"]) == pos[:10]
    st.close()


@pytest.mark.parametrize("top", [10, 16])
def test_prefix_with_top_live_rows_decides_and_one_less_falls_back(qb, top):
    """Every row of the first third deleted but `top` strong ones: the sample holds exactly `top` live rows and decides.  With one more
    deleted it cannot give a threshold, and the search falls back on the device."""
    rng = np.random.default_rng(top)
    dim = 96
    base = rng.standard_normal((N, dim), dtype=np.float32)
    q = rng.standard_normal(dim).astype(np.float32)
    keep = [100 + 3000 * i for i in range(top)]              # inside the prefix
    base[keep] = q[None, :] * (3.0 + 0.01 * np.arange(top, dtype=np.float32))[:, None]
    deleted = np.zeros(N, bool)
    deleted[: N // 3] = True
    deleted[keep] = False
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    got, stats = search_both_ways(qb, st, [q], top, 0, deleted)
    assert stats == (1, 0)
    assert sorted(got[0]["idx"]) == keep
    deleted[keep[0]] = True
    _, stats = search_both_ways(qb, st, [q], top, 0, deleted)
    assert stats == (1, 1)
    st.close()


def test_per_call_deletions_inside_the_prefix(qb):
    """The prefix's best rows by far are deleted per call: the sample must skip them, or its threshold would be above every live row."""
    rng = np.random.default_rng(17)
    dim = 96
    base = rng.standard_normal((N, dim), dtype=np.float32)
    q = rng.standard_normal(dim).astype(np.float32)
    strong = np.arange(200, 60_000, 2_000)
    base[strong] = q * 4.0
    deleted = np.zeros(N, bool)
    deleted[strong] = True
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    got, stats = search_both_ways(qb, st, [q], 10, 0, deleted)
    assert stats == (1, 0)
    assert not set(got[0]["idx"]) & set(strong.tolist())
    st.close()


def test_approximate_ranking_that_overstates_scores(qb):
    """Rows whose 6-bit codes are exact but whose 5-bit reconstruction is off by +1/2 in the direction of the query: their approximate score
    is about one sigma above the exact one, so every warp's sample list fills with them.  Their exact scores (about 3 sigma) then make the
    threshold, which is lower than the prefix's true top-k but still lets few enough rows through."""
    rng = np.random.default_rng(23)
    dim = 96
    base = rng.standard_normal((N, dim), dtype=np.float32)
    q = rng.standard_normal(dim).astype(np.float32)
    # z: odd (low code bit 0, 5-bit code rounds up) where q > 0, even (rounds down) where q < 0; one entry of 31 sets the row's scale
    z = np.where(q > 0, 1.0, 0.0).astype(np.float32)
    j = int(np.argmax(q))
    z[j] = 31.0
    alpha = np.float32(3.0 * np.linalg.norm(q) / float(q @ z))
    adv = np.arange(0, N // 8, 17)
    base[adv] = z * alpha
    st = qb.DenseVectorStorage(base, qb.Distance.Dot)
    got, stats = search_both_ways(qb, st, [q], 10, 0)
    assert stats == (1, 0)
    assert not set(got[0]["idx"]) & set(adv.tolist())
    st.close()
