"""The block-scaled 4-bit first stage (f32_to_q4b_rows_kernel, dense_q4b_filter_kernel; qb_prefilter.cu): the row record's layout and the
kernel's dp4a operands restated in numpy, and its upper bound checked row by row against the exact f32 score the oracle computes, on random
and adversarial rows, on the CPU (as tests/test_prefilter_bounds_q5.py does for the 5-bit stage)."""
import numpy as np
import pytest

from tests.test_prefilter_bounds_q5 import operand_bytes
from tests.test_prefilter_bounds_q6 import q6_rows, q8_query

F = np.float32


def d_pad_of(dim):
    return -(-dim // 32) * 32


def q4b_stride(d_pad):
    return -(-((d_pad // 2 + d_pad // 16 + 3) // 4 * 4 + 8) // 8) * 8


def q4b_rows(x):
    """f32_to_q4b_rows_kernel in f32 arithmetic: s_r = max / 7, per 16-dimension chunk k_b = ceil(max_b * (255 / max)) in [1, 255] (0 for an
    all-zero chunk), c = rint(x * (255 / (s_r k_b))) in [-7, 7]; rows below 1e-30 keep codes 0, k_b = 255, s_r = 2 max.  rho4 = ||x - x^||_2
    (f64, rounded up to f32) with x^ = s_r k_b / 255 c."""
    n, dim = x.shape
    d_pad = d_pad_of(dim)
    xp = np.zeros((n, d_pad), F)
    xp[:, :dim] = x
    mx = np.abs(x).max(axis=1).astype(F)
    tiny = ~(mx >= F(1e-30))
    mb = np.abs(xp).reshape(n, d_pad // 16, 16).max(axis=2)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        sr = np.where(tiny, mx * F(2), (mx / F(7)).astype(F)).astype(F)
        kr = np.where(tiny, F(0), (F(255) / mx).astype(F)).astype(F)
        kb = np.where(mb > 0, np.clip(np.ceil((mb * kr[:, None]).astype(F)), 1, 255), 0).astype(np.int64)
        kb[tiny] = 255
        inv = np.where(tiny[:, None] | (kb == 0), F(0), (F(255) / (sr[:, None] * kb.astype(F)).astype(F)).astype(F)).astype(F)
    c = np.clip(np.rint((xp * np.repeat(inv, 16, axis=1)).astype(F)), -7, 7).astype(np.int64)
    kd = np.repeat(kb, 16, axis=1)
    r = (xp.astype(np.float64) * 255 - sr.astype(np.float64)[:, None] * (kd * c)) / 255
    rho = np.nextafter((np.sqrt((r * r).sum(axis=1)) * (1 + 2.0 ** -40)).astype(F), F(np.inf))
    return c, kb, sr, rho


def pack_q4b(c, kb, sr, rho):
    """The row record: codes (byte 8v + 4k + j: c + 8 of dims 16v + 8k + j in the low nibble and + 4 in the high one), k_b per chunk, then
    s_r and rho4 at the next 4-byte boundary, zero padding up to a multiple of 8 bytes."""
    n, d_pad = c.shape
    u = c + 8
    ab = np.arange(d_pad // 2)
    d = (ab >> 3) * 16 + ((ab >> 2) & 1) * 8 + (ab & 3)
    rec = np.zeros((n, q4b_stride(d_pad)), np.uint8)
    rec[:, : d_pad // 2] = u[:, d] | (u[:, d + 4] << 4)
    rec[:, d_pad // 2 : d_pad // 2 + d_pad // 16] = kb
    meta = (d_pad // 2 + d_pad // 16 + 3) // 4 * 4
    rec[:, meta : meta + 8] = np.stack([sr, rho], axis=1).astype("<f4").view(np.uint8)
    return rec


def kernel_operands(rec, d_pad):
    """dense_q4b_filter_kernel's dp4a operands (x & 0x0F0F0F0F, (x >> 4) & 0x0F0F0F0F of a chunk's two words) decoded per dimension, and k_b."""
    w = np.ascontiguousarray(rec[:, : d_pad // 2]).view("<u4").astype(np.int64)
    lo, hi = w[:, 0::2], w[:, 1::2]
    ops = [lo & 0x0F0F0F0F, (lo >> 4) & 0x0F0F0F0F, hi & 0x0F0F0F0F, (hi >> 4) & 0x0F0F0F0F]
    return operand_bytes(ops, rec.shape[0], d_pad), rec[:, d_pad // 2 : d_pad // 2 + d_pad // 16].astype(np.int64)


def q4b_upper_bound(x, q):
    """The kernel's per-row upper bound (f64 here; the kernel rounds every term towards "pass") and the 6-bit plane's slack:
    approx = sum_b s_b s_q (H_b + L_b / 254), + min(t1, t2) + ev."""
    n, dim = x.shape
    d_pad = d_pad_of(dim)
    c, kb, sr, rho = q4b_rows(x)
    _, _, _, mxn = q6_rows(x)
    sq, h, l = q8_query(q)
    qp, hp, lp = (np.zeros(d_pad), np.zeros(d_pad, np.int64), np.zeros(d_pad, np.int64))
    qp[:dim], hp[:dim], lp[:dim] = q, h, l
    nb = d_pad // 16
    Hb = (c.reshape(n, nb, 16) * hp.reshape(nb, 16)).sum(axis=2)
    Lb = (c.reshape(n, nb, 16) * lp.reshape(nb, 16)).sum(axis=2)
    assert np.abs(254 * Hb + Lb).max() < 2 ** 22                   # exact through the kernel's exponent trick
    sb = sr.astype(np.float64)[:, None] * kb / 255.0
    approx = (sb * float(sq) * (Hb + Lb / 254.0)).sum(axis=1)
    n_b = np.clip(dim - 16 * np.arange(nb), 0, 16)
    Eb = np.abs(qp).reshape(nb, 16).sum(axis=1) * (0.5 + 2.0 ** -13) + float(sq) * 0.014 * n_b
    t1 = (sb * Eb).sum(axis=1)
    qn = np.sqrt((q.astype(np.float64) ** 2).sum())
    e2 = float(sq) * np.sqrt(dim) * 0.00202
    rho64 = rho.astype(np.float64)
    t2 = rho64 * (qn + e2) + e2 * mxn
    ev = 2.0 ** -19 * (qn + e2) * (mxn + rho64)
    slack = 2 * (dim * 2.0 ** -22 + 2.0 ** -17) * qn * mxn + 1e-37
    return approx + np.minimum(t1, t2) + ev, slack, c, kb, rho64


@pytest.mark.parametrize("dim", [32, 40, 200, 768, 1000])
def test_row_record_round_trips(dim):
    rng = np.random.default_rng(dim)
    x = rng.standard_normal((9, dim)).astype(F)
    x[0, : min(dim, 16)] = 0.0                                       # an all-zero chunk
    c, kb, sr, rho = q4b_rows(x)
    d_pad = d_pad_of(dim)
    rec = pack_q4b(c, kb, sr, rho)
    assert rec.shape[1] % 8 == 0 and (dim != 768 or rec.shape[1] == 440)
    u, k = kernel_operands(rec, d_pad)
    assert u.max() <= 15 and u.min() >= 1                            # non-negative int8 operands
    np.testing.assert_array_equal(u - 8, c)
    np.testing.assert_array_equal(k, kb)
    assert (c[:, dim:] == 0).all() and kb[0, 0] == 0 and (kb[:, (dim + 15) // 16 :] == 0).all()
    assert (kb.max(axis=1) == 255).all()                             # the chunk holding the row's maximum


def test_u8_scale_rounding_edges():
    """k_b rounds up: a chunk maximum at exactly k / 255 of the row's, or one f32 step above or below it, keeps every code in [-7, 7] with
    |x - s_b c| <= s_b (1/2 + 2^-13)."""
    dim = 64
    rows = []
    for k in (1, 2, 17, 128, 254, 255):
        for step in (-1, 0, 1):
            x = np.zeros(dim, F)
            x[0] = F(7.0)
            x[16:32] = np.nextafter(F(7.0 * k / 255), F(np.inf) if step > 0 else F(-np.inf)) if step else F(7.0 * k / 255)
            x[32:48] = -x[16:32]
            x[48] = F(1e-40)                                          # a denormal alone in its chunk
            rows.append(x)
    x = np.stack(rows)
    c, kb, sr, _ = q4b_rows(x)
    assert (np.abs(c) <= 7).all()
    sb = np.repeat(sr.astype(np.float64)[:, None] * kb / 255.0, 16, axis=1)
    err = np.abs(x.astype(np.float64) - sb * c)
    assert (err <= sb * (0.5 + 2.0 ** -13)).all()
    assert (kb[:, 3] == 1).all()


CASES = ["gauss", "unit", "spiky", "one_high_block", "zero_blocks", "mixed_scale", "denormal", "sparse_query", "residual_along_q", "extreme_scale"]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("dim", [40, 200, 768, 1000])
def test_q4b_stage_upper_bound_covers_the_exact_score(oracle, case, dim):
    rng = np.random.default_rng(dim + 5 * sum(map(ord, case)))
    n = 3000
    x = rng.standard_normal((n, dim)).astype(F)
    q = rng.standard_normal(dim).astype(F)
    if case == "unit":
        x = oracle.preprocess_rows_f32(oracle.COSINE, x); q = oracle.preprocess_f32(oracle.COSINE, q)
    elif case == "spiky":
        x[:, rng.integers(0, dim, 3)] *= F(300.0)
    elif case == "one_high_block":
        x[:, 16:] *= F(1e-3)                                          # the first chunk's maximum far above every other chunk's
    elif case == "zero_blocks":
        x[:, 16 : dim // 2] = 0.0
    elif case == "mixed_scale":
        x *= (10.0 ** rng.uniform(-8, 8, (n, 1))).astype(F)
    elif case == "denormal":
        x[: n // 2] *= F(1e-38); x[n // 2 : n // 2 + 10] = 0; x[n // 2 + 10 : n // 2 + 20] *= F(1e-31)
    elif case == "sparse_query":
        q[rng.random(dim) < 0.9] = 0
    elif case == "residual_along_q":
        # residuals of almost half a step on the side q points to, in every chunk: x = s_b (k +- (1/2 - 1e-4)) with s_b = 1
        q = np.sign(q).astype(F)
        k = rng.integers(-6, 7, (n, dim))
        x = (k + np.where(q > 0, 0.5 - 1e-4, -0.5 + 1e-4)).astype(F)
        x[:, ::16] = F(7) * np.sign(q[::16])                          # pins every chunk's maximum: k_b = 255, s_b = 1
    elif case == "extreme_scale":
        x *= np.where(rng.random((n, 1)) < 0.5, F(1e30), F(1e-29)).astype(F)
        q *= F(1e-6)
    exact = oracle.score_points_f32(oracle.DOT, x, q, np.arange(n, dtype=np.uint32)).astype(np.float64)
    up, slack, c, kb, rho = q4b_upper_bound(x, q)
    worst = (exact - slack - up).max()
    assert worst <= 0, f"{case} dim={dim}: exact exceeds the stage-1 upper bound by {worst}"
    if case == "residual_along_q":
        assert (kb[:, : dim // 16] == 255).all()
        # q . r reaches ||q||_2 rho4 up to the pinned dims, which carry no residual: q . r = sqrt(1 - pinned / dim) ||q||_2 rho4
        pinned = len(range(0, dim, 16))
        assert np.median((up - exact) / (rho * np.sqrt(dim))) < 1 - np.sqrt(1 - pinned / dim) + 0.01


def test_block_scales_pass_fewer_rows_than_one_row_scale(oracle):
    """On unit-norm Gaussian rows at dim 768 with a top-10 threshold of a 1/8 sample, the block-scaled bound passes far fewer rows than the
    same 4-bit codes with one scale per row would (about half of them here, where the sample is small), and every row whose exact score
    reaches the threshold."""
    rng = np.random.default_rng(7)
    x = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((16384, 768)).astype(F))
    q = oracle.preprocess_f32(oracle.COSINE, rng.standard_normal(768).astype(F))
    exact = oracle.score_points_f32(oracle.DOT, x, q, np.arange(len(x), dtype=np.uint32)).astype(np.float64)
    thr = np.sort(exact[:2048])[-10]
    up, slack, _, _, _ = q4b_upper_bound(x, q)
    passed = up >= thr - slack
    assert passed[exact >= thr].all()
    # one scale per row: s_r = max / 7, rho4 of those codes
    sr = np.abs(x).max(axis=1).astype(np.float64) / 7
    r = x - sr[:, None] * np.clip(np.rint(x / sr[:, None]), -7, 7)
    rho_row = np.sqrt((r * r).sum(axis=1))
    up_row = (x - r) @ q.astype(np.float64) + rho_row * np.sqrt((q.astype(np.float64) ** 2).sum())
    assert passed.sum() < 0.6 * (up_row >= thr - slack).sum()
