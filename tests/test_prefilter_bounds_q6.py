"""The 6-bit shadow plane of the single-query prefilter (f32_to_q6_rows_kernel / dense_q6_filter_kernel, qb_prefilter.cu): the kernels'
arithmetic restated in numpy — same quantisation steps, same constants — and the upper bound checked row by row against the exact f32 score
the oracle computes, on random and adversarial rows, on the CPU (as tests/test_prefilter_bounds.py does for the int8 and bf16 planes)."""
import numpy as np
import pytest

F = np.float32


def q6_rows(x):
    """f32_to_q6_rows_kernel: c = rint(x * (31 / max)) in [-31, 31], s_r = max / 31, rho_r = ||x - s_r c||_2 (f64) rounded up to f32;
    rows below 1e-30 keep all-zero codes, s_r = 2 max and rho_r = ||x||.  Also returns the plane's max row norm (f64, rounded up)."""
    mx = np.abs(x).max(axis=1).astype(F)
    tiny = ~(mx >= F(1e-30))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        sr = np.where(tiny, mx * F(2), (mx / F(31)).astype(F)).astype(F)
        inv = np.where(tiny, F(0), (F(31) / mx).astype(F)).astype(F)
    c = np.clip(np.rint((x * inv[:, None]).astype(F)), -31, 31).astype(np.int64)
    r = x.astype(np.float64) - sr.astype(np.float64)[:, None] * c
    up = lambda v: np.nextafter(v.astype(F), F(np.inf))       # f64 -> f32 rounded up (the kernel: __double2float_ru)
    rho = up(np.sqrt((r * r).sum(axis=1)) * (1 + 2.0 ** -40))
    mxn = up(np.sqrt((x.astype(np.float64) ** 2).sum(axis=1)).max() * (1 + 2.0 ** -40))
    return c, sr, rho, float(mxn)


def pack_q6(c, dim):
    """The row record's code bytes: u = c + 31 = 4 a + b; a-plane byte 8v + 4w + j holds dims 16v + 8w + j (low nibble) and + 4 (high);
    b-plane byte 4v + j holds dim 16v + 4k + j in bits [2k, 2k + 2)."""
    d_pad = -(-dim // 32) * 32
    u = np.full((c.shape[0], d_pad), 31, np.int64)
    u[:, :dim] = c + 31
    a, b = u >> 2, u & 3
    ab = np.arange(d_pad // 2)
    d = (ab >> 3) * 16 + ((ab >> 2) & 1) * 8 + (ab & 3)
    a_plane = a[:, d] | (a[:, d + 4] << 4)
    bb = np.arange(d_pad // 4)
    d = (bb >> 2) * 16 + (bb & 3)
    b_plane = sum(b[:, d + 4 * k] << (2 * k) for k in range(4))
    return np.concatenate([a_plane, b_plane], axis=1).astype(np.uint8)


def unpack_q6(codes, dim):
    """dense_q6_filter_kernel's view of a row: the dp4a operands of chunk v, m = 0..3, against query bytes of dims 16v + 4m + j."""
    d_pad = codes.shape[1] // 3 * 4
    a_plane, b_plane = codes[:, : d_pad // 2].astype(np.int64), codes[:, d_pad // 2 :].astype(np.int64)
    u = np.zeros((codes.shape[0], d_pad), np.int64)
    for v in range(d_pad // 16):
        w0, w1 = a_plane[:, 8 * v : 8 * v + 4], a_plane[:, 8 * v + 4 : 8 * v + 8]
        a = [w0 & 15, w0 >> 4, w1 & 15, w1 >> 4]
        wb = b_plane[:, 4 * v : 4 * v + 4]
        for m in range(4):
            u[:, 16 * v + 4 * m : 16 * v + 4 * m + 4] = 4 * a[m] + ((wb >> (2 * m)) & 3)
    return u[:, :dim] - 31


def q8_query(q):
    """The two int8 levels of the query, q ~ s_q (h + l / 254) (shared with the int8 plane's kernel)."""
    qmax = F(np.abs(q).max())
    sq = (qmax / F(127)).astype(F) if qmax > 0 else F(0)
    inv = (F(127) / qmax).astype(F) if qmax > 0 else F(0)
    y = (q * inv).astype(F)
    h = np.clip(np.rint(y), -127, 127).astype(F)
    l = np.clip(np.rint(((y - h).astype(F) * F(254)).astype(F)), -127, 127)
    return sq, h.astype(np.int64), l.astype(np.int64)


def q6_upper_bound(x, q):
    """The kernel's per-row upper bound of the exact score and its threshold slack (f64 here; the kernel rounds every term towards "pass")."""
    dim = x.shape[1]
    c, sr, rho, mxn = q6_rows(x)
    sq, h, l = q8_query(q)
    H, L = c @ h, c @ l
    q1, qn = np.abs(q).astype(np.float64).sum(), np.sqrt((q.astype(np.float64) ** 2).sum())
    e1 = q1 * (0.5 + 2.0 ** -13) + float(sq) * dim * 0.066
    e2 = float(sq) * np.sqrt(dim) * 0.00202
    sr64, rho64 = sr.astype(np.float64), rho.astype(np.float64)
    bound = np.minimum(sr64 * e1, rho64 * (qn + e2) + e2 * mxn)
    up = sr64 * float(sq) * (H + L / 254.0) + bound
    slack = 2 * (dim * 2.0 ** -22 + 2.0 ** -17) * qn * mxn + 1e-37
    return up, slack, c, rho


def test_row_record_round_trips():
    rng = np.random.default_rng(1)
    for dim in (32, 40, 200, 768, 1000):
        c = rng.integers(-31, 32, (7, dim))
        codes = pack_q6(c, dim)
        assert codes.shape[1] == -(-dim // 32) * 24
        np.testing.assert_array_equal(unpack_q6(codes, dim), c)


@pytest.mark.parametrize("case", ["gauss", "unit", "spiky", "mixed_scale", "denormal", "sparse_query", "flat", "residual_along_q", "extreme_scale"])
@pytest.mark.parametrize("dim", [64, 200, 768, 1000])
def test_q6_plane_upper_bound_covers_the_exact_score(oracle, case, dim):
    rng = np.random.default_rng(dim + sum(map(ord, case)))
    n = 3000
    x = rng.standard_normal((n, dim)).astype(F)
    q = rng.standard_normal(dim).astype(F)
    if case == "unit":
        x = oracle.preprocess_rows_f32(oracle.COSINE, x); q = oracle.preprocess_f32(oracle.COSINE, q)
    elif case == "spiky":
        x[:, rng.integers(0, dim, 3)] *= F(300.0)
    elif case == "mixed_scale":
        x *= (10.0 ** rng.uniform(-8, 8, (n, 1))).astype(F)
    elif case == "denormal":
        x[: n // 2] *= F(1e-38); x[n // 2 : n // 2 + 10] = 0
    elif case == "sparse_query":
        q[rng.random(dim) < 0.9] = 0
    elif case == "flat":
        x = np.sign(x).astype(F) * F(0.37); q = np.sign(q).astype(F)
    elif case == "residual_along_q":
        # every coordinate sits just below a rounding boundary (code + 0.5 - tiny) on the side q points to: the residual is parallel to
        # sign(q) with |r_i| ~ s_r / 2, so |q . r| meets ||q||_1 max|r_i| and the L2 term is near its worst case for flat q
        q = np.sign(q).astype(F) * F(1.0)
        s = F(31.0) / F(31)                                    # max |x| = 31 s  ->  s_r = s
        k = rng.integers(-30, 30, (n, dim)).astype(np.float64)
        x = ((k + 0.5 - 1e-4 * np.sign(q)) * s).astype(F)
        x[:, 0] = F(31) * s * np.sign(q[0])                    # pins the max
    elif case == "extreme_scale":
        x *= np.where(rng.random((n, 1)) < 0.5, F(1e30), F(1e-29)).astype(F)
        q *= F(1e-6)
    exact = oracle.score_points_f32(oracle.DOT, x, q, np.arange(n, dtype=np.uint32)).astype(np.float64)
    up, slack, c, rho = q6_upper_bound(x, q)
    assert np.abs(c).max() <= 31
    worst = (exact - slack - up).max()
    assert worst <= 0, f"{case} dim={dim}: exact exceeds the kernel's upper bound by {worst}"
    if case == "residual_along_q":
        # the bound is nearly met: q . r reaches ||q||_2 rho_r (and ||q||_1 max|r_i|) to within a percent
        assert np.median((up - exact) / (rho.astype(np.float64) * np.sqrt(dim))) < 0.01
    if case in ("gauss", "unit"):
        assert np.median(up - exact) < 1.5 * exact.std()


def test_q6_plane_is_tighter_than_the_l1_bound_alone(oracle):
    """On unit-norm Gaussian rows the Cauchy-Schwarz term ||q|| rho_r decides: about 0.9 sigma of the score spread at dim 768."""
    rng = np.random.default_rng(5)
    x = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((2000, 768)).astype(F))
    q = oracle.preprocess_f32(oracle.COSINE, rng.standard_normal(768).astype(F))
    exact = oracle.score_points_f32(oracle.DOT, x, q, np.arange(2000, dtype=np.uint32)).astype(np.float64)
    up, _, c, rho = q6_upper_bound(x, q)
    _, sr, _, _ = q6_rows(x)
    l1 = sr.astype(np.float64) * np.abs(q).astype(np.float64).sum() * 0.5
    l2 = rho.astype(np.float64) * np.sqrt((q.astype(np.float64) ** 2).sum())
    assert (l2 < l1).all()
    assert np.median(l2) < 1.0 * exact.std()
