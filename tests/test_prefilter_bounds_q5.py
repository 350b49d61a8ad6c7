"""The 5-bit cascade over the 6-bit shadow plane (f32_to_q6_rows_kernel, dense_q5_filter_kernel, dense_q6_rescreen_kernel; qb_prefilter.cu):
the row record's layout and the kernels' dp4a operands restated in numpy, the stage-1 sums plus the side plane's sums checked against the 6-bit
sums, and the stage-1 upper bound checked row by row against the exact f32 score the oracle computes, on random and adversarial rows, on the CPU
(as tests/test_prefilter_bounds_q6.py does for the 6-bit test that stage 2 applies)."""
import numpy as np
import pytest

from tests.test_prefilter_bounds_q6 import q6_rows, q8_query

F = np.float32
P = (0, 2, 1, 3)           # byte j of a spread u16 holds its nibble P[j]


def pack_q5(c, dim):
    """f32_to_q6_rows_kernel's code bytes for codes c: (main record: a plane then b plane, side plane of low bits e); u = c + 31 = 4a + 2b + e,
    padded dims hold u = 31.  a-plane byte 8v + 4k + j: dims 16v + 8k + j (low nibble) and + 4 (high); u16 v of the b plane and of the side
    plane: bit 4 P[j] + m = dim 16v + 4m + j."""
    n, d_pad = c.shape[0], -(-dim // 32) * 32
    u = np.full((n, d_pad), 31, np.int64)
    u[:, :dim] = c + 31
    a = u >> 2
    ab = np.arange(d_pad // 2)
    d = (ab >> 3) * 16 + ((ab >> 2) & 1) * 8 + (ab & 3)
    a_plane = (a[:, d] | (a[:, d + 4] << 4)).astype(np.uint8)

    def bit_plane(b):
        words = np.zeros((n, d_pad // 16), np.int64)
        for j in range(4):
            for m in range(4):
                words |= b[:, np.arange(d_pad // 16) * 16 + 4 * m + j] << (4 * P[j] + m)
        return np.ascontiguousarray(words.astype("<u2")).view(np.uint8)

    return np.concatenate([a_plane, bit_plane((u >> 1) & 1)], axis=1), bit_plane(u & 1)


def spread(t):
    return (t | (t << 12)) & 0x0F0F0F0F


def operand_bytes(ops, n, d_pad):
    """[n, d_pad]: byte j of operand m of chunk v -> dim 16v + 4m + j"""
    out = np.zeros((n, d_pad), np.int64)
    for m in range(4):
        for j in range(4):
            out[:, np.arange(d_pad // 16) * 16 + 4 * m + j] = (ops[m] >> (8 * j)) & 0xFF
    return out


def stage1_codes(main, d_pad):
    """dense_q5_filter_kernel's dp4a operands (2a + b per byte), decoded to the 5-bit code w of every dimension."""
    n = main.shape[0]
    wa = np.ascontiguousarray(main[:, : d_pad // 2]).view("<u4").astype(np.int64)
    y = spread(np.ascontiguousarray(main[:, d_pad // 2 : d_pad // 2 + d_pad // 8]).view("<u2").astype(np.int64))
    lo, hi = wa[:, 0::2], wa[:, 1::2]
    ops = [((lo << 1) & 0x1E1E1E1E) | (y & 0x01010101), ((lo >> 3) & 0x1E1E1E1E) | ((y >> 1) & 0x01010101),
           ((hi << 1) & 0x1E1E1E1E) | ((y >> 2) & 0x01010101), ((hi >> 3) & 0x1E1E1E1E) | ((y >> 3) & 0x01010101)]
    return operand_bytes(ops, n, d_pad)


def stage2_bits(side, d_pad):
    """dense_q6_rescreen_kernel's dp4a operands, decoded to the low bit e of every dimension."""
    y = spread(np.ascontiguousarray(side).view("<u2").astype(np.int64))
    return operand_bytes([(y >> m) & 0x01010101 for m in range(4)], side.shape[0], d_pad)


def q5_upper_bound(x, q):
    """dense_q5_filter_kernel's per-row upper bound of the exact score and its threshold slack (f64 here; the kernel rounds every term towards
    "pass"): approx = s_r s_q (H5 + L5 / 254) / 2 over the 2 c5 = 4w - 61 of the 5-bit code, + min(t1, t2) with the half-step s_r (1 + 2^-13)
    and rho5 >= ||x - s_r c5||_2."""
    dim = x.shape[1]
    c, sr, _, mxn = q6_rows(x)
    w = (c + 31) >> 1
    c5 = 2 * w + 0.5 - 31
    sr64 = sr.astype(np.float64)
    r5 = x.astype(np.float64) - sr64[:, None] * c5
    rho5 = np.nextafter((np.sqrt((r5 * r5).sum(axis=1)) * (1 + 2.0 ** -40)).astype(F), F(np.inf)).astype(np.float64)
    sq, h, l = q8_query(q)
    H5, L5 = (4 * w - 61) @ h, (4 * w - 61) @ l
    assert np.abs(H5).max() < 2 ** 24 and np.abs(L5).max() < 2 ** 24
    q1, qn = np.abs(q).astype(np.float64).sum(), np.sqrt((q.astype(np.float64) ** 2).sum())
    e1_5 = q1 * (1 + 2.0 ** -13) + float(sq) * dim * 0.066
    e2 = float(sq) * np.sqrt(dim) * 0.00202
    bound = np.minimum(sr64 * e1_5, rho5 * (qn + e2) + e2 * mxn)
    up = sr64 * float(sq) * (H5 + L5 / 254.0) / 2 + bound
    slack = 2 * (dim * 2.0 ** -22 + 2.0 ** -17) * qn * mxn + 1e-37
    return up, slack, c, rho5


@pytest.mark.parametrize("dim", [32, 40, 200, 768, 1000])
def test_row_record_round_trips(dim):
    rng = np.random.default_rng(dim)
    c = rng.integers(-31, 32, (9, dim))
    c[0], c[1] = -31, 31
    main, side = pack_q5(c, dim)
    d_pad = -(-dim // 32) * 32
    assert main.shape[1] == 5 * d_pad // 8 and side.shape[1] == d_pad // 8
    stride = -(-(5 * d_pad // 8 + 12) // 8) * 8                  # + s_r, rho5, rho6; two records are a multiple of 16 bytes
    assert (2 * stride) % 16 == 0 and (dim != 768 or stride == 496)
    w, lb = stage1_codes(main, d_pad), stage2_bits(side, d_pad)
    assert w.max() < 32 and lb.max() <= 1                       # non-negative int8 operands
    np.testing.assert_array_equal(2 * w[:, :dim] + lb[:, :dim] - 31, c)
    assert (w[:, dim:] == 15).all() and (lb[:, dim:] == 1).all()   # padding decodes to c = 0 (and meets a zero query)


@pytest.mark.parametrize("dim", [40, 200, 768, 1000])
def test_stage1_sums_plus_low_bits_give_the_6bit_sums(dim):
    rng = np.random.default_rng(dim + 1)
    c = rng.integers(-31, 32, (64, dim))
    c[0], c[1], c[2] = 31, -31, 30                                # extreme and all-even / all-odd u rows
    main, side = pack_q5(c, dim)
    d_pad = -(-dim // 32) * 32
    w, lb = stage1_codes(main, d_pad), stage2_bits(side, d_pad)
    for q in (rng.standard_normal(dim).astype(F), np.full(dim, -1.0, F)):
        _, h, l = q8_query(q)
        hp, lp = np.zeros(d_pad, np.int64), np.zeros(d_pad, np.int64)
        hp[:dim], lp[:dim] = h, l
        for qq in (hp, lp):
            s_w = w @ qq
            partial = 2 * s_w - 31 * qq.sum()                         # what stage 1 appends
            np.testing.assert_array_equal(partial + lb @ qq, c @ qq[:dim])
            h5 = 4 * s_w - 61 * qq.sum()                              # stage 1's sum over 2 c5
            np.testing.assert_array_equal(h5, (4 * w - 61) @ qq)
            assert np.abs(h5).max() < 2 ** 24 and np.abs(4 * s_w).max() < 2 ** 31


CASES = ["gauss", "unit", "spiky", "mixed_scale", "denormal", "sparse_query", "residual_along_q", "low_bits_zero", "low_bits_one", "extreme_scale"]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("dim", [40, 200, 768, 1000])
def test_q5_stage_upper_bound_covers_the_exact_score(oracle, case, dim):
    rng = np.random.default_rng(dim + 3 * sum(map(ord, case)))
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
        x[: n // 2] *= F(1e-38); x[n // 2 : n // 2 + 10] = 0; x[n // 2 + 10 : n // 2 + 20] *= F(1e-31)
    elif case == "sparse_query":
        q[rng.random(dim) < 0.9] = 0
    elif case == "residual_along_q":
        # the 5-bit residual r5_i = r_i + s_r (e_i - 1/2) at its largest, on the side q points to: codes whose low bit is 1 with x just below
        # code + 1/2 where q > 0, codes whose low bit is 0 with x just above code - 1/2 where q < 0, so that |r5_i| ~ s_r along sign(q)
        q = np.sign(q).astype(F)
        k = rng.integers(-29, 29, (n, dim))
        want_odd_u = q > 0                                         # u = k + 31 odd  <=>  k even
        k += ((k % 2 == 0) != want_odd_u).astype(np.int64)
        x = ((k + np.where(q > 0, 0.5 - 1e-4, -0.5 + 1e-4)) * 1.0).astype(F)
        x[:, 0] = F(31) * np.sign(q[0])                            # pins the max: s_r = 1
    elif case in ("low_bits_zero", "low_bits_one"):
        k = rng.integers(-30, 30, (n, dim))
        k += ((k % 2 == 0) == (case == "low_bits_zero")).astype(np.int64)   # low bit of u = k + 31 is 0 for odd k
        x = (k + rng.uniform(-0.45, 0.45, (n, dim))).astype(F)
        x[:, 0] = F(31)                                            # pins the max (u = 62: low bit 0) so that s_r = 1 and the codes are k
    elif case == "extreme_scale":
        x *= np.where(rng.random((n, 1)) < 0.5, F(1e30), F(1e-29)).astype(F)
        q *= F(1e-6)
    exact = oracle.score_points_f32(oracle.DOT, x, q, np.arange(n, dtype=np.uint32)).astype(np.float64)
    up, slack, c, rho5 = q5_upper_bound(x, q)
    if case in ("low_bits_zero", "low_bits_one"):
        assert (((c[:, 1:] + 31) & 1) == (case == "low_bits_one")).all()
    worst = (exact - slack - up).max()
    assert worst <= 0, f"{case} dim={dim}: exact exceeds the stage-1 upper bound by {worst}"
    if case == "residual_along_q":
        # the bound is nearly met: q . r5 reaches ||q||_2 rho5 (and ||q||_1 max|r5_i|) to within a percent
        assert np.median((up - exact) / (rho5 * np.sqrt(dim))) < 0.01


def test_q5_stage_lets_through_every_row_the_6bit_test_passes(oracle):
    """Both tests bound the same exact score; on unit-norm Gaussian rows at dim 768 with a top-10 threshold of a 1/8 sample, every row that
    the 6-bit test passes also passes the 5-bit one, which passes a few times more rows."""
    from tests.test_prefilter_bounds_q6 import q6_upper_bound

    rng = np.random.default_rng(7)
    x = oracle.preprocess_rows_f32(oracle.COSINE, rng.standard_normal((16384, 768)).astype(F))
    q = oracle.preprocess_f32(oracle.COSINE, rng.standard_normal(768).astype(F))
    exact = oracle.score_points_f32(oracle.DOT, x, q, np.arange(len(x), dtype=np.uint32)).astype(np.float64)
    thr = np.sort(exact[:2048])[-10]
    up5, slack, _, _ = q5_upper_bound(x, q)
    up6, _, _, _ = q6_upper_bound(x, q)
    pass5, pass6 = up5 >= thr - slack, up6 >= thr - slack
    assert pass6.sum() > 0 and not (pass6 & ~pass5).any()
    assert pass5.sum() > pass6.sum()
