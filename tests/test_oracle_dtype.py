"""CPU pins for the oracle's Float16 / Uint8 helpers: the two query conversions against literal expected values, and the
whole-storage scans against the per-row similarity loop they restate."""
import numpy as np
import pytest

from tests.util import pack_bitmap


def f32(bits):
    return np.array([bits], np.uint32).view(np.float32)[0]


# (f32 input, f16 bits): round to nearest even, overflow to inf, subnormals and signed zeros kept
F16_CASES = [
    (1.0, 0x3C00),
    (-2.0, 0xC000),
    (0.1, 0x2E66),
    (65504.0, 0x7BFF),                   # the largest finite f16
    (65519.0, 0x7BFF),                   # below the midpoint to 65536: rounds down
    (65520.0, 0x7C00),                   # the midpoint: ties to the even neighbour, which is 2^16 = inf
    (-65520.0, 0xFC00),
    (1e6, 0x7C00),
    (np.inf, 0x7C00),
    (-np.inf, 0xFC00),
    (2.0 ** -14, 0x0400),                # the smallest normal
    (2.0 ** -14 - 2.0 ** -25, 0x0400),   # rounds up into the normal range
    (2.0 ** -24, 0x0001),                # the smallest subnormal
    (1.5 * 2.0 ** -24, 0x0002),          # tie: to the even 2
    (2.5 * 2.0 ** -24, 0x0002),          # tie: to the even 2
    (2.0 ** -25, 0x0000),                # tie between 0 and 2^-24: to the even 0
    (f32(0x33000001), 0x0001),           # just above that tie
    (2.0 ** -26, 0x0000),
    (-(2.0 ** -26), 0x8000),
    (0.0, 0x0000),
    (-0.0, 0x8000),
    (1.0 + 2.0 ** -11, 0x3C00),          # tie: to the even mantissa
    (1.0 + 3 * 2.0 ** -11, 0x3C02),      # tie: to the even mantissa (up)
    (1.0 + 2.0 ** -11 + 2.0 ** -20, 0x3C01),
]

# (f32 input, u8): `x as u8`
U8_CASES = [(np.nan, 0), (-np.nan, 0), (np.inf, 255), (-np.inf, 0), (-0.0, 0), (0.0, 0), (-3.7, 0), (-0.5, 0), (0.99, 0), (3.7, 3),
            (254.99, 254), (255.0, 255), (255.5, 255), (256.0, 255), (1e30, 255), (-1e30, 0)]


def test_to_f16_query_literals(oracle):
    x = np.array([c[0] for c in F16_CASES], np.float32)
    want = np.array([c[1] for c in F16_CASES], np.uint16)
    got = oracle.to_f16_query(oracle.DOT, x).view(np.uint16)
    for xi, g, w in zip(x, got, want):
        assert g == w, f"f16({xi!r}) = {g:#06x}, expected {w:#06x}"
    # NaN stays NaN, whatever its sign
    nan = oracle.to_f16_query(oracle.EUCLID, np.array([np.nan, -np.nan, f32(0x7F800001)], np.float32))
    assert np.isnan(nan).all()


def test_to_f16_query_preprocesses_in_f32_first(oracle):
    """Cosine normalises the f32 query before the conversion: a query whose values overflow f16 stays finite."""
    q = np.array([65504.0, 65519.0, 65520.0, 1e6, 2.0 ** -24, 2.0 ** -26, -3.0, 0.5], np.float32)
    dot = oracle.to_f16_query(oracle.DOT, q)
    assert dot.view(np.uint16)[:4].tolist() == [0x7BFF, 0x7BFF, 0x7C00, 0x7C00]
    cos = oracle.to_f16_query(oracle.COSINE, q)
    assert np.isfinite(cos).all()
    np.testing.assert_array_equal(cos.view(np.uint16), oracle.to_f16_query(oracle.DOT, oracle.preprocess_f32(oracle.COSINE, q)).view(np.uint16))


def test_to_f16_query_matches_an_independent_conversion(oracle):
    """Every f32 exponent that can reach f16, random mantissas: the restatement equals numpy's IEEE conversion."""
    rng = np.random.default_rng(0)
    exps = np.repeat(np.arange(95, 145, dtype=np.uint32), 2000)
    bits = (exps << 23) | rng.integers(0, 1 << 23, exps.size, dtype=np.uint32) | (rng.integers(0, 2, exps.size, dtype=np.uint32) << 31)
    x = bits.view(np.float32)
    with np.errstate(over="ignore"):
        want = x.astype(np.float16).view(np.uint16)
    np.testing.assert_array_equal(oracle.to_f16_query(oracle.DOT, x).view(np.uint16), want)


def test_to_u8_query_literals(oracle):
    x = np.array([c[0] for c in U8_CASES], np.float32)
    got = oracle.to_u8_query(x)
    for xi, g, (_, w) in zip(x, got, U8_CASES):
        assert g == w, f"u8({xi!r}) = {g}, expected {w}"


@pytest.mark.parametrize("dim", [1, 8, 15, 16, 17, 31, 32, 33, 100])
@pytest.mark.parametrize("dist", ["COSINE", "DOT", "EUCLID", "MANHATTAN"])
def test_scans_equal_the_per_row_loop(oracle, dist, dim):
    d = getattr(oracle, dist)
    rng = np.random.default_rng(dim)
    n = 300
    deleted = rng.random(n) < 0.3
    bm = pack_bitmap(deleted)
    live = np.flatnonzero(~deleted)
    ids = rng.choice(n, 50).astype(np.uint32)

    def check(rows, queries, score_rows, scan, sim):
        for q in queries:
            want = np.array([sim(d, q, rows[i]) for i in range(n)], np.float32)
            np.testing.assert_array_equal(score_rows(d, rows, q).view(np.uint32), want.view(np.uint32))
            np.testing.assert_array_equal(score_rows(d, rows, q, ids).view(np.uint32), want[ids].view(np.uint32))
        for top in (1, 10, n + 5):
            for got, q in zip(scan(d, rows, queries, top), queries):
                want = np.array([sim(d, q, rows[i]) for i in range(n)], np.float32)
                np.testing.assert_array_equal(got, oracle.topk(want, top))
            for got, q in zip(scan(d, rows, queries, top, deleted=bm), queries):
                want = np.array([sim(d, q, rows[i]) for i in live], np.float32)
                np.testing.assert_array_equal(got, oracle.topk(want, top, live))

    rows8 = rng.integers(0, 256, (n, dim), dtype=np.uint8)
    q8 = np.stack([oracle.to_u8_query(rng.uniform(-10, 300, dim).astype(np.float32)) for _ in range(3)])
    check(rows8, q8, oracle.score_rows_u8, oracle.scan_u8, oracle.similarity_u8)
    rows16 = rng.standard_normal((n, dim)).astype(np.float16)
    q16 = np.stack([oracle.to_f16_query(d, rng.standard_normal(dim).astype(np.float32)) for _ in range(3)])
    check(rows16, q16, oracle.score_rows_f16, oracle.scan_f16, oracle.similarity_f16)
