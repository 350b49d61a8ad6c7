"""Committed golden vectors = outputs of the reference's OWN C kernels (tests/golden/make_golden.py ran them from a
qdrant source tree, which is not part of this repository).  CPU: the oracle's restatement reproduces them.  GPU: the CUDA path
reproduces them through the C ABI."""
import ctypes as C
import os

import numpy as np
import pytest

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "simd_utils_r01.npz"))
u8p = C.POINTER(C.c_uint8)


def test_golden_sq8_inner_loops_vs_oracle(oracle):
    L = oracle.lib()
    for c in range(G["sq8_dim"].size):
        dim = int(G["sq8_dim"][c])
        q, v = np.ascontiguousarray(G["sq8_q"][c]), np.ascontiguousarray(G["sq8_v"][c])
        assert np.float32(L.qo_sq8_dot_avx(q.ctypes.data_as(u8p), v.ctypes.data_as(u8p), dim)) == G["sq8_dot_avx"][c], (c, dim)
        assert np.float32(L.qo_sq8_l1_avx(q.ctypes.data_as(u8p), v.ctypes.data_as(u8p), dim)) == G["sq8_l1_avx"][c], (c, dim)
        if dim <= 1040:  # inside the exactness window every tier is the plain integer sum (SURVEY Appendix A)
            exact = int(np.dot(q[:dim].astype(np.int64), v[:dim].astype(np.int64)))
            assert G["sq8_dot_avx"][c] == np.float32(exact) == G["sq8_dot_sse"][c]
        l1 = int(np.abs(q[:dim].astype(np.int64) - v[:dim].astype(np.int64)).sum())
        assert G["sq8_l1_avx"][c] == np.float32(l1)  # u16 lanes of the AVX2 tier cannot overflow below dim 8256
        # reference quirk, recorded not reproduced: the SSE tier's final HSUM128_EPI16 keeps 16 bits (cpp/sse.c:504-512), so its
        # L1 wraps modulo 65536; the bench host dispatches the AVX2 tier (encoded_vectors_u8.rs:471-490), which is what the path restates
        if dim <= 2000:
            assert G["sq8_l1_sse"][c] == np.float32(l1 % 65536)


def test_golden_sq8_end_to_end_vs_oracle(oracle):
    """EncodedVectorsU8 scoring of a whole segment: restated encode_query + score == reference kernel + postprocess_score."""
    rows = np.ascontiguousarray(G["e2e_rows"])
    base_like = np.zeros((rows.shape[0], 768), np.float32)
    sq = oracle.SQ8.encode(base_like, oracle.QD_DOT, False, alpha=G["e2e_meta"][0], offset=G["e2e_meta"][1])
    assert np.float32(sq.meta.multiplier) == G["e2e_meta"][2]
    sq.rows = rows
    for qi, q in enumerate(G["e2e_queries"]):
        code, off = sq.encode_query(oracle.preprocess_f32(oracle.COSINE, q))
        np.testing.assert_array_equal(code, G["e2e_query_codes"][qi])
        assert off == G["e2e_query_offs"][qi]
        np.testing.assert_array_equal(sq.score_all(code, off), G["e2e_scores"][qi])


def test_golden_bq_popcounts_vs_oracle(oracle):
    dim = int(G["bq_dim"][0])
    data, q = G["bq_data"], G["bq_query_f32"]
    for tag, qenc, bits in (("s8", oracle.BQQ_SCALAR8, 8), ("s4", oracle.BQQ_SCALAR4, 4), ("bin", oracle.BQQ_SAME, 1)):
        bq = oracle.BQ.encode(data, oracle.BQ_ONE, qenc, oracle.QD_DOT, False)
        np.testing.assert_array_equal(np.asarray(bq.rows), G["bq_rows"])
        qe = bq.encode_query(q)
        np.testing.assert_array_equal(np.asarray(qe), G["bq_query_" + tag])
        for i in range(data.shape[0]):
            x = np.float32(G["bq_xor_" + tag][i])
            xf = x / np.float32((1 << bits) - 1) if bits > 1 else x
            assert bq.score(qe, i) == (np.float32(dim) - xf) - xf  # calculate_metric, Dot: zeros - xor (encoded_vectors_binary.rs:766-810)


@pytest.mark.gpu
def test_golden_sq8_end_to_end_on_gpu():
    from qdrant_b200 import scorer as qb

    rows = np.ascontiguousarray(G["e2e_rows"])
    alpha, offset, mult = (float(x) for x in G["e2e_meta"])
    st = qb.ScalarQuantizedVectors(rows, 768, alpha, offset, mult, qb.Distance.Cosine)
    ids = np.arange(rows.shape[0], dtype=np.uint32)
    for qi, q in enumerate(G["e2e_queries"]):
        sc = st.raw_scorer(q)
        np.testing.assert_array_equal(sc.score_points(ids), G["e2e_scores"][qi])
        sc.close()
    got = st.search_batch(G["e2e_queries"], 10)
    for qi in range(3):
        order = np.argsort(-G["e2e_scores"][qi], kind="stable")[:10]
        np.testing.assert_array_equal(got[qi]["score"], G["e2e_scores"][qi][order])
    st.close()


@pytest.mark.gpu
def test_golden_bq_scores_on_gpu():
    from qdrant_b200 import scorer as qb

    dim = int(G["bq_dim"][0])
    rows = np.ascontiguousarray(G["bq_rows"])
    ids = np.arange(rows.shape[0], dtype=np.uint32)
    for tag, qenc, bits in (("s8", qb.BQQueryEncoding.Scalar8bits, 8), ("s4", qb.BQQueryEncoding.Scalar4bits, 4), ("bin", qb.BQQueryEncoding.SameAsStorage, 1)):
        st = qb.BinaryQuantizedVectors(rows, dim, qb.Distance.Dot, qb.BQEncoding.OneBit, qenc, None)
        x = G["bq_xor_" + tag].astype(np.float32)
        xf = x / np.float32((1 << bits) - 1) if bits > 1 else x
        want = (np.float32(dim) - xf) - xf
        sc = st.raw_scorer(G["bq_query_f32"])
        np.testing.assert_array_equal(sc.score_points(ids), want.astype(np.float32))
        sc.close()
        st.close()
