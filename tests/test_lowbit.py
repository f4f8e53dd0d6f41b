"""Low-bit weight GEMM (ternary I2X4 and binary I1X8 x I8 / U8 -> I32, MXFP4X2 x I8 -> F32 / BF16), the parts that need no GPU:

  * the restatement oracle/oracle_lowbit.c equals the reference's libxsmm_reference_gemm bit for bit for the six tuples, all four
    batch-reduce modes and beta 0 / 1, with ld > dim and m, n not multiples of 32; A covers every byte value (every 2-bit code, bit
    pattern and nibble table entry), B the int8 extremes, the E8M0 scales include 0 and 254; NaN positions are excluded;
  * the committed fixture tests/golden/lowbit.npz is what the oracle computes, and what the reference computes where it exists;
  * dispatch: every accepted form gives a handle on the CUDA-core backend, every declined clause gives NULL, and the declines pinned
    by other tests still hold;
  * the batch entry points' refusals, without a device."""
import os
import zlib

import numpy as np
import pytest

import libxsmm_b200 as X
from lowbit_ffi import (BETA_0, BF16, F32, I1, I2, I8, I32, INTLV_A, MXFP4, TRANS_A, TRANS_B, TUPLES, U8, VNNI_A, VNNI_B, VNNI_C, LbCase,
                        case_from_meta, meta, oracle_gemm_lowbit, ref_gemm_lowbit, same_c)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lowbit.npz")
need_ref = pytest.mark.skipif(ref_gemm_lowbit is None, reason="the reference build (oracle/_ref/libxsmm_ref_lowbit.so) is not present")


def parity_cases():
    out = []
    for ta, tb, tc in TUPLES:
        for br_type in (0, 1, 2, 3):
            for beta0 in (True, False):
                m = {I2: 44, I1: 46, MXFP4: 45}[ta]
                k = 96 if ta == MXFP4 else 52
                out.append(LbCase(ta, tb, tc, m, 37, k, lda=m + 6, ldb=k + 8, ldc=m + 3, beta0=beta0, br_type=br_type, br=3))
    return out


@need_ref
@pytest.mark.parametrize("case", parity_cases(), ids=repr)
def test_oracle_equals_reference_bit_for_bit(case):
    A, B, C0, SA, SB = case.operands(np.random.default_rng(zlib.crc32(repr(case).encode())))
    rc_r, want = case.run(ref_gemm_lowbit, A, B, C0, SA, SB)
    rc_o, got = case.run(oracle_gemm_lowbit, A, B, C0, SA, SB)
    assert rc_r == 0 and rc_o == 0
    assert same_c(case, want, got), case
    assert not np.array_equal(want.view(np.uint8), C0.view(np.uint8))


def test_inputs_cover_every_byte_extreme_and_scale():
    case = LbCase(MXFP4, I8, F32, 45, 37, 96, lda=51, ldb=104, ldc=48, br_type=3, br=3)
    A, B, C0, SA, SB = case.operands(np.random.default_rng(1))
    assert set(np.unique(A)) == set(range(256))
    assert B.view(np.int8).min() == -128 and B.view(np.int8).max() == 127
    assert 0 in SA and 254 in SA and 0.0 in SB
    case = LbCase(I2, U8, I32, 44, 37, 52, lda=50, ldb=60, ldc=47)
    _, B, C0, _, _ = case.operands(np.random.default_rng(2))
    assert B.min() == 0 and B.max() == 255 and C0.min() == -2 ** 31 and C0.max() == 2 ** 31 - 1


def test_ternary_and_binary_decoding():
    """the 2-bit codes 0, 1, 2, 3 mean 0, +1, -1, -1 in bit pairs of rows i, i + m/4, i + m/2, i + 3m/4; a clear bit is +1"""
    case = LbCase(I2, I8, I32, 4, 1, 4, lda=4, ldb=4, ldc=4)
    A = np.array([0b11100100, 0, 0, 0], np.uint8)             # k = 0: rows 0..3 hold codes 0, 1, 2, 3
    B = np.array([5, 0, 0, 0], np.uint8)
    _, c = case.run(oracle_gemm_lowbit, A, B, np.zeros(4, np.int32), np.zeros(1, np.uint8), np.zeros(1, np.float32))
    assert list(c) == [0, 5, -5, -5]
    if ref_gemm_lowbit is not None:
        assert list(case.run(ref_gemm_lowbit, A, B, np.zeros(4, np.int32), np.zeros(1, np.uint8), np.zeros(1, np.float32))[1]) == [0, 5, -5, -5]
    case = LbCase(I1, I8, I32, 2, 1, 4, lda=2, ldb=4, ldc=2)
    A = np.array([0b10100001], np.uint8)                      # row 0: k0 set; row 1: k1, k3 set
    B = np.array([1, 2, 4, 8], np.uint8)
    _, c = case.run(oracle_gemm_lowbit, A, B, np.zeros(2, np.int32), np.zeros(1, np.uint8), np.zeros(1, np.float32))
    assert list(c) == [-1 + 2 + 4 + 8, 1 - 2 + 4 - 8]


def golden_cases():
    g = np.load(GOLDEN)
    return [(case_from_meta(g["meta%d" % t]), [g["%s%d" % (nm, t)] for nm in ("a", "b", "c0", "sa", "sb")], g["c%d" % t])
            for t in range(int(g["ncases"]))]


def test_golden_fixture_is_what_the_oracle_computes():
    cases = golden_cases()
    assert len(cases) >= 12
    assert {(c.ta, c.tb, c.tc) for c, _, _ in cases} == set(TUPLES)
    for ta in (I2, I1, MXFP4):
        assert {c.br_type for c, _, _ in cases if c.ta == ta} == {0, 1, 2, 3}
    for case, ops, want in cases:
        rc, c = case.run(oracle_gemm_lowbit, *ops)
        assert rc == 0 and same_c(case, want, c), case


@need_ref
def test_golden_fixture_reproduces_from_the_reference():
    import sys
    sys.path.insert(0, os.path.dirname(GOLDEN))
    import make_golden_lowbit
    g = np.load(GOLDEN)
    assert int(g["ncases"]) == len(make_golden_lowbit.CASES)
    for t, case in enumerate(make_golden_lowbit.CASES):
        ops = case.operands(np.random.default_rng(7170 + t))
        for nm, x in zip(("a", "b", "c0", "sa", "sb"), ops):
            assert np.array_equal(g["%s%d" % (nm, t)], x), (t, nm)
        assert np.array_equal(g["meta%d" % t], meta(case))
        rc, c = case.run(ref_gemm_lowbit, *ops)
        assert rc == 0 and np.array_equal(g["c%d" % t].view(np.uint8), c.view(np.uint8)), case   # NaN bits included


# ---- dispatch (no device needed) -------------------------------------------------------------------------------------------
def _dispatch(ta, tb, tc, m=16, n=8, k=32, lda=16, ldb=32, ldc=16, flags=None, br=None, sa=0, sb=0, comp=I32):
    sh = X.libxsmm_create_gemm_shape(m, n, k, lda, ldb, ldc, ta, tb, tc, comp)
    flags = (VNNI_A if ta == I1 else VNNI_A | INTLV_A) if flags is None else flags
    if br is None:
        return X.libxsmm_dispatch_gemm(sh, flags, 0)
    return X.libxsmm_dispatch_brgemm(sh, flags, 0, X.libxsmm_create_gemm_batch_reduce_config(br, sa, sb, 0))


def test_dispatch_accepts_the_defined_forms_on_the_cuda_core_backend():
    for ta, tb, tc in TUPLES:
        base = VNNI_A if ta == I1 else VNNI_A | INTLV_A
        for beta in (0, BETA_0):
            for br in (None, X.GEMM_BATCH_REDUCE_NONE, X.GEMM_BATCH_REDUCE_ADDRESS, X.GEMM_BATCH_REDUCE_OFFSET, X.GEMM_BATCH_REDUCE_STRIDE):
                h = _dispatch(ta, tb, tc, flags=base | beta, br=br, sa=512, sb=1024)
                assert h and X.libxsmm_b200_kernel_backend(h) == X.BACKEND_SIMT, (ta, tb, tc, beta, br)
    assert _dispatch(I2, I8, I32, m=12, lda=20, k=8, ldb=9, ldc=13)          # ld > dim
    assert _dispatch(I1, U8, I32, m=6, lda=10, k=4, ldb=4, ldc=6)
    assert _dispatch(MXFP4, I8, BF16, m=7, lda=9, k=64, ldb=70, ldc=8)


def test_dispatch_declines_every_undefined_form():
    for ta, tb, tc in TUPLES:
        base = VNNI_A if ta == I1 else VNNI_A | INTLV_A
        assert _dispatch(ta, tb, tc, flags=base)                              # the control
        for extra, kw in ((TRANS_A, {}), (TRANS_B, {}), (VNNI_B, {}), (VNNI_C, {}), (524288, {})):   # 524288: bitmap-compressed A
            assert not _dispatch(ta, tb, tc, flags=base | extra, **kw), (ta, tb, tc, extra)
        assert not _dispatch(ta, tb, tc, flags=base, lda=15)                 # lda >= m
        assert not _dispatch(ta, tb, tc, flags=base, ldb=31)                 # ldb >= k
        assert not _dispatch(ta, tb, tc, flags=0)                            # the packed layouts need VNNI_A
        # no fused form
        sh = X.libxsmm_create_gemm_shape(16, 8, 32, 16, 32, 16, ta, tb, tc, I32)
        assert not X.libxsmm_dispatch_brgemm_ext(sh, base, 0, X.libxsmm_create_gemm_batch_reduce_config(0, 0, 0, 0),
                                                 X.libxsmm_create_gemm_ext_unary_argops(0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
                                                 X.libxsmm_create_gemm_ext_binary_postops(0, 0, 0, 0))
    assert not _dispatch(I2, I8, I32, flags=VNNI_A)                         # I2 needs INTLV_A_FORMAT as well
    assert not _dispatch(I2, I8, I32, m=18, lda=18)                         # m % 4: rows past 4*(m/4) are never written
    assert not _dispatch(I2, I8, I32, k=30, ldb=30)                         # k % 4
    assert not _dispatch(I1, I8, I32, flags=VNNI_A | INTLV_A)               # ignored by the reference: declined
    assert not _dispatch(I1, I8, I32, m=15, lda=16)                         # rows in pairs
    assert not _dispatch(I1, I8, I32, lda=17)                               # lda even
    assert not _dispatch(I1, I8, I32, k=30, ldb=32)                         # k % 4
    assert not _dispatch(MXFP4, I8, F32, flags=VNNI_A)                      # the int8-B form is the interleaved one
    assert not _dispatch(MXFP4, I8, F32, k=48, ldb=48)                      # k % 32
    assert not _dispatch(MXFP4, U8, F32) and not _dispatch(MXFP4, U8, BF16)   # no such branch: the bytes would be read as signed
    # comp and C types outside the tuples
    assert not _dispatch(I2, I8, F32) and not _dispatch(I1, U8, F32) and not _dispatch(MXFP4, I8, I32)
    assert not _dispatch(I2, I8, I32, comp=F32) and not _dispatch(MXFP4, I8, F32, comp=F32)
    assert not _dispatch(I2, I2, I32) and not _dispatch(I1, I1, I32)
    # declines pinned elsewhere: MXFP4 x BF16, MXFP4 x MXFP4, int4 x U8 with k = 12
    assert not _dispatch(MXFP4, BF16, F32, comp=F32, flags=VNNI_A) and not _dispatch(MXFP4, BF16, BF16, comp=F32, flags=VNNI_A)
    assert not _dispatch(MXFP4, MXFP4, F32, comp=F32, flags=VNNI_A)
    assert not _dispatch(18, U8, I32, k=12, ldb=12, flags=VNNI_A | INTLV_A)


def test_batch_refusals_without_a_device():
    nb = -6                                            # LIBXSMM_B200_ERROR_NOT_BATCHABLE
    for tc in (F32, BF16):
        h = _dispatch(MXFP4, I8, tc)
        assert h
        assert X.libxsmm_b200_gemm_batch_strided(h, 16, 16, 16, 0, 0, 0, 1, 1) == nb
        assert X.libxsmm_b200_gemm_batch_strided_multi(h, 16, 16, 16, 0, 0, 0, 1, 1, 1) == nb
        assert not X.libxsmm_b200_gemm_plan_create(h, None, 1)
        params = (X.GemmParam * 1)()                   # per-tile form: a tile without block scales is refused before any launch
        assert X.libxsmm_b200_gemm_batch(h, params, 1) == -1
        assert X.libxsmm_b200_gemm_batch_strided_scaled(h, 16, 16, 16, 0, 0, 0, 16, None, None, 0, 0, 0, 1, 1) == -1   # B scales missing
    h = _dispatch(MXFP4, I8, F32, br=X.GEMM_BATCH_REDUCE_OFFSET)
    assert X.libxsmm_b200_gemm_batch_strided_scaled(h, 16, 16, 16, 0, 0, 0, 16, 16, None, 0, 0, 0, 1, 1) == -2
    # I2 / I1 carry no per-call scales: the scaled form does not take them
    for ta, tb in ((I2, I8), (I1, U8)):
        assert X.libxsmm_b200_gemm_batch_strided_scaled(_dispatch(ta, tb, I32), 16, 16, 16, 0, 0, 0, 16, 16, None, 0, 0, 0, 1, 1) == -1
