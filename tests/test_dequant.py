"""Dequantising GEMM (I8 x BF16, I8 / I4 / U4 / BF8 x F16 with per-row scales and zero points), the parts that need no GPU:

  * the restatement oracle/oracle_dq.c equals the reference's libxsmm_reference_gemm bit for bit for every tuple, comp (F16 / F32 /
    IMPLICIT), beta 0 / 1, all four batch-reduce modes, ld > dim and TRANS_B where the reference honours it; A covers every int8,
    int4 and bf8 byte, the scales 0, negative values and values that overflow f16 under the replacement FMA, the zero points sit on
    f16 rounding ties; NaN positions are excluded;
  * the reference's quirks the dispatch rules rest on: U8 bytes are used as signed, I8 x F16 ignores zero points, IMPLICIT is F16
    comp on an SPR host;
  * the committed fixture tests/golden/dequant.npz is what the oracle computes, and what the reference computes where it exists;
  * dispatch: every accepted form gives a handle on the exact-order kernel, every declined clause gives NULL;
  * the batch entry points' refusals, without a device."""
import os

import numpy as np
import pytest

import libxsmm_b200 as X
from dq_ffi import (BETA_0, BF8, BF16, F16, F32, I4, I8, IMPLICIT, TRANS_A, TRANS_B, U4, U8, VNNI_A, VNNI_B, DqCase, case_from_meta, meta,
                    oracle_gemm_dq, ref_gemm_dq, same_c)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dequant.npz")
need_ref = pytest.mark.skipif(ref_gemm_dq is None, reason="the reference build (oracle/_ref/libxsmm_ref_dq.so) is not present")

TUPLES = [(I8, BF16, F32, F32), (I8, BF16, F32, BF16)] + \
         [(ta, F16, comp, tc) for ta in (I8, I4, U4, BF8) for comp in (F16, F32, IMPLICIT) for tc in (F16, F32)]


def parity_cases():
    out = []
    for ta, tb, comp, tc in TUPLES:
        for br_type in (0, 1, 2, 3):
            for beta0 in (True, False):
                trans = (False, True) if tb == F16 else (False,)
                for tr in trans:
                    vn = [None] if ta != BF8 else [False, True]
                    for v in vn:
                        out.append(DqCase(ta, tb, comp, tc, 11, 6, 26, lda=13, ldb=(9 if tr else 30), ldc=12, beta0=beta0, trans_b=tr,
                                          vnni_a=v, br_type=br_type, br=3))
    return out


@need_ref
@pytest.mark.parametrize("case", parity_cases(), ids=repr)
def test_oracle_equals_reference_bit_for_bit(case):
    rng = np.random.default_rng(case.m * 1000 + case.k + case.ta * 7 + case.comp * 3 + case.br_type + 17 * case.beta0)
    ops = case.operands(rng)
    rc_o, c_o = case.run(oracle_gemm_dq, *ops)
    rc_r, c_r = case.run(ref_gemm_dq, *ops)
    assert rc_o == 0 and rc_r == 0
    assert same_c(case, c_r, c_o)
    assert case.nan_mask(c_o).mean() < 0.5                       # not vacuous


@need_ref
def test_inputs_cover_every_byte_and_the_overflow_scales():
    """one long k per form: every int8 / int4 / bf8 byte value appears in A; under comp F16 a scale of 900 turns 127 * 900 into +-inf
    (f16 overflow) where comp F32 keeps it finite; the results still agree with the reference"""
    for ta, tb, tc in ((I8, BF16, BF16), (I8, F16, F16), (I4, F16, F32), (U4, F16, F16), (BF8, F16, F32)):
        for comp in ((F32,) if tb == BF16 else (F16, F32, IMPLICIT)):
            case = DqCase(ta, tb, comp, tc, 16, 4, 512, beta0=False)
            rng = np.random.default_rng(ta * 100 + comp)
            A, B, C0, S, Z = case.operands(rng)
            A[:256] = np.arange(256, dtype=np.uint8)
            assert len(np.unique(A)) == 256
            rc_o, c_o = case.run(oracle_gemm_dq, A, B, C0, S, Z)
            rc_r, c_r = case.run(ref_gemm_dq, A, B, C0, S, Z)
            assert rc_o == 0 and rc_r == 0 and same_c(case, c_r, c_o), case
    # overflow under the replacement FMA: A = 127 everywhere, B = 1, scale 900
    case16, case32 = DqCase(I8, F16, F16, F32, 4, 2, 2), DqCase(I8, F16, F32, F32, 4, 2, 2)
    A = np.full(case16.size_a, 127, np.uint8); B = np.full(case16.size_b, 0x3C00, np.uint16)
    S = np.full(4, 0x6308, np.uint16)                             # f16 900
    for case, want_inf in ((case16, True), (case32, False)):
        _, c_r = case.run(ref_gemm_dq, A, B, np.zeros(case.size_c, np.float32), S, None)
        _, c_o = case.run(oracle_gemm_dq, A, B, np.zeros(case.size_c, np.float32), S, None)
        assert np.all(np.isinf(c_r) == want_inf) and same_c(case, c_r, c_o)


@need_ref
def test_reference_quirks_the_dispatch_rules_rest_on():
    rng = np.random.default_rng(3)
    # U8 A: the same bytes give the I8 results (the branches read A as char, :1703 / :1907 / :1979) -- dispatch declines U8
    for tb, tc in ((BF16, F32), (F16, F16), (F16, F32)):
        ci = DqCase(I8, tb, F32, tc, 9, 5, 20, beta0=False)
        cu = DqCase(U8, tb, F32, tc, 9, 5, 20, beta0=False)
        ops = ci.operands(rng)
        assert np.any(ops[0] >= 128)
        _, c_i = ci.run(ref_gemm_dq, *ops)
        _, c_u = cu.run(ref_gemm_dq, *ops)
        assert same_c(ci, c_i, c_u)
    # I8 x F16: a.quaternary is never read (fuse_zpt_sub is 0 for I8, :430 / :473)
    case = DqCase(I8, F16, F16, F16, 9, 5, 20)
    A, B, C0, S, Z = case.operands(rng)
    _, c1 = case.run(ref_gemm_dq, A, B, C0, S, Z)
    _, c2 = case.run(ref_gemm_dq, A, B, C0, S, (Z.astype(np.int32) ^ 0x1234).astype(np.uint16))
    assert np.array_equal(c1, c2)
    # IMPLICIT is the replacement FMA (F16 comp) as resolved on an SPR host, and differs from F32 comp
    res = {}
    for comp in (F16, IMPLICIT, F32):
        case = DqCase(I4, F16, comp, F32, 16, 8, 128)
        _, res[comp] = case.run(ref_gemm_dq, *case.operands(np.random.default_rng(11)))
    assert np.array_equal(res[F16], res[IMPLICIT]) and not np.array_equal(res[F16], res[F32])


def golden_cases():
    g = np.load(GOLDEN)
    return [(case_from_meta(g["meta%d" % t]), [g["%s%d" % (nm, t)] for nm in ("a", "b", "c0", "s", "z")], g["c%d" % t])
            for t in range(int(g["ncases"]))]


def test_golden_fixture_is_what_the_oracle_computes():
    cases = golden_cases()
    assert len(cases) >= 10
    assert {c.ta for c, _, _ in cases} == {I8, I4, U4, BF8} and {c.br_type for c, _, _ in cases} == {0, 1, 2, 3}
    for case, ops, want in cases:
        rc, c = case.run(oracle_gemm_dq, *ops)
        assert rc == 0 and same_c(case, want, c), case


@need_ref
def test_golden_fixture_reproduces_from_the_reference():
    import sys
    sys.path.insert(0, os.path.dirname(GOLDEN))
    import make_golden_dq
    g = np.load(GOLDEN)
    assert int(g["ncases"]) == len(make_golden_dq.CASES)
    for t, case in enumerate(make_golden_dq.CASES):
        ops = case.operands(np.random.default_rng(5150 + t))
        for nm, x in zip(("a", "b", "c0", "s", "z"), ops):
            assert np.array_equal(g["%s%d" % (nm, t)], x), (t, nm)
        assert np.array_equal(g["meta%d" % t], meta(case))
        rc, c = case.run(ref_gemm_dq, *ops)
        assert rc == 0 and np.array_equal(g["c%d" % t].view(np.uint8), c.view(np.uint8)), case   # NaN bits included


# ---- dispatch (no device needed) -------------------------------------------------------------------------------------------
def _dispatch(ta, tb, comp, tc, m=16, n=8, k=32, lda=16, ldb=32, ldc=16, flags=0, br=None, sa=0, sb=0):
    sh = X.libxsmm_create_gemm_shape(m, n, k, lda, ldb, ldc, ta, tb, tc, comp)
    if br is None:
        return X.libxsmm_dispatch_gemm(sh, flags, 0)
    return X.libxsmm_dispatch_brgemm(sh, flags, 0, X.libxsmm_create_gemm_batch_reduce_config(br, sa, sb, 0))


def test_dispatch_accepts_the_defined_forms_on_the_exact_order_kernel():
    for ta, tb, comp, tc in TUPLES:
        vn = VNNI_A if ta in (I4, U4) else 0
        for extra in ([0, TRANS_B] if tb == F16 else [0]):
            for beta in (0, BETA_0):
                flags = vn | extra | beta
                ldb = 8 if extra else 32
                for br in (None, X.GEMM_BATCH_REDUCE_NONE, X.GEMM_BATCH_REDUCE_ADDRESS, X.GEMM_BATCH_REDUCE_OFFSET, X.GEMM_BATCH_REDUCE_STRIDE):
                    h = _dispatch(ta, tb, comp, tc, ldb=ldb, flags=flags, br=br, sa=512, sb=1024)
                    assert h and X.libxsmm_b200_kernel_backend(h) == X.BACKEND_SIMT, (ta, tb, comp, tc, flags, br)
    assert _dispatch(BF8, F16, F16, F16, flags=VNNI_A)          # VNNI2 bf8 A
    assert _dispatch(I8, F16, F32, F32, m=7, lda=9, ldc=11, k=5, ldb=6)   # ld > dim, odd k for a flat A


def test_dispatch_declines_every_undefined_form():
    assert _dispatch(I8, BF16, F32, BF16)                                      # the controls
    assert _dispatch(I4, F16, F16, F16, flags=VNNI_A)
    # U8 A: the reference would use the bytes as signed
    for tb, comp, tc in ((BF16, F32, F32), (BF16, F32, BF16), (F16, F16, F16), (F16, F32, F32), (F16, IMPLICIT, F16)):
        assert not _dispatch(U8, tb, comp, tc)
    # flags the reference would ignore rather than obey
    assert not _dispatch(I8, BF16, F32, BF16, flags=TRANS_B, ldb=8) and not _dispatch(I8, BF16, F32, BF16, flags=VNNI_A)
    assert not _dispatch(I8, F16, F16, F16, flags=VNNI_A)
    for ta, tb, comp, tc, base in ((I8, BF16, F32, F32, 0), (I8, F16, F16, F16, 0), (I4, F16, F16, F32, VNNI_A), (BF8, F16, F32, F16, 0)):
        assert _dispatch(ta, tb, comp, tc, flags=base)
        assert not _dispatch(ta, tb, comp, tc, flags=base | TRANS_A, lda=32)
        assert not _dispatch(ta, tb, comp, tc, flags=base | VNNI_B)
        assert not _dispatch(ta, tb, comp, tc, flags=base | X.GEMM_FLAG_VNNI_C)
        assert not _dispatch(ta, tb, comp, tc, flags=base | 524288)          # bitmap-compressed A
        assert not _dispatch(ta, tb, comp, tc, flags=base, lda=15)          # lda >= m
        assert not _dispatch(ta, tb, comp, tc, flags=base, ldb=31)          # ldb >= k
        if tb == F16:
            assert not _dispatch(ta, tb, comp, tc, flags=base | TRANS_B, ldb=7)   # ldb >= n under TRANS_B
    assert not _dispatch(I4, F16, F16, F16)                                  # int4 x f16 is the VNNI_A form only
    assert not _dispatch(U4, F16, F16, F16, flags=VNNI_A | 262144)          # INTLV_A_FORMAT: the int8-B form
    assert not _dispatch(I4, F16, F16, F16, flags=VNNI_A, k=31, ldb=31)     # odd k in pairs
    assert not _dispatch(BF8, F16, F16, F16, flags=VNNI_A, k=31, ldb=31)
    assert _dispatch(BF8, F16, F16, F16, k=31, ldb=31)                      # flat bf8: any k
    # comp / C types outside the tuples
    assert not _dispatch(I8, BF16, BF16, BF16) and not _dispatch(I8, BF16, F32, F16) and not _dispatch(I8, F16, F32, BF16)
    assert not _dispatch(I8, F16, BF16, F16) and not _dispatch(BF8, F16, F32, BF8) and not _dispatch(I4, F16, F32, BF16, flags=VNNI_A)
    # no fused form
    sh = X.libxsmm_create_gemm_shape(16, 8, 32, 16, 32, 16, I8, BF16, BF16, F32)
    assert not X.libxsmm_dispatch_brgemm_ext(sh, 0, 0, X.libxsmm_create_gemm_batch_reduce_config(0, 0, 0, 0),
                                             X.libxsmm_create_gemm_ext_unary_argops(0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
                                             X.libxsmm_create_gemm_ext_binary_postops(0, 0, 0, 0))


def test_batch_refusals_without_a_device():
    nb = -6                                            # LIBXSMM_B200_ERROR_NOT_BATCHABLE
    for ta, tb, comp, tc, fl in ((I8, BF16, F32, BF16, 0), (I8, F16, F16, F32, 0), (I4, F16, F16, F16, VNNI_A), (U4, F16, F32, F32, VNNI_A)):
        h = _dispatch(ta, tb, comp, tc, flags=fl)
        assert h
        assert X.libxsmm_b200_gemm_batch_strided(h, 16, 16, 16, 0, 0, 0, 1, 1) == nb
        assert X.libxsmm_b200_gemm_batch_strided_multi(h, 16, 16, 16, 0, 0, 0, 1, 1, 1) == nb
        assert not X.libxsmm_b200_gemm_plan_create(h, None, 1)
        params = (X.GemmParam * 1)()                   # per-tile form: a tile without row scales is refused before any launch
        assert X.libxsmm_b200_gemm_batch(h, params, 1) == -1
    # the scaled strided form takes the int8 handles only; int4 needs zero points per tile, bf8 has no scales
    for ta, tb, comp, tc, fl in ((I4, F16, F16, F16, VNNI_A), (BF8, F16, F16, F16, 0)):
        assert X.libxsmm_b200_gemm_batch_strided_scaled(_dispatch(ta, tb, comp, tc, flags=fl), 16, 16, 16, 0, 0, 0, 16, 0, 0, 0, 0, 0, 1, 1) == -1
    h = _dispatch(I8, BF16, F32, BF16)
    assert X.libxsmm_b200_gemm_batch_strided_scaled(h, 16, 16, 16, 0, 0, 0, None, 0, 0, 0, 0, 0, 1, 1) == -1   # scales missing
    h = _dispatch(I8, F16, F16, F16, br=X.GEMM_BATCH_REDUCE_ADDRESS)
    assert X.libxsmm_b200_gemm_batch_strided_scaled(h, 16, 16, 16, 0, 0, 0, 16, 0, 0, 0, 0, 0, 1, 1) == -2
    assert X.TYPESIZE[I4] == 1 and X.TYPESIZE[U4] == 1
