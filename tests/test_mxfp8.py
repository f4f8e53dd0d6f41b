"""MX fp8 GEMM (MXBF8 x MXBF8 / MXHF8 x MXHF8 with E8M0 block scales), the parts that need no GPU:

  * the restatement oracle/oracle_mx.c equals the reference's libxsmm_reference_gemm bit for bit (both types, F32 / MXBF8 C,
    beta 0 / 1, no batch-reduce / stride, k = 32 .. 320, ldc > m, every fp8 byte pattern, scale bytes 0, 0xFF and 127 +- 20);
  * the committed fixture tests/golden/mxfp8.npz is what the oracle computes (and what the reference computes, where it exists);
  * dispatch: every accepted form gives a handle on the exact-order kernel, every declined clause gives NULL;
  * the batch entry points refuse MX handles (NOT_BATCHABLE), and the scaled entry point refuses every other handle."""
import os

import numpy as np
import pytest

import libxsmm_b200 as X
from mx_ffi import (BETA_0, F32, MX_FLAGS, MXBF8, MXHF8, TRANS_A, TRANS_B, VNNI_A, VNNI_B, MxCase, image_nan, oracle_e8m0_to_f32,
                    oracle_f32_to_mxbf8_block, oracle_gemm_mx, ref_gemm_mx, same_bits, same_mxbf8)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mxfp8.npz")
need_ref = pytest.mark.skipif(ref_gemm_mx is None, reason="the reference build (oracle/_ref/libxsmm_ref_mx.so) is not present")


def parity_cases():
    out = []
    for ta in (MXBF8, MXHF8):
        for k in (32, 64, 96, 320):
            out.append(MxCase(ta, F32, 7, 5, k, lda=9, ldb=6, ldc=11, beta0=True))
            out.append(MxCase(ta, F32, 12, 3, k, lda=12, ldb=4, ldc=13, beta0=False, br_type=3, br=3))
        out.append(MxCase(ta, F32, 33, 17, 128, lda=40, ldb=17, ldc=35, beta0=False))
    for k in (32, 160):
        out.append(MxCase(MXBF8, MXBF8, 32, 5, k, lda=33, ldb=7, ldc=64, beta0=True))
        out.append(MxCase(MXBF8, MXBF8, 64, 3, k, lda=64, ldb=3, ldc=96, beta0=True, br_type=3, br=2))
    return out


@need_ref
@pytest.mark.parametrize("case", parity_cases(), ids=repr)
def test_oracle_equals_reference_bit_for_bit(case):
    rng = np.random.default_rng(case.m * 1000 + case.k + case.ta)
    ops = case.operands(rng)
    rc_o, c_o, cs_o = case.run(oracle_gemm_mx, *ops)
    rc_r, c_r, cs_r = case.run(ref_gemm_mx, *ops)
    assert rc_o == 0 and rc_r == 0
    if case.tc == F32:
        assert same_bits(c_r, c_o)
        assert np.isnan(c_o).mean() < 0.7                        # the comparison is not vacuous (a 0xFF scale of B turns a column to NaN)
    else:
        assert same_mxbf8(c_r, c_o, image_nan(case, ops[0], ops[1], ops[3], ops[4])) and np.array_equal(cs_r, cs_o)


@need_ref
def test_scale_byte_quirks_match_the_reference():
    """scale 0 is +0 (not 2^-127) and 0xFF is +inf (not NaN): with A = B = 1.0 everywhere, a block with a zero scale adds
    +0 and one with 0xFF adds +inf"""
    for ta, one in ((MXBF8, 0x3C), (MXHF8, 0x38)):
        case = MxCase(ta, F32, 4, 3, 64, beta0=True)
        A = np.full(case.size_a, one, np.uint8); B = np.full(case.size_b, one, np.uint8)
        As = np.full(case.size_as, 127, np.uint8); Bs = np.full(case.size_bs, 127, np.uint8)
        As[0] = 0                        # row 0, first 32-k block: the block adds (32 * 0) * 1
        As[case.lda + 1] = 0xFF          # row 1, second 32-k block: (32 * inf) * 1
        ops = case.operands(np.random.default_rng(0), A, B, (As, Bs))
        for fn in (oracle_gemm_mx, ref_gemm_mx):
            rc, c, _ = case.run(fn, *ops)
            assert rc == 0
            c = c.reshape(case.n, case.ldc)
            assert c[0, 0] == 32.0 and c[0, 1] == np.inf and c[0, 2] == 64.0, c[0]
    assert oracle_e8m0_to_f32(0) == 0.0 and oracle_e8m0_to_f32(0xFF) == np.inf and oracle_e8m0_to_f32(127) == 1.0


@need_ref
def test_mxbf8_c_quantiser_matches_the_reference_on_edge_blocks():
    """the C quantiser through the reference GEMM: an all-zero block (scale byte 0, data bytes from 0 * inf), a tiny block
    (shared exponent clamped to 0), a huge block (exponent 254 clamp) and ordinary ones"""
    case = MxCase(MXBF8, MXBF8, 32, 4, 32, beta0=True)
    A = np.zeros(case.size_a, np.uint8); B = np.zeros(case.size_b, np.uint8)
    A[:] = 0x3C                                    # 1.0
    for j, bb in enumerate((0x00, 0x04, 0x7B, 0x3D)):   # B column j: 0, a subnormal, 57344, 1.25
        B.reshape(case.k // 4, case.ldb, 4)[:, j, :] = bb
    As = np.full(case.size_as, 127, np.uint8); Bs = np.array([127, 1, 254, 127], np.uint8)
    ops = case.operands(np.random.default_rng(1), A, B, (As, Bs))
    rc_o, c_o, cs_o = case.run(oracle_gemm_mx, *ops)
    rc_r, c_r, cs_r = case.run(ref_gemm_mx, *ops)
    assert rc_o == 0 and rc_r == 0
    assert np.array_equal(c_r, c_o) and np.array_equal(cs_r, cs_o), (c_r.reshape(4, 32)[:, :2], c_o.reshape(4, 32)[:, :2], cs_r, cs_o)


def test_mxbf8_block_quantiser_pins():
    """the quantiser's choices, stated without the reference: a zero block -> scale 0 and 0xFB bytes (0 * inf is x86's negative
    default NaN, clamped); 1.0 -> scale 127 - 15 and the bf8 code of 2^15 (0x78)"""
    out = np.zeros(32, np.uint8); sc = np.zeros(1, np.uint8)
    oracle_f32_to_mxbf8_block(np.zeros(32, np.float32).ctypes.data, out.ctypes.data, sc.ctypes.data)
    assert sc[0] == 0 and np.all(out == 0xFB)
    oracle_f32_to_mxbf8_block(np.ones(32, np.float32).ctypes.data, out.ctypes.data, sc.ctypes.data)
    assert sc[0] == 112 and np.all(out == 0x78)


def test_golden_fixture_is_what_the_oracle_computes():
    g = np.load(GOLDEN)
    n = int(g["ncases"])
    assert n >= 6
    for t in range(n):
        meta = g["meta%d" % t]
        case = MxCase(*[int(v) for v in meta])
        ops = [g["%s%d" % (nm, t)] for nm in ("a", "b", "c0", "as", "bs", "cs0")]
        rc, c, cs = case.run(oracle_gemm_mx, *ops)
        assert rc == 0
        if case.tc == F32:
            assert same_bits(g["c%d" % t], c), case
        else:
            assert same_mxbf8(g["c%d" % t], c, image_nan(case, ops[0], ops[1], ops[3], ops[4])) and np.array_equal(g["cs%d" % t], cs), case


# ---- dispatch (no device needed) -------------------------------------------------------------------------------------------
def _dispatch(ta, tc, m, n, k, lda, ldb, ldc, flags, br=None, sa=0, sb=0, tb=None, comp=F32):
    sh = X.libxsmm_create_gemm_shape(m, n, k, lda, ldb, ldc, ta, ta if tb is None else tb, tc, comp)
    if br is None:
        return X.libxsmm_dispatch_gemm(sh, flags, 0)
    return X.libxsmm_dispatch_brgemm(sh, flags, 0, X.libxsmm_create_gemm_batch_reduce_config(br, sa, sb, 0))


def test_dispatch_accepts_the_defined_forms_on_the_exact_order_kernel():
    for ta in (MXBF8, MXHF8):
        for flags in (MX_FLAGS, MX_FLAGS | BETA_0):
            h = _dispatch(ta, F32, 20, 9, 64, 24, 9, 21, flags)
            assert h and X.libxsmm_b200_kernel_backend(h) == X.BACKEND_SIMT
            h = _dispatch(ta, F32, 20, 9, 64, 24, 9, 21, flags, X.GEMM_BATCH_REDUCE_STRIDE, 24 * 64, 9 * 64)
            assert h and X.libxsmm_b200_kernel_backend(h) == X.BACKEND_SIMT
            h = _dispatch(ta, F32, 20, 9, 64, 24, 9, 21, flags, X.GEMM_BATCH_REDUCE_NONE)
            assert h
    h = _dispatch(MXBF8, MXBF8, 64, 9, 64, 64, 9, 96, MX_FLAGS | BETA_0)
    assert h and X.libxsmm_b200_kernel_backend(h) == X.BACKEND_SIMT


def test_dispatch_declines_every_undefined_form():
    base = dict(ta=MXBF8, tc=F32, m=32, n=8, k=64, lda=32, ldb=8, ldc=32, flags=MX_FLAGS)

    def d(**kw):
        a = dict(base); a.update(kw)
        return _dispatch(**a)
    assert d()                                                              # the control
    assert not d(flags=MX_FLAGS & ~VNNI_A) and not d(flags=MX_FLAGS & ~VNNI_B) and not d(flags=MX_FLAGS & ~TRANS_B)
    assert not d(flags=MX_FLAGS | TRANS_A)
    assert not d(flags=MX_FLAGS | X.GEMM_FLAG_VNNI_C) and not d(flags=MX_FLAGS | 524288)   # VNNI C, bitmap-compressed A
    assert not d(k=48) and not d(k=16)                                      # k % 32
    assert not d(lda=31) and not d(ldb=7)                                   # lda >= m, ldb >= n
    assert not d(tb=MXHF8) and not d(ta=MXHF8, tb=MXBF8)                    # mixed
    assert not d(ta=MXHF8, tc=MXHF8, flags=MX_FLAGS | BETA_0)               # MXHF8 C
    assert not d(comp=MXBF8) and not d(tc=2)                                # comp F32, C F32 / MXBF8
    for t in (16, 17, 20):                                                  # MXBF6, MXHF6, MXFP4
        assert not d(ta=t)
    assert not d(br=X.GEMM_BATCH_REDUCE_ADDRESS) and not d(br=X.GEMM_BATCH_REDUCE_OFFSET)
    assert d(br=X.GEMM_BATCH_REDUCE_STRIDE, sa=32 * 64, sb=8 * 64)
    assert not d(br=X.GEMM_BATCH_REDUCE_STRIDE, sa=32 * 64 + 16, sb=8 * 64) and not d(br=X.GEMM_BATCH_REDUCE_STRIDE, sa=32 * 64, sb=8 * 64 * 2)
    # MXBF8 C: BETA_0, m % 32, ldc % 32
    assert d(tc=MXBF8, flags=MX_FLAGS | BETA_0)
    assert not d(tc=MXBF8) and not d(tc=MXBF8, flags=MX_FLAGS | BETA_0, m=48, lda=48, ldc=64)
    assert not d(tc=MXBF8, flags=MX_FLAGS | BETA_0, ldc=48)
    # fused MX does not exist
    sh = X.libxsmm_create_gemm_shape(32, 8, 64, 32, 8, 32, MXBF8, MXBF8, F32, F32)
    assert not X.libxsmm_dispatch_brgemm_ext(sh, MX_FLAGS, 0, X.libxsmm_create_gemm_batch_reduce_config(0, 0, 0, 0),
                                             X.libxsmm_create_gemm_ext_unary_argops(0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0),
                                             X.libxsmm_create_gemm_ext_binary_postops(0, 0, 0, 0))


def test_batch_entry_points_refuse_mx_handles_and_scaled_refuses_others():
    h = _dispatch(MXHF8, F32, 32, 8, 64, 32, 8, 32, MX_FLAGS)
    nb = -6                                            # LIBXSMM_B200_ERROR_NOT_BATCHABLE
    assert X.libxsmm_b200_gemm_batch_strided(h, 16, 16, 16, 0, 0, 0, 1, 1) == nb
    assert X.libxsmm_b200_gemm_batch_strided_multi(h, 16, 16, 16, 0, 0, 0, 1, 1, 1) == nb
    assert X.libxsmm_b200_gemm_batch(h, None, 1) == nb
    other = X.libxsmm_dispatch_gemm(X.libxsmm_create_gemm_shape(8, 8, 8, 8, 8, 8, F32, F32, F32, F32), 0, 0)
    assert other
    assert X.libxsmm_b200_gemm_batch_strided_scaled(other, 16, 16, 16, 0, 0, 0, 16, 16, 16, 0, 0, 0, 1, 1) == -1
    assert X.libxsmm_b200_gemm_batch_strided_scaled(None, 16, 16, 16, 0, 0, 0, 16, 16, 16, 0, 0, 0, 1, 1) == -1
    assert X.TYPESIZE[MXBF8] == 1 and X.TYPESIZE[MXHF8] == 1
