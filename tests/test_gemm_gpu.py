"""GPU parity of the dense GEMM/BRGEMM path through the C ABI.

 * exact-order CUDA-core kernel: bit-identical to the oracle (and to the reference itself where
   oracle/_ref is present) for every precision tuple / layout flag / batch-reduce mode of the first bar;
 * tensor-core (wgmma) kernel: within the reference's acceptance norms (samples/xgemm/gemm_kernel.c:5312-5414:
   f32 out < 1.2e-5, bf16/f16 out < 5e-3 relative Frobenius error)."""
import ctypes as C

import numpy as np
import pytest
import torch

import cases
import gen
import libxsmm_b200 as X
import gpu_util
from gpu_util import dev, dispatch, host, run_single_calls
from oracle_ffi import iarr, oracle, ref, run_gemm

pytestmark = pytest.mark.gpu


def test_simt_every_tuple_bit_exact():
    X.libxsmm_b200_set_force_simt(1)
    try:
        n = 0
        for case in cases.small_cases():
            ops = cases.Operands(case, seed=100 + n)
            kernel = dispatch(case, ops)
            assert kernel, case
            assert X.libxsmm_b200_kernel_backend(kernel) == X.BACKEND_SIMT
            d_a, d_b, d_c = dev(ops.a), dev(ops.b), dev(ops.c0)
            run_single_calls(kernel, case, ops, d_a, d_b, d_c)
            got = host(d_c, gen.NP_OF[case.tc])
            want = cases.ref_result(oracle, case, ops, run_gemm)
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), case
            if ref is not None and n % 7 == 0:
                assert np.array_equal(got.view(np.uint8), cases.ref_result(ref, case, ops, run_gemm).view(np.uint8)), case
            n += 1
    finally:
        X.libxsmm_b200_set_force_simt(0)


def test_hello_host_pointers_f64_and_f32():
    """samples/hello/hello.c: plain host memory, 1000 calls C += A_i * B_i of a 13x5x7 kernel"""
    for t in (gen.F64, gen.F32):
        case = cases.GemmCase(13, 5, 7, t, t, t, t)
        ops = cases.Operands(case, count=50)
        kernel = dispatch(case, ops)
        assert kernel
        c = np.zeros(case.size_c, dtype=gen.NP_OF[t]); want = c.copy()
        fn = X.GEMMFUNCTION(kernel)
        for i in range(ops.count):
            p = X.GemmParam()
            p.a.primary = ops.a.ctypes.data + i * ops.tile_a; p.b.primary = ops.b.ctypes.data + i * ops.tile_b; p.c.primary = c.ctypes.data
            fn(C.byref(p))
            run_gemm(oracle, case.dims, case.types, 0, 0, 0, 0, 1, ops.a[i * case.size_a:], ops.b[i * case.size_b:], want)
        X.check()
        assert np.array_equal(c, want)


TC_SHAPES = [(64, 64, 64), (64, 64, 32), (32, 64, 64), (64, 32, 64), (48, 40, 80), (128, 64, 64), (96, 128, 64),
             (128, 128, 128), (16, 16, 16), (64, 256, 64), (64, 64, 128), (24, 72, 200), (32, 40, 96), (16, 24, 48), (32, 128, 64)]   # m = 16 / 32: small tiles in an m64 instruction


@pytest.mark.parametrize("ta,tc", [(gen.BF16, gen.F32), (gen.BF16, gen.BF16), (gen.F16, gen.F32), (gen.F16, gen.F16)])
def test_tcgen05_brgemm_within_reference_norm(ta, tc):
    thr = 1.2e-5 if tc == gen.F32 else 5e-3
    n = 0
    for (m, n_, k) in TC_SHAPES:
        for br_type, br, beta0, count in ((3, 8, 1, 37), (3, 3, 0, 5), (0, 1, 1, 300), (3, 1, 0, 2)):
            if m * n_ * k >= 128 ** 3 and count > 40:
                count = 40
            case = cases.GemmCase(m, n_, k, ta, ta, gen.F32, tc, flags=(cases.FLAG_BETA_0 if beta0 else 0), br_type=br_type, br=br,
                                  lda=(m + 7) // 8 * 8, ldb=(k + 7) // 8 * 8, ldc=m + (3 if n % 2 else 0))
            ops = cases.Operands(case, seed=900 + n, count=count)
            kernel = dispatch(case, ops)
            assert kernel and X.libxsmm_b200_kernel_backend(kernel) == X.BACKEND_TCGEN05, case
            d_a, d_b, d_c = dev(ops.a), dev(ops.b), dev(ops.c0)
            rc = X.libxsmm_b200_gemm_batch_strided(kernel, d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(),
                                                   ops.tile_a, ops.tile_b, ops.tile_c, case.br, count)
            assert rc == 0, (case, X.libxsmm_b200_last_error_string())
            got = host(d_c, gen.NP_OF[tc])
            want = cases.ref_result(oracle, case, ops, run_gemm)
            err = gen.normf_rel(gen.to_f64(want, tc), gen.to_f64(got, tc))
            assert err <= thr, (case, count, err)
            # untouched padding of C (ldc > m) must be preserved
            if case.ldc > case.m:
                g = got.reshape(count, case.n, case.ldc)[:, :, case.m:]; w = ops.c0.reshape(count, case.n, case.ldc)[:, :, case.m:]
                assert np.array_equal(g, w), case
            n += 1


def test_tcgen05_single_call_matches_batch():
    case = cases.GemmCase(64, 64, 64, gen.BF16, gen.BF16, gen.F32, gen.F32, flags=cases.FLAG_BETA_0, br_type=3, br=8)
    ops = cases.Operands(case, count=3)
    kernel = dispatch(case, ops)
    d_a, d_b, d_c = dev(ops.a), dev(ops.b), dev(ops.c0)
    run_single_calls(kernel, case, ops, d_a, d_b, d_c)
    got = host(d_c, np.float32)
    want = cases.ref_result(oracle, case, ops, run_gemm)
    assert gen.normf_rel(want, got) <= 1.2e-5


def test_batch_plan_address_mode():
    """general batch entry point: one reference argument struct per tile, address batch-reduce"""
    case = cases.GemmCase(32, 24, 16, gen.F32, gen.F32, gen.F32, gen.F32, flags=0, br_type=1, br=4)
    ops = cases.Operands(case, count=9); ops.case_br = case.br
    kernel = dispatch(case, ops)
    d_a, d_b, d_c = dev(ops.a), dev(ops.b), dev(ops.c0)
    params = (X.GemmParam * ops.count)(); keep = []
    for t in range(ops.count):
        aa, ab = ops.addr_arrays(d_a.data_ptr(), d_b.data_ptr(), t); br = C.c_ulonglong(case.br); keep += [aa, ab, br]
        params[t].op.tertiary = C.addressof(br)
        params[t].a.primary, params[t].b.primary = C.addressof(aa), C.addressof(ab)
        params[t].c.primary = d_c.data_ptr() + t * ops.tile_c
    assert X.libxsmm_b200_gemm_batch(kernel, params, ops.count) == 0
    X.check()
    assert np.array_equal(host(d_c, np.float32), cases.ref_result(oracle, case, ops, run_gemm))


def test_int8_full_size_linearity_property():
    """size-independent property at a BASELINE size (int8 128^3, batch 4096): C(A, B1+B2) == C(A,B1) + C(A,B2) exactly"""
    case = cases.GemmCase(128, 128, 128, gen.I8, gen.I8, gen.I32, gen.I32, flags=cases.FLAG_BETA_0 | cases.FLAG_VNNI_A)
    count = 4096
    rng = np.random.default_rng(11)
    a = rng.integers(-20, 20, size=case.size_a * count, dtype=np.int8)
    b1 = rng.integers(-20, 20, size=case.size_b * count, dtype=np.int8); b2 = rng.integers(-20, 20, size=case.size_b * count, dtype=np.int8)
    ops = cases.Operands(case, count=1)
    kernel = dispatch(case, ops)
    outs = []
    for b in (b1, b2, (b1 + b2).astype(np.int8)):
        d_a, d_b = dev(a), dev(b); d_c = torch.zeros(case.size_c * count * 4, dtype=torch.uint8, device="cuda")
        assert X.libxsmm_b200_gemm_batch_strided(kernel, d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), case.size_a, case.size_b, case.size_c * 4, 1, count) == 0
        outs.append(host(d_c, np.int32))
    assert np.array_equal(outs[0] + outs[1], outs[2])


@pytest.mark.parametrize("pinned", [False, True])
def test_host_resident_batch_goes_through_the_copy_pipeline(pinned, monkeypatch):
    """libxsmm_b200_gemm_batch_strided with HOST buffers (the e2e path of bench.py): chunks of the batch are staged through
    three streams; many small chunks (1 MB) exercise slot reuse; beta=1 needs C copied in as well."""
    monkeypatch.setenv("LIBXSMM_B200_CHUNK_MB", "1")
    for (t, beta0, count) in (((gen.BF16, gen.BF16, gen.F32, gen.F32), 1, 150), ((gen.BF16, gen.BF16, gen.F32, gen.BF16), 0, 90),
                              ((gen.U8, gen.I8, gen.I32, gen.I32), 0, 70)):
        flags = (cases.FLAG_BETA_0 if beta0 else 0) | (cases.FLAG_VNNI_A if t[0] == gen.U8 else 0)
        case = cases.GemmCase(64, 64, 64, *t, flags=flags, br_type=3, br=4)
        ops = cases.Operands(case, seed=31, count=count)
        kernel = dispatch(case, ops)
        assert kernel
        want = cases.ref_result(oracle, case, ops, run_gemm)
        if pinned:
            ha, hb, hc = (torch.from_numpy(x.view(np.uint8).copy()).pin_memory() for x in (ops.a, ops.b, ops.c0))
            pa, pb, pc = ha.data_ptr(), hb.data_ptr(), hc.data_ptr()
        else:
            ha, hb, hc = ops.a.copy(), ops.b.copy(), ops.c0.copy()
            pa, pb, pc = ha.ctypes.data, hb.ctypes.data, hc.ctypes.data
        rc = X.libxsmm_b200_gemm_batch_strided(kernel, pa, pb, pc, ops.tile_a, ops.tile_b, ops.tile_c, case.br, count)
        assert rc == 0, X.libxsmm_b200_last_error_string()
        X.check()
        got = hc.numpy().view(gen.NP_OF[case.tc]) if pinned else hc
        if case.tc == gen.I32:
            assert np.array_equal(got, want)
        else:
            assert gen.normf_rel(gen.to_f64(want, case.tc), gen.to_f64(got, case.tc)) <= (1.2e-5 if case.tc == gen.F32 else 5e-3)


@pytest.mark.parametrize("types", [(gen.F32, gen.F32, gen.F32, gen.F32), (gen.BF16, gen.BF16, gen.F32, gen.BF16), (gen.BF16, gen.BF16, gen.F32, gen.F32),
                                   (gen.F16, gen.F16, gen.F32, gen.F16), (gen.U8, gen.I8, gen.I32, gen.F32)])
def test_fused_brgemm_ext_matches_oracle(types):
    """libxsmm_dispatch_brgemm_ext: column-bias pre-op, ReLU (+bitmask) / sigmoid post-op, VNNI-packed C, over the matrix of
    samples/xgemm/kernel_test/gemm_kernel_fused.tpl (beta x batch-reduce mode x fusion). ReLU / bias / packing are bit-exact
    (same operation order and rounding points as the reference); sigmoid within 1 ulp of the output type (device tanhf)."""
    import ctypes as C
    from oracle_ffi import oracle
    rng = np.random.default_rng(89)
    ta, tb, tcomp, tc = types
    for (m, n, k, pad) in ((32, 16, 32, 0), (13, 6, 8, 3), (64, 64, 64, 0)):
        for beta0 in (1, 0):
            for br_type, br in ((0, 1), (3, 3)):
                for fuse in cases.fused_variants():
                    if fuse[3] and (tc == gen.F32 or n % 2):
                        continue
                    vnni_a = ta in (gen.I8, gen.U8) or (ta != gen.F32 and k % 2 == 0 and m % 2 == 0)   # int8: VNNI4 A, k % 4 == 0
                    flags = (cases.FLAG_BETA_0 if beta0 else 0) | (cases.FLAG_VNNI_A if vnni_a else 0)
                    case = cases.GemmCase(m, n, k, ta, tb, tcomp, tc, flags=flags, br_type=br_type, br=br, pad=pad)
                    ops = cases.Operands(case, seed=int(rng.integers(1 << 30)))
                    bias = gen.values(rng, m, tc)
                    mask0 = rng.integers(0, 256, size=((case.ldc + 15) // 16 * 16) // 8 * n + 8, dtype=np.uint8)
                    scf = C.c_float(ops.scf)     # int8 -> f32 scale, read from c.tertiary
                    want, wmask = ops.c0.copy(), mask0.copy()
                    assert cases.run_gemm_ext(oracle, case, ops, fuse, bias if fuse[0] else None, wmask if fuse[2] else None, want) == 0
                    argops = X.libxsmm_create_gemm_ext_unary_argops(0, 0, 0, 0, 0, 0, 0, 0, case.ldc, fuse[1], X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT if fuse[2] else 0, 0)
                    postops = X.libxsmm_create_gemm_ext_binary_postops(case.ldc, tc, X.MELTW_TYPE_BINARY_ADD if fuse[0] else 0,
                                                                       X.MELTW_FLAG_BINARY_BCAST_COL_IN_0 if fuse[0] else 0)
                    brt = {0: X.GEMM_BATCH_REDUCE_NONE, 3: X.GEMM_BATCH_REDUCE_STRIDE}[br_type]
                    cfg = X.libxsmm_create_gemm_batch_reduce_config(brt, ops.stride_a, ops.stride_b, 0)
                    k_ext = X.libxsmm_dispatch_brgemm_ext(gpu_util.shape_of(case), case.flags | (cases.FLAG_VNNI_C if fuse[3] else 0), 0, cfg, argops, postops)
                    assert k_ext, (case, fuse)
                    for resident in (1, 0):      # device buffers, then host buffers through the staging path
                        if resident:
                            d_a, d_b, d_c, d_bias, d_m = dev(ops.a), dev(ops.b), dev(ops.c0), dev(bias), dev(mask0)
                            pa, pb, pc, pd, pm = d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), d_bias.data_ptr(), d_m.data_ptr()
                        else:
                            hc, hm = ops.c0.copy(), mask0.copy()
                            pa, pb, pc, pd, pm = ops.a.ctypes.data, ops.b.ctypes.data, hc.ctypes.data, bias.ctypes.data, hm.ctypes.data
                        p = X.GemmExtParam(); brv = C.c_ulonglong(case.br)
                        p.op.tertiary = C.addressof(brv); p.a.primary, p.b.primary, p.c.primary = pa, pb, pc
                        p.c.tertiary = C.addressof(scf)
                        if fuse[0]:
                            p.d.primary = pd
                        if fuse[2]:
                            p.c.secondary = pm
                        X.GEMMFUNCTION_EXT(k_ext)(C.byref(p)); X.check()
                        got = host(d_c, gen.NP_OF[tc]) if resident else hc
                        gm = host(d_m, np.uint8) if resident else hm
                        if fuse[1] == cases.SIGMOID:
                            g64, w64 = gen.to_f64(got, tc), gen.to_f64(want, tc)
                            tol = {gen.F32: 3e-7, gen.BF16: 8e-3, gen.F16: 1e-3}[tc]
                            assert np.allclose(g64, w64, rtol=tol, atol=tol), (case, fuse, resident)
                        else:
                            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (case, fuse, resident)
                        if fuse[2]:
                            assert np.array_equal(gm, wmask), (case, fuse, resident, "relu mask")


def test_int4_gemm_with_zero_points_bit_exact():
    """U4 x U8 -> I32 (reference :1273-1321) through libxsmm_dispatch_gemm / _brgemm: device and host operands"""
    import ctypes as C
    from test_oracle_vs_ref import FLAG_COL_VEC_ZPT, FLAG_INTLV_A, FLAG_MXK_ZPT, I4X2, int4_case
    rng = np.random.default_rng(92)
    for (m, n, k, pad) in ((32, 16, 32, 0), (13, 6, 8, 3), (64, 64, 64, 0), (5, 3, 16, 1)):
        for br_type, br in ((0, 1), (3, 4)):
            for beta0 in (0, 1):
                dims, a, b, zpt, c0, blk_a, blk_b = int4_case(rng, m, n, k, br, pad)
                flags = (cases.FLAG_BETA_0 if beta0 else 0) | cases.FLAG_VNNI_A | FLAG_INTLV_A | (FLAG_MXK_ZPT if br_type else FLAG_COL_VEC_ZPT)
                want = c0.copy()
                assert oracle["gemm_i4"](iarr(*dims), flags, br_type, blk_a, blk_b, br, a.ctypes.data, b.ctypes.data, want.ctypes.data, zpt.ctypes.data) == 0
                sh = X.libxsmm_create_gemm_shape(*dims, I4X2, gen.U8, gen.I32, gen.I32)
                if br_type:
                    kern = X.libxsmm_dispatch_brgemm(sh, flags, 0, X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, blk_a, blk_b, 0))
                else:
                    kern = X.libxsmm_dispatch_gemm(sh, flags, 0)
                assert kern and X.libxsmm_b200_kernel_backend(kern) == X.BACKEND_SIMT
                for resident in (1, 0):
                    if resident:
                        d_a, d_b, d_c, d_z = dev(a), dev(b), dev(c0), dev(zpt)
                        pa, pb, pc, pz = d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), d_z.data_ptr()
                    else:
                        hc = c0.copy(); pa, pb, pc, pz = a.ctypes.data, b.ctypes.data, hc.ctypes.data, zpt.ctypes.data
                    p = X.GemmParam(); brv = C.c_ulonglong(br)
                    p.op.tertiary = C.addressof(brv); p.a.primary, p.b.primary, p.c.primary, p.a.quaternary = pa, pb, pc, pz
                    X.GEMMFUNCTION(kern)(C.byref(p)); X.check()
                    got = host(d_c, np.int32) if resident else hc
                    assert np.array_equal(got, want), (dims, br_type, beta0, resident)
                if br_type:   # per-tile batch: each record carries its own tile's zero points (a.quaternary)
                    zpt2 = ((zpt + 7) % 16).astype(np.uint8); want2 = c0.copy()
                    assert oracle["gemm_i4"](iarr(*dims), flags, br_type, blk_a, blk_b, br, a.ctypes.data, b.ctypes.data, want2.ctypes.data, zpt2.ctypes.data) == 0
                    d_a, d_b, d_zs, d_cs = dev(a), dev(b), (dev(zpt), dev(zpt2)), (dev(c0), dev(c0))
                    params = (X.GemmParam * 2)(); brv = C.c_ulonglong(br)
                    for t in range(2):
                        params[t].op.tertiary = C.addressof(brv)
                        params[t].a.primary, params[t].b.primary, params[t].c.primary, params[t].a.quaternary = d_a.data_ptr(), d_b.data_ptr(), d_cs[t].data_ptr(), d_zs[t].data_ptr()
                    assert X.libxsmm_b200_gemm_batch(kern, params, 2) == 0; X.check()
                    assert np.array_equal(host(d_cs[0], np.int32), want) and np.array_equal(host(d_cs[1], np.int32), want2), (dims, beta0, "batch")
    # what the reference cannot build answers NULL here too: no zero-point layout for address mode in this kernel, k % 8 != 0
    sh = X.libxsmm_create_gemm_shape(16, 16, 12, 16, 12, 16, I4X2, gen.U8, gen.I32, gen.I32)
    assert not X.libxsmm_dispatch_gemm(sh, cases.FLAG_VNNI_A | FLAG_INTLV_A | FLAG_COL_VEC_ZPT, 0)


def test_bitmap_compressed_a_bit_exact():
    """DECOMPRESS_A_VIA_BITMASK (reference :857-948): compressed A + bitmap in a.secondary; device and host operands"""
    import ctypes as C
    from test_oracle_vs_ref import FLAG_BITMASK_A, bitmap_case
    rng = np.random.default_rng(93)
    for ta, tb, tc in ((gen.F32, gen.F32, gen.F32), (gen.BF16, gen.BF16, gen.F32), (gen.BF16, gen.BF16, gen.BF16), (gen.F16, gen.F16, gen.F16)):
        for (m, n, k, pad) in ((32, 16, 32, 0), (16, 6, 8, 3), (64, 64, 64, 0), (128, 40, 256, 0)):
            for beta0 in (0, 1):
                dims, a, b, bitmap, c0 = bitmap_case(rng, m, n, k, ta, tb, tc, pad=pad)
                flags = (cases.FLAG_BETA_0 if beta0 else 0) | FLAG_BITMASK_A | (cases.FLAG_VNNI_A if ta != gen.F32 else 0)
                want = c0.copy()
                assert oracle["gemm_bitmap"](iarr(*dims), iarr(ta, tb, gen.F32, tc), flags, a.ctypes.data, b.ctypes.data, want.ctypes.data, bitmap.ctypes.data) == 0
                kern = X.libxsmm_dispatch_gemm(X.libxsmm_create_gemm_shape(*dims, ta, tb, tc, gen.F32), flags, 0)
                assert kern, (dims, ta)
                for resident in (1, 0):
                    if resident:
                        d_a, d_b, d_c, d_m = dev(a), dev(b), dev(c0), dev(bitmap)
                        pa, pb, pc, pm = d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), d_m.data_ptr()
                    else:
                        hc = c0.copy(); pa, pb, pc, pm = a.ctypes.data, b.ctypes.data, hc.ctypes.data, bitmap.ctypes.data
                    p = X.GemmParam()
                    p.a.primary, p.b.primary, p.c.primary, p.a.secondary = pa, pb, pc, pm
                    X.GEMMFUNCTION(kern)(C.byref(p)); X.check()
                    got = host(d_c, gen.NP_OF[tc]) if resident else hc
                    assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (dims, (ta, tb, tc), beta0, resident)


@pytest.mark.parametrize("types", [(gen.U8, gen.I8, gen.I32, gen.I32), (gen.I8, gen.U8, gen.I32, gen.I32), (gen.I8, gen.I8, gen.I32, gen.I32), (gen.U8, gen.U8, gen.I32, gen.I32),
                                   (gen.U8, gen.I8, gen.I32, gen.F32), (gen.BF16, gen.BF16, gen.F32, gen.F32), (gen.BF16, gen.BF16, gen.F32, gen.BF16),
                                   (gen.F16, gen.F16, gen.F32, gen.F16)])
def test_vnni_a_on_tensor_cores(types):
    """VNNI-packed A (the reference's canonical low-precision layout) as wgmma register fragments (gemm_tc.cu): int8 /
    16-bit. Integer tuples bit-exact against the oracle (integer sums are order-free), I8->F32 exact as well (one
    int->float conversion and one multiply), 16-bit tuples within the reference drivers' norms. Batches through the strided API."""
    rng = np.random.default_rng(97)
    ta, tb, tcomp, tc = types
    is8 = ta in (gen.I8, gen.U8)
    shapes = [(64, 64, 64, 3, 8, 0), (128, 128, 128, 0, 1, 0), (16, 16, 16, 0, 1, 0), (32, 48, 96, 3, 2, 16), (12, 20, 48 if is8 else 40, 0, 1, 0),
              (128, 64, 256 + 32, 3, 2, 0), (64, 128, 32, 0, 1, 0), (8, 8, 16, 0, 1, 0), (24, 16, 32, 3, 3, 0), (4, 32, 64, 0, 1, 0)]   # m <= 32: small tiles in an m64 instruction
    for (m, n, k, br_type, br, pad) in shapes:
        for beta0 in (1, 0):
            flags = (cases.FLAG_BETA_0 if beta0 else 0) | cases.FLAG_VNNI_A
            case = cases.GemmCase(m, n, k, ta, tb, tcomp, tc, flags=flags, br_type=br_type, br=br, pad=pad)
            count = 37
            ops = cases.Operands(case, seed=int(rng.integers(1 << 30)), count=count)
            kernel = dispatch(case, ops)
            assert kernel, case
            assert X.libxsmm_b200_kernel_backend(kernel) == X.BACKEND_TCGEN05, case
            d_a, d_b, d_c = dev(ops.a), dev(ops.b), dev(ops.c0)
            if tc == gen.F32 and is8:      # the scalar scale travels with the call: per-call path
                run_single_calls(kernel, case, ops, d_a, d_b, d_c)
            else:
                assert X.libxsmm_b200_gemm_batch_strided(kernel, d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), ops.tile_a, ops.tile_b, ops.tile_c, case.br, count) == 0
                X.check()
            want = cases.ref_result(oracle, case, ops, run_gemm)
            got = host(d_c, gen.NP_OF[tc])
            if is8:
                assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (case, beta0)
            else:
                thr = 1.2e-5 if tc == gen.F32 else 5e-3
                assert gen.normf_rel(gen.to_f64(want, tc), gen.to_f64(got, tc)) <= thr, (case, beta0)


@pytest.mark.parametrize("tc", [gen.F32, gen.BF16])
def test_address_mode_pool_on_tensor_cores(tc):
    """ADDRESS batch-reduce whose pointers walk a pool of block-sets (mode R of the benchmark): the plan recognises the pool and
    runs the tensor-core kernel (set index = tensor-map coordinate, tiles visited sorted by set pair, two tiles that share B
    in one item). Every tile against the oracle called exactly like the reference (pointer arrays)."""
    rng = np.random.default_rng(98)
    for (m, n, k, br, nsets, count) in ((64, 64, 64, 8, 5, 300), (32, 48, 64, 2, 3, 41), (128, 64, 128, 3, 4, 57), (64, 64, 64, 1, 2, 9),
                                        (64, 64, 64, 2, 7, 3001), (48, 80, 96, 2, 6, 2000)):   # many items per CTA: set changes, buffer swaps, odd tails
        case = cases.GemmCase(m, n, k, gen.BF16, gen.BF16, gen.F32, tc, flags=cases.FLAG_BETA_0, br_type=1, br=br)
        blk_a, blk_b = m * k * 2, k * n * 2
        pool_a = gen.values(rng, nsets * br * m * k, gen.BF16); pool_b = gen.values(rng, nsets * br * k * n, gen.BF16)
        c0 = gen.values(rng, count * m * n, tc)
        sa = rng.integers(0, nsets, size=count); sb = rng.integers(0, nsets, size=count)
        kernel = dispatch(case, None)
        assert kernel
        d_a, d_b, d_c = dev(pool_a), dev(pool_b), dev(c0)
        params = (X.GemmParam * count)(); keep = []
        tsc = gen.TS[tc]
        for t in range(count):
            aa = (C.c_void_p * br)(*[d_a.data_ptr() + (int(sa[t]) * br + r) * blk_a for r in range(br)])
            ab = (C.c_void_p * br)(*[d_b.data_ptr() + (int(sb[t]) * br + r) * blk_b for r in range(br)])
            brv = C.c_ulonglong(br); keep += [aa, ab, brv]
            params[t].op.tertiary = C.addressof(brv)
            params[t].a.primary, params[t].b.primary = C.addressof(aa), C.addressof(ab)
            params[t].c.primary = d_c.data_ptr() + t * m * n * tsc
        plan = X.libxsmm_b200_gemm_plan_create(kernel, params, count)
        assert plan and X.libxsmm_b200_gemm_plan_is_pooled(plan) == 1, (m, n, k, br)
        for rep in range(2):
            assert X.libxsmm_b200_gemm_plan_run(plan) == 0
            X.check()
        got = host(d_c, gen.NP_OF[tc])
        want = c0.copy()
        for t in range(count):
            ha = (C.c_void_p * br)(*[pool_a.ctypes.data + (int(sa[t]) * br + r) * blk_a for r in range(br)])
            hb = (C.c_void_p * br)(*[pool_b.ctypes.data + (int(sb[t]) * br + r) * blk_b for r in range(br)])
            cv = want[t * m * n:(t + 1) * m * n]
            assert run_gemm(oracle, case.dims, case.types, case.flags, 1, 0, 0, br, ha, hb, cv) == 0
        thr = 1.2e-5 if tc == gen.F32 else 5e-3
        assert gen.normf_rel(gen.to_f64(want, tc), gen.to_f64(got, tc)) <= thr, (m, n, k, br, tc)
        X.libxsmm_b200_gemm_plan_destroy(plan)


def test_offset_mode_pool_on_tensor_cores():
    """OFFSET batch-reduce (block r = a.primary + a.secondary[r]) over the same kind of operand pool: recognised by the plan like the
    ADDRESS form and run by the tensor-core kernel"""
    rng = np.random.default_rng(99)
    tc = gen.BF16
    for (m, n, k, br, nsets, count) in ((64, 64, 64, 4, 4, 777), (32, 32, 128, 2, 3, 50)):
        case = cases.GemmCase(m, n, k, gen.BF16, gen.BF16, gen.F32, tc, flags=cases.FLAG_BETA_0, br_type=2, br=br)
        blk_a, blk_b = m * k * 2, k * n * 2
        pool_a = gen.values(rng, nsets * br * m * k, gen.BF16); pool_b = gen.values(rng, nsets * br * k * n, gen.BF16)
        c0 = gen.values(rng, count * m * n, tc)
        sa = rng.integers(0, nsets, size=count); sb = rng.integers(0, nsets, size=count)
        kernel = dispatch(case, None)
        assert kernel
        d_a, d_b, d_c = dev(pool_a), dev(pool_b), dev(c0)
        offs_a = (C.c_ulonglong * br)(*[r * blk_a for r in range(br)]); offs_b = (C.c_ulonglong * br)(*[r * blk_b for r in range(br)])
        brv = C.c_ulonglong(br)
        params = (X.GemmParam * count)()
        for t in range(count):
            params[t].op.tertiary = C.addressof(brv)
            params[t].a.primary = d_a.data_ptr() + int(sa[t]) * br * blk_a; params[t].a.secondary = C.addressof(offs_a)
            params[t].b.primary = d_b.data_ptr() + int(sb[t]) * br * blk_b; params[t].b.secondary = C.addressof(offs_b)
            params[t].c.primary = d_c.data_ptr() + t * m * n * gen.TS[tc]
        plan = X.libxsmm_b200_gemm_plan_create(kernel, params, count)
        assert plan and X.libxsmm_b200_gemm_plan_is_pooled(plan) == 1, (m, n, k, br)
        assert X.libxsmm_b200_gemm_plan_run(plan) == 0
        X.check()
        got = host(d_c, gen.NP_OF[tc])
        want = c0.copy()
        for t in range(count):
            ha = (C.c_void_p * br)(*[pool_a.ctypes.data + (int(sa[t]) * br + r) * blk_a for r in range(br)])
            hb = (C.c_void_p * br)(*[pool_b.ctypes.data + (int(sb[t]) * br + r) * blk_b for r in range(br)])
            cv = want[t * m * n:(t + 1) * m * n]
            assert run_gemm(oracle, case.dims, case.types, case.flags, 1, 0, 0, br, ha, hb, cv) == 0     # same blocks through the ADDRESS form of the oracle
        assert gen.normf_rel(gen.to_f64(want, tc), gen.to_f64(got, tc)) <= 5e-3, (m, n, k, br)
        X.libxsmm_b200_gemm_plan_destroy(plan)


def test_multi_device_strided_batch_from_host_buffers():
    """libxsmm_b200_gemm_batch_strided_multi: a host-resident strided batch cut into one contiguous range per device (all visible GPUs,
    one worker thread and stream each). On a one-GPU box this is the ndevices = 1 path."""
    import torch
    ndev = max(1, min(4, torch.cuda.device_count()))
    rng = np.random.default_rng(100)
    case = cases.GemmCase(64, 64, 64, gen.BF16, gen.BF16, gen.F32, gen.F32, flags=cases.FLAG_BETA_0, br_type=3, br=2)
    count = 1001
    ops = cases.Operands(case, seed=int(rng.integers(1 << 30)), count=count)
    kernel = dispatch(case, ops)
    assert kernel
    a, b, c = ops.a.copy(), ops.b.copy(), ops.c0.copy()
    rc = X.libxsmm_b200_gemm_batch_strided_multi(kernel, a.ctypes.data, b.ctypes.data, c.ctypes.data, ops.tile_a, ops.tile_b, ops.tile_c, case.br, count, ndev)
    assert rc == 0, X.libxsmm_b200_last_error_string()
    want = cases.ref_result(oracle, case, ops, run_gemm)
    assert gen.normf_rel(want, c) <= 1.2e-5, ndev
