"""CPU-only: pins oracle/oracle.c (the restatement) against the UNMODIFIED reference built from
/root/reference (oracle/_ref/libxsmm_ref.so) on seeded inputs -- bit for bit -- and against the
reference's JIT path (AMX/AVX-512 on this host) within the reference's own acceptance norms."""
import ctypes as C

import numpy as np
import pytest

import cases
import gen
from oracle_ffi import iarr, oracle, ref, run_gemm

needs_ref = pytest.mark.skipif(ref is None, reason="oracle/_ref/libxsmm_ref.so not built (no /root/reference here)")


def _cpu_flags():
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("flags"):
                    return set(line.split(":", 1)[1].split())
    except OSError:
        pass
    return set()


CPU_FLAGS = _cpu_flags()
# the reference JIT fuses multiply and add only where the host has FMA, and runs C-sparse on 16 lanes only with AVX-512; the oracle
# states that path (oracle/oracle.c), so elsewhere the two are not expected to agree bit for bit
needs_fma = pytest.mark.skipif("fma" not in CPU_FLAGS, reason="host without FMA: the reference JIT rounds product and sum separately")


@needs_ref
def test_conversions_match_reference():
    rng = np.random.default_rng(1)
    bits = np.concatenate([rng.integers(0, 2**32, size=20000, dtype=np.uint64).astype(np.uint32),
                           np.array([0, 0x80000000, 0x7f800000, 0xff800000, 0x7fc00000, 0x7f800001, 0x00000001, 0x007fffff,
                                     0x38800000, 0x387fffff, 0x33000000, 0x33000001, 0x477fe000, 0x477ff000, 0x47800000], dtype=np.uint32)])
    for u in bits:
        f = float(np.array([u], dtype=np.uint32).view(np.float32)[0])
        assert oracle["f32_to_bf16"](f) == ref["f32_to_bf16"](f), hex(u)
        assert oracle["f32_to_f16"](f) == ref["f32_to_f16"](f), hex(u)
    for h in range(0, 65536, 7):
        a, b = oracle["f16_to_f32"](h), ref["f16_to_f32"](h)
        assert (a == b) or (a != a and b != b), h
        a, b = oracle["bf16_to_f32"](h), ref["bf16_to_f32"](h)
        assert (a == b) or (a != a and b != b), h


@needs_ref
def test_gemm_restatement_is_bit_exact():
    n = 0
    for case in cases.small_cases():
        ops = cases.Operands(case, seed=555 + n)
        want = cases.ref_result(ref, case, ops, run_gemm)
        got = cases.ref_result(oracle, case, ops, run_gemm)
        assert np.array_equal(want.view(np.uint8), got.view(np.uint8)), case
        n += 1
    assert n > 300


@needs_ref
def test_reference_jit_agrees_with_reference_kernel():
    """the JIT'ed x86 kernels (the CPU baseline) against the C kernel, reference thresholds (gemm_kernel.c:5312-5414)"""
    for t, thr in (((gen.F32, gen.F32, gen.F32, gen.F32), 1.2e-5), ((gen.BF16, gen.BF16, gen.F32, gen.F32), 1.2e-5),
                   ((gen.BF16, gen.BF16, gen.F32, gen.BF16), 5e-3), ((gen.U8, gen.I8, gen.I32, gen.I32), 0.0)):
        flags = cases.FLAG_BETA_0 | (cases.FLAG_VNNI_A if t[0] != gen.F32 else 0)
        case = cases.GemmCase(64, 64, 64, *t, flags=flags, br_type=3, br=8)
        ops = cases.Operands(case)
        c_ref = ops.c0.copy(); c_jit = ops.c0.copy()
        assert run_gemm(ref, case.dims, case.types, case.flags, 3, ops.stride_a, ops.stride_b, 8, ops.a, ops.b, c_ref, mode=0) == 0
        rc = run_gemm(ref, case.dims, case.types, case.flags, 3, ops.stride_a, ops.stride_b, 8, ops.a, ops.b, c_jit, mode=1)
        assert rc in (0, 2)
        assert gen.normf_rel(gen.to_f64(c_ref, t[3]), gen.to_f64(c_jit, t[3])) <= thr


@needs_ref
def test_int8_full_range_restatement_is_bit_exact():
    """U8 in [0, 255] and I8 in [-128, 127] in all four sign combinations (gen.values stays within +-20), VNNI4 and flat A, I32 C over the
    whole int32 range (beta = 1 wraps) and the scaled F32 C; plus one U8 x U8 case of 255s whose sums pass 2^31 and wrap"""
    rng = np.random.default_rng(23)
    for ta, tb in ((gen.U8, gen.U8), (gen.U8, gen.I8), (gen.I8, gen.U8), (gen.I8, gen.I8)):
        for tc, vnni in ((gen.I32, 1), (gen.I32, 0), (gen.F32, 1)):
            for beta0 in (0, 1):
                flags = (cases.FLAG_BETA_0 if beta0 else 0) | (cases.FLAG_VNNI_A if vnni else 0)
                case = cases.GemmCase(24, 13, 36, ta, tb, gen.I32, tc, flags=flags, br_type=3, br=3, pad=2)
                ops = cases.Operands(case, seed=int(rng.integers(1 << 30)), count=2)
                ops.a = rng.integers(-128 if ta == gen.I8 else 0, 128 if ta == gen.I8 else 256, size=ops.a.size).astype(gen.NP_OF[ta])
                ops.b = rng.integers(-128 if tb == gen.I8 else 0, 128 if tb == gen.I8 else 256, size=ops.b.size).astype(gen.NP_OF[tb])
                if tc == gen.I32:
                    ops.c0 = rng.integers(-2 ** 31, 2 ** 31, size=ops.c0.size).astype(np.int32)
                want = cases.ref_result(ref, case, ops, run_gemm)
                got = cases.ref_result(oracle, case, ops, run_gemm)
                assert np.array_equal(want.view(np.uint8), got.view(np.uint8)), case
    case = cases.GemmCase(16, 4, 1024, gen.U8, gen.U8, gen.I32, gen.I32, flags=cases.FLAG_BETA_0 | cases.FLAG_VNNI_A, br_type=3, br=36)
    ops = cases.Operands(case, count=1)
    ops.a[:] = 255; ops.b[:] = 255
    want = cases.ref_result(ref, case, ops, run_gemm)
    assert np.all(want == np.int32(255 * 255 * 1024 * 36 - 2 ** 32)), "255^2 * 36864 wraps to a negative int32"
    assert np.array_equal(want, cases.ref_result(oracle, case, ops, run_gemm))


def _bcsc_inputs(rng, ta, tb, tc, mblocks, M, K, N, bk, bn, density, vnni_a=True, trans_a=False):
    nbr, nbc = K // bk, N // bn
    keep = rng.random((nbc, nbr)) < density
    colptr = np.zeros(nbc + 1, dtype=np.uint32); rowidx = []
    for j in range(nbc):
        rows = np.nonzero(keep[j])[0]
        rowidx.extend(rows.tolist()); colptr[j + 1] = len(rowidx)
    rowidx = np.array(rowidx if rowidx else [0], dtype=np.uint32)
    nnzb = int(colptr[-1])
    bvals = gen.values(rng, max(nnzb, 1) * bk * bn, tb)
    a = gen.values(rng, mblocks * K * M, ta)
    c0 = gen.values(rng, mblocks * N * M, tc)
    return a, bvals, colptr, rowidx, c0


def _run_bcsc(side, types, geo, flags, a, bvals, colptr, rowidx, c):
    from oracle_ffi import iarr
    return side["bcsc"](iarr(*types), iarr(*geo), flags, a.ctypes.data, bvals.ctypes.data, colptr.ctypes.data, rowidx.ctypes.data, c.ctypes.data)


@needs_ref
@needs_fma
def test_bcsc_oracle_matches_reference_jit():
    """no portable C kernel exists for BCSC in the reference (no fallback for this build kind): the x86 JIT is the second opinion.
    f32 accumulates in the same order with one FMA per product (VFMADD231PS), so it agrees bit for bit, like the integer paths; bf16
    runs through the JIT's dot-product instructions, which pair k differently (the reference drivers' norm)."""
    rng = np.random.default_rng(3)
    for (ta, tb, tcomp, tc), thr in (((gen.F32, gen.F32, gen.F32, gen.F32), 0.0), ((gen.BF16, gen.BF16, gen.F32, gen.BF16), 5e-3),
                                      ((gen.U8, gen.I8, gen.I32, gen.I32), 0.0), ((gen.I8, gen.U8, gen.I32, gen.I32), 0.0)):
        for beta0 in (1, 0):
            mblocks, M, K, N, bk, bn = 3, 32, 128, 64, 32 if ta != gen.F32 else 16, 16
            flags = (cases.FLAG_BETA_0 if beta0 else 0) | (cases.FLAG_VNNI_A if ta != gen.F32 else 0)
            a, bvals, colptr, rowidx, c0 = _bcsc_inputs(rng, ta, tb, tc, mblocks, M, K, N, bk, bn, 0.5)
            geo = (mblocks, M, K, N, bk, bn)
            c_o, c_r = c0.copy(), c0.copy()
            assert _run_bcsc(oracle, (ta, tb, tcomp, tc), geo, flags, a, bvals, colptr, rowidx, c_o) == 0
            rc = _run_bcsc(ref, (ta, tb, tcomp, tc), geo, flags, a, bvals, colptr, rowidx, c_r)
            if rc != 0:
                pytest.skip("reference JIT cannot build BCSC for this host ISA")
            if thr == 0.0:
                assert np.array_equal(c_r.view(np.uint8), c_o.view(np.uint8)), ((ta, tb, tc), beta0)
            else:
                err = gen.normf_rel(gen.to_f64(c_r, tc), gen.to_f64(c_o, tc))
                assert err <= thr, ((ta, tb, tc), beta0, err)


@needs_ref
def test_bcsc_trans_a_oracle_matches_reference_jit():
    """f32 BCSC with TRANS_A (the reference's AT_CT kernel): A read as [M][K], C written as [M][N], like the reference driver's gold
    (samples/xgemm_sparse/spmm_kernel.c:92-101) and the oracle. The JIT places k across vector lanes and reduces horizontally at
    the end, while the oracle sums k in ascending order, so elements differ in their last bits; where the ascending sum cancels to
    exactly zero, the JIT's residual makes the relative error look huge. What must hold is the layout: every element within
    4 ulp-of-1 of sum_k |a||b| + |c0| of the oracle, with dense, sparse and empty block columns, beta 0 and 1."""
    rng = np.random.default_rng(8)
    T = (gen.F32,) * 4
    eps = float(np.finfo(np.float32).eps)
    for geo, dens in (((1, 16, 32, 32, 16, 16), 0.5), ((1, 32, 64, 64, 16, 16), 0.5), ((3, 32, 128, 64, 16, 16), 0.5), ((1, 5, 7, 6, 1, 2), 0.6),
                      ((2, 16, 32, 32, 4, 4), 0.4), ((1, 13, 48, 32, 16, 8), 0.5), ((2, 8, 32, 32, 16, 16), 1.0)):
        for beta0 in (1, 0):
            mblocks, M, K, N, bk, bn = geo
            flags = (cases.FLAG_BETA_0 if beta0 else 0) | cases.FLAG_TRANS_A
            a, bvals, colptr, rowidx, c0 = _bcsc_inputs(rng, gen.F32, gen.F32, gen.F32, mblocks, M, K, N, bk, bn, dens)
            c_o, c_r, c_abs = c0.copy(), c0.copy(), np.abs(c0)
            assert _run_bcsc(oracle, T, geo, flags, a, bvals, colptr, rowidx, c_o) == 0
            if _run_bcsc(ref, T, geo, flags, a, bvals, colptr, rowidx, c_r) != 0:
                pytest.skip("reference JIT cannot build BCSC for this host ISA")
            assert _run_bcsc(oracle, T, geo, flags, np.abs(a), np.abs(bvals), colptr, rowidx, c_abs) == 0
            bound = 4 * eps * c_abs.astype(np.float64)
            assert np.all(np.abs(c_r.astype(np.float64) - c_o) <= bound), (geo, beta0)


@needs_ref
def test_fsspmdm_oracle_matches_reference():
    rng = np.random.default_rng(4)
    for dtype, eps in ((gen.F32, 1e-4), (gen.F64, 1e-8)):
        for beta in (0.0, 1.0):
            M, K, N = 24, 40, 96
            npdt = gen.NP_OF[dtype]
            a = (gen.values(rng, M * K, gen.F64) * (rng.random(M * K) < 0.2)).astype(npdt)
            b = gen.values(rng, K * N, dtype); c0 = gen.values(rng, M * N, dtype)
            alpha = np.array([1.5], dtype=npdt); bt = np.array([beta], dtype=npdt)
            c_o, c_r = c0.copy(), c0.copy()
            args = (dtype, M, N, K, K, N, N, alpha.ctypes.data, bt.ctypes.data, a.ctypes.data, b.ctypes.data)
            assert oracle["fsspmdm"](*args, c_o.ctypes.data) == 0
            assert ref["fsspmdm"](*args, c_r.ctypes.data) == 0
            assert gen.normf_rel(c_r, c_o) <= eps
    # invalid inputs answer "no handle" on both sides (N not a multiple of the vector length, beta=2, empty A)
    M, K, N = 8, 8, 24
    a = np.ones(M * K, dtype=np.float32); b = np.ones(K * N, dtype=np.float32); c = np.zeros(M * N, dtype=np.float32)
    one = np.array([1.0], dtype=np.float32); two = np.array([2.0], dtype=np.float32)
    for side in (oracle, ref):
        assert side["fsspmdm"](gen.F32, M, N, K, K, N, N, one.ctypes.data, one.ctypes.data, a.ctypes.data, b.ctypes.data, c.ctypes.data) != 0
        assert side["fsspmdm"](gen.F32, M, 32, K, K, 32, 32, one.ctypes.data, two.ctypes.data, a.ctypes.data, b.ctypes.data, c.ctypes.data) != 0
        z = np.zeros(M * K, dtype=np.float32)
        assert side["fsspmdm"](gen.F32, M, 32, K, K, 32, 32, one.ctypes.data, one.ctypes.data, z.ctypes.data, b.ctypes.data, c.ctypes.data) != 0


@needs_ref
@pytest.mark.parametrize("dtype", [gen.F32, gen.F64])
def test_fsspmdm_oracle_is_bit_exact_on_exact_operands(dtype):
    """Family E of tests/test_fsspmdm_exact_gpu.py (cases.fsspmdm_exact_operands: every partial sum exact), on which the GPU kernels are
    compared with oracle["fsspmdm"] bit for bit: the oracle, the reference and the float64 product must agree exactly, every alpha of the
    family, beta 0 and 1, rows with 0 to 9 non-zeros. Zeros compare by value (the reference's dense kernel may produce -0)."""
    rng = np.random.default_rng(6)
    npdt = gen.NP_OF[dtype]
    M, K, N = 24, 40, 96
    for alpha in cases.FSSPMDM_EXACT_ALPHAS:
        for beta in (0.0, 1.0):
            mask = cases.fsspmdm_pattern(rng, M, K, row_nnz=[(3 + 7 * i) % 10 for i in range(M)])
            a, b, c0 = cases.fsspmdm_exact_operands(rng, dtype, mask, N, N, N, alpha)
            al, bt = np.array([alpha], dtype=npdt), np.array([beta], dtype=npdt)
            args = (dtype, M, N, K, K, N, N, al.ctypes.data, bt.ctypes.data, a.ctypes.data, b.ctypes.data)
            c_o, c_r = c0.copy(), c0.copy()
            assert oracle["fsspmdm"](*args, c_o.ctypes.data) == 0
            assert ref["fsspmdm"](*args, c_r.ctypes.data) == 0
            exact, _ = cases.fsspmdm_reference(cases.fsspmdm_fold(dtype, a, alpha), b, c0, N, beta)
            assert np.array_equal(c_r, exact.astype(npdt)), (alpha, beta, "reference vs float64")
            assert np.array_equal(c_o, c_r), (alpha, beta, "oracle vs reference")


@needs_ref
@needs_fma
@pytest.mark.parametrize("kind", ["a_csr", "b_csr", "b_csc", "c_csc"])
def test_packed_sparse_oracle_matches_reference_jit(kind):
    """oracle_packed_sp (restated driver golds, samples/xgemm_norm_packed/*.c, one FMA per product) against the reference's own JIT
    of libxsmm_create_packed_spgemm_csr/_csc (src/libxsmm_main.c:3553-3638) -- EDGE sizes and P = 13, f32/f64, beta 0/1, bit for bit."""
    rng = np.random.default_rng(77)
    ran = 0
    if kind == "c_csc" and "avx512f" not in CPU_FLAGS:
        pytest.skip("host without AVX-512: the reference's C-sparse kernel runs 8 lanes, the oracle states the 16-lane schedule")
    for dtype in (gen.F32, gen.F64):
        for (M, N, K, P) in ((9, 9, 9, 8), (20, 9, 35, 16), (56, 9, 56, 64), (35, 20, 9, 16), (6, 5, 7, 13), (35, 20, 9, 48)):
            for beta0 in (0, 1):
                is_csc, dims, ptr, idx, a, b, c0 = cases.packed_sp_case(rng, kind, dtype, M, N, K, P)
                flags = cases.FLAG_BETA_0 if beta0 else 0
                vals = a if kind == "a_csr" else b if kind.startswith("b_") else c0
                c_o, c_r = c0.copy(), c0.copy()
                args = (is_csc, dtype, iarr(*dims), flags, P, ptr.ctypes.data, idx.ctypes.data, vals.ctypes.data, a.ctypes.data, b.ctypes.data)
                rc_o = oracle["packed_sp"](*args, c_o.ctypes.data)
                rc = ref["packed_sp"](*args, c_r.ctypes.data)
                if kind == "c_csc" and (dtype != gen.F32 or P % 16):
                    assert rc_o != 0          # C-sparse exists for f32 and whole 16-lane vectors only
                    continue
                assert rc_o == 0
                if rc != 0:
                    continue          # the JIT declines this (kind, precision, width) on this host
                if kind == "c_csc" and beta0:
                    continue          # reference defect: with BETA_0 the 16-accumulator path stores zmm1 while the sums sit in
                                      # zmm0 (..._csc_csparse_avx_avx2_avx512.c:567-590); the oracle overwrites as documented
                ran += 1
                assert np.array_equal(c_r.view(np.uint8), c_o.view(np.uint8)), (kind, dtype, (M, N, K, P), beta0)
    assert ran > 0, "the reference JIT built none of the cases"


@needs_ref
@pytest.mark.parametrize("types", [(gen.F32, gen.F32, gen.F32, gen.F32), (gen.BF16, gen.BF16, gen.F32, gen.BF16), (gen.BF16, gen.BF16, gen.F32, gen.F32),
                                   (gen.F16, gen.F16, gen.F32, gen.F16), (gen.U8, gen.I8, gen.I32, gen.F32)])
def test_fused_gemm_restatement_matches_reference(types):
    """oracle_gemm_ext against libxsmm_reference_gemm on the extended ABI: column-bias pre-op, ReLU (+bitmask) / sigmoid post-op,
    VNNI-packed C (generator_gemm_reference_impl.c:255-372, 2803-2842) -- bit for bit (same libm on the same host).
    int8 -> f32 reads A as VNNI4 (every k here is a multiple of 4) and scales the product by c.tertiary."""
    rng = np.random.default_rng(88)
    ta, tb, tcomp, tc = types
    for (m, n, k, pad) in ((32, 16, 32, 0), (13, 6, 8, 3), (64, 64, 64, 0)):
        for beta0 in (1, 0):
            for br_type, br in ((0, 1), (3, 3)):
                for fuse in cases.fused_variants():
                    if fuse[3] and (tc == gen.F32 or n % 2):
                        continue
                    vnni_a = ta in (gen.I8, gen.U8) or (ta != gen.F32 and k % 2 == 0 and m % 2 == 0)
                    flags = (cases.FLAG_BETA_0 if beta0 else 0) | (cases.FLAG_VNNI_A if vnni_a else 0)
                    case = cases.GemmCase(m, n, k, ta, tb, tcomp, tc, flags=flags, br_type=br_type, br=br, pad=pad)
                    ops = cases.Operands(case, seed=int(rng.integers(1 << 30)))
                    bias = gen.values(rng, m, tc)
                    mask0 = rng.integers(0, 256, size=((case.ldc + 15) // 16 * 16) // 8 * n + 8, dtype=np.uint8)
                    outs = []
                    for side in (ref, oracle):
                        c = ops.c0.copy(); mk = mask0.copy()
                        assert cases.run_gemm_ext(side, case, ops, fuse, bias if fuse[0] else None, mk if fuse[2] else None, c) == 0, (case, fuse)
                        outs.append((c, mk))
                    assert np.array_equal(outs[0][0].view(np.uint8), outs[1][0].view(np.uint8)), (case, fuse)
                    assert np.array_equal(outs[0][1], outs[1][1]), (case, fuse, "mask")


I4X2 = 18
FLAG_COL_VEC_ZPT, FLAG_INTLV_A, FLAG_BITMASK_A, FLAG_MXK_ZPT = 131072, 262144, 524288, 1048576


def int4_case(rng, m, n, k, br, pad=0):
    lda, ldb, ldc = m + pad, k + pad, m + pad
    blk_a, blk_b = (k // 8) * lda * 4, n * ldb
    a = rng.integers(0, 256, size=blk_a * br, dtype=np.uint8)
    b = rng.integers(0, 256, size=blk_b * br, dtype=np.uint8)
    zpt = rng.integers(0, 16, size=max(m, (blk_a * 2 // k) * br + m), dtype=np.uint8)
    c0 = rng.integers(-1000, 1000, size=n * ldc).astype(np.int32)
    return (m, n, k, lda, ldb, ldc), a, b, zpt, c0, blk_a, blk_b


@needs_ref
def test_int4_gemm_restatement_is_bit_exact():
    """U4 x U8 -> I32 with zero points (reference :1273-1321): plain and stride batch-reduce, beta 0/1"""
    rng = np.random.default_rng(90)
    for (m, n, k, pad) in ((32, 16, 32, 0), (13, 6, 8, 3), (64, 64, 64, 0), (5, 3, 16, 1)):
        for br_type, br in ((0, 1), (3, 4)):
            for beta0 in (0, 1):
                dims, a, b, zpt, c0, blk_a, blk_b = int4_case(rng, m, n, k, br, pad)
                flags = (cases.FLAG_BETA_0 if beta0 else 0) | cases.FLAG_VNNI_A | FLAG_INTLV_A | (FLAG_MXK_ZPT if br_type else FLAG_COL_VEC_ZPT)
                c_o, c_r = c0.copy(), c0.copy()
                assert oracle["gemm_i4"](iarr(*dims), flags, br_type, blk_a, blk_b, br, a.ctypes.data, b.ctypes.data, c_o.ctypes.data, zpt.ctypes.data) == 0
                assert ref["gemm_aux"](iarr(*dims), iarr(I4X2, gen.U8, gen.I32, gen.I32), flags, br_type, blk_a, blk_b, br, a.ctypes.data, b.ctypes.data,
                                       c_r.ctypes.data, 1, zpt.ctypes.data) == 0
                assert np.array_equal(c_o, c_r), (dims, br_type, beta0)


def bitmap_case(rng, m, n, k, ta, tb, tc, density=0.4, pad=0):
    kb = 1 if ta == gen.F32 else 2
    ldb, ldc = k + pad, m + pad
    bits = rng.random((k // kb) * m * kb) < density
    bitmap = np.packbits(bits, bitorder="little")
    bitmap = np.concatenate([bitmap, np.zeros(8, dtype=np.uint8)])
    a = gen.values(rng, int(bits.sum()) + 4, ta)
    b = gen.values(rng, n * ldb, tb); c0 = gen.values(rng, n * ldc, tc)
    return (m, n, k, m, ldb, ldc), a, b, bitmap, c0


@needs_ref
def test_bitmap_sparse_a_restatement_is_bit_exact():
    """bitmap-compressed A (DECOMPRESS_A_VIA_BITMASK, reference :857-948): F32 and 16-bit operands, beta 0/1"""
    rng = np.random.default_rng(91)
    for ta, tb, tc in ((gen.F32, gen.F32, gen.F32), (gen.BF16, gen.BF16, gen.F32), (gen.BF16, gen.BF16, gen.BF16), (gen.F16, gen.F16, gen.F16)):
        for (m, n, k, pad) in ((32, 16, 32, 0), (16, 6, 8, 3), (64, 64, 64, 0)):
            for beta0 in (0, 1):
                dims, a, b, bitmap, c0 = bitmap_case(rng, m, n, k, ta, tb, tc, pad=pad)
                flags = (cases.FLAG_BETA_0 if beta0 else 0) | FLAG_BITMASK_A | (cases.FLAG_VNNI_A if ta != gen.F32 else 0)
                c_o, c_r = c0.copy(), c0.copy()
                assert oracle["gemm_bitmap"](iarr(*dims), iarr(ta, tb, gen.F32, tc), flags, a.ctypes.data, b.ctypes.data, c_o.ctypes.data, bitmap.ctypes.data) == 0
                assert ref["gemm_aux"](iarr(*dims), iarr(ta, tb, gen.F32, tc), flags, 0, 0, 0, 1, a.ctypes.data, b.ctypes.data, c_r.ctypes.data, 2, bitmap.ctypes.data) == 0
                assert np.array_equal(c_o.view(np.uint8), c_r.view(np.uint8)), (dims, (ta, tb, tc), beta0)


@needs_ref
@needs_fma
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_packed_dense_oracle_matches_reference_jit(kind):
    """libxsmm_create_packed_gemm / _ac_rm / _bc_rm (include/libxsmm.h:195-214): restated driver golds (one FMA per product, k
    ascending) against the reference JIT, bit for bit, padded leading dimensions included"""
    rng = np.random.default_rng(94)
    ran = 0
    for dtype in (gen.F32, gen.F64):
        for (M, N, K, P, pad) in ((9, 9, 9, 8, 0), (20, 9, 35, 16, 0), (56, 9, 56, 16, 0), (4, 3, 5, 8, 0), (16, 16, 16, 8, 0), (9, 7, 11, 16, 3)):
            if dtype == gen.F32 and P == 8:
                P = 16
            for beta0 in (0, 1):
                dims, a, b, c0 = cases.packed_dense_case(rng, kind, dtype, M, N, K, P, pad)
                flags = cases.FLAG_BETA_0 if beta0 else 0
                c_o, c_r = c0.copy(), c0.copy()
                assert oracle["packed_dense"](kind, dtype, iarr(*dims), flags, P, a.ctypes.data, b.ctypes.data, c_o.ctypes.data) == 0
                if ref["packed_dense"](kind, dtype, iarr(*dims), flags, P, a.ctypes.data, b.ctypes.data, c_r.ctypes.data) != 0:
                    continue
                ran += 1
                assert np.array_equal(c_r.view(np.uint8), c_o.view(np.uint8)), (kind, dtype, dims, P, beta0)
    assert ran > 0, "the reference JIT built none of the cases"
