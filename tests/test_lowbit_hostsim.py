"""Low-bit weight GEMM through the host half of the library on the simulated device: the host_*.c objects, tests/c/hostsim_runtime.c
and tests/c/hostsim_lowbit.c (low-bit tiles answered by oracle/oracle_lowbit.c) linked into tests/c/_hostsim/lowbit/libxsmm.so. What this
checks is the host code: dispatch of the forms the reference's driver uses, staging of pageable A / B / C and of the MXFP4 block scales
(address mode: arrays of pointers), the copy back of C, the batch forms' per-tile scales, and the missing-scale error. The reference's
unmodified samples/xgemm/gemm_kernel.c (oracle/ref_drivers.py) runs against it for the six tuples with nobr, strdbr, addrbr and offsbr
and must pass by its own verdict."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import lowbit_ffi  # noqa: F401  (builds oracle/liboracle.so and oracle/liboracle_lowbit.so)
from lowbit_ffi import BF16, F32, I1, I2, I8, I32, MXFP4, U8, LbCase, oracle_gemm_lowbit, same_c
from test_hostsim import CSRC, DRV, HOST_C, ORACLE, ROOT

OUT = os.path.join(ROOT, "tests", "c", "_hostsim", "lowbit")


def build_sim_lowbit():
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, "libxsmm.so")
    srcs = [os.path.join(CSRC, f) for f in HOST_C] + [os.path.join(ROOT, "tests", "c", f) for f in ("hostsim_runtime.c", "hostsim_lowbit.c")]
    deps = srcs + [os.path.join(CSRC, "xb_internal.h")]
    if os.path.exists(so) and all(os.path.getmtime(s) < os.path.getmtime(so) for s in deps):
        return so
    cmd = ["gcc", "-O1", "-std=gnu99", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-Wl,--wrap=xb_gemm_simt_launch", "-o", so] + \
        srcs + ["-L" + ORACLE, "-loracle_lowbit", "-loracle", "-Wl,-rpath," + ORACLE, "-lpthread", "-ldl", "-lm"]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    return so


# samples/xgemm/gemm_kernel.c: A B Comp C  M N K LDA LDB LDC  alpha beta  alignA alignC  trA trB  vnniA vnniB vnniC  prefetch  br-kind br-count
# br-unroll  reps  tilecfg. The driver sets VNNI_A (and INTLV_A_FORMAT for I2 / MXFP4) itself, and packs its I2 operand in the
# reference's layout for m = 32 and m = 64 only. ldb is a multiple of 32: the driver's gold places B's MXFP4 scales of block r at
# r * (ldb/32) * n floats, the reference at r * stride_b / 32, and the two agree only then.
def driver_args(types, br):
    beta = 0 if br in ("strdbr", "offsbr") else 1
    return tuple(types.split()) + (64, 24, 64, 72, 96, 68, 1, beta, 0, 0, 0, 0, 0, 0, 0, "nopf", br, 1 if br == "nobr" else 3, 0, 3, 0)


TYPES = ["I2 I8 I32 I32", "I2 U8 I32 I32", "I1 I8 I32 I32", "I1 U8 I32 I32", "MXFP4 I8 I32 F32", "MXFP4 I8 I32 BF16"]
BRS = ["nobr", "strdbr", "addrbr", "offsbr"]


@pytest.mark.parametrize("br", BRS)
@pytest.mark.parametrize("types", TYPES, ids=lambda t: t.replace(" ", "_"))
def test_reference_gemm_kernel_driver_against_the_simulated_device(types, br):
    exe = os.path.join(DRV, "gemm_kernel")
    if not os.path.exists(exe):
        pytest.skip("gemm_kernel was not prebuilt (no reference tree in the build container?)")
    build_sim_lowbit()
    args = driver_args(types, br)
    env = dict(os.environ, LD_LIBRARY_PATH=OUT + ":" + ORACLE + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="2")
    p = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=300, env=env, cwd=DRV)
    assert p.returncode == 0, (args, p.stdout[-1500:], p.stderr[-600:])
    assert "hostsim:" not in p.stderr and "JIT failed" not in p.stdout, (args, p.stdout[-1500:], p.stderr[-600:])
    if types.split()[0] in ("I2", "I1"):
        assert "Total Max Error 0.0000" in p.stdout, (args, p.stdout[-1500:])   # integer results: the driver's gold is exact


def _lib():
    import libxsmm_b200 as X
    lib = C.CDLL(build_sim_lowbit())
    lib.libxsmm_dispatch_gemm.restype, lib.libxsmm_dispatch_gemm.argtypes = C.c_void_p, [X.GemmShape, C.c_uint, C.c_uint]
    lib.libxsmm_dispatch_brgemm.restype = C.c_void_p
    lib.libxsmm_dispatch_brgemm.argtypes = [X.GemmShape, C.c_uint, C.c_uint, X.BatchReduceConfig]
    lib.libxsmm_b200_gemm_batch.restype, lib.libxsmm_b200_gemm_batch.argtypes = C.c_int, [C.c_void_p, C.POINTER(X.GemmParam), C.c_longlong]
    lib.libxsmm_b200_gemm_batch_strided.restype = C.c_int
    lib.libxsmm_b200_gemm_batch_strided.argtypes = [C.c_void_p] * 4 + [C.c_longlong] * 3 + [C.c_ulonglong, C.c_longlong]
    lib.libxsmm_b200_gemm_batch_strided_scaled.restype = C.c_int
    lib.libxsmm_b200_gemm_batch_strided_scaled.argtypes = [C.c_void_p] * 4 + [C.c_longlong] * 3 + [C.c_void_p] * 3 + [C.c_longlong] * 3 + [C.c_ulonglong, C.c_longlong]
    lib.libxsmm_b200_last_error.restype = C.c_int
    lib.libxsmm_b200_launch_count.restype = C.c_ulonglong
    return X, lib


def _handle(X, lib, case):
    sh = X.GemmShape(case.m, case.n, case.k, case.lda, case.ldb, case.ldc, case.ta, case.tb, case.tc, I32)
    if case.br_type == 0:
        h = lib.libxsmm_dispatch_gemm(sh, case.flags, 0)
    else:
        kind = {1: X.GEMM_BATCH_REDUCE_ADDRESS, 2: X.GEMM_BATCH_REDUCE_OFFSET, 3: X.GEMM_BATCH_REDUCE_STRIDE}[case.br_type]
        h = lib.libxsmm_dispatch_brgemm(sh, case.flags, 0, X.libxsmm_create_gemm_batch_reduce_config(kind, case.stride_a, case.stride_b, 0))
    assert h
    return h


def _call(X, lib, case, A, B, c, SA, SB):
    """one call like the reference's drivers make it: address mode passes arrays of pointers for A, B and both scales"""
    keep = []
    p = X.GemmParam()
    brc = C.c_ulonglong(case.br)
    p.op.tertiary = C.addressof(brc)
    p.c.primary = c.ctypes.data
    if case.br_type == 1:
        arrs = [(C.c_void_p * case.br)(*[base + r * step for r in range(case.br)])
                for base, step in ((A.ctypes.data, case.block_a), (B.ctypes.data, case.block_b), (SA.ctypes.data, case.block_sa),
                                   (SB.ctypes.data, 4 * case.block_sb))]
        keep += arrs
        p.a.primary, p.b.primary, p.a.tertiary, p.b.tertiary = [C.addressof(x) for x in arrs]
    else:
        p.a.primary, p.b.primary, p.a.tertiary, p.b.tertiary = A.ctypes.data, B.ctypes.data, SA.ctypes.data, SB.ctypes.data
        if case.br_type == 2:
            oa = np.array([(case.br - 1 - r) * case.block_a for r in range(case.br)], np.int64)
            ob = np.array([(case.br - 1 - r) * case.block_b for r in range(case.br)], np.int64)
            keep += [oa, ob]
            p.a.secondary, p.b.secondary = oa.ctypes.data, ob.ctypes.data
    if not case.mx():
        p.a.tertiary = p.b.tertiary = None
    X.GEMMFUNCTION(lib_fn(lib, X, case))(C.byref(p))


_handles = {}


def lib_fn(lib, X, case):
    return _handles[repr(case)]


@pytest.mark.parametrize("br_type", [0, 1, 2, 3])
@pytest.mark.parametrize("ta,tb,tc", [(I2, U8, I32), (I1, I8, I32), (MXFP4, I8, F32), (MXFP4, I8, BF16)])
def test_single_pageable_call_stages_operands_and_scales(ta, tb, tc, br_type):
    """one call with pageable A / B / C / scales in every batch-reduce mode: C equals the oracle, C's padding rows keep their contents"""
    X, lib = _lib()
    m = {I2: 20, I1: 22, MXFP4: 21}[ta]
    case = LbCase(ta, tb, tc, m, 7, 64, lda=m + 4, ldb=72, ldc=m + 5, beta0=False, br_type=br_type, br=3)
    A, B, C0, SA, SB = case.operands(np.random.default_rng(4 + br_type))
    _handles[repr(case)] = _handle(X, lib, case)
    c = C0.copy()
    _call(X, lib, case, A, B, c, SA, SB)
    _, want = case.run(oracle_gemm_lowbit, A, B, C0, SA, SB)
    assert same_c(case, want, c), case
    pad = np.asarray(c).reshape(case.n, case.ldc)[:, case.m:]
    assert np.array_equal(pad.view(np.uint8), C0.reshape(case.n, case.ldc)[:, case.m:].view(np.uint8))


def test_missing_scales_are_a_noted_error_not_a_launch():
    X, lib = _lib()
    case = LbCase(MXFP4, I8, F32, 8, 4, 32)
    A, B, C0, SA, SB = case.operands(np.random.default_rng(5))
    h = _handle(X, lib, case)
    lib.libxsmm_b200_last_error()                                  # clears the simulated runtime's error
    n0 = lib.libxsmm_b200_launch_count()
    c = C0.copy()
    X.call_gemm(h, A, B, c, a_scales=SA)                           # b.tertiary missing
    assert lib.libxsmm_b200_last_error() != 0 and lib.libxsmm_b200_launch_count() == n0
    assert np.array_equal(c.view(np.uint8), C0.view(np.uint8))


def test_batch_forms():
    """I2 / I1: the plain strided form; MXFP4: libxsmm_b200_gemm_batch with each tile's a.tertiary / b.tertiary, and
    libxsmm_b200_gemm_batch_strided_scaled with scf + t*stride, stride 0 sharing one set of scales"""
    X, lib = _lib()
    rng = np.random.default_rng(6)
    count = 3
    for ta, tb, tc in ((I2, I8, I32), (I1, U8, I32)):
        case = LbCase(ta, tb, tc, 12, 5, 16, lda=14, ldb=20, ldc=13, beta0=False, br_type=3, br=2)
        h = _handle(X, lib, case)
        tiles = [case.operands(rng) for _ in range(count)]
        A = np.concatenate([t[0] for t in tiles]); B = np.concatenate([t[1] for t in tiles]); Cb = np.concatenate([t[2] for t in tiles])
        assert lib.libxsmm_b200_gemm_batch_strided(h, A.ctypes.data, B.ctypes.data, Cb.ctypes.data, case.size_a, case.size_b, 4 * case.size_c,
                                                   case.br, count) == 0
        for t in range(count):
            want = case.run(oracle_gemm_lowbit, *tiles[t])[1]
            assert same_c(case, want, Cb[t * case.size_c:(t + 1) * case.size_c]), (ta, t)
    case = LbCase(MXFP4, I8, BF16, 10, 6, 64, lda=12, ldb=64, ldc=11, beta0=False, br_type=2, br=2)
    h = _handle(X, lib, case)
    tiles = [case.operands(rng) for _ in range(count)]
    cs = [t[2].copy() for t in tiles]
    params = (X.GemmParam * count)()
    brc = C.c_ulonglong(case.br)
    oa = np.array([(case.br - 1 - r) * case.block_a for r in range(case.br)], np.int64)
    ob = np.array([(case.br - 1 - r) * case.block_b for r in range(case.br)], np.int64)
    for t, (A, B, C0, SA, SB) in enumerate(tiles):
        p = params[t]
        p.op.tertiary = C.addressof(brc)
        p.a.primary, p.b.primary, p.c.primary = A.ctypes.data, B.ctypes.data, cs[t].ctypes.data
        p.a.secondary, p.b.secondary = oa.ctypes.data, ob.ctypes.data
        p.a.tertiary, p.b.tertiary = SA.ctypes.data, SB.ctypes.data
    assert lib.libxsmm_b200_gemm_batch(h, params, count) == 0
    for t, (A, B, C0, SA, SB) in enumerate(tiles):
        assert same_c(case, case.run(oracle_gemm_lowbit, A, B, C0, SA, SB)[1], cs[t]), t
    case = LbCase(MXFP4, I8, F32, 10, 6, 64, lda=12, ldb=64, ldc=11, beta0=False)
    h = _handle(X, lib, case)
    tiles = [case.operands(rng) for _ in range(count)]
    A = np.concatenate([t[0] for t in tiles]); B = np.concatenate([t[1] for t in tiles])
    SA = np.concatenate([t[3] for t in tiles]); SB = np.concatenate([t[4] for t in tiles])
    for shared in (False, True):
        Cb = np.concatenate([t[2] for t in tiles])
        os.environ["XB_HOSTSIM_PTR_KIND"] = "1"       # the scaled form takes device-accessible operands only
        try:
            rc = lib.libxsmm_b200_gemm_batch_strided_scaled(h, A.ctypes.data, B.ctypes.data, Cb.ctypes.data, case.size_a, case.size_b, 4 * case.size_c,
                                                            SA.ctypes.data, SB.ctypes.data, None, 0 if shared else case.size_sa,
                                                            0 if shared else 4 * case.size_sb, 0, 1, count)
        finally:
            del os.environ["XB_HOSTSIM_PTR_KIND"]
        assert rc == 0
        for t in range(count):
            want = case.run(oracle_gemm_lowbit, tiles[t][0], tiles[t][1], tiles[t][2], tiles[0][3] if shared else tiles[t][3],
                            tiles[0][4] if shared else tiles[t][4])[1]
            assert same_c(case, want, Cb[t * case.size_c:(t + 1) * case.size_c]), (shared, t)
