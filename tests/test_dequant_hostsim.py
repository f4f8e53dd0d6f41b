"""Dequantising GEMM through the host half of the library on the simulated device: the host_*.c objects, tests/c/hostsim_runtime.c and
tests/c/hostsim_dq.c (dequantising tiles answered by oracle/oracle_dq.c) linked into tests/c/_hostsim/dq/libxsmm.so. What this checks
is the host code: dispatch of the forms the reference's driver uses, staging of pageable A / B / C and of the row scales and zero
points, the copy back of C, the batch forms' per-tile scales, and the missing-scale error. The reference's unmodified
samples/xgemm/gemm_kernel.c (oracle/ref_drivers.py) runs against it for every tuple with nobr, strdbr, addrbr and offsbr and must pass
by its own verdict; where the driver's gold follows the reference's order it also reports a zero error."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import dq_ffi  # noqa: F401  (builds oracle/liboracle.so and oracle/liboracle_dq.so)
from dq_ffi import BF16, F16, F32, I4, I8, U4, DqCase, oracle_gemm_dq, same_c
from test_hostsim import CSRC, DRV, HOST_C, ORACLE, ROOT

OUT = os.path.join(ROOT, "tests", "c", "_hostsim", "dq")


def build_sim_dq():
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, "libxsmm.so")
    srcs = [os.path.join(CSRC, f) for f in HOST_C] + [os.path.join(ROOT, "tests", "c", f) for f in ("hostsim_runtime.c", "hostsim_dq.c")]
    deps = srcs + [os.path.join(CSRC, "xb_internal.h")]
    if os.path.exists(so) and all(os.path.getmtime(s) < os.path.getmtime(so) for s in deps):
        return so
    cmd = ["gcc", "-O1", "-std=gnu99", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-Wl,--wrap=xb_gemm_simt_launch", "-o", so] + \
        srcs + ["-L" + ORACLE, "-loracle_dq", "-loracle", "-Wl,-rpath," + ORACLE, "-lpthread", "-ldl", "-lm"]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    return so


# samples/xgemm/gemm_kernel.c: A B Comp C  M N K LDA LDB LDC  alpha beta  alignA alignC  trA trB  vnniA vnniB vnniC  prefetch  br-kind br-count
# br-unroll  reps  tilecfg
def _gk(types, beta, br, trb=0, vnnia=0, m=64, n=48, k=64, lda=64, ldb=64, ldc=64):
    return tuple(types.split()) + (m, n, k, lda, ldb, ldc, 1, beta, 0, 0, 0, trb, vnnia, 0, 0, "nopf", br, 1 if br == "nobr" else 3, 0, 3, 0)


TYPES = ["I8 BF16 F32 F32", "I8 BF16 F32 BF16"] + ["%s F16 %s %s" % (a, comp, c) for a in ("I8", "I4", "U4", "BF8")
                                                  for comp in ("F16", "F32", "IMPLICIT") for c in ("F16", "F32")]
BRS = ["nobr", "strdbr", "addrbr", "offsbr"]


def _driver_args(types, br):
    a = types.split()[0]
    vnnia = 1 if a in ("I4", "U4", "BF8") else 0
    beta = 0 if br in ("strdbr", "offsbr") else 1
    return _gk(types, beta, br, vnnia=vnnia, m=40, n=24, k=64, lda=48, ldb=72, ldc=44)


# the driver's own gold (gemm_kernel.c :1835-2060) restates the reference's order for these; the others it computes differently
EXACT = {"I8 BF16 F32 F32", "I8 BF16 F32 BF16"} | {"%s F16 %s %s" % (a, comp, c) for a in ("I8", "I4", "U4") for comp in ("F16", "F32", "IMPLICIT")
                                                  for c in ("F16", "F32")}


@pytest.mark.parametrize("br", BRS)
@pytest.mark.parametrize("types", TYPES, ids=lambda t: t.replace(" ", "_"))
def test_reference_gemm_kernel_driver_against_the_simulated_device(types, br):
    exe = os.path.join(DRV, "gemm_kernel")
    if not os.path.exists(exe):
        pytest.skip("gemm_kernel was not prebuilt (no reference tree in the build container?)")
    build_sim_dq()
    args = _driver_args(types, br)
    env = dict(os.environ, LD_LIBRARY_PATH=OUT + ":" + ORACLE + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="2",
               LIBXSMM_TARGET="spr")
    p = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=300, env=env, cwd=DRV)
    assert p.returncode == 0, (args, p.stdout[-1500:], p.stderr[-600:])
    assert "hostsim:" not in p.stderr and "JIT failed" not in p.stdout, (args, p.stdout[-1500:], p.stderr[-600:])
    if types in EXACT:
        assert "Total Max Error 0.0000" in p.stdout, (args, p.stdout[-1500:])


def _lib():
    import libxsmm_b200 as X
    lib = C.CDLL(build_sim_dq())
    lib.libxsmm_dispatch_gemm.restype, lib.libxsmm_dispatch_gemm.argtypes = C.c_void_p, [X.GemmShape, C.c_uint, C.c_uint]
    lib.libxsmm_b200_gemm_batch.restype, lib.libxsmm_b200_gemm_batch.argtypes = C.c_int, [C.c_void_p, C.POINTER(X.GemmParam), C.c_longlong]
    lib.libxsmm_b200_gemm_batch_strided_scaled.restype = C.c_int
    lib.libxsmm_b200_gemm_batch_strided_scaled.argtypes = [C.c_void_p] * 4 + [C.c_longlong] * 3 + [C.c_void_p] * 3 + [C.c_longlong] * 3 + [C.c_ulonglong, C.c_longlong]
    lib.libxsmm_b200_last_error.restype = C.c_int
    lib.libxsmm_b200_launch_count.restype = C.c_ulonglong
    return X, lib


def _handle(X, lib, case):
    h = lib.libxsmm_dispatch_gemm(X.GemmShape(case.m, case.n, case.k, case.lda, case.ldb, case.ldc, case.ta, case.tb, case.tc, case.comp), case.flags, 0)
    assert h
    return h


@pytest.mark.parametrize("ta,tb,comp,tc", [(I8, BF16, F32, BF16), (I8, F16, F16, F32), (I4, F16, F32, F16), (U4, F16, 25, F32)])
def test_single_pageable_call_stages_scales_and_leaves_c_padding_alone(ta, tb, comp, tc):
    """one call with pageable A / B / C / scales / zero points: C equals the oracle, C's padding rows keep their contents"""
    X, lib = _lib()
    case = DqCase(ta, tb, comp, tc, 21, 7, 34, lda=25, ldb=36, ldc=30, beta0=False)
    A, B, C0, S, Z = case.operands(np.random.default_rng(4))
    c = C0.copy()
    X.call_gemm(_handle(X, lib, case), A, B, c, a_scales=S, a_zero_points=Z if ta != I8 else None)
    _, want = case.run(oracle_gemm_dq, A, B, C0, S, Z)
    assert same_c(case, want, c)
    pad = np.asarray(c).reshape(case.n, case.ldc)[:, case.m:]
    assert np.array_equal(pad.view(np.uint8), C0.reshape(case.n, case.ldc)[:, case.m:].view(np.uint8))


def test_missing_scales_are_a_noted_error_not_a_launch():
    X, lib = _lib()
    for ta, tb, comp, tc, give_s in ((I8, BF16, F32, F32, False), (I4, F16, F16, F16, True)):
        case = DqCase(ta, tb, comp, tc, 8, 4, 16)
        A, B, C0, S, Z = case.operands(np.random.default_rng(5))
        lib.libxsmm_b200_last_error()                                  # clears the simulated runtime's error
        n0 = lib.libxsmm_b200_launch_count()
        c = C0.copy()
        X.call_gemm(_handle(X, lib, case), A, B, c, a_scales=S if give_s else None)   # int4: zero points missing
        assert lib.libxsmm_b200_last_error() != 0 and lib.libxsmm_b200_launch_count() == n0
        assert np.array_equal(c.view(np.uint8), C0.view(np.uint8))


def test_batch_forms_carry_per_tile_scales():
    """libxsmm_b200_gemm_batch: each tile's a.tertiary / a.quaternary; libxsmm_b200_gemm_batch_strided_scaled: scf_a + t*stride, and
    stride 0 shares one set of scales"""
    X, lib = _lib()
    rng = np.random.default_rng(6)
    case = DqCase(I4, F16, F16, F32, 12, 5, 20, lda=14, ldb=22, ldc=13, beta0=False, br_type=3, br=2)
    sh = X.GemmShape(case.m, case.n, case.k, case.lda, case.ldb, case.ldc, case.ta, case.tb, case.tc, case.comp)
    lib.libxsmm_dispatch_brgemm.restype = C.c_void_p
    lib.libxsmm_dispatch_brgemm.argtypes = [X.GemmShape, C.c_uint, C.c_uint, X.BatchReduceConfig]
    h = lib.libxsmm_dispatch_brgemm(sh, case.flags, 0, X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, case.stride_a, case.stride_b, 0))
    assert h
    tiles = [case.operands(rng) for _ in range(4)]
    cs = [t[2].copy() for t in tiles]
    params = (X.GemmParam * 4)()
    brc = C.c_ulonglong(case.br)
    for t, (A, B, C0, S, Z) in enumerate(tiles):
        p = params[t]
        p.op.tertiary = C.addressof(brc)
        p.a.primary, p.b.primary, p.c.primary = A.ctypes.data, B.ctypes.data, cs[t].ctypes.data
        p.a.tertiary, p.a.quaternary = S.ctypes.data, Z.ctypes.data
    assert lib.libxsmm_b200_gemm_batch(h, params, 4) == 0
    for t, (A, B, C0, S, Z) in enumerate(tiles):
        assert same_c(case, case.run(oracle_gemm_dq, A, B, C0, S, Z)[1], cs[t]), t
    # strided scaled, I8 x BF16 -> BF16, per-tile and shared scales
    case = DqCase(I8, BF16, F32, BF16, 10, 6, 18, lda=12, ldb=20, ldc=11, beta0=False)
    h = _handle(X, lib, case)
    count = 3
    tiles = [case.operands(rng) for _ in range(count)]
    A = np.concatenate([t[0] for t in tiles]); B = np.concatenate([t[1] for t in tiles]); S = np.concatenate([t[3] for t in tiles])
    for shared in (False, True):
        Cb = np.concatenate([t[2] for t in tiles])
        os.environ["XB_HOSTSIM_PTR_KIND"] = "1"       # the scaled form takes device-accessible operands only
        try:
            rc = lib.libxsmm_b200_gemm_batch_strided_scaled(h, A.ctypes.data, B.ctypes.data, Cb.ctypes.data, case.size_a, 2 * case.size_b, 2 * case.size_c,
                                                            S.ctypes.data, None, None, 0 if shared else 4 * case.m, 0, 0, 1, count)
        finally:
            del os.environ["XB_HOSTSIM_PTR_KIND"]
        assert rc == 0
        for t in range(count):
            want = case.run(oracle_gemm_dq, tiles[t][0], tiles[t][1], tiles[t][2], tiles[0][3] if shared else tiles[t][3], None)[1]
            assert same_c(case, want, Cb[t * case.size_c:(t + 1) * case.size_c]), (shared, t)
