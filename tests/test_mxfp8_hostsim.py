"""MX fp8 GEMM through the host half of the library on the simulated device: the host_*.c objects, tests/c/hostsim_runtime.c and
tests/c/hostsim_mx.c (MX tiles answered by the MX oracle) linked into tests/c/_hostsim/mx/libxsmm.so. What this checks is the host
code: dispatch of the forms the reference's driver uses, staging of pageable A / B / C and of the three scale arrays, and the copy
back of C's data and scale bytes. The reference's unmodified samples/xgemm/gemm_kernel.c (oracle/ref_drivers.py) runs against it
for MXBF8_MXBF8_F32_F32, MXHF8_MXHF8_F32_F32 and MXBF8_MXBF8_F32_MXBF8 with nobr and strdbr and must pass by its own verdict."""
import os
import subprocess

import numpy as np
import pytest

import mx_ffi  # noqa: F401  (builds oracle/liboracle.so and oracle/liboracle_mx.so)
from test_hostsim import CSRC, DRV, HOST_C, ORACLE, ROOT

OUT = os.path.join(ROOT, "tests", "c", "_hostsim", "mx")


def build_sim_mx():
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, "libxsmm.so")
    srcs = [os.path.join(CSRC, f) for f in HOST_C] + [os.path.join(ROOT, "tests", "c", f) for f in ("hostsim_runtime.c", "hostsim_mx.c")]
    deps = srcs + [os.path.join(CSRC, "xb_internal.h")]
    if os.path.exists(so) and all(os.path.getmtime(s) < os.path.getmtime(so) for s in deps):
        return so
    cmd = ["gcc", "-O1", "-std=gnu99", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-Wl,--wrap=xb_gemm_simt_launch", "-o", so] + \
        srcs + ["-L" + ORACLE, "-loracle_mx", "-loracle", "-Wl,-rpath," + ORACLE, "-lpthread", "-ldl", "-lm"]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    return so


# samples/xgemm/gemm_kernel.c: A B Comp C  M N K LDA LDB LDC  alpha beta  alignA alignC  trA trB  vnniA vnniB vnniC  prefetch  br-kind br-count
# br-unroll  reps  tilecfg
def _gk(types, m, n, k, lda, ldb, ldc, beta, br, brn):
    return tuple(types.split()) + (m, n, k, lda, ldb, ldc, 1, beta, 0, 0, 0, 1, 1, 1, 0, "nopf", br, brn, 0, 3, 0)


RUNS = [_gk("MXBF8 MXBF8 F32 F32", 64, 48, 64, 64, 48, 64, 1, "nobr", 1), _gk("MXBF8 MXBF8 F32 F32", 40, 24, 96, 48, 32, 44, 0, "strdbr", 3),
        _gk("MXHF8 MXHF8 F32 F32", 64, 48, 64, 64, 48, 64, 1, "nobr", 1), _gk("MXHF8 MXHF8 F32 F32", 40, 24, 96, 48, 32, 44, 0, "strdbr", 3),
        _gk("MXBF8 MXBF8 F32 MXBF8", 64, 48, 64, 64, 48, 64, 0, "nobr", 1), _gk("MXBF8 MXBF8 F32 MXBF8", 64, 24, 96, 64, 32, 96, 0, "strdbr", 3)]


@pytest.mark.parametrize("args", RUNS, ids=lambda a: "%s_%s_%s" % (a[0], a[3], a[20]))
def test_reference_gemm_kernel_driver_against_the_simulated_device(args):
    exe = os.path.join(DRV, "gemm_kernel")
    if not os.path.exists(exe):
        pytest.skip("gemm_kernel was not prebuilt (no reference tree in the build container?)")
    build_sim_mx()
    env = dict(os.environ, LD_LIBRARY_PATH=OUT + ":" + ORACLE + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="2")
    p = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=300, env=env, cwd=DRV)
    assert p.returncode == 0, (args, p.stdout[-1500:], p.stderr[-600:])
    assert "hostsim:" not in p.stderr and "JIT failed" not in p.stdout, (args, p.stdout[-1500:], p.stderr[-600:])
    assert "Total Max Error 0.0000" in p.stdout, (args, p.stdout[-1500:])


def test_single_call_stages_host_operands_and_copies_scales_back():
    """one MXBF8 -> MXBF8 call with pageable A / B / C and scale arrays through the simulation: C's data and scale bytes equal the oracle's,
    C's padding rows and the scale bytes past m/32 of each column keep their contents"""
    import ctypes as C
    import libxsmm_b200 as X
    from mx_ffi import MXBF8, MxCase, oracle_gemm_mx
    lib = C.CDLL(build_sim_mx())
    lib.libxsmm_dispatch_gemm.restype, lib.libxsmm_dispatch_gemm.argtypes = C.c_void_p, [X.GemmShape, C.c_uint, C.c_uint]
    case = MxCase(MXBF8, MXBF8, 64, 5, 96, lda=70, ldb=6, ldc=128)
    A, B, C0, As, Bs, Cs = case.operands(np.random.default_rng(9))
    C0[:] = 0x33; Cs[:] = 0x44
    h = lib.libxsmm_dispatch_gemm(X.GemmShape(case.m, case.n, case.k, case.lda, case.ldb, case.ldc, MXBF8, MXBF8, MXBF8, 1), case.flags, 0)
    assert h
    c, cs = C0.copy(), Cs.copy()
    X.call_gemm(h, A, B, c, a_scales=As, b_scales=Bs, c_scales=cs)
    _, want_c, want_cs = case.run(oracle_gemm_mx, A, B, C0, As, Bs, Cs)
    assert np.array_equal(c, want_c)
    got = cs.reshape(case.n, case.ldc // 32)
    assert np.array_equal(got[:, :case.m // 32], want_cs.reshape(case.n, case.ldc // 32)[:, :case.m // 32])
    assert np.all(got[:, case.m // 32:] == 0x44) and np.all(c.reshape(case.n, case.ldc)[:, case.m:] == 0x33)
