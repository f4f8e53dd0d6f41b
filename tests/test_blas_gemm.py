"""libxsmm_dgemm / libxsmm_sgemm, their Fortran-77 symbols and the C++ libxsmm_gemm overloads, without a GPU.

* Simulated device (the host_*.c sources linked with tests/c/hostsim_runtime.c, see tests/test_hostsim.py; every GEMM tile is answered by
  the oracle): the reference's argument rules -- transpose characters, beta = 0 vs accumulate, ignored alpha, NULL defaults -- the
  staging of host operands, and C's padding rows, bit for bit against the oracle under those rules.
* Four threads updating row blocks of one pageable C: only the m x n block a call owns may be copied back.
* The reference's own libxsmm_dgemm / libxsmm_sgemm (oracle/_ref/libxsmm_ref_blas.so) on exact-by-construction operands pins the rules
  to the reference itself.
* Relink: a C caller (tests/c/blas_demo.c), a C++ caller of the overloads (tests/c/blas_overloads.cpp, -Wall -Werror) and the
  reference's samples/magazine/magazine_xsmm.c, unmodified."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import blas_cases as B
import gen
from oracle_ffi import oracle, run_gemm
from test_hostsim import ORACLE, OUT as SIM_DIR, build_sim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "libxsmm_b200", "lib")
BUILD = os.path.join(ROOT, "build")
REF_BLAS_SO = os.path.join(ROOT, "oracle", "_ref", "libxsmm_ref_blas.so")
MAGAZINE_DIR = os.path.join(ROOT, "oracle", "_ref", "blas")
SIM_ENV = dict(os.environ, LD_LIBRARY_PATH=SIM_DIR + ":" + ORACLE + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="4")


@pytest.fixture(scope="module")
def sim():
    lib = B.bind(C.CDLL(build_sim()))
    for name in ("libxsmm_dgemm_", "libxsmm_sgemm_"):
        getattr(lib, name).argtypes = lib.libxsmm_dgemm.argtypes
    lib.libxsmm_b200_launch_count_backend.restype, lib.libxsmm_b200_launch_count_backend.argtypes = C.c_ulonglong, [C.c_int]
    return lib


def build_caller(src, exe, cxx=False):
    """a caller of the public headers, linked with -lxsmm like a relinking user"""
    os.makedirs(BUILD, exist_ok=True)
    cmd = (["g++", "-std=c++11"] if cxx else ["gcc", "-std=c99"]) + ["-O1", "-ffp-contract=off", "-Wall", "-Werror", "-I" + INCLUDE,
                                                                      os.path.join(ROOT, "tests", "c", src), "-L" + LIBDIR, "-lxsmm",
                                                                      "-Wl,-rpath," + LIBDIR, "-lm", "-o", os.path.join(BUILD, exe)]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    return os.path.join(BUILD, exe)


@pytest.mark.parametrize("dtype", [gen.F64, gen.F32], ids=["f64", "f32"])
def test_reference_argument_rules_on_the_simulated_device(sim, dtype):
    """every transpose character (N n T t NULL) on both sides x beta {0, 1, 0.5, NULL} x alpha {1, 3, NULL} on ragged and padded shapes
    and on NULL k / n / leading dimensions: C equals the oracle under the reference's rules bit for bit, padding rows included"""
    rng = np.random.default_rng(1 + dtype)
    ran = 0
    for shape_id, (transa, transb, m, n, k, lda, ldb, ldc, beta, alpha) in B.parity_cases():
        e = B.resolve(transa, transb, m, n, k, lda, ldb, ldc, beta)
        a, b, c0 = B.operands(rng, dtype, e)
        want = B.expected(dtype, e, a, b, c0)
        c = c0.copy()
        before = sim.libxsmm_b200_launch_count_backend(1)
        B.call(sim, dtype, transa, transb, m, n, k, alpha, a.ctypes.data, lda, b.ctypes.data, ldb, beta, c.ctypes.data, ldc)
        assert sim.libxsmm_b200_launch_count_backend(1) == before + 1
        assert np.array_equal(c.view(np.uint8), want.view(np.uint8)), (shape_id, transa, transb, beta, alpha)
        ran += 1
    assert ran == len(B.SHAPES) * 25 * 12


@pytest.mark.parametrize("dtype", [gen.F64, gen.F32], ids=["f64", "f32"])
def test_beta_one_half_accumulates_like_one_and_alpha_is_ignored(sim, dtype):
    """the two quirks a BLAS user would not expect, stated directly: beta = 0.5 and beta = 1 give the same bytes, and so do alpha 1 / 3 / NULL"""
    rng = np.random.default_rng(7)
    e = B.resolve(b"N", b"N", 37, 13, 29, 37, 29, 40, 0.5)
    a, b, c0 = B.operands(rng, dtype, e)
    outs = []
    for beta, alpha in ((1.0, 1.0), (0.5, 1.0), (0.5, 3.0), (None, None), (2.0, -1.0)):
        c = c0.copy()
        B.call(sim, dtype, b"N", b"N", 37, 13, 29, alpha, a.ctypes.data, 37, b.ctypes.data, 29, beta, c.ctypes.data, 40)
        outs.append(c)
    assert all(np.array_equal(o.view(np.uint8), outs[0].view(np.uint8)) for o in outs)
    assert np.array_equal(outs[0].view(np.uint8), B.expected(dtype, e, a, b, c0).view(np.uint8))


def test_fortran_symbols_forward(sim):
    rng = np.random.default_rng(8)
    for dtype, symbol in ((gen.F64, "libxsmm_dgemm_"), (gen.F32, "libxsmm_sgemm_")):
        e = B.resolve(b"T", b"n", 21, 6, 10, 10, 10, 24, 0.0)
        a, b, c0 = B.operands(rng, dtype, e)
        c = c0.copy()
        B.call(sim, dtype, b"T", b"n", 21, 6, 10, 1.0, a.ctypes.data, 10, b.ctypes.data, 10, 0.0, c.ctypes.data, 24, symbol=symbol)
        assert np.array_equal(c.view(np.uint8), B.expected(dtype, e, a, b, c0).view(np.uint8)), symbol


def test_rejected_shape_prints_the_reference_message_and_leaves_c_alone(sim, capfd):
    """lda < m (given explicitly) and m = 0 fail in the descriptor: "LIBXSMM_GEMM failed" on stdout, C untouched, nothing launched"""
    libc = C.CDLL(None)
    for dtype in (gen.F64, gen.F32):
        npdt = gen.NP_OF[dtype]
        a, b = np.ones(64, dtype=npdt), np.ones(64, dtype=npdt)
        c = np.full(64, 7, dtype=npdt)
        before = sim.libxsmm_b200_launch_count_backend(1)
        B.call(sim, dtype, b"N", b"N", 8, 4, 4, 1.0, a.ctypes.data, 4, b.ctypes.data, None, 1.0, c.ctypes.data, None)
        B.call(sim, dtype, None, None, 0, 4, 4, 1.0, a.ctypes.data, None, b.ctypes.data, None, 1.0, c.ctypes.data, None)
        libc.fflush(None)
        assert sim.libxsmm_b200_launch_count_backend(1) == before
        assert np.all(c == 7)
    assert capfd.readouterr().out.count("LIBXSMM_GEMM failed\n") == 4


def test_four_threads_update_row_blocks_of_one_pageable_c(sim):
    """Four threads each run libxsmm_sgemm eight times on their own row block of ONE host C (ldc = 5m: four owned blocks, one block of
    padding rows). Every call stages C through the device; a copy-back of the contiguous span (n-1)*ldc + m would carry the other blocks
    back as they were when the call started, over the results their threads wrote meanwhile."""
    c, want = B.four_thread_row_blocks(sim)
    for t in range(B.THREADS):
        blk = slice(t * B.ROWS, (t + 1) * B.ROWS)
        assert np.array_equal(c[:, blk], want[:, blk]), ("row block", t, int((c[:, blk] != want[:, blk]).sum()))
    assert np.all(c[:, B.THREADS * B.ROWS:] == B.SENTINEL)


@pytest.mark.skipif(not os.path.exists(REF_BLAS_SO), reason="oracle/_ref/libxsmm_ref_blas.so was not built (no reference tree at build time)")
@pytest.mark.parametrize("dtype", [gen.F64, gen.F32], ids=["f64", "f32"])
def test_the_reference_blas_entry_points_follow_the_same_rules(dtype):
    """The reference's own libxsmm_dgemm / libxsmm_sgemm (its JIT, which contracts to FMA) on exact-by-construction operands: A = +-(1..7)/8,
    B on the grid 2^-fb, C on 2^-q with every partial sum representable (cases.FSSPMDM_EXACT), so any summation order and FMA give the same
    bits. It equals the oracle under the rules above for beta 0, 1, 0.5, NULL and alpha 1, 3: "alpha ignored, beta != 0 acts as 1" is
    the reference's behaviour, not a reading of it."""
    import cases
    ref = C.CDLL(REF_BLAS_SO)
    symbol = "ref_blas_dgemm" if dtype == gen.F64 else "ref_blas_sgemm"
    getattr(ref, symbol).argtypes = [C.c_char_p, C.c_char_p] + [C.c_void_p] * 11
    p, q, fb = cases.FSSPMDM_EXACT[dtype]
    rng = np.random.default_rng(9)
    bmax = 2 ** (fb + 1) - 1

    def dyadic(kind, shape):
        if kind == "a":
            return rng.integers(1, 8, size=shape) * rng.choice([-1.0, 1.0], size=shape) / 8.0
        if kind == "b":
            return rng.integers(-bmax, bmax + 1, size=shape) * 2.0 ** -fb
        return rng.integers(-2 ** (q + 1), 2 ** (q + 1) + 1, size=shape) * 2.0 ** -q
    for (m, n, k, lda, ldb, ldc) in ((37, 13, 29, 40, 31, 41), (1, 5, 7, 1, 7, 3), (64, 48, 64, 64, 64, 64)):
        assert k * 7 / 8 * bmax * 2.0 ** -fb + 2 < 2.0 ** (p - q)
        for transa, transb in ((b"N", b"N"), (b"t", b"N"), (b"N", b"T"), (None, b"t")):
            ta, tb = transa not in (None, b"N", b"n"), transb not in (None, b"N", b"n")
            la, lb = (max(lda, k) if ta else lda), (max(ldb, n) if tb else ldb)
            for beta in (0.0, 1.0, 0.5, None):
                for alpha in (1.0, 3.0):
                    e = B.resolve(transa, transb, m, n, k, la, lb, ldc, beta)
                    a, b, c0 = B.operands(rng, dtype, e, values=dyadic)
                    c = c0.copy()
                    B.call(ref, dtype, transa, transb, m, n, k, alpha, a.ctypes.data, la, b.ctypes.data, lb, beta, c.ctypes.data, ldc, symbol=symbol)
                    assert np.array_equal(c.view(np.uint8), B.expected(dtype, e, a, b, c0).view(np.uint8)), (m, transa, transb, beta, alpha)


def test_c_caller_links_and_rejects_without_a_gpu():
    """the C caller links against the real library (both C and Fortran-77 symbols) and its rejected shapes need no device"""
    exe = build_caller("blas_demo.c", "blas_demo")
    p = subprocess.run([exe, "reject"], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0 and "reject ok" in p.stdout, p.stdout + p.stderr
    assert p.stdout.count("LIBXSMM_GEMM failed") == 4, p.stdout


def test_cxx_overloads_compile_warning_free_and_reject_without_a_gpu():
    exe = build_caller("blas_overloads.cpp", "blas_overloads", cxx=True)
    p = subprocess.run([exe, "reject"], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0 and "reject ok" in p.stdout, p.stdout + p.stderr
    assert p.stdout.count("LIBXSMM_GEMM failed") == 4, p.stdout


@pytest.mark.parametrize("src,exe", [("blas_demo.c", "blas_demo"), ("blas_overloads.cpp", "blas_overloads")])
def test_callers_against_the_simulated_device(src, exe):
    """the same binaries with the simulation library first on the loader's path: every product matches its triple loop exactly"""
    path = build_caller(src, exe, cxx=src.endswith(".cpp"))
    build_sim()
    p = subprocess.run([path, "run"], capture_output=True, text=True, timeout=300, env=SIM_ENV)
    assert p.returncode == 0 and "max_abs_diff 0.000e+00" in p.stdout, p.stdout + p.stderr[-600:]
    assert "hostsim:" not in p.stderr, p.stderr[-600:]


# ---- samples/magazine/magazine_xsmm.c, unmodified ---------------------------------------------------------------------------------
MAGAZINE_BATCH, MAGAZINE_MNK = 500, (13, 5, 7)       # the driver's default shape; batch given on the command line


def magazine_check():
    """The driver's checksum: the largest Kahan sum of |C_i| after C_i += A_i B_i (beta = 1) over its own seeded fill (magazine.h init /
    norm, restated), every product by the oracle in the exact-order kernel's order. Printed by the driver as "%f (check)"."""
    m, n, k = MAGAZINE_MNK
    scale = 1.0 / MAGAZINE_BATCH

    def init(seed, nrows, ncols):
        seed1 = scale * seed + scale
        return np.array([seed1 * float(i * nrows + j + 1) for i in range(ncols) for j in range(nrows)], dtype=np.float64)
    check = 0.0
    for i in range(MAGAZINE_BATCH):
        a, b, c = init(25 + i, m, k), init(75 + i, k, n), init(42 + i, m, n)
        assert run_gemm(oracle, (m, n, k, m, k, m), (gen.F64,) * 4, 0, 0, 0, 0, 1, a, b, c) == 0
        result = comp = 0.0
        for v in c.tolist():
            x = abs(v) - comp
            y = result + x
            comp = (y - result) - x
            result = y
        check = max(check, result)
    return "%f (check)" % check


def run_magazine(env):
    """both builds of the sample: as shipped (one dispatched kernel) and with -DAUTO (every matrix through libxsmm_dgemm)"""
    want = magazine_check()
    for name in ("magazine_xsmm", "magazine_xsmm_auto"):
        exe = os.path.join(MAGAZINE_DIR, name)
        m, n, k = MAGAZINE_MNK
        p = subprocess.run([exe, str(MAGAZINE_BATCH), str(m), str(n), str(k)], capture_output=True, text=True, timeout=300, env=env)
        assert p.returncode == 0, (name, p.stdout[-800:], p.stderr[-800:])
        assert want in p.stdout, (name, want, p.stdout[-800:])
        assert "LIBXSMM_GEMM failed" not in p.stdout


@pytest.mark.skipif(not os.path.exists(os.path.join(MAGAZINE_DIR, "magazine_xsmm_auto")), reason="samples/magazine was not built (no reference tree at build time)")
def test_magazine_sample_against_the_simulated_device():
    build_sim()
    run_magazine(SIM_ENV)
