"""-m gpu: libxsmm_dgemm / libxsmm_sgemm on the H100, bit for bit against the oracle under the reference's argument rules
(tests/blas_cases.py), with A, B and C in pageable host, pinned, managed and device memory. F64 and F32 run on the exact-order
gemm_simt_kernel family: every call must launch exactly one kernel, of that family. Plus four threads on row blocks of one pageable C,
the C and C++ callers and samples/magazine/magazine_xsmm.c on the device."""
import os
import subprocess

import numpy as np
import pytest

import blas_cases as B
import gen
import libxsmm_b200 as X
from test_blas_gemm import MAGAZINE_DIR, build_caller, run_magazine

pytestmark = pytest.mark.gpu
KINDS = ("host", "pinned", "managed", "device")
ARENA = 32 << 20


class Arena:
    """one allocation of a memory kind; operands are copied in at 256-byte aligned offsets and read back after the call"""
    def __init__(self, kind):
        self.kind = kind
        self.base = {"pinned": X.libxsmm_b200_host_malloc, "managed": X.libxsmm_malloc, "device": X.libxsmm_b200_device_malloc}[kind](ARENA)
        assert self.base
        self.top = 0

    def place(self, arr):
        ptr = self.base + self.top
        self.top += (arr.nbytes + 255) // 256 * 256
        assert self.top <= ARENA
        assert X.libxsmm_b200_memcpy(ptr, arr.ctypes.data, arr.nbytes) == 0
        return ptr

    def fetch(self, ptr, like):
        out = np.empty_like(like)
        assert X.libxsmm_b200_memcpy(out.ctypes.data, ptr, out.nbytes) == 0
        return out

    def free(self):
        {"pinned": X.libxsmm_b200_host_free, "managed": X.libxsmm_free, "device": X.libxsmm_b200_device_free}[self.kind](self.base)


@pytest.fixture(scope="module")
def arenas():
    X.libxsmm_b200_set_device(0)
    made = {kind: Arena(kind) for kind in KINDS if kind != "host"}
    yield made
    for a in made.values():
        a.free()


def run_everywhere(arenas, dtype, args, a, b, c0):
    """the call `args` (blas_cases.parity_cases order, a/b/c replaced by the operands) from every memory kind; yields (kind, C after)"""
    transa, transb, m, n, k, lda, ldb, ldc, beta, alpha = args
    for kind in KINDS:
        counts = [X.libxsmm_b200_launch_count()] + [X.libxsmm_b200_launch_count_backend(f) for f in (X.BACKEND_SIMT, X.BACKEND_TCGEN05, X.BACKEND_STREAM)]
        if kind == "host":
            c = c0.copy()
            B.call(X.lib, dtype, transa, transb, m, n, k, alpha, a.ctypes.data, lda, b.ctypes.data, ldb, beta, c.ctypes.data, ldc)
        else:
            ar = arenas[kind]
            ar.top = 0
            pa, pb, pc = ar.place(a), ar.place(b), ar.place(c0)
            B.call(X.lib, dtype, transa, transb, m, n, k, alpha, pa, lda, pb, ldb, beta, pc, ldc)
            c = ar.fetch(pc, c0)
        X.check()
        after = [X.libxsmm_b200_launch_count()] + [X.libxsmm_b200_launch_count_backend(f) for f in (X.BACKEND_SIMT, X.BACKEND_TCGEN05, X.BACKEND_STREAM)]
        assert [y - x for x, y in zip(counts, after)] == [1, 1, 0, 0], (kind, counts, after)
        yield kind, c


@pytest.mark.parametrize("dtype", [gen.F64, gen.F32], ids=["f64", "f32"])
def test_reference_argument_rules_from_every_memory_kind(arenas, dtype):
    """the CPU tier's grid (every transpose character on both sides x beta {0, 1, 0.5, NULL} x alpha {1, 3, NULL}, ragged and padded
    shapes, NULL k / n / leading dimensions) on the device, from host, pinned, managed and device pointers"""
    rng = np.random.default_rng(101 + dtype)
    for shape_id, args in B.parity_cases():
        transa, transb, m, n, k, lda, ldb, ldc, beta, alpha = args
        e = B.resolve(transa, transb, m, n, k, lda, ldb, ldc, beta)
        a, b, c0 = B.operands(rng, dtype, e)
        want = B.expected(dtype, e, a, b, c0)
        for kind, c in run_everywhere(arenas, dtype, args, a, b, c0):
            assert np.array_equal(c.view(np.uint8), want.view(np.uint8)), (kind, shape_id, transa, transb, beta, alpha)


@pytest.mark.parametrize("dtype", [gen.F64, gen.F32], ids=["f64", "f32"])
def test_larger_product_with_padded_c(arenas, dtype):
    """1024 x 768 x 512, ldc = 1040, beta 1 and beta 0 with A transposed"""
    rng = np.random.default_rng(7 + dtype)
    for args in ((b"N", b"N", 1024, 768, 512, 1024, 512, 1040, 1.0, 1.0), (b"T", b"N", 1024, 768, 512, 520, 512, 1040, 0.0, 2.0)):
        e = B.resolve(*args[:8], args[8])
        a, b, c0 = B.operands(rng, dtype, e)
        want = B.expected(dtype, e, a, b, c0)
        for kind, c in run_everywhere(arenas, dtype, args, a, b, c0):
            assert np.array_equal(c.view(np.uint8), want.view(np.uint8)), (kind, args[:2])


def test_four_threads_update_row_blocks_of_one_pageable_c():
    X.libxsmm_b200_set_device(0)
    c, want = B.four_thread_row_blocks(X.lib)
    X.check()
    for t in range(B.THREADS):
        blk = slice(t * B.ROWS, (t + 1) * B.ROWS)
        assert np.array_equal(c[:, blk], want[:, blk]), ("row block", t, int((c[:, blk] != want[:, blk]).sum()))
    assert np.all(c[:, B.THREADS * B.ROWS:] == B.SENTINEL)


@pytest.mark.parametrize("src,exe", [("blas_demo.c", "blas_demo"), ("blas_overloads.cpp", "blas_overloads")])
def test_callers_run_on_host_buffers(src, exe):
    path = build_caller(src, exe, cxx=src.endswith(".cpp"))
    p = subprocess.run([path, "run"], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and "max_abs_diff 0.000e+00" in p.stdout, p.stdout + p.stderr[-600:]


@pytest.mark.skipif(not os.path.exists(os.path.join(MAGAZINE_DIR, "magazine_xsmm_auto")), reason="samples/magazine was not built (no reference tree at build time)")
def test_magazine_sample_on_the_device():
    """buffers from libxsmm_aligned_malloc (managed memory), OpenMP threads calling libxsmm_dgemm / the dispatched kernel"""
    run_magazine(dict(os.environ, OMP_NUM_THREADS="4"))
