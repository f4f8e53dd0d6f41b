"""TEST INFRASTRUCTURE: the BLAS-style GEMM (libxsmm_dgemm / libxsmm_sgemm) as the reference defines it, restated for the tests
of tests/test_blas_gemm.py (simulated device, reference pin) and tests/test_blas_gemm_gpu.py (H100).

LIBXSMM_XGEMM (reference src/libxsmm_main.h:215-240): only 'N' / 'n' (or NULL) means "as is"; alpha is never read; beta == 0 selects
BETA_0 and any other beta (0.5 too, NULL means 1) accumulates; k defaults to m, n to k, lda to m (k under TRANS_A), ldb to k (n under
TRANS_B), ldc to m, every leading dimension at least 1. `resolve` restates that, `expected` asks the oracle for the product."""
import ctypes as C
import threading

import numpy as np

import gen
from oracle_ffi import oracle, run_gemm

FLAG_TRANS_A, FLAG_TRANS_B, FLAG_BETA_0 = 1, 2, 4
TRANS = (b"N", b"n", b"T", b"t", None)
BETAS = (0.0, 1.0, 0.5, None)
ALPHAS = (1.0, 3.0, None)
SENTINEL = -1234.5           # C's padding rows; must come back unchanged
# (m, n, k, lda, ldb, ldc) as passed; a leading dimension of None is passed as NULL. lda/ldb given as (as is, transposed) pairs.
SHAPES = [(1, 5, 7, (3, 9), (9, 6), 4), (37, 13, 29, (40, 31), (31, 16), 41), (16, 16, 16, (None, None), (None, None), None),
          (12, None, None, (None, None), (None, None), None), (9, None, 5, (None, None), (None, None), 11)]   # k = m, n = k


def bind(lib):
    for name in ("libxsmm_dgemm", "libxsmm_sgemm"):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = None, [C.c_char_p, C.c_char_p] + [C.c_void_p] * 11
    return lib


def resolve(transa, transb, m, n, k, lda, ldb, ldc, beta):
    """the shape, flags and leading dimensions the reference derives from the arguments"""
    ta = transa is not None and transa not in (b"N", b"n")
    tb = transb is not None and transb not in (b"N", b"n")
    kk = m if k is None else k
    nn = kk if n is None else n
    return dict(ta=ta, tb=tb, m=m, n=nn, k=kk,
                lda=max(lda if lda is not None else (kk if ta else m), 1), ldb=max(ldb if ldb is not None else (nn if tb else kk), 1),
                ldc=max(ldc if ldc is not None else m, 1),
                flags=(FLAG_TRANS_A if ta else 0) | (FLAG_TRANS_B if tb else 0) | (FLAG_BETA_0 if beta is not None and beta == 0 else 0))


def operands(rng, dtype, e, values=None):
    """(a, b, c0) column-major for the resolved call `e`: NaN in the padding of A and B, SENTINEL in C's padding rows. The used elements
    are values(which, shape) with which in "abc", standard normal by default."""
    npdt = gen.NP_OF[dtype]
    draw = values or (lambda which, shape: rng.standard_normal(shape))
    a = np.full((e["m"] if e["ta"] else e["k"], e["lda"]), np.nan, dtype=npdt)
    a[:, :(e["k"] if e["ta"] else e["m"])] = draw("a", (a.shape[0], e["k"] if e["ta"] else e["m"]))
    b = np.full((e["k"] if e["tb"] else e["n"], e["ldb"]), np.nan, dtype=npdt)
    b[:, :(e["n"] if e["tb"] else e["k"])] = draw("b", (b.shape[0], e["n"] if e["tb"] else e["k"]))
    c0 = np.full((e["n"], e["ldc"]), SENTINEL, dtype=npdt)
    c0[:, :e["m"]] = draw("c", (e["n"], e["m"]))
    return a.ravel(), b.ravel(), c0.ravel()


def expected(dtype, e, a, b, c0):
    want = c0.copy()
    assert run_gemm(oracle, (e["m"], e["n"], e["k"], e["lda"], e["ldb"], e["ldc"]), (dtype,) * 4, e["flags"], 0, 0, 0, 1, a, b, want) == 0
    return want


def call(lib, dtype, transa, transb, m, n, k, alpha, a, lda, b, ldb, beta, c, ldc, symbol=None):
    """libxsmm_dgemm / libxsmm_sgemm (or `symbol`) with every scalar by reference; None is passed as NULL; a, b, c are addresses"""
    I = C.c_int
    S = C.c_double if dtype == gen.F64 else C.c_float
    fn = getattr(lib, symbol or ("libxsmm_dgemm" if dtype == gen.F64 else "libxsmm_sgemm"))

    def ref(v, T):
        return None if v is None else C.byref(T(v))
    fn(transa, transb, ref(m, I), ref(n, I), ref(k, I), ref(alpha, S), a, ref(lda, I), b, ref(ldb, I), ref(beta, S), c, ref(ldc, I))


def parity_cases():
    """every transpose pair x beta x alpha on each shape, the leading dimensions matching the transposes"""
    for shape_id, (m, n, k, ldas, ldbs, ldc) in enumerate(SHAPES):
        for transa in TRANS:
            for transb in TRANS:
                ta = transa is not None and transa not in (b"N", b"n")
                tb = transb is not None and transb not in (b"N", b"n")
                for beta in BETAS:
                    for alpha in ALPHAS:
                        yield shape_id, (transa, transb, m, n, k, ldas[ta], ldbs[tb], ldc, beta, alpha)


# ---- four threads, four row blocks of ONE pageable C ------------------------------------------------------------------------------
ROWS, COLS, DEPTH, THREADS, LOOPS = 64, 48, 96, 4, 8
LDC = (THREADS + 1) * ROWS    # four owned row blocks and one block of padding rows


def four_thread_row_blocks(lib, seed=31):
    """each thread runs LOOPS times C[rows of block t] += A_t B_t through libxsmm_sgemm (host numpy buffers: staged through the device).
    Returns (c, want): every block accumulated LOOPS times in order, the padding rows SENTINEL."""
    rng = np.random.default_rng(seed)
    a = [rng.standard_normal(ROWS * DEPTH).astype(np.float32) for _ in range(THREADS)]
    b = [rng.standard_normal(DEPTH * COLS).astype(np.float32) for _ in range(THREADS)]
    c = np.full((COLS, LDC), SENTINEL, dtype=np.float32)
    c[:, :THREADS * ROWS] = rng.standard_normal((COLS, THREADS * ROWS))
    want = c.copy()
    e = resolve(b"N", b"N", ROWS, COLS, DEPTH, ROWS, DEPTH, LDC, 1.0)
    for t in range(THREADS):
        view = want.ravel()[t * ROWS:]
        for _ in range(LOOPS):
            assert run_gemm(oracle, (ROWS, COLS, DEPTH, ROWS, DEPTH, LDC), (gen.F32,) * 4, e["flags"], 0, 0, 0, 1, a[t], b[t], view) == 0
    start = threading.Barrier(THREADS)

    def work(t):
        start.wait()
        for _ in range(LOOPS):
            call(lib, gen.F32, b"N", b"N", ROWS, COLS, DEPTH, 1.0, a[t].ctypes.data, ROWS, b[t].ctypes.data, DEPTH, 1.0,
                 c.ctypes.data + t * ROWS * 4, LDC)
    threads = [threading.Thread(target=work, args=(t,)) for t in range(THREADS)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    return c, want
