"""GPU parity of the sparse kernels through the C ABI: fsspmdm, BCSC, packed CSR/CSC."""
import ctypes as C

import numpy as np
import pytest
import torch

import cases
import gen
import libxsmm_b200 as X
from gpu_util import dev, host
from oracle_ffi import iarr, oracle, ref
from test_oracle_vs_ref import _bcsc_inputs, _run_bcsc

pytestmark = pytest.mark.gpu


def _fsspmdm_case(rng, dtype, M, K, N, density, lda=None, ldb=None, ldc=None, uniq=True):
    npdt = gen.NP_OF[dtype]
    lda, ldb, ldc = lda or K, ldb or N, ldc or N
    a = np.zeros(M * lda, dtype=npdt)
    vals = gen.values(rng, M * K, gen.F64) if uniq else rng.standard_normal(M * K)
    a.reshape(M, lda)[:, :K] = (vals * (rng.random(M * K) < density)).reshape(M, K).astype(npdt)
    b = rng.standard_normal(K * ldb).astype(npdt); c0 = rng.standard_normal(M * ldc).astype(npdt)
    return a, b, c0, lda, ldb, ldc


@pytest.mark.parametrize("dtype,eps", [(gen.F32, 1e-4), (gen.F64, 1e-8)])
def test_fsspmdm_matches_oracle(dtype, eps):
    """thresholds of samples/xgemm_sparse_Ainregs/pyfr_driver_asp_reg.c:18-20 (matdiff epsilon)"""
    rng = np.random.default_rng(21)
    for (M, K, N, dens, pad) in ((32, 128, 4096, 0.15, 0), (192, 96, 1024, 0.02, 0), (7, 5, 64, 0.6, 16), (48, 200, 2048 + 64, 0.1, 0),
                                 (33, 300, 512, 0.05, 0), (64, 700, 256, 0.03, 0)):
        for beta in (0.0, 1.0):
            a, b, c0, lda, ldb, ldc = _fsspmdm_case(rng, dtype, M, K, N, dens, ldb=N + pad, ldc=N + pad)
            npdt = gen.NP_OF[dtype]
            alpha = np.array([0.5], dtype=npdt); bt = np.array([beta], dtype=npdt)
            h = X.libxsmm_fsspmdm_create(dtype, M, N, K, lda, ldb, ldc, alpha.ctypes.data, bt.ctypes.data, a.ctypes.data, 0, None)
            assert h, (M, K, N)
            d_b, d_c = dev(b), dev(c0)
            X.libxsmm_fsspmdm_execute(h, d_b.data_ptr(), d_c.data_ptr()); X.check()
            got = host(d_c, npdt)
            want = c0.copy()
            assert oracle["fsspmdm"](dtype, M, N, K, lda, ldb, ldc, alpha.ctypes.data, bt.ctypes.data, a.ctypes.data, b.ctypes.data, want.ctypes.data) == 0
            g, w = got.reshape(M, ldc), want.reshape(M, ldc)
            assert gen.normf_rel(w[:, :N], g[:, :N]) <= eps, (M, K, N, beta)
            assert np.array_equal(g[:, N:], c0.reshape(M, ldc)[:, N:])
            # host-pointer execution (the reference calling convention) gives the same result
            c_h = c0.copy()
            X.libxsmm_fsspmdm_execute(h, b.ctypes.data, c_h.ctypes.data); X.check()
            assert np.array_equal(c_h, got)
            X.libxsmm_fsspmdm_destroy(h)


def test_fsspmdm_invalid_inputs_return_null():
    a = np.ones(64, dtype=np.float32); one = np.array([1.0], dtype=np.float32); two = np.array([2.0], dtype=np.float32)
    assert not X.libxsmm_fsspmdm_create(gen.F32, 8, 24, 8, 8, 24, 24, one.ctypes.data, one.ctypes.data, a.ctypes.data, 0, None)   # N % 16
    assert not X.libxsmm_fsspmdm_create(gen.F32, 8, 32, 8, 8, 32, 32, one.ctypes.data, two.ctypes.data, a.ctypes.data, 0, None)   # beta = 2
    assert not X.libxsmm_fsspmdm_create(gen.F32, 8, 32, 8, 4, 32, 32, one.ctypes.data, one.ctypes.data, a.ctypes.data, 0, None)   # lda < K
    z = np.zeros(64, dtype=np.float32)
    assert not X.libxsmm_fsspmdm_create(gen.F32, 8, 32, 8, 8, 32, 32, one.ctypes.data, one.ctypes.data, z.ctypes.data, 0, None)   # empty A
    assert not X.libxsmm_fsspmdm_create(gen.F32, 8, 32, 8, 8, 32, 32, one.ctypes.data, one.ctypes.data, None, 0, None)


@pytest.mark.parametrize("types", [(gen.F32, gen.F32, gen.F32, gen.F32), (gen.BF16, gen.BF16, gen.F32, gen.BF16),
                                   (gen.U8, gen.I8, gen.I32, gen.I32), (gen.I8, gen.U8, gen.I32, gen.I32)])
def test_bcsc_bit_exact_vs_oracle(types):
    rng = np.random.default_rng(31)
    ta, tb, tcomp, tc = types
    for (mblocks, M, K, N, bk, bn, dens) in ((5, 32, 128, 64, 32, 16, 0.5), (3, 16, 64, 96, 16, 32, 0.3), (2, 64, 256, 128, 32, 32, 0.5), (4, 8, 32, 32, 8, 8, 0.9)):
        if ta != gen.F32 and bk % (2 if ta == gen.BF16 else 4):
            continue
        for beta0, trans_a in ((1, 0), (0, 0), (1, 1)):
            flags = (cases.FLAG_BETA_0 if beta0 else 0) | (cases.FLAG_VNNI_A if (ta != gen.F32 and not trans_a) else 0) | (cases.FLAG_TRANS_A if trans_a else 0)
            a, bvals, colptr, rowidx, c0 = _bcsc_inputs(rng, ta, tb, tc, mblocks, M, K, N, bk, bn, dens)
            sh = X.libxsmm_create_gemm_shape(mblocks, 0, K, K, 0, N, ta, tb, tc, tcomp)
            cfg = X.SpgemmConfig(M, bk, bn)
            kernel = X.libxsmm_create_packed_spgemm_bcsc(sh, flags, 0, cfg)
            assert kernel
            d_a, d_b, d_cp, d_ri, d_c = dev(a), dev(bvals), dev(colptr), dev(rowidx), dev(c0)
            X.call_gemm(kernel, d_a, d_b, d_c, colptr=d_cp, rowidx=d_ri, nblocks=N // bn); X.check()
            got = host(d_c, gen.NP_OF[tc])
            want = c0.copy()
            assert _run_bcsc(oracle, types, (mblocks, M, K, N, bk, bn), flags, a, bvals, colptr, rowidx, want) == 0
            if tc == gen.I32:
                assert np.array_equal(got, want), (types, mblocks, M, K, N)
            else:
                thr = 5e-3 if tc == gen.BF16 else 1e-4          # spmm_kernel.c:1019-1029
                assert gen.normf_rel(gen.to_f64(want, tc), gen.to_f64(got, tc)) <= thr, (types, mblocks, M, K, N, beta0, trans_a)
            X.libxsmm_release_kernel(kernel)


def _bcsc_bf16_run(rng, mblocks, M, K, N, bk, bn, dens, beta0, expect_variant, thr=5e-3):
    ta = gen.BF16
    types = (ta, ta, gen.F32, ta)
    flags = (cases.FLAG_BETA_0 if beta0 else 0) | cases.FLAG_VNNI_A
    a, bvals, colptr, rowidx, c0 = _bcsc_inputs(rng, ta, ta, ta, mblocks, M, K, N, bk, bn, dens)
    sh = X.libxsmm_create_gemm_shape(mblocks, 0, K, K, 0, N, ta, ta, ta, gen.F32)
    kernel = X.libxsmm_create_packed_spgemm_bcsc(sh, flags, 0, X.SpgemmConfig(M, bk, bn))
    assert kernel
    assert X.libxsmm_b200_bcsc_variant(kernel, N // bn) == expect_variant, (mblocks, M, K, N, bk, bn, X.libxsmm_b200_bcsc_variant(kernel, N // bn))
    assert X.libxsmm_b200_kernel_backend(kernel) == (X.BACKEND_TCGEN05 if expect_variant else X.BACKEND_SIMT)
    d_a, d_b, d_cp, d_ri, d_c = dev(a), dev(bvals), dev(colptr), dev(rowidx), dev(c0)
    want = c0.copy()
    assert _run_bcsc(oracle, types, (mblocks, M, K, N, bk, bn), flags, a, bvals, colptr, rowidx, want) == 0
    for rep in range(2):     # a second call on the same handle gives the same result
        d_c.copy_(dev(c0))
        X.call_gemm(kernel, d_a, d_b, d_c, colptr=d_cp, rowidx=d_ri, nblocks=N // bn); X.check()
        err = gen.normf_rel(gen.to_f64(want, ta), gen.to_f64(host(d_c, np.uint16), ta))
        assert err <= thr, ((mblocks, M, K, N, bk, bn, dens, beta0), rep, err)
    X.libxsmm_release_kernel(kernel)


# (m_blocks, M, K, N, bk, bn, density): packed widths 16..128, all three block depths, ragged groups (m_blocks not a multiple of
# 128/M), K not a multiple of 64, N not a multiple of the 128-column part, empty block-columns (low density), dense B
_BCSC_TC_GEOMETRIES = ((4, 32, 64, 64, 32, 32, 1.0), (4, 32, 128, 64, 32, 32, 0.5), (5, 32, 512, 512, 32, 32, 0.5), (3, 16, 64, 96, 16, 32, 0.5),
                       (2, 64, 256, 128, 32, 16, 0.5), (3, 32, 128, 128, 64, 32, 0.5), (9, 32, 96, 320, 32, 32, 0.4), (3, 128, 160, 64, 16, 16, 0.6),
                       (7, 32, 512, 512, 32, 32, 0.1), (6, 64, 448, 384, 64, 128, 0.7), (11, 16, 192, 48, 16, 48, 0.8))


def test_bcsc_bf16_tensor_core_kernel():
    """the wgmma BCSC kernel against the oracle, incl. the BASELINE configs[3] geometry (M=32, N=K=512, 32x32 blocks, 50%) at a
    small m_blocks; thresholds of samples/xgemm_sparse/spmm_kernel.c:1019-1029"""
    rng = np.random.default_rng(77)
    for geo in _BCSC_TC_GEOMETRIES:
        for beta0 in (1, 0):
            _bcsc_bf16_run(rng, *geo, beta0, expect_variant=1)


def test_bcsc_bf16_kernel_selection_by_geometry(monkeypatch):
    """K > 512, N > 512 and bn > 128 are all served by the tensor-core kernel; K < 64 or an unsupported block shape -> exact-order
    kernel"""
    rng = np.random.default_rng(5)
    _bcsc_bf16_run(rng, 5, 32, 640, 256, 32, 32, 0.5, 1, expect_variant=1)
    _bcsc_bf16_run(rng, 5, 32, 256, 1024, 32, 32, 0.4, 1, expect_variant=1)
    _bcsc_bf16_run(rng, 3, 32, 128, 512, 32, 256, 0.6, 0, expect_variant=1)
    _bcsc_bf16_run(rng, 3, 32, 32, 64, 16, 16, 0.6, 0, expect_variant=0)
    _bcsc_bf16_run(rng, 3, 8, 64, 64, 32, 32, 0.6, 1, expect_variant=0)


def test_bcsc_handle_is_reentrant_across_streams():
    """one handle, two host threads on two streams with different B values and patterns: results must not mix
    (reference handles are re-entrant, SURVEY.md 8b; scratch is kept per stream, launches are enqueued under the handle's lock)"""
    import threading
    ta = gen.BF16
    mblocks, M, K, N, bk, bn = 64, 32, 256, 256, 32, 32
    flags = cases.FLAG_BETA_0 | cases.FLAG_VNNI_A
    sh = X.libxsmm_create_gemm_shape(mblocks, 0, K, K, 0, N, ta, ta, ta, gen.F32)
    kernel = X.libxsmm_create_packed_spgemm_bcsc(sh, flags, 0, X.SpgemmConfig(M, bk, bn))
    assert kernel
    jobs = []
    for t in range(2):
        rng = np.random.default_rng(100 + t)
        a, bvals, colptr, rowidx, c0 = _bcsc_inputs(rng, ta, ta, ta, mblocks, M, K, N, bk, bn, 0.3 + 0.4 * t)
        want = c0.copy()
        assert _run_bcsc(oracle, (ta, ta, gen.F32, ta), (mblocks, M, K, N, bk, bn), flags, a, bvals, colptr, rowidx, want) == 0
        jobs.append(dict(d=[dev(x) for x in (a, bvals, colptr, rowidx, c0)], want=want, stream=torch.cuda.Stream(), errs=[]))
    torch.cuda.synchronize()

    def worker(job):
        X.libxsmm_b200_set_device(0)
        X.libxsmm_b200_set_stream(job["stream"].cuda_stream)
        X.libxsmm_b200_set_blocking(0)
        d_a, d_b, d_cp, d_ri, d_c = job["d"]
        for _ in range(20):
            X.call_gemm(kernel, d_a, d_b, d_c, colptr=d_cp, rowidx=d_ri, nblocks=N // bn)
            job["stream"].synchronize()
            job["errs"].append(gen.normf_rel(gen.to_f64(job["want"], ta), gen.to_f64(host(d_c, np.uint16), ta)))
    threads = [threading.Thread(target=worker, args=(j,)) for j in jobs]
    [th.start() for th in threads]; [th.join() for th in threads]
    X.check()
    for j in jobs:
        assert len(j["errs"]) == 20 and max(j["errs"]) <= 5e-3, j["errs"]
    X.libxsmm_release_kernel(kernel)


@pytest.mark.parametrize("kind", ["a_csr", "b_csr", "b_csc", "c_csc"])
@pytest.mark.parametrize("dtype", [gen.F32, gen.F64])
def test_packed_csr_csc_all_four_kinds(kind, dtype):
    """SOA-packed sparse x dense (EDGE/SeisSol sizes): A-sparse CSR, B-sparse CSR, B-sparse CSC (bit-exact against the
    oracle: same summation order) and C-sparse CSC (packed dimension summed away; shuffle tree => tolerance 2e-6)."""
    rng = np.random.default_rng(41)
    npdt = gen.NP_OF[dtype]
    for (M, N, K, P) in ((9, 9, 9, 8), (20, 9, 35, 16), (56, 9, 56, 64), (35, 20, 9, 16), (4, 3, 5, 1)):
        for beta0 in (0, 1):
            flags = cases.FLAG_BETA_0 if beta0 else 0
            is_csc, dims, ptr, idx, a, b, c0 = cases.packed_sp_case(rng, kind, dtype, M, N, K, P, density=0.25)
            vals = a if kind == "a_csr" else b if kind.startswith("b_") else c0
            create = X.libxsmm_create_packed_spgemm_csc if is_csc else X.libxsmm_create_packed_spgemm_csr
            k = create(X.libxsmm_create_gemm_shape(*dims, dtype, dtype, dtype, dtype), flags, 0, P, ptr.ctypes.data, idx.ctypes.data, vals.ctypes.data)
            want = c0.copy()
            rc = oracle["packed_sp"](is_csc, dtype, iarr(*dims), flags, P, ptr.ctypes.data, idx.ctypes.data, vals.ctypes.data,
                                     a.ctypes.data, b.ctypes.data, want.ctypes.data)
            if rc != 0:                      # C-sparse outside f32 / 16-lane widths: no kernel on either side
                assert kind == "c_csc" and not k
                continue
            assert k, (kind, dtype, (M, N, K, P))
            assert X.libxsmm_b200_kernel_backend(k) == X.BACKEND_STREAM
            d_a, d_b, d_c = dev(a), dev(b), dev(c0)
            X.call_gemm(k, d_a, d_b, d_c); X.check()
            got = host(d_c, npdt)
            if kind == "c_csc":
                assert gen.normf_rel(want, got) <= 2e-6, (kind, (M, N, K, P), beta0)
            else:
                assert np.array_equal(got, want), (kind, dtype, (M, N, K, P), beta0)
            # host-resident operands go through the staging path and must give the same bits
            c_h = c0.copy()
            X.call_gemm(k, a.ctypes.data, b.ctypes.data, c_h.ctypes.data); X.check()
            assert np.array_equal(c_h, got), (kind, "host pointers")
            X.libxsmm_release_kernel(k)


@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("dtype", [gen.F32, gen.F64])
def test_packed_dense_gemm_matches_oracle(kind, dtype):
    """packed dense GEMM, the three layouts of include/libxsmm.h:195-214; FMA vs separate multiply-add => tolerance"""
    rng = np.random.default_rng(95)
    create = (X.libxsmm_create_packed_gemm, X.libxsmm_create_packed_gemm_ac_rm, X.libxsmm_create_packed_gemm_bc_rm)[kind]
    for (M, N, K, P, pad) in ((9, 9, 9, 8, 0), (20, 9, 35, 16, 2), (56, 9, 56, 64, 0), (4, 3, 5, 1, 1)):
        for beta0 in (0, 1):
            dims, a, b, c0 = cases.packed_dense_case(rng, kind, dtype, M, N, K, P, pad)
            flags = cases.FLAG_BETA_0 if beta0 else 0
            k = create(X.libxsmm_create_gemm_shape(*dims, dtype, dtype, dtype, dtype), flags, 0, P)
            assert k, (kind, dims)
            want = c0.copy()
            assert oracle["packed_dense"](kind, dtype, iarr(*dims), flags, P, a.ctypes.data, b.ctypes.data, want.ctypes.data) == 0
            d_a, d_b, d_c = dev(a), dev(b), dev(c0)
            X.call_gemm(k, d_a, d_b, d_c); X.check()
            got = host(d_c, gen.NP_OF[dtype])
            assert gen.normf_rel(want, got) <= (3e-6 if dtype == gen.F32 else 1e-14), (kind, dims, P, beta0)
            hc = c0.copy()
            X.call_gemm(k, a.ctypes.data, b.ctypes.data, hc.ctypes.data); X.check()
            assert np.array_equal(hc, got), "host operands through the staging path"
            X.libxsmm_release_kernel(k)
