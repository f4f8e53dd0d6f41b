"""Golden vectors: outputs of the UNMODIFIED reference (tests/golden/make_golden.py, generated in the build
container) for seeded inputs. They pin
  * the CPU oracle (oracle/oracle.c)                 -- `-m "not gpu"`, runs anywhere;
  * the CUDA kernels through the C ABI               -- `-m gpu`, also on a box without /root/reference.
Bars: bit-exact for GEMM (the reference C kernel defines the operation order, which oracle and the exact-order CUDA
kernel both keep). BCSC, EDGE and fsspmdm fixtures come from the reference's x86 JIT. The f32 BCSC and the EDGE packed kernels
keep the oracle's order with one FMA per product, so they are bit-exact too, like the integer cases; bf16 BCSC (dot-product
instructions) and fsspmdm (kernel picked by timing) are held to the reference drivers' norms."""
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import cases  # noqa: E402
import gen  # noqa: E402
import golden_cases as G  # noqa: E402
from oracle_ffi import oracle, run_gemm  # noqa: E402

GEMM = np.load(os.path.join(HERE, "golden", "gemm.npz"))
INT8 = np.load(os.path.join(HERE, "golden", "int8.npz"))
SPARSE = np.load(os.path.join(HERE, "golden", "sparse.npz"))
MTX = np.load(os.path.join(HERE, "golden", "mtx.npz"))


def crc(*arrs):
    c = 0
    for a in arrs:
        c = zlib.crc32(np.ascontiguousarray(a).view(np.uint8).tobytes(), c)
    return np.uint32(c)


def sparse_thr(tc, kind):
    if tc in (gen.I32,):
        return 0.0
    return {gen.BF16: 5e-3, gen.F32: 1e-4, gen.F64: 1e-8}[tc]


def test_gemm_golden_pins_the_oracle():
    lst = G.gemm_cases()
    assert len(lst) * 2 == len(GEMM.files)
    for i, (case, seed, count) in enumerate(lst):
        ops = cases.Operands(case, seed=seed, count=count)
        assert crc(ops.a, ops.b, ops.c0) == GEMM["gemm_%03d_crc" % i], "input generator drifted: regenerate the fixtures"
        got = cases.ref_result(oracle, case, ops, run_gemm)
        assert np.array_equal(got.view(np.uint8), GEMM["gemm_%03d" % i].view(np.uint8)), case


def test_int8_full_range_golden_pins_the_oracle():
    case, ops = G.int8_full_range()
    assert crc(ops.a, ops.b, ops.c0) == INT8["crc"], "input generator drifted: regenerate the fixtures"
    assert np.array_equal(cases.ref_result(oracle, case, ops, run_gemm), INT8["gemm"]), case


def test_sparse_golden_pins_the_oracle():
    for i, cfg in enumerate(G.bcsc_cases()):
        inp = G.bcsc_inputs(cfg)
        assert crc(inp["a"], inp["bvals"], inp["colptr"], inp["rowidx"], inp["c0"]) == SPARSE["bcsc_%02d_crc" % i]
        c = inp["c0"].copy()
        assert G.run_bcsc(oracle, cfg, inp, c) == 0
        tc = cfg["types"][3]
        if tc == gen.F32:
            assert np.array_equal(SPARSE["bcsc_%02d" % i].view(np.uint8), c.view(np.uint8)), cfg
        assert gen.normf_rel(gen.to_f64(SPARSE["bcsc_%02d" % i], tc), gen.to_f64(c, tc)) <= sparse_thr(tc, "bcsc"), cfg
    for i, cfg in enumerate(G.fsspmdm_cases()):
        inp = G.fsspmdm_inputs(cfg)
        assert crc(inp["a"], inp["b"], inp["c0"]) == SPARSE["fsspmdm_%02d_crc" % i]
        c = inp["c0"].copy()
        assert G.run_fsspmdm(oracle, cfg, inp, c) == 0
        assert gen.normf_rel(SPARSE["fsspmdm_%02d" % i], c) <= sparse_thr(cfg["dtype"], "fsspmdm"), cfg


def test_reference_operator_files_pin_the_oracle():
    """PyFR (samples/xgemm_sparse_Ainregs/mats) and EDGE (samples/xgemm_norm_packed/mats) operators: reference JIT output
    stored in mtx.npz against the oracle restatement on the same seeded dense operands; EDGE bit for bit"""
    for i, cfg in enumerate(G.pyfr_cases()):
        inp = G.pyfr_inputs(cfg)
        assert crc(inp["a"], inp["b"], inp["c0"]) == MTX["pyfr_%02d_crc" % i]
        c = inp["c0"].copy()
        assert G.run_pyfr(oracle, cfg, inp, c) == 0
        assert gen.normf_rel(MTX["pyfr_%02d" % i], c) <= sparse_thr(cfg["dtype"], "fsspmdm"), cfg
    for i, cfg in enumerate(G.edge_cases()):
        inp = G.edge_inputs(cfg)
        assert crc(inp["ptr"], inp["idx"], inp["a"], inp["b"], inp["c0"]) == MTX["edge_%02d_crc" % i]
        c = inp["c0"].copy()
        assert G.run_edge(oracle, cfg, inp, c) == 0
        assert np.array_equal(MTX["edge_%02d" % i].view(np.uint8), c.view(np.uint8)), cfg


@pytest.mark.gpu
def test_reference_operator_files_on_gpu():
    import libxsmm_b200 as X
    from gpu_util import dev, host
    for i, cfg in enumerate(G.pyfr_cases()):
        inp = G.pyfr_inputs(cfg)
        M, K, N = inp["M"], inp["K"], cfg["N"]
        h = X.libxsmm_fsspmdm_create(cfg["dtype"], M, N, K, K, N, N, inp["alpha"].ctypes.data, inp["beta"].ctypes.data, inp["a"].ctypes.data, 0, None)
        assert h, cfg
        d_b, d_c = dev(inp["b"]), dev(inp["c0"])
        X.libxsmm_fsspmdm_execute(h, d_b.data_ptr(), d_c.data_ptr()); X.check()
        assert gen.normf_rel(MTX["pyfr_%02d" % i], host(d_c, gen.NP_OF[cfg["dtype"]])) <= sparse_thr(cfg["dtype"], "fsspmdm"), cfg
        X.libxsmm_fsspmdm_destroy(h)
    for i, cfg in enumerate(G.edge_cases()):
        inp = G.edge_inputs(cfg)
        dt = cfg["dtype"]
        create = X.libxsmm_create_packed_spgemm_csc if inp["is_csc"] else X.libxsmm_create_packed_spgemm_csr
        k = create(X.libxsmm_create_gemm_shape(*inp["dims"], dt, dt, dt, dt), inp["flags"], 0, cfg["P"], inp["ptr"].ctypes.data, inp["idx"].ctypes.data,
                   inp["vals"].ctypes.data)
        assert k, cfg
        d_a, d_b, d_c = dev(inp["a"]), dev(inp["b"]), dev(inp["c0"])
        X.call_gemm(k, d_a, d_b, d_c); X.check()
        assert np.array_equal(MTX["edge_%02d" % i].view(np.uint8), host(d_c, np.uint8)), cfg
        X.libxsmm_release_kernel(k)


@pytest.mark.gpu
def test_gemm_golden_on_gpu():
    import libxsmm_b200 as X
    from gpu_util import dev, dispatch, host, run_single_calls
    for force_simt in (1, 0):
        X.libxsmm_b200_set_force_simt(force_simt)
        try:
            for i, (case, seed, count) in enumerate(G.gemm_cases()):
                ops = cases.Operands(case, seed=seed, count=count)
                kernel = dispatch(case, ops)
                assert kernel, case
                d_a, d_b, d_c = dev(ops.a), dev(ops.b), dev(ops.c0)
                run_single_calls(kernel, case, ops, d_a, d_b, d_c)
                got = host(d_c, gen.NP_OF[case.tc])
                want = GEMM["gemm_%03d" % i]
                if X.libxsmm_b200_kernel_backend(kernel) == X.BACKEND_TCGEN05:
                    thr = 1.2e-5 if case.tc == gen.F32 else 5e-3
                    assert gen.normf_rel(gen.to_f64(want, case.tc), gen.to_f64(got, case.tc)) <= thr, case
                else:
                    assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), case
        finally:
            X.libxsmm_b200_set_force_simt(0)


@pytest.mark.gpu
def test_int8_full_range_golden_on_gpu():
    """the full-range int8 vector on the wgmma kernel (strided batch) and on the dp4a kernel (forced exact-order): bit for bit"""
    import libxsmm_b200 as X
    from gpu_util import dev, dispatch, host
    case, ops = G.int8_full_range()
    for force_simt, backend in ((0, X.BACKEND_TCGEN05), (1, X.BACKEND_SIMT)):
        X.libxsmm_b200_set_force_simt(force_simt)
        try:
            kernel = dispatch(case, ops)
        finally:
            X.libxsmm_b200_set_force_simt(0)
        assert kernel and X.libxsmm_b200_kernel_backend(kernel) == backend
        d_a, d_b, d_c = dev(ops.a), dev(ops.b), dev(ops.c0)
        before = X.libxsmm_b200_launch_count_backend(backend)
        assert X.libxsmm_b200_gemm_batch_strided(kernel, d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), ops.tile_a, ops.tile_b, ops.tile_c, case.br, ops.count) == 0
        X.check()
        assert X.libxsmm_b200_launch_count_backend(backend) > before
        assert np.array_equal(host(d_c, np.int32), INT8["gemm"]), backend


@pytest.mark.gpu
def test_sparse_golden_on_gpu():
    import ctypes as C
    import libxsmm_b200 as X
    from gpu_util import dev, host
    for i, cfg in enumerate(G.bcsc_cases()):
        inp = G.bcsc_inputs(cfg)
        ta, tb, tcomp, tc = cfg["types"]
        mblocks, M, K, N, bk, bn = cfg["geo"]
        sh = X.libxsmm_create_gemm_shape(mblocks, 0, K, K, 0, N, ta, tb, tc, tcomp)
        k = X.libxsmm_create_packed_spgemm_bcsc(sh, G.bcsc_flags(cfg), 0, X.SpgemmConfig(M, bk, bn))
        assert k, cfg
        d_a, d_b, d_c = dev(inp["a"]), dev(inp["bvals"]), dev(inp["c0"])
        X.call_gemm(k, d_a, d_b, d_c, colptr=inp["colptr"], rowidx=inp["rowidx"], nblocks=N // bn)   # host-side pattern, device matrices
        X.check()
        got = host(d_c, gen.NP_OF[tc])
        if tc == gen.F32:                  # the exact-order kernel, one FMA per product like the reference's VFMADD231PS
            assert np.array_equal(SPARSE["bcsc_%02d" % i].view(np.uint8), got.view(np.uint8)), cfg
        assert gen.normf_rel(gen.to_f64(SPARSE["bcsc_%02d" % i], tc), gen.to_f64(got, tc)) <= sparse_thr(tc, "bcsc"), cfg
        X.libxsmm_release_kernel(k)
    for i, cfg in enumerate(G.fsspmdm_cases()):
        inp = G.fsspmdm_inputs(cfg)
        M, K, N = cfg["M"], cfg["K"], cfg["N"]
        h = X.libxsmm_fsspmdm_create(cfg["dtype"], M, N, K, K, N, N, inp["alpha"].ctypes.data, inp["beta"].ctypes.data, inp["a"].ctypes.data, 0, None)
        assert h, cfg
        d_b, d_c = dev(inp["b"]), dev(inp["c0"])
        X.libxsmm_fsspmdm_execute(h, d_b.data_ptr(), d_c.data_ptr())
        X.check()
        got = host(d_c, gen.NP_OF[cfg["dtype"]])
        assert gen.normf_rel(SPARSE["fsspmdm_%02d" % i], got) <= sparse_thr(cfg["dtype"], "fsspmdm"), cfg
        X.libxsmm_fsspmdm_destroy(h)
