"""Low-bit weight GEMM (I2X4 / I1X8 x I8 / U8 -> I32, MXFP4X2 x I8 -> F32 / BF16) on the GPU: the dp4a kernel, element by element.

 * The fixture tests/golden/lowbit.npz (bytes computed by the reference) and the oracle (oracle/oracle_lowbit.c) must be matched bit
   for bit, NaN positions excepted (the sign of a NaN made from inf - inf is the host's choice), for device, pinned and pageable
   operands in every batch-reduce mode; C padding rows (ldc > m) come back untouched.
 * Every handle reports the CUDA-core backend and every call runs exactly one CUDA-core launch and no tensor-core kernel.
 * The batch forms equal one call per tile: I2 / I1 through the plain strided form (host and device operands), _multi with one device
   and libxsmm_b200_gemm_batch; MXFP4 through libxsmm_b200_gemm_batch_strided_scaled (per-tile and shared scales) and
   libxsmm_b200_gemm_batch. The refused forms return -6 and leave C untouched.
 * The reference's own samples/xgemm/gemm_kernel.c driver, unmodified, passes by its own verdict for each tuple."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import libxsmm_b200 as X
from gpu_util import dev, host
from lowbit_ffi import BF16, F32, I1, I2, I8, I32, MXFP4, TUPLES, U8, LbCase, case_from_meta, oracle_gemm_lowbit, same_c

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lowbit.npz")
SIMT, TC = X.BACKEND_SIMT, X.BACKEND_TCGEN05
NOT_BATCHABLE = -6                                 # LIBXSMM_B200_ERROR_NOT_BATCHABLE
BRT = {0: None, 1: X.GEMM_BATCH_REDUCE_ADDRESS, 2: X.GEMM_BATCH_REDUCE_OFFSET, 3: X.GEMM_BATCH_REDUCE_STRIDE}


class Launches:
    def __init__(self):
        self.simt, self.tc = X.libxsmm_b200_launch_count_backend(SIMT), X.libxsmm_b200_launch_count_backend(TC)

    def expect(self, simt):
        assert X.libxsmm_b200_launch_count_backend(SIMT) - self.simt == simt
        assert X.libxsmm_b200_launch_count_backend(TC) == self.tc


def handle(case):
    sh = X.libxsmm_create_gemm_shape(case.m, case.n, case.k, case.lda, case.ldb, case.ldc, case.ta, case.tb, case.tc, I32)
    if case.br_type == 0:
        h = X.libxsmm_dispatch_gemm(sh, case.flags, 0)
    else:
        h = X.libxsmm_dispatch_brgemm(sh, case.flags, 0, X.libxsmm_create_gemm_batch_reduce_config(BRT[case.br_type], case.stride_a, case.stride_b, 0))
    assert h and X.libxsmm_b200_kernel_backend(h) == SIMT
    return h


def fill_param(case, p, pa, pb, pc, psa, psb, keep):
    """a libxsmm_gemm_param for one call on operands at addresses pa / pb / pc and scales at psa / psb (block r right after block r-1)"""
    br = C.c_ulonglong(case.br); keep.append(br)
    p.op.tertiary = C.addressof(br)
    p.a.primary, p.b.primary, p.c.primary = pa, pb, pc
    if case.mx():
        p.a.tertiary, p.b.tertiary = psa, psb
    if case.br_type == 1:                  # host arrays of block addresses (and of the blocks' scales)
        arrs = [(C.c_void_p * case.br)(*[base + r * step for r in range(case.br)])
                for base, step in ((pa, case.block_a), (pb, case.block_b), (psa, case.block_sa), (psb, 4 * case.block_sb))]
        keep += arrs
        p.a.primary, p.b.primary = C.addressof(arrs[0]), C.addressof(arrs[1])
        if case.mx():
            p.a.tertiary, p.b.tertiary = C.addressof(arrs[2]), C.addressof(arrs[3])
    elif case.br_type == 2:                # blocks in reverse order, host offset arrays
        oa = np.array([(case.br - 1 - r) * case.block_a for r in range(case.br)], np.int64)
        ob = np.array([(case.br - 1 - r) * case.block_b for r in range(case.br)], np.int64)
        keep += [oa, ob]
        p.a.secondary, p.b.secondary = oa.ctypes.data, ob.ctypes.data


def run_single(case, ops, where="device"):
    """one call with operands in device memory, pinned host memory or pageable host memory; returns C"""
    A, B, C0, SA, SB = ops
    h = handle(case)
    cnt = Launches()
    keep = []
    p = X.GemmParam()
    if where == "pageable":
        c = C0.copy()
        fill_param(case, p, A.ctypes.data, B.ctypes.data, c.ctypes.data, SA.ctypes.data, SB.ctypes.data, keep)
        X.GEMMFUNCTION(h)(C.byref(p)); X.check()
        out = c
    else:
        if where == "device":
            bufs = [dev(x) for x in (A, B, C0, SA, SB)]
        else:
            bufs = [torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).copy()).pin_memory() for x in (A, B, C0, SA, SB)]
        fill_param(case, p, *[t.data_ptr() for t in bufs], keep)
        X.GEMMFUNCTION(h)(C.byref(p))
        torch.cuda.synchronize(); X.check()
        out = host(bufs[2], C0.dtype) if where == "device" else bufs[2].numpy().view(C0.dtype).copy()
    cnt.expect(1)
    return out


def golden_cases():
    g = np.load(GOLDEN)
    return [(case_from_meta(g["meta%d" % t]), [g["%s%d" % (nm, t)] for nm in ("a", "b", "c0", "sa", "sb")], g["c%d" % t])
            for t in range(int(g["ncases"]))]


@pytest.mark.parametrize("where", ["device", "pinned", "pageable"])
def test_kernel_equals_the_reference_fixture(where):
    for case, ops, want in golden_cases():
        got = run_single(case, ops, where)
        assert same_c(case, want, got), (where, case)
        pad = got.reshape(case.n, case.ldc)[:, case.m:]
        assert np.array_equal(pad.view(np.uint8), ops[2].reshape(case.n, case.ldc)[:, case.m:].view(np.uint8)), case


def parity_cases():
    out = []
    for ta, tb, tc in TUPLES:
        for br_type in (0, 1, 2, 3):
            for beta0 in (True, False):
                m = {I2: 76, I1: 70, MXFP4: 45}[ta]
                k = 288 if ta == MXFP4 else 268          # past one 128-k panel of B
                out.append(LbCase(ta, tb, tc, m, 37, k, lda=m + 8, ldb=k + 4, ldc=m + 3, beta0=beta0, br_type=br_type, br=3))
    out.append(LbCase(I2, U8, I32, 8, 300, 36, lda=8, ldb=37, ldc=9, beta0=False))          # two panels of columns, unaligned B rows
    out.append(LbCase(I1, I8, I32, 2, 1, 4, beta0=False))
    out.append(LbCase(MXFP4, I8, BF16, 1, 259, 32, lda=3, ldb=33, ldc=1, beta0=False, br_type=3, br=2))
    return out


@pytest.mark.parametrize("case", parity_cases(), ids=repr)
def test_kernel_equals_the_oracle(case):
    ops = case.operands(np.random.default_rng(case.m * 1000 + case.n + case.br_type))
    want = case.run(oracle_gemm_lowbit, *ops)[1]
    assert same_c(case, want, run_single(case, ops, "device")), case


def _strided(case, count, rng):
    tiles = [case.operands(rng) for _ in range(count)]
    return tiles, [np.concatenate([t[i] for t in tiles]) for i in range(5)]


@pytest.mark.parametrize("ta,tb", [(I2, I8), (I1, U8)])
def test_integer_forms_batch_in_every_form(ta, tb):
    rng = np.random.default_rng(11)
    count = 9
    case = LbCase(ta, tb, I32, 64, 64, 256, beta0=False, br_type=3, br=2)
    h = handle(case)
    tiles, (A, B, Cs, _, _) = _strided(case, count, rng)
    wants = [case.run(oracle_gemm_lowbit, *t)[1] for t in tiles]
    sa, sb, sc = case.size_a, case.size_b, 4 * case.size_c
    check = lambda got: [same_c(case, wants[t], got[t * case.size_c:(t + 1) * case.size_c]) for t in range(count)]
    d = [dev(x) for x in (A, B, Cs)]
    cnt = Launches()
    assert X.libxsmm_b200_gemm_batch_strided(h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), sa, sb, sc, case.br, count) == 0
    X.check(); cnt.expect(1)
    assert all(check(host(d[2], np.int32)))
    c = Cs.copy()
    assert X.libxsmm_b200_gemm_batch_strided(h, A.ctypes.data, B.ctypes.data, c.ctypes.data, sa, sb, sc, case.br, count) == 0
    X.check()
    assert all(check(c))
    c = Cs.copy()
    assert X.libxsmm_b200_gemm_batch_strided_multi(h, A.ctypes.data, B.ctypes.data, c.ctypes.data, sa, sb, sc, case.br, count, 1) == 0
    X.check()
    assert all(check(c))
    d = [dev(x) for x in (A, B, Cs)]
    params = (X.GemmParam * count)()
    brc = C.c_ulonglong(case.br)
    for t in range(count):
        params[t].op.tertiary = C.addressof(brc)
        params[t].a.primary, params[t].b.primary = d[0].data_ptr() + t * sa, d[1].data_ptr() + t * sb
        params[t].c.primary = d[2].data_ptr() + t * sc
    assert X.libxsmm_b200_gemm_batch(h, params, count) == 0
    torch.cuda.synchronize(); X.check()
    assert all(check(host(d[2], np.int32)))
    plan = X.libxsmm_b200_gemm_plan_create(h, params, count)
    assert plan
    X.libxsmm_b200_gemm_plan_destroy(plan)


@pytest.mark.parametrize("tc", [F32, BF16])
def test_mxfp4_batches_through_the_scaled_and_per_tile_forms(tc):
    rng = np.random.default_rng(12)
    count = 7
    case = LbCase(MXFP4, I8, tc, 64, 64, 256, beta0=False, br_type=3, br=2)
    h = handle(case)
    tiles, (A, B, Cs, SA, SB) = _strided(case, count, rng)
    d = [dev(x) for x in (A, B, Cs, SA, SB)]
    for shared in (False, True):
        wants = [case.run(oracle_gemm_lowbit, tiles[t][0], tiles[t][1], tiles[t][2], tiles[0][3] if shared else tiles[t][3],
                          tiles[0][4] if shared else tiles[t][4])[1] for t in range(count)]
        d[2].copy_(dev(Cs))
        cnt = Launches()
        assert X.libxsmm_b200_gemm_batch_strided_scaled(h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), case.size_a, case.size_b,
                                                        case.size_c * Cs.itemsize, d[3].data_ptr(), d[4].data_ptr(), None,
                                                        0 if shared else case.size_sa, 0 if shared else 4 * case.size_sb, 0, case.br, count) == 0
        torch.cuda.synchronize(); X.check(); cnt.expect(1)
        got = host(d[2], Cs.dtype)
        for t in range(count):
            assert same_c(case, wants[t], got[t * case.size_c:(t + 1) * case.size_c]), (shared, t)
    # per-tile records, address mode: each record's a.tertiary / b.tertiary are host arrays of block pointers
    case = LbCase(MXFP4, I8, tc, 40, 24, 96, lda=44, ldb=96, ldc=41, beta0=False, br_type=1, br=3)
    h = handle(case)
    tiles, (A, B, Cs, SA, SB) = _strided(case, count, rng)
    wants = [case.run(oracle_gemm_lowbit, *t)[1] for t in tiles]
    d = [dev(x) for x in (A, B, Cs, SA, SB)]
    params = (X.GemmParam * count)()
    keep = []
    for t in range(count):
        fill_param(case, params[t], d[0].data_ptr() + t * case.size_a, d[1].data_ptr() + t * case.size_b,
                   d[2].data_ptr() + t * case.size_c * Cs.itemsize, d[3].data_ptr() + t * case.size_sa, d[4].data_ptr() + t * 4 * case.size_sb, keep)
    cnt = Launches()
    assert X.libxsmm_b200_gemm_batch(h, params, count) == 0
    torch.cuda.synchronize(); X.check(); cnt.expect(1)
    got = host(d[2], Cs.dtype)
    for t in range(count):
        assert same_c(case, wants[t], got[t * case.size_c:(t + 1) * case.size_c]), t
    assert not X.libxsmm_b200_gemm_plan_create(h, params, count)


def test_refused_forms_leave_c_untouched():
    case = LbCase(MXFP4, I8, F32, 32, 16, 64, beta0=False)
    h = handle(case)
    A, B, C0, SA, SB = case.operands(np.random.default_rng(13))
    d = [dev(x) for x in (A, B, C0, SA, SB)]
    cnt = Launches()
    assert X.libxsmm_b200_gemm_batch_strided(h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), 0, 0, 0, 1, 1) == NOT_BATCHABLE
    assert X.libxsmm_b200_gemm_batch_strided_multi(h, A.ctypes.data, B.ctypes.data, C0.ctypes.data, 0, 0, 0, 1, 1, 1) == NOT_BATCHABLE
    torch.cuda.synchronize(); cnt.expect(0)
    assert np.array_equal(host(d[2], np.uint8), C0.view(np.uint8))


# samples/xgemm/gemm_kernel.c: A B Comp C  M N K LDA LDB LDC  alpha beta  alignA alignC  trA trB  vnniA vnniB vnniC  prefetch  br-kind br-count
# br-unroll  reps  tilecfg. ldb is a multiple of 32 (the driver's gold places B's MXFP4 scales per block at (ldb/32) * n floats).
DRIVER_RUNS = [("I2 I8 I32 I32", "nobr"), ("I2 U8 I32 I32", "strdbr"), ("I1 I8 I32 I32", "addrbr"), ("I1 U8 I32 I32", "offsbr"),
               ("MXFP4 I8 I32 F32", "strdbr"), ("MXFP4 I8 I32 BF16", "addrbr")]


@pytest.mark.parametrize("types,br", DRIVER_RUNS, ids=lambda x: x.replace(" ", "_"))
def test_reference_gemm_kernel_driver_passes(types, br):
    import subprocess
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    from ref_drivers import LIBDIR, OUT
    exe = os.path.join(OUT, "gemm_kernel")
    if not os.path.exists(exe):
        pytest.skip("gemm_kernel was not built: build() compiles the drivers where the reference sources exist")
    beta = 0 if br in ("strdbr", "offsbr") else 1
    args = types.split() + [64, 48, 128, 64, 128, 64, 1, beta, 0, 0, 0, 0, 0, 0, 0, "nopf", br, 1 if br == "nobr" else 4, 0, 3, 0]
    env = dict(os.environ, LD_LIBRARY_PATH=LIBDIR + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="4")
    p = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=300, env=env, cwd=OUT)
    assert p.returncode == 0, (p.stdout[-1500:], p.stderr[-800:])
    assert "JIT failed" not in p.stdout and "FAILED" not in p.stdout.upper(), p.stdout[-1500:]
    if types.split()[0] in ("I2", "I1"):
        assert "Total Max Error 0.0000" in p.stdout, p.stdout[-1500:]
