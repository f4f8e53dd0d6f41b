"""Dequantising GEMM (I8 x BF16, I8 / I4 / U4 / BF8 x F16 with per-row scales and zero points) on the GPU: the exact-order kernel,
element by element.

 * The fixture tests/golden/dequant.npz (bytes computed by the reference) and the oracle (oracle/oracle_dq.c) must be matched bit for
   bit, NaN positions excepted (the sign of a NaN made from 0 * inf is the host's choice: x86's default NaN is negative), for device,
   pinned and pageable operands; C padding rows (ldc > m) come back untouched.
 * Every tuple, comp, beta and batch-reduce mode against the oracle; beta = 0 over a NaN-filled C.
 * The batch forms equal one call per tile: libxsmm_b200_gemm_batch (per-tile scales and zero points),
   libxsmm_b200_gemm_batch_strided_scaled (per-tile and shared scales), and the plain strided forms for BF8 x F16, which has no scales.
 * Every call checks the launch counts: one exact-order launch per call or batch, and no tensor-core kernel runs.
 * The reference's own samples/xgemm/gemm_kernel.c driver, unmodified, passes by its own verdict."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import libxsmm_b200 as X
from dq_ffi import BF8, BF16, F16, F32, I4, I8, IMPLICIT, U4, DqCase, case_from_meta, oracle_gemm_dq, same_c
from gpu_util import dev, host

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dequant.npz")
SIMT, TC = X.BACKEND_SIMT, X.BACKEND_TCGEN05
SENTINEL = 0xA5
NOT_BATCHABLE = -6                                 # LIBXSMM_B200_ERROR_NOT_BATCHABLE
BRT = {0: None, 1: X.GEMM_BATCH_REDUCE_ADDRESS, 2: X.GEMM_BATCH_REDUCE_OFFSET, 3: X.GEMM_BATCH_REDUCE_STRIDE}


class Launches:
    def __init__(self):
        self.simt, self.tc = X.libxsmm_b200_launch_count_backend(SIMT), X.libxsmm_b200_launch_count_backend(TC)

    def expect(self, simt):
        assert X.libxsmm_b200_launch_count_backend(SIMT) - self.simt == simt
        assert X.libxsmm_b200_launch_count_backend(TC) == self.tc


def handle(case):
    sh = X.libxsmm_create_gemm_shape(case.m, case.n, case.k, case.lda, case.ldb, case.ldc, case.ta, case.tb, case.tc, case.comp)
    if case.br_type == 0:
        h = X.libxsmm_dispatch_gemm(sh, case.flags, 0)
    else:
        h = X.libxsmm_dispatch_brgemm(sh, case.flags, 0, X.libxsmm_create_gemm_batch_reduce_config(BRT[case.br_type], case.stride_a, case.stride_b, 0))
    assert h and X.libxsmm_b200_kernel_backend(h) == SIMT
    return h


def fill_param(case, p, pa, pb, pc, ps, pz, keep):
    """a libxsmm_gemm_param for one call on operands at addresses pa / pb / pc (block r of A / B right after block r-1)"""
    br = C.c_ulonglong(case.br); keep.append(br)
    p.op.tertiary = C.addressof(br)
    p.a.primary, p.b.primary, p.c.primary = pa, pb, pc
    if case.br_type == 1:                  # host arrays of block addresses
        aa = (C.c_void_p * case.br)(*[pa + r * case.block_a for r in range(case.br)])
        ab = (C.c_void_p * case.br)(*[pb + 2 * r * case.block_b for r in range(case.br)])
        keep += [aa, ab]
        p.a.primary, p.b.primary = C.addressof(aa), C.addressof(ab)
    elif case.br_type == 2:                # blocks in reverse order, host offset arrays
        oa = np.array([(case.br - 1 - r) * case.block_a for r in range(case.br)], np.int64)
        ob = np.array([2 * (case.br - 1 - r) * case.block_b for r in range(case.br)], np.int64)
        keep += [oa, ob]
        p.a.secondary, p.b.secondary = oa.ctypes.data, ob.ctypes.data
    if case.needs_scales():
        p.a.tertiary = ps
    if case.ta in (I4, U4):
        p.a.quaternary = pz


def run_single(case, ops, where="device"):
    """one call with operands in device memory, pinned host memory or pageable host memory; returns C"""
    A, B, C0, S, Z = ops
    h = handle(case)
    cnt = Launches()
    keep = []
    p = X.GemmParam()
    if where == "pageable":
        c = C0.copy()
        fill_param(case, p, A.ctypes.data, B.ctypes.data, c.ctypes.data, S.ctypes.data, Z.ctypes.data, keep)
        X.GEMMFUNCTION(h)(C.byref(p)); X.check()
        out = c
    else:
        if where == "device":
            bufs = [dev(x) for x in (A, B, C0, S, Z)]
        else:
            bufs = [torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).copy()).pin_memory() for x in (A, B, C0, S, Z)]
        fill_param(case, p, *[t.data_ptr() for t in bufs], keep)
        X.GEMMFUNCTION(h)(C.byref(p))
        torch.cuda.synchronize(); X.check()
        out = host(bufs[2], C0.dtype) if where == "device" else bufs[2].numpy().view(C0.dtype).copy()
    cnt.expect(1)
    return out


def golden_cases():
    g = np.load(GOLDEN)
    return [(case_from_meta(g["meta%d" % t]), [g["%s%d" % (nm, t)] for nm in ("a", "b", "c0", "s", "z")], g["c%d" % t])
            for t in range(int(g["ncases"]))]


@pytest.mark.parametrize("where", ["device", "pinned", "pageable"])
def test_exact_order_kernel_equals_the_reference_fixture(where):
    for case, ops, want in golden_cases():
        c = run_single(case, ops, where)
        assert same_c(case, want, c), (case, where)
        assert same_c(case, case.run(oracle_gemm_dq, *ops)[1], c), case
        pad = c.reshape(case.n, case.ldc)[:, case.m:]               # padding rows untouched
        assert np.array_equal(pad.view(np.uint8), ops[2].reshape(case.n, case.ldc)[:, case.m:].view(np.uint8)), case


TUPLES = [(I8, BF16, F32, F32), (I8, BF16, F32, BF16)] + \
         [(ta, F16, comp, tc) for ta in (I8, I4, U4, BF8) for comp in (F16, F32, IMPLICIT) for tc in (F16, F32)]


def parity_cases():
    out = []
    for n, (ta, tb, comp, tc) in enumerate(TUPLES):
        for br_type in (0, 1, 2, 3):
            tr = tb == F16 and (n + br_type) % 2 == 1
            out.append(DqCase(ta, tb, comp, tc, 37, 19, 64, lda=40, ldb=(21 if tr else 66), ldc=41, beta0=(br_type % 2 == 0), trans_b=tr,
                              vnni_a=(None if ta != BF8 else br_type >= 2), br_type=br_type, br=3))
    return out


@pytest.mark.parametrize("case", parity_cases(), ids=repr)
def test_exact_order_kernel_equals_the_oracle(case):
    ops = case.operands(np.random.default_rng(case.ta * 1000 + case.comp * 10 + case.tc + case.br_type))
    c = run_single(case, ops)
    assert same_c(case, case.run(oracle_gemm_dq, *ops)[1], c)
    assert case.nan_mask(c).mean() < 0.5


def test_beta0_runs_over_a_nan_c():
    for ta, tb, comp, tc in ((I8, BF16, F32, BF16), (I8, F16, F16, F32), (I4, F16, IMPLICIT, F16), (BF8, F16, F32, F32)):
        case = DqCase(ta, tb, comp, tc, 20, 9, 32, ldc=24, beta0=True)
        A, B, C0, S, Z = case.operands(np.random.default_rng(ta + tc))
        C0 = np.full(case.size_c, np.nan, np.float32) if tc == F32 else np.full(case.size_c, 0x7E00 if tc == F16 else 0x7FC0, np.uint16)
        c = run_single(case, [A, B, C0, S, Z])
        want = case.run(oracle_gemm_dq, A, B, C0, S, Z)[1]
        assert same_c(case, want, c), case


def _pack(arrs, pad):
    """tiles back to back, each followed by `pad` sentinel bytes; returns (buffer, stride in bytes)"""
    size = arrs[0].nbytes + pad
    buf = np.full(size * len(arrs), SENTINEL, np.uint8)
    for t, x in enumerate(arrs):
        buf[t * size:t * size + x.nbytes] = x.view(np.uint8)
    return buf, size


@pytest.mark.parametrize("tb,comp,tc", [(BF16, F32, BF16), (F16, F16, F32)])
def test_scaled_strided_batch_equals_one_call_per_tile(tb, comp, tc):
    case = DqCase(I8, tb, comp, tc, 40, 24, 64, lda=44, ldb=64, ldc=48, beta0=False, br_type=3, br=2)
    count, rng = 7, np.random.default_rng(21)
    tiles = [case.operands(rng) for _ in range(count)]
    packed = [_pack([t[i] for t in tiles], 32) for i in range(4)]
    h = handle(case)
    for shared in (False, True):
        d = [dev(p[0]) for p in packed]
        cnt = Launches()
        rc = X.libxsmm_b200_gemm_batch_strided_scaled(h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), packed[0][1], packed[1][1], packed[2][1],
                                                      d[3].data_ptr(), None, None, 0 if shared else packed[3][1], 0, 0, case.br, count)
        torch.cuda.synchronize()
        assert rc == 0
        X.check()
        cnt.expect(1)
        got = host(d[2], np.uint8)
        sc = packed[2][1]
        for t in range(count):
            ops = list(tiles[t])
            if shared:
                ops[3] = tiles[0][3]
            c = got[t * sc:t * sc + tiles[t][2].nbytes].view(tiles[t][2].dtype)
            assert np.array_equal(c.view(np.uint8), run_single(case, ops).view(np.uint8)), (shared, t)
            assert same_c(case, case.run(oracle_gemm_dq, *ops)[1], c)
            assert np.all(got[t * sc + tiles[t][2].nbytes:(t + 1) * sc] == SENTINEL)
    # the other strided forms refuse the handle and launch nothing
    before = host(d[2], np.uint8)
    cnt = Launches()
    assert X.libxsmm_b200_gemm_batch_strided(h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), packed[0][1], packed[1][1], packed[2][1],
                                             case.br, count) == NOT_BATCHABLE
    assert X.libxsmm_b200_gemm_batch_strided_multi(h, packed[0][0].ctypes.data, packed[1][0].ctypes.data, packed[2][0].ctypes.data,
                                                   packed[0][1], packed[1][1], packed[2][1], case.br, count, 1) == NOT_BATCHABLE
    torch.cuda.synchronize()
    cnt.expect(0)
    assert np.array_equal(before, host(d[2], np.uint8))


@pytest.mark.parametrize("ta,br_type", [(I4, 1), (U4, 2), (I8, 3)])
def test_per_tile_batch_equals_one_call_per_tile(ta, br_type):
    """libxsmm_b200_gemm_batch: each tile brings its own row scales and zero points (and its batch-reduce arrays)"""
    case = DqCase(ta, F16, F16 if ta != U4 else IMPLICIT, F32, 24, 12, 40, lda=26, ldb=42, ldc=25, beta0=False, br_type=br_type, br=3)
    count, rng = 5, np.random.default_rng(31 + ta)
    tiles = [case.operands(rng) for _ in range(count)]
    bufs = [[dev(x) for x in t] for t in tiles]
    params = (X.GemmParam * count)()
    keep = []
    for t in range(count):
        fill_param(case, params[t], *[b.data_ptr() for b in bufs[t]], keep)
    cnt = Launches()
    assert X.libxsmm_b200_gemm_batch(handle(case), params, count) == 0
    X.check()
    cnt.expect(1)
    assert not X.libxsmm_b200_gemm_plan_create(handle(case), params, count)        # a plan does not take per-call scales
    for t in range(count):
        c = host(bufs[t][2], np.float32)
        assert np.array_equal(c.view(np.uint8), run_single(case, tiles[t]).view(np.uint8)), t
        assert same_c(case, case.run(oracle_gemm_dq, *tiles[t])[1], c), t


def test_bf8_batches_in_every_form():
    """BF8 x F16 has no per-call operands: the plain strided batch (device and pageable host operands) and a plan run it"""
    case = DqCase(BF8, F16, F16, F16, 32, 16, 48, lda=32, ldb=48, ldc=36, beta0=False, vnni_a=True, br_type=3, br=2)
    count, rng = 6, np.random.default_rng(41)
    tiles = [case.operands(rng) for _ in range(count)]
    packed = [_pack([t[i] for t in tiles], 0) for i in range(3)]
    h = handle(case)
    wants = [case.run(oracle_gemm_dq, *t)[1] for t in tiles]
    d = [dev(p[0]) for p in packed]
    cnt = Launches()
    assert X.libxsmm_b200_gemm_batch_strided(h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), packed[0][1], packed[1][1], packed[2][1],
                                             case.br, count) == 0
    X.check()
    cnt.expect(1)
    host_c = packed[2][0].copy()
    assert X.libxsmm_b200_gemm_batch_strided(h, packed[0][0].ctypes.data, packed[1][0].ctypes.data, host_c.ctypes.data, packed[0][1],
                                             packed[1][1], packed[2][1], case.br, count) == 0
    X.check()
    got = host(d[2], np.uint8)
    sc = packed[2][1]
    for t in range(count):
        assert same_c(case, wants[t], got[t * sc:(t + 1) * sc].view(np.uint16)), t
        assert same_c(case, wants[t], host_c[t * sc:(t + 1) * sc].view(np.uint16)), t


# samples/xgemm/gemm_kernel.c: A B Comp C  M N K LDA LDB LDC  alpha beta  alignA alignC  trA trB  vnniA vnniB vnniC  prefetch  br-kind br-count
# br-unroll  reps  tilecfg
DRIVER_RUNS = [("I8 BF16 F32 F32", "nobr"), ("I8 BF16 F32 BF16", "strdbr"), ("I8 F16 F16 F16", "addrbr"), ("I8 F16 IMPLICIT F32", "offsbr"),
               ("I4 F16 F16 F16", "strdbr"), ("U4 F16 F32 F32", "nobr"), ("BF8 F16 F16 F16", "offsbr"), ("BF8 F16 F32 F32", "addrbr")]


@pytest.mark.parametrize("types,br", DRIVER_RUNS, ids=lambda x: x.replace(" ", "_"))
def test_reference_gemm_kernel_driver_passes(types, br):
    import subprocess
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    from ref_drivers import LIBDIR, OUT
    exe = os.path.join(OUT, "gemm_kernel")
    if not os.path.exists(exe):
        pytest.skip("gemm_kernel was not built: build() compiles the drivers where the reference sources exist")
    vnnia = 1 if types.split()[0] in ("I4", "U4", "BF8") else 0
    beta = 0 if br in ("strdbr", "offsbr") else 1
    args = types.split() + [64, 48, 64, 64, 64, 64, 1, beta, 0, 0, 0, 0, vnnia, 0, 0, "nopf", br, 1 if br == "nobr" else 4, 0, 3, 0]
    env = dict(os.environ, LD_LIBRARY_PATH=LIBDIR + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="4", LIBXSMM_TARGET="spr")
    p = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=300, env=env, cwd=OUT)
    assert p.returncode == 0, (p.stdout[-1500:], p.stderr[-800:])
    assert "JIT failed" not in p.stdout and "FAILED" not in p.stdout.upper(), p.stdout[-1500:]
    assert "Total Max Error 0.0000" in p.stdout, p.stdout[-1500:]
