"""MX fp8 GEMM (MXBF8 x MXBF8 / MXHF8 x MXHF8 with E8M0 block scales) on the GPU: the exact-order kernel, element by element.

 * The fixture tests/golden/mxfp8.npz (bytes computed by the reference) and the oracle (oracle/oracle_mx.c) must be matched bit for
   bit, NaN positions excepted (the sign of a NaN created from two NaNs is the compiler's choice on x86; for an MXBF8 C only the
   magnitude of the clamped byte is compared there). MXBF8 C scale bytes must match exactly.
 * Device pointers and pageable host pointers (staged per call); C padding rows (ldc > m) and everything around the operands must
   come back untouched.
 * libxsmm_b200_gemm_batch_strided_scaled equals one call per tile; the gaps between tiles keep their sentinel. The older batch
   forms return NOT_BATCHABLE and leave C alone.
 * Every call checks the launch counts: F32 C launches one exact-order kernel, MXBF8 C two (the product and the quantiser), and no
   tensor-core kernel runs.
 * The reference's own samples/xgemm/gemm_kernel.c driver, unmodified, passes by its own verdict for the three tuples."""
import os

import numpy as np
import pytest
import torch

import libxsmm_b200 as X
from gpu_util import dev, host
from mx_ffi import F32, MXBF8, MXHF8, MxCase, image_nan, oracle_gemm_mx, same_bits, same_mxbf8

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mxfp8.npz")
SIMT, TC = X.BACKEND_SIMT, X.BACKEND_TCGEN05
SENTINEL = 0xA5
NOT_BATCHABLE = -6                                 # LIBXSMM_B200_ERROR_NOT_BATCHABLE


class Launches:
    def __init__(self):
        self.simt, self.tc = X.libxsmm_b200_launch_count_backend(SIMT), X.libxsmm_b200_launch_count_backend(TC)

    def expect(self, simt):
        assert X.libxsmm_b200_launch_count_backend(SIMT) - self.simt == simt
        assert X.libxsmm_b200_launch_count_backend(TC) == self.tc


def handle(case):
    sh = X.libxsmm_create_gemm_shape(case.m, case.n, case.k, case.lda, case.ldb, case.ldc, case.ta, case.ta, case.tc, F32)
    if case.br_type == 0:
        h = X.libxsmm_dispatch_gemm(sh, case.flags, 0)
    else:
        cfg = X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, case.lda * case.k, case.ldb * case.k, 0)
        h = X.libxsmm_dispatch_brgemm(sh, case.flags, 0, cfg)
    assert h and X.libxsmm_b200_kernel_backend(h) == SIMT
    return h


def launches_per_call(case):
    return 2 if case.tc == MXBF8 else 1


def check(case, ops, c, cs, want_c=None, want_cs=None):
    if want_c is None:
        _, want_c, want_cs = case.run(oracle_gemm_mx, *ops)
    if case.tc == F32:
        assert same_bits(want_c, c), case
    else:
        assert same_mxbf8(want_c, c, image_nan(case, ops[0], ops[1], ops[3], ops[4])), case
        assert np.array_equal(want_cs, cs), (case, want_cs, cs)


def run_single(case, ops, on_device=True):
    A, B, C0, As, Bs, Cs = ops
    h = handle(case)
    cnt = Launches()
    if on_device:
        bufs = [dev(x) for x in (A, B, C0, As, Bs, Cs)]
        X.call_gemm(h, bufs[0], bufs[1], bufs[2], br_count=case.br, a_scales=bufs[3], b_scales=bufs[4],
                    c_scales=bufs[5] if case.tc == MXBF8 else None)
        torch.cuda.synchronize(); X.check()
        c, cs = host(bufs[2], C0.dtype), host(bufs[5], np.uint8)
    else:
        c, cs = C0.copy(), Cs.copy()
        X.call_gemm(h, A, B, c, br_count=case.br, a_scales=As, b_scales=Bs, c_scales=cs if case.tc == MXBF8 else None)
        X.check()
    cnt.expect(launches_per_call(case))
    return c, cs[:case.size_cs]


def golden_cases():
    g = np.load(GOLDEN)
    return [(MxCase(*[int(v) for v in g["meta%d" % t]]), [g["%s%d" % (nm, t)] for nm in ("a", "b", "c0", "as", "bs", "cs0")],
             g["c%d" % t], g["cs%d" % t]) for t in range(int(g["ncases"]))]


@pytest.mark.parametrize("on_device", [True, False], ids=["device", "host"])
def test_exact_order_kernel_equals_the_reference_fixture(on_device):
    for case, ops, want_c, want_cs in golden_cases():
        c, cs = run_single(case, ops, on_device)
        check(case, ops, c, cs, want_c, want_cs)


def parity_cases():
    out = []
    for ta in (MXBF8, MXHF8):
        for k in (32, 64, 320):
            out.append(MxCase(ta, F32, 7, 5, k, lda=9, ldb=6, ldc=11, beta0=True))
            out.append(MxCase(ta, F32, 12, 3, k, lda=12, ldb=4, ldc=13, beta0=False, br_type=3, br=3))
        out.append(MxCase(ta, F32, 100, 70, 256, lda=104, ldb=70, ldc=101, beta0=False, br_type=3, br=2))
    for k in (32, 160):
        out.append(MxCase(MXBF8, MXBF8, 32, 5, k, lda=33, ldb=7, ldc=64, beta0=True))
        out.append(MxCase(MXBF8, MXBF8, 96, 33, k, lda=96, ldb=40, ldc=128, beta0=True, br_type=3, br=2))
    return out


@pytest.mark.parametrize("case", parity_cases(), ids=repr)
def test_exact_order_kernel_equals_the_oracle(case):
    rng = np.random.default_rng(case.m * 7919 + case.k + case.ta + case.br)
    ops = case.operands(rng)
    c, cs = run_single(case, ops, on_device=True)
    check(case, ops, c, cs)
    if case.tc == F32:
        assert np.isnan(c).mean() < 0.7                          # not vacuous (a 0xFF scale of B turns a column to NaN)


def test_beta0_runs_over_a_nan_c_and_scale_quirks_hold():
    """beta = 0 never reads C; a zero scale adds +0, a 0xFF scale +inf; an all-zero MXBF8 block gives scale 0 and 0xFB bytes"""
    case = MxCase(MXHF8, F32, 4, 3, 64, beta0=True)
    A = np.full(case.size_a, 0x38, np.uint8); B = np.full(case.size_b, 0x38, np.uint8)
    As = np.full(case.size_as, 127, np.uint8); Bs = np.full(case.size_bs, 127, np.uint8)
    As[0] = 0; As[case.lda + 1] = 0xFF
    C0 = np.full(case.size_c, np.nan, np.float32)
    c, _ = run_single(case, [A, B, C0, As, Bs, np.zeros(1, np.uint8)])
    c = c.reshape(case.n, case.ldc)
    assert c[0, 0] == 32.0 and c[0, 1] == np.inf and c[0, 2] == 64.0 and c[0, 3] == 64.0, c[0]
    zc = MxCase(MXBF8, MXBF8, 32, 2, 32, beta0=True)
    ops = [np.zeros(zc.size_a, np.uint8), np.zeros(zc.size_b, np.uint8), np.full(zc.size_c, 0x11, np.uint8),
           np.full(zc.size_as, 127, np.uint8), np.full(zc.size_bs, 127, np.uint8), np.full(zc.size_cs, 0x11, np.uint8)]
    c, cs = run_single(zc, ops)
    assert np.all(c == 0xFB) and np.all(cs == 0)
    check(zc, ops, c, cs)


@pytest.mark.parametrize("tc", [F32, MXBF8], ids=["f32c", "mxbf8c"])
def test_scaled_batch_equals_one_call_per_tile(tc):
    case = MxCase(MXBF8 if tc == MXBF8 else MXHF8, tc, 64, 24, 128, lda=68, ldb=24, ldc=96, beta0=(tc == MXBF8), br_type=3, br=2)
    count, rng = 9, np.random.default_rng(77)
    tiles = [case.operands(rng) for _ in range(count)]
    pad = 48                                          # a sentinel gap after every tile of every operand

    def pack(idx, dtype):
        size = tiles[0][idx].nbytes + pad
        buf = np.full(size * count, SENTINEL, np.uint8)
        for t in range(count):
            buf[t * size:t * size + tiles[t][idx].nbytes] = tiles[t][idx].view(np.uint8)
        return buf, size
    packed = [pack(i, tiles[0][i].dtype) for i in range(6)]
    d = [dev(p[0]) for p in packed]
    h = handle(case)
    cnt = Launches()
    rc = X.libxsmm_b200_gemm_batch_strided_scaled(h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), packed[0][1], packed[1][1], packed[2][1],
                                                  d[3].data_ptr(), d[4].data_ptr(), d[5].data_ptr(), packed[3][1], packed[4][1], packed[5][1], case.br, count)
    torch.cuda.synchronize()
    assert rc == 0
    X.check()
    cnt.expect(launches_per_call(case))
    got_c, got_cs = host(d[2], np.uint8), host(d[5], np.uint8)
    for t in range(count):
        sc, sz = packed[2][1], tiles[t][2].nbytes
        c = got_c[t * sc:t * sc + sz].view(tiles[t][2].dtype)
        ssz = tiles[t][5].nbytes
        cs = got_cs[t * packed[5][1]:t * packed[5][1] + ssz][:case.size_cs]
        single_c, single_cs = run_single(case, tiles[t])
        assert np.array_equal(c.view(np.uint8), single_c.view(np.uint8)) and np.array_equal(cs, single_cs), t
        check(case, tiles[t], c, cs)
        assert np.all(got_c[t * sc + sz:(t + 1) * sc] == SENTINEL)
    # pageable host operands are refused, the older batch forms refuse the handle, C stays as it was
    assert X.libxsmm_b200_gemm_batch_strided_scaled(h, packed[0][0].ctypes.data, d[1].data_ptr(), d[2].data_ptr(), packed[0][1], packed[1][1], packed[2][1],
                                                    d[3].data_ptr(), d[4].data_ptr(), d[5].data_ptr(), packed[3][1], packed[4][1], packed[5][1], case.br, count) == -4
    before = host(d[2], np.uint8)
    cnt = Launches()
    assert X.libxsmm_b200_gemm_batch_strided(h, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), packed[0][1], packed[1][1], packed[2][1],
                                             case.br, count) == NOT_BATCHABLE
    assert X.libxsmm_b200_gemm_batch_strided_multi(h, packed[0][0].ctypes.data, packed[1][0].ctypes.data, packed[2][0].ctypes.data,
                                                   packed[0][1], packed[1][1], packed[2][1], case.br, count, 1) == NOT_BATCHABLE
    torch.cuda.synchronize()
    cnt.expect(0)
    assert np.array_equal(before, host(d[2], np.uint8))


# samples/xgemm/gemm_kernel.c: A B Comp C  M N K LDA LDB LDC  alpha beta  alignA alignC  trA trB  vnniA vnniB vnniC  prefetch  br-kind br-count
# br-unroll  reps  tilecfg
@pytest.mark.parametrize("types,beta,br", [("MXBF8 MXBF8 F32 F32", 1, "nobr"), ("MXBF8 MXBF8 F32 F32", 0, "strdbr"),
                                           ("MXHF8 MXHF8 F32 F32", 1, "nobr"), ("MXHF8 MXHF8 F32 F32", 0, "strdbr"),
                                           ("MXBF8 MXBF8 F32 MXBF8", 0, "nobr"), ("MXBF8 MXBF8 F32 MXBF8", 0, "strdbr")])
def test_reference_gemm_kernel_driver_passes(types, beta, br):
    import subprocess
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    from ref_drivers import LIBDIR, OUT
    exe = os.path.join(OUT, "gemm_kernel")
    if not os.path.exists(exe):
        pytest.skip("gemm_kernel was not built: build() compiles the drivers where the reference sources exist")
    args = types.split() + [64, 64, 64, 64, 64, 64, 1, beta, 0, 0, 0, 1, 1, 1, 0, "nopf", br, 4 if br != "nobr" else 1, 0, 3, 0]
    env = dict(os.environ, LD_LIBRARY_PATH=LIBDIR + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="4")
    p = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=300, env=env, cwd=OUT)
    assert p.returncode == 0, (p.stdout[-1500:], p.stderr[-800:])
    assert "JIT failed" not in p.stdout and "FAILED" not in p.stdout.upper(), p.stdout[-1500:]


def test_scaled_batch_with_mxbf8_c_runs_in_chunks():
    """an MXBF8 C is quantised from an f32 image in scratch, at most 64 MiB of it per chunk: 128 x 128 tiles (64 KiB of image) make
    1024 tiles a chunk, so 1100 tiles cross one chunk boundary; tiles on both sides and the last one must equal the oracle"""
    case = MxCase(MXBF8, MXBF8, 128, 128, 32, beta0=True)
    count, rng = 1100, np.random.default_rng(5)
    ops0 = case.operands(rng)
    A = np.concatenate([ops0[0]] + [case.operands(rng)[0] for _ in range(7)])      # 8 distinct A tiles, cycled
    a = np.tile(A, count // 8 + 1)[:count * case.size_a]
    b = rng.integers(0, 256, count * case.size_b, dtype=np.uint8)
    b[(b & 0x7C) == 0x7C] ^= 0x40
    as_ = rng.integers(117, 138, count * case.size_as, dtype=np.uint8)
    bs_ = rng.integers(117, 138, count * case.size_bs, dtype=np.uint8)
    d_a, d_b, d_as, d_bs = dev(a), dev(b), dev(as_), dev(bs_)
    d_c = torch.full((count * case.size_c,), SENTINEL, dtype=torch.uint8, device="cuda")
    d_cs = torch.full((count * case.size_cs,), SENTINEL, dtype=torch.uint8, device="cuda")
    h = handle(case)
    cnt = Launches()
    rc = X.libxsmm_b200_gemm_batch_strided_scaled(h, d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), case.size_a, case.size_b, case.size_c,
                                                  d_as.data_ptr(), d_bs.data_ptr(), d_cs.data_ptr(), case.size_as, case.size_bs, case.size_cs, 1, count)
    assert rc == 0
    X.check()
    cnt.expect(2 * 2)                                  # two chunks, product + quantiser each
    got_c, got_cs = host(d_c, np.uint8), host(d_cs, np.uint8)
    for t in (0, 1, 1022, 1023, 1024, 1025, count - 1):
        ops = [a[t * case.size_a:(t + 1) * case.size_a], b[t * case.size_b:(t + 1) * case.size_b], np.zeros(case.size_c, np.uint8),
               as_[t * case.size_as:(t + 1) * case.size_as], bs_[t * case.size_bs:(t + 1) * case.size_bs], np.zeros(case.size_cs, np.uint8)]
        check(case, ops, got_c[t * case.size_c:(t + 1) * case.size_c], got_cs[t * case.size_cs:(t + 1) * case.size_cs])
