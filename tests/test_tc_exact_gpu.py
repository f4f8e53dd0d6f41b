"""The tensor-core kernels (gemm_tc.cu: SS16 / RS16 / RS8 forms of gemm_wg_kernel and the pooled plan; bcsc_tc.cu) and the int8
exact-order kernels, element by element against a float64 / int64 reference decoded from the very bytes handed to the kernel.

 * Family E (exact by construction): operands and old C are dyadic values on one grid 2^-q and every element satisfies
   sum |a*b| + |c0| < 2^(24-q), so every partial sum is an f32 value and the result cannot depend on the summation order. The
   kernel must then equal the reference after ONE round-to-nearest-even to the output type, bit for bit, and equal the oracle.
   The results carry more significant bits than bf16 / f16 hold, so the output rounding (ties included) is exercised.
 * Family R (full mantissas): per-element bound |got - exact| <= K*2^-23*sum|a||b| + ulp_out(|exact| + that)/2.
 * Padding of A and B (lda > m, ldb > k), gaps between batch-reduce blocks and between tiles hold NaN (0x80 / 0xff for int8);
   C padding, gaps between C tiles and a guard band after the last tile hold a sentinel and must come back byte-identical;
   beta = 0 runs over an all-NaN C.
 * Every call checks which kernel family ran (libxsmm_b200_launch_count_backend): a launch-time fallback to the exact-order
   kernel would otherwise pass every tensor-core test."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import gen
import libxsmm_b200 as X
from oracle_ffi import oracle, run_gemm

pytestmark = pytest.mark.gpu

BF16, F16, F32, I32, I8, U8 = gen.BF16, gen.F16, gen.F32, gen.I32, gen.I8, gen.U8
BETA_0, VNNI_A = X.GEMM_FLAG_BETA_0, X.GEMM_FLAG_VNNI_A
ES = {BF16: 2, F16: 2, F32: 4, I32: 4, I8: 1, U8: 1}
UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32}
POISON = {F32: 0x7FC00000, BF16: 0x7FC0, F16: 0x7E00, I8: 0x80, U8: 0xFF}       # NaN for the floating-point types
NAN_C = {F32: 0x7FC00000, BF16: 0x7FC0, F16: 0x7E00}
SENTINEL = 0xA5
TC, SIMT = X.BACKEND_TCGEN05, X.BACKEND_SIMT


def up(x, a):
    return (x + a - 1) // a * a


def decode(bits, t):
    """element bits (unsigned array) -> float64 values, int64 for the integer types"""
    bits = np.ascontiguousarray(bits)
    if t == BF16:
        return gen.bf16_bits_to_f32(bits).astype(np.float64)
    if t == F16:
        return bits.view(np.float16).astype(np.float64)
    if t == F32:
        return bits.view(np.float32).astype(np.float64)
    if t == I8:
        return bits.view(np.int8).astype(np.int64)
    if t == I32:
        return bits.view(np.int32).astype(np.int64)
    return bits.astype(np.int64)


def encode(vals, t):
    """float64 values exactly representable in type t -> bits"""
    if t == BF16:
        f = np.asarray(vals, dtype=np.float32)
        assert np.array_equal(f.astype(np.float64), vals)
        return gen.f32_to_bf16_bits(f)
    if t == F16:
        return np.asarray(vals, dtype=np.float16).view(np.uint16)
    if t == F32:
        return np.asarray(vals, dtype=np.float32).view(np.uint32)
    if t in (I8, U8):
        return np.asarray(vals, dtype=np.int64).astype(np.uint8)
    return np.asarray(vals, dtype=np.int64).astype(np.uint32)


def round_out(x, tc):
    """one round-to-nearest-even of f32-representable float64 values to the output type"""
    f = x.astype(np.float32)
    if tc == F32:
        return f.view(np.uint32)
    if tc == BF16:
        return gen.f32_to_bf16_bits(f)
    return f.astype(np.float16).view(np.uint16)


def wrap32(x):
    return ((np.asarray(x, dtype=np.int64) + (1 << 31)) % (1 << 32) - (1 << 31)).astype(np.int64)


def ulp_out(x, tc):
    """spacing of the output type at |x| (normal range; the subnormal spacing below)"""
    mant, emin = {F32: (23, -126), BF16: (7, -126), F16: (10, -14)}[tc]
    e = np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** emin)))
    return np.exp2(e - mant)


class Launches:
    """kernels launched per family while the block runs"""

    def __enter__(self):
        self.t0, self.s0 = X.libxsmm_b200_launch_count_backend(TC), X.libxsmm_b200_launch_count_backend(SIMT)
        return self

    def __exit__(self, *exc):
        self.tc = X.libxsmm_b200_launch_count_backend(TC) - self.t0
        self.simt = X.libxsmm_b200_launch_count_backend(SIMT) - self.s0

    def expect(self, backend, what):
        if backend == TC:
            assert self.tc > 0 and self.simt == 0, ("the tensor-core kernel did not run", what, self.tc, self.simt)
        else:
            assert self.simt > 0 and self.tc == 0, ("the exact-order kernel did not run", what, self.tc, self.simt)


def dev(arr):
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).copy()).cuda()


def back(t, like):
    return t.cpu().numpy().view(like.dtype).copy()


class Batch:
    """A strided batch laid out with poisoned padding and gaps. A: flat (vnni 1) or VNNI-packed (2, 4) column-major m x k blocks,
    B: column-major k x n blocks, `br` blocks per tile `blk_gap` bytes apart, tiles `tile_gap` bytes apart; C: column-major m x n
    tiles, sentinel everywhere outside the logical elements, `guard` bytes after the last tile."""

    def __init__(self, m, n, k, ta, tb, tc, beta0, count=1, br=1, vnni=1, lda=None, ldb=None, ldc=None, blk_gap=0, tile_gap=0, guard=256):
        self.m, self.n, self.k, self.ta, self.tb, self.tc, self.beta0, self.count, self.br, self.vnni = m, n, k, ta, tb, tc, beta0, count, br, vnni
        self.lda, self.ldb, self.ldc = lda or m, ldb or k, ldc or m
        ea, eb, ec = ES[ta], ES[tb], ES[tc]
        foot_a = (((k // vnni - 1) * self.lda * vnni + m * vnni) if vnni > 1 else ((k - 1) * self.lda + m)) * ea
        foot_b = ((n - 1) * self.ldb + k) * eb
        self.bsa, self.bsb = up(foot_a + blk_gap, 16), up(foot_b + blk_gap, 16)
        self.sta, self.stb = up(self.bsa * max(br, 1) + tile_gap, 16), up(self.bsb * max(br, 1) + tile_gap, 16)
        self.stc = up(((n - 1) * self.ldc + m) * ec + tile_gap, 16)
        t4 = np.arange(count)[:, None, None, None]; r4 = np.arange(br)[None, :, None, None]
        i, kk, j = np.arange(m), np.arange(k), np.arange(n)
        ia = ((kk[None, :] // vnni) * self.lda * vnni + i[:, None] * vnni + kk[None, :] % vnni) if vnni > 1 else (kk[None, :] * self.lda + i[:, None])
        self.idx_a = (t4 * self.sta + r4 * self.bsa) // ea + ia[None, None]                      # [count][br][m][k]
        self.idx_b = (t4 * self.stb + r4 * self.bsb) // eb + (j[None, :] * self.ldb + kk[:, None])[None, None]   # [count][br][k][n]
        self.idx_c = (np.arange(count)[:, None, None] * self.stc) // ec + (j[None, :] * self.ldc + i[:, None])[None]   # [count][m][n]
        self.buf_a = np.full(max(count * self.sta // ea, 16), POISON[ta], dtype=UINT[ea])
        self.buf_b = np.full(max(count * self.stb // eb, 16), POISON[tb], dtype=UINT[eb])
        self.buf_c = np.full(count * self.stc + guard, SENTINEL, dtype=np.uint8).view(UINT[ec])

    def fill(self, a_bits, b_bits, c_bits):
        self.buf_a[self.idx_a] = a_bits
        self.buf_b[self.idx_b] = b_bits
        self.buf_c[self.idx_c] = c_bits if not self.beta0 else NAN_C.get(self.tc, 0)
        return self

    def operands(self):
        return decode(self.buf_a[self.idx_a], self.ta), decode(self.buf_b[self.idx_b], self.tb)

    def old_c(self):
        """old C as the epilogue sees it (f16 inputs with f32 C round it through f16 first)"""
        c = decode(self.buf_c[self.idx_c], self.tc)
        if self.ta == F16 and self.tc == F32:
            c = c.astype(np.float16).astype(np.float64)
        return c

    def product(self):
        """(sum_r A_r B_r, sum_r |A_r||B_r|) per tile in float64 (int64 for int8)"""
        A, B = self.operands()
        acc = np.zeros((self.count, self.m, self.n), dtype=A.dtype); mag = np.zeros_like(acc)
        for r in range(self.br):
            acc += np.matmul(A[:, r], B[:, r]); mag += np.matmul(np.abs(A[:, r]), np.abs(B[:, r]))
        return acc, mag

    def dispatch(self, force_simt=False):
        flags = (BETA_0 if self.beta0 else 0) | (VNNI_A if self.vnni > 1 else 0)
        tcomp = I32 if self.ta in (I8, U8) else F32
        sh = X.libxsmm_create_gemm_shape(self.m, self.n, self.k, self.lda, self.ldb, self.ldc, self.ta, self.tb, self.tc, tcomp)
        X.libxsmm_b200_set_force_simt(1 if force_simt else 0)
        try:
            cfg = X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, self.bsa, self.bsb, 0)
            kern = X.libxsmm_dispatch_brgemm(sh, flags, 0, cfg)
        finally:
            X.libxsmm_b200_set_force_simt(0)
        assert kern, self
        return kern

    def run(self, backend, force_simt=False):
        """one strided batch call; returns the C buffer after it. Asserts which kernel family ran."""
        kern = self.dispatch(force_simt)
        d_a, d_b, d_c = dev(self.buf_a), dev(self.buf_b), dev(self.buf_c)
        with Launches() as L:
            rc = X.libxsmm_b200_gemm_batch_strided(kern, d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), self.sta, self.stb, self.stc, self.br, self.count)
            assert rc == 0, (self, X.libxsmm_b200_last_error_string())
            X.check()
        L.expect(backend, self)
        return back(d_c, self.buf_c)

    def oracle_c(self, scf=0.0):
        """the oracle, one call per tile on the same bytes"""
        c = self.buf_c.copy()
        flags = (BETA_0 if self.beta0 else 0) | (VNNI_A if self.vnni > 1 else 0)
        tcomp = I32 if self.ta in (I8, U8) else F32
        a8, b8, c8 = self.buf_a.view(np.uint8), self.buf_b.view(np.uint8), c.view(np.uint8)
        for t in range(self.count):
            assert run_gemm(oracle, (self.m, self.n, self.k, self.lda, self.ldb, self.ldc), (self.ta, self.tb, tcomp, self.tc), flags, 3, self.bsa, self.bsb,
                            self.br, a8[t * self.sta:], b8[t * self.stb:], c8[t * self.stc:], scf=scf) == 0
        return c

    def __repr__(self):
        return "batch(m%d n%d k%d ld%d/%d/%d %s->%s vnni%d br%d x%d beta0=%d)" % (self.m, self.n, self.k, self.lda, self.ldb, self.ldc, self.ta,
                                                                            self.tc, self.vnni, self.br, self.count, self.beta0)


def grid_ints(rng, shape, lim):
    return rng.integers(-lim, lim + 1, size=shape)


def family_e(rng, bt, c_scale=1):
    """operands i/4 with |i| <= 15, old C on the 2^-4 grid of the products: representable in bf16 and f16"""
    a = grid_ints(rng, bt.idx_a.shape, 15) / 4.0
    b = grid_ints(rng, bt.idx_b.shape, 15) / 4.0
    lim = {BF16: 255, F16: 2047, F32: 255 * c_scale}[bt.tc]
    c = grid_ints(rng, bt.idx_c.shape, lim) / 16.0
    if bt.ta == F16 and bt.tc == F32:
        c = grid_ints(rng, bt.idx_c.shape, 1 << 19) / 16.0     # f32 old C with more bits than f16: the epilogue rounds it through f16
    return bt.fill(encode(a, bt.ta), encode(b, bt.tb), encode(c, bt.tc))


def expect_exact(bt, got, q=4):
    """family E: the exactness premise, one RNE rounding of the float64 result, the untouched bytes, and the oracle"""
    acc, mag = bt.product()
    old = np.zeros_like(acc) if bt.beta0 else bt.old_c()
    assert np.all((mag + np.abs(old)) * 2.0 ** q < 2.0 ** 24), "the operands break the exactness premise"
    exact = acc + old
    want = round_out(exact, bt.tc)
    g = got[bt.idx_c]
    bad = np.nonzero((g != want).reshape(bt.count, -1).any(axis=1))[0]
    if len(bad):
        t = int(bad[0]); e = np.argwhere(g[t] != want[t])[0]
        pytest.fail("%r: %d of %d tiles differ, first tile %d element (m=%d, n=%d): got %s want %s (exact %r)"
                    % (bt, len(bad), bt.count, t, e[0], e[1], hex(int(g[t][tuple(e)])), hex(int(want[t][tuple(e)])), exact[t][tuple(e)]))
    expect_untouched(bt, got)
    assert np.array_equal(got.view(np.uint8), bt.oracle_c().view(np.uint8)), ("oracle", bt)
    return exact


def expect_untouched(bt, got):
    mask = np.ones(got.shape, dtype=bool); mask[bt.idx_c] = False
    assert np.all(got.view(np.uint8).reshape(-1, ES[bt.tc])[mask] == SENTINEL), ("C padding, gaps or guard band written", bt)
    if bt.beta0 and bt.tc != I32:
        assert not np.isnan(decode(got[bt.idx_c], bt.tc)).any(), ("beta = 0 read the old C", bt)


# ---- shape grid at the eligibility edges ---------------------------------------------------------------------------------
# SS16 (flat A): m 16..128, n 16..256, k 16..4096, lda % 8 == 0. A covering set of the edges, not their product.
SS16_SHAPES = [(16, 17, 63), (17, 16, 16), (63, 31, 65), (64, 33, 130), (65, 65, 17), (72, 129, 63), (100, 200, 16), (127, 256, 65),
               (128, 16, 130), (16, 256, 4096), (100, 31, 4096), (64, 129, 17), (127, 33, 16), (65, 200, 130)]
SS16_TYPES = [(BF16, F32), (BF16, BF16), (F16, F32), (F16, F16)]


@pytest.mark.parametrize("ta,tc", SS16_TYPES)
def test_ss16_exact_at_the_edges(ta, tc):
    rng = np.random.default_rng(1000 + 10 * ta + tc)
    for s, (m, n, k) in enumerate(SS16_SHAPES):
        beta0, br = s % 2, (1, 3, 2)[s % 3] if k < 4096 else 1
        bt = family_e(rng, Batch(m, n, k, ta, ta, tc, beta0, count=3 if k < 4096 else 2, br=br, lda=up(m + 3, 8), ldb=up(k + 1, 8),
                                 ldc=m + 5, blk_gap=96, tile_gap=64))
        expect_exact(bt, bt.run(TC))


RS_M, RS_N = (4, 60, 68, 124, 128), (1, 7, 15, 17, 33, 128)


def rs_shapes(ta):
    ks = (2, 18, 66, 8192) if ta != U8 and ta != I8 else (4, 36, 132, 8192)
    return [(RS_M[s % len(RS_M)], RS_N[s % len(RS_N)], ks[s % len(ks)]) for s in range(12)]


@pytest.mark.parametrize("ta,tc", SS16_TYPES)
def test_rs16_exact_at_the_edges(ta, tc):
    rng = np.random.default_rng(2000 + 10 * ta + tc)
    for s, (m, n, k) in enumerate(rs_shapes(ta)):
        beta0, br = s % 2, (2 if k < 8192 else 1)
        bt = family_e(rng, Batch(m, n, k, ta, ta, tc, beta0, count=3, br=br, vnni=2, lda=m + 4, ldb=up(k + 3, 8), ldc=m + 3, blk_gap=48, tile_gap=80))
        expect_exact(bt, bt.run(TC))


def test_just_outside_eligibility_runs_the_exact_order_kernel_bit_exact():
    """m = 129, n = 257 (SS16) / 129 (RS), k = 4097 (SS16) / 8194 (RS), lda % 8 != 0 (SS16), m % 4 != 0 (RS): the exact-order kernel"""
    rng = np.random.default_rng(3000)
    for (m, n, k, vnni, lda) in ((129, 16, 32, 1, 136), (32, 257, 32, 1, 32), (16, 16, 4097, 1, 16), (20, 24, 64, 1, 22),
                                 (132, 16, 32, 2, 132), (32, 129, 32, 2, 32), (16, 16, 8194, 2, 16), (30, 16, 32, 2, 30)):
        for beta0 in (0, 1):
            bt = family_e(rng, Batch(m, n, k, BF16, BF16, BF16, beta0, count=2, br=2 if k < 4000 else 1, vnni=vnni, lda=lda, ldb=up(k, 8), ldc=m + 2,
                                     blk_gap=32, tile_gap=32))
            expect_exact(bt, bt.run(SIMT))


def test_int8_just_outside_eligibility_runs_the_exact_order_kernel():
    rng = np.random.default_rng(3001)
    for (m, n, k) in ((132, 16, 64), (32, 129, 64), (16, 16, 8196), (30, 16, 64)):
        bt = Batch(m, n, k, U8, I8, I32, 0, count=2, br=1, vnni=4, ldc=m + 1, tile_gap=32)
        full_range_int8(rng, bt)
        expect_int8(bt, bt.run(SIMT))


@pytest.mark.parametrize("vnni", [1, 2])
def test_br_count_zero(vnni):
    """an empty batch-reduce: beta = 0 zeroes C, beta = 1 keeps it"""
    rng = np.random.default_rng(3002)
    for beta0 in (0, 1):
        bt = family_e(rng, Batch(64, 32, 64, BF16, BF16, BF16, beta0, count=3, br=0, vnni=vnni, ldc=70, tile_gap=16))
        got = bt.run(SIMT)
        want = np.zeros_like(got[bt.idx_c]) if beta0 else bt.buf_c[bt.idx_c]
        assert np.array_equal(got[bt.idx_c], want), beta0
        expect_untouched(bt, got)
        assert np.array_equal(got.view(np.uint8), bt.oracle_c().view(np.uint8))


# ---- the persistent schedule ------------------------------------------------------------------------------------------------
def ring_and_grid(m, n, wg_forced=None, rs_m=None):
    """mirror of gemm_tc.cu plan_stages: (stages, CTAs per SM) of an SS16 (rs_m None) or RS16 launch"""
    nt = 16 if n <= 16 else 32 if n <= 32 else 64 if n <= 64 else 128 if n <= 128 else 256
    wg = 1 if m <= 64 else 2
    stage = (wg * 8192 if rs_m is None else up(rs_m * 128, 1024)) + nt * 128
    c = 3 if (nt == 64 and wg == 1) or nt < 64 else 1
    while c > 1 and 2 * stage + 2048 > (227 * 1024) // c:
        c -= 1
    st = min(8, max(2, ((227 * 1024) // c - 2048) // stage))
    return st, c


@pytest.mark.parametrize("ta,vnni", [(BF16, 1), (F16, 1), (BF16, 2), (F16, 2)])
def test_persistent_schedule_many_tiles_per_cta(ta, vnni):
    """counts around multiples of the SM count and ~3x the grid plus a prime; loads per tile (br x k-chunks) coprime with the ring
    size, so that the mbarrier phase carries across tile boundaries at every offset. Each tile checked on its own (family E)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(4000 + ta + vnni)
    m, n, k = 64, 48, 64
    stages, ctas = ring_and_grid(m, n, rs_m=(m if vnni == 2 else None))
    kchunks = (k + 63) // 64
    br = next(b for b in (3, 5, 7, 9, 11) if math.gcd(b * kchunks, stages) == 1)
    grid = sms * ctas
    for count in (1, sms - 1, sms, sms + 1, 2 * sms + 1, grid - 1, grid, grid + 1, 3 * grid + 13):
        bt = family_e(rng, Batch(m, n, k, ta, ta, ta, count % 2, count=count, br=br, vnni=vnni, ldc=m + 2, tile_gap=16))
        expect_exact(bt, bt.run(TC))


# ---- the pooled plan (address batch-reduce over a pool of block-sets) -------------------------------------------------------
@pytest.mark.parametrize("m", [64, 100])
def test_pooled_plan_exact_f16_beta1_padded_c(m):
    """mode R: f16 -> f16, beta = 1, ldc > m, tiles that share a B set paired (m <= 64) with some sets used an odd number of times so
    that items travel alone (second C pointer NULL); every C tile padded and surrounded by sentinels"""
    rng = np.random.default_rng(5000 + m)
    n, k, br, nsets, ldc = 40, 96, 3, 5, m + 6
    lda = up(m, 8)
    blk_a, blk_b = up(k * lda * 2, 16), up(n * k * 2, 16)
    a = grid_ints(rng, (nsets, br, k, lda), 15) / 4.0; b = grid_ints(rng, (nsets, br, n, k), 15) / 4.0
    a[:, :, :, m:] = np.nan
    pool_a = np.full(nsets * br * blk_a // 2, POISON[F16], np.uint16); pool_b = np.full(nsets * br * blk_b // 2, POISON[F16], np.uint16)
    for s in range(nsets):
        for r in range(br):
            o = (s * br + r) * blk_a // 2; pool_a[o:o + k * lda] = a[s, r].astype(np.float16).view(np.uint16).ravel()
            o = (s * br + r) * blk_b // 2; pool_b[o:o + n * k] = b[s, r].astype(np.float16).view(np.uint16).ravel()
    count = 41
    sb = np.concatenate([np.full(c, s) for s, c in enumerate((9, 7, 12, 5, 8))])       # odd counts: unpaired items
    sa = rng.integers(0, nsets, size=count)
    rng.shuffle(sb)
    stc = up(n * ldc * 2 + 32, 16)
    c0 = grid_ints(rng, (count, n, ldc), 2047) / 16.0
    cbuf = np.full(count * stc + 256, SENTINEL, np.uint8)
    for t in range(count):
        v = cbuf[t * stc:t * stc + n * ldc * 2].view(np.uint16).reshape(n, ldc)
        v[:, :m] = c0[t, :, :m].astype(np.float16).view(np.uint16)
    case_kern = X.libxsmm_dispatch_brgemm(X.libxsmm_create_gemm_shape(m, n, k, lda, k, ldc, F16, F16, F16, F32), 0, 0,
                                          X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_ADDRESS, 0, 0, 0))
    assert case_kern
    d_a, d_b, d_c = dev(pool_a), dev(pool_b), dev(cbuf)
    params = (X.GemmParam * count)(); keep = []
    for t in range(count):
        aa = (C.c_void_p * br)(*[d_a.data_ptr() + (int(sa[t]) * br + r) * blk_a for r in range(br)])
        ab = (C.c_void_p * br)(*[d_b.data_ptr() + (int(sb[t]) * br + r) * blk_b for r in range(br)])
        brv = C.c_ulonglong(br); keep += [aa, ab, brv]
        params[t].op.tertiary = C.addressof(brv); params[t].a.primary, params[t].b.primary = C.addressof(aa), C.addressof(ab)
        params[t].c.primary = d_c.data_ptr() + t * stc
    plan = X.libxsmm_b200_gemm_plan_create(case_kern, params, count)
    assert plan and X.libxsmm_b200_gemm_plan_is_pooled(plan) == 1
    with Launches() as L:
        assert X.libxsmm_b200_gemm_plan_run(plan) == 0
        X.check()
    L.expect(TC, "pooled plan")
    X.libxsmm_b200_gemm_plan_destroy(plan)
    got = d_c.cpu().numpy()
    want = cbuf.copy()
    for t in range(count):
        A = np.nan_to_num(a[sa[t]][:, :, :m])             # [br][k][m]
        acc = sum(b[sb[t], r] @ A[r] for r in range(br))  # C^T[n][m]
        mag = sum(np.abs(b[sb[t], r]) @ np.abs(A[r]) for r in range(br))
        old = c0[t, :, :m].astype(np.float16).astype(np.float64)
        assert np.all((mag + np.abs(old)) * 16 < 2.0 ** 24)
        v = want[t * stc:t * stc + n * ldc * 2].view(np.uint16).reshape(n, ldc)
        v[:, :m] = round_out(acc + old, F16)
    bad = [t for t in range(count) if not np.array_equal(got[t * stc:(t + 1) * stc], want[t * stc:(t + 1) * stc])]
    assert not bad, ("first failing tile", bad[0], len(bad))
    assert np.array_equal(got, want)


# ---- family R: full mantissas, per-element bound ----------------------------------------------------------------------------
R_WORST = {}


@pytest.mark.parametrize("ta,tc,vnni", [(BF16, F32, 1), (BF16, BF16, 1), (F16, F32, 1), (F16, F16, 1), (BF16, BF16, 2), (F16, F16, 2), (F16, F32, 2)])
def test_full_mantissa_rounding_per_element(ta, tc, vnni):
    rng = np.random.default_rng(6000 + 10 * ta + tc + vnni)
    worst = 0.0
    for (m, n, k, br, beta0) in ((64, 64, 64, 4, 1), (100, 33, 130, 2, 0), (17 if vnni == 1 else 20, 129 if vnni == 1 else 120, 256, 1, 1), (128, 200 if vnni == 1 else 128, 512, 2, 0)):
        bt = Batch(m, n, k, ta, ta, tc, beta0, count=3, br=br, vnni=vnni, lda=up(m + 1, 8), ldb=up(k + 1, 8), ldc=m + 1, blk_gap=16, tile_gap=16)
        scale_b = np.exp2(rng.integers(-6, 5, size=(3, br, 1, n)))                  # per-column scales 2^[-6, 4]: f16 C stays finite
        a = rng.standard_normal(bt.idx_a.shape); b = rng.standard_normal(bt.idx_b.shape) * scale_b
        c = rng.standard_normal(bt.idx_c.shape) * 4
        rt = (lambda x: gen.bf16_bits_to_f32(gen.f32_to_bf16_bits(x.astype(np.float32))).astype(np.float64)) if ta == BF16 else (lambda x: x.astype(np.float16).astype(np.float64))
        a, b = rt(a), rt(b)
        cb = gen.f32_to_bf16_bits(c.astype(np.float32)) if tc == BF16 else (c.astype(np.float16).view(np.uint16) if tc == F16 else c.astype(np.float32).view(np.uint32))
        bt.fill(encode(a, ta), encode(b, ta), cb)
        got = bt.run(TC)
        acc, mag = bt.product()
        old = np.zeros_like(acc) if beta0 else bt.old_c()
        exact = acc + old
        term = k * br * 2.0 ** -23 * (mag + np.abs(old))
        bound = term + 0.5 * ulp_out(np.abs(exact) + term, tc)
        err = np.abs(decode(got[bt.idx_c], tc) - exact)
        ratio = float((err / bound).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, (bt, "max err/bound", ratio, np.unravel_index(np.argmax(err / bound), err.shape))
        expect_untouched(bt, got)
    R_WORST[(ta, tc, vnni)] = worst
    print("family R %s->%s vnni%d: max err/bound %.4f" % (ta, tc, vnni, worst))


# ---- int8 over the full range ------------------------------------------------------------------------------------------------
def full_range_int8(rng, bt, fill_a=None, fill_b=None):
    lo = lambda t: -128 if t == I8 else 0
    hi = lambda t: 127 if t == I8 else 255
    a = rng.integers(lo(bt.ta), hi(bt.ta) + 1, size=bt.idx_a.shape) if fill_a is None else np.full(bt.idx_a.shape, fill_a)
    b = rng.integers(lo(bt.tb), hi(bt.tb) + 1, size=bt.idx_b.shape) if fill_b is None else np.full(bt.idx_b.shape, fill_b)
    c = rng.integers(-(1 << 31), 1 << 31, size=bt.idx_c.shape) if bt.tc == I32 else rng.integers(-1000, 1000, size=bt.idx_c.shape) / 8.0
    return bt.fill(encode(a, bt.ta), encode(b, bt.tb), encode(c, bt.tc) if bt.tc == I32 else c.astype(np.float32).view(np.uint32))


def expect_int8(bt, got, scf=0.0):
    acc, _ = bt.product()
    if bt.tc == I32:
        want = encode(wrap32(acc if bt.beta0 else acc + decode(bt.buf_c[bt.idx_c], I32)), I32)
    else:
        f = wrap32(acc).astype(np.float32) * np.float32(scf)
        want = (f if bt.beta0 else f + decode(bt.buf_c[bt.idx_c], F32).astype(np.float32)).view(np.uint32)
    g = got[bt.idx_c]
    assert np.array_equal(g, want), (bt, int(np.count_nonzero(g != want)), "of", g.size)
    expect_untouched(bt, got)
    assert np.array_equal(got.view(np.uint8), bt.oracle_c(scf).view(np.uint8)), ("oracle", bt)


SIGNS = [(U8, U8), (U8, I8), (I8, U8), (I8, I8)]


@pytest.mark.parametrize("ta,tb", SIGNS)
def test_int8_full_range_rs8(ta, tb):
    rng = np.random.default_rng(7000 + 10 * ta + tb)
    for s, (m, n, k) in enumerate(rs_shapes(I8)):
        bt = full_range_int8(rng, Batch(m, n, k, ta, tb, I32, s % 2, count=3, br=2 if k < 8192 else 1, vnni=4, lda=m + 4, ldb=up(k + 5, 16), ldc=m + 3,
                                        blk_gap=32, tile_gap=48))
        expect_int8(bt, bt.run(TC))


@pytest.mark.parametrize("ta,tb", SIGNS)
def test_int8_full_range_exact_order_kernels(ta, tb):
    """gemm_i8_kernel (VNNI4 A, dp4a) and the exact-order kernel (flat A)"""
    rng = np.random.default_rng(7100 + 10 * ta + tb)
    for (m, n, k, vnni, br) in ((64, 64, 64, 4, 3), (37, 19, 132, 4, 1), (128, 128, 256, 4, 2), (33, 40, 36, 1, 2), (64, 17, 128, 1, 1)):
        for beta0 in (0, 1):
            bt = full_range_int8(rng, Batch(m, n, k, ta, tb, I32, beta0, count=5, br=br, vnni=vnni, ldc=m + 2, tile_gap=16))
            expect_int8(bt, bt.run(SIMT, force_simt=True))


def test_int32_accumulation_wraps_on_tensor_cores():
    """U8 x U8 filled with 255, k * br = 40960: every sum is 255^2 * 40960 = 2.66e9 > 2^31; the reference's int32 wraps"""
    rng = np.random.default_rng(7200)
    bt = full_range_int8(rng, Batch(64, 16, 8192, U8, U8, I32, 1, count=2, br=5, vnni=4), fill_a=255, fill_b=255)
    got = bt.run(TC)
    acc, _ = bt.product()
    assert acc.max() > 2 ** 31
    g = decode(got[bt.idx_c], I32)
    assert np.all(g == wrap32(acc)), ("wgmma int32 accumulation did not wrap", int(g.ravel()[0]), int(wrap32(acc).ravel()[0]))


@pytest.mark.parametrize("ta,tb", SIGNS)
def test_int8_to_f32_with_power_of_two_scales(ta, tb):
    """single calls (the scale in c.tertiary) on the tensor cores, and libxsmm_b200_gemm_batch with a different scale per tile"""
    rng = np.random.default_rng(7300 + 10 * ta + tb)
    m, n, k, count = 64, 40, 128, 6
    for beta0 in (0, 1):
        bt = full_range_int8(rng, Batch(m, n, k, ta, tb, F32, beta0, count=count, br=1, vnni=4, ldc=m + 2, tile_gap=32))
        kern = bt.dispatch()
        scales = [2.0 ** -(3 + t) for t in range(count)]
        d_a, d_b, d_c = dev(bt.buf_a), dev(bt.buf_b), dev(bt.buf_c)
        for route in ("single", "batch"):
            d_c.copy_(dev(bt.buf_c))
            keep = [C.c_float(s) for s in scales]; params = (X.GemmParam * count)()
            for t in range(count):
                params[t].a.primary, params[t].b.primary = d_a.data_ptr() + t * bt.sta, d_b.data_ptr() + t * bt.stb
                params[t].c.primary, params[t].c.tertiary = d_c.data_ptr() + t * bt.stc, C.addressof(keep[t])
            with Launches() as L:
                if route == "single":
                    for t in range(count):
                        X.GEMMFUNCTION(kern)(C.byref(params[t]))
                else:
                    assert X.libxsmm_b200_gemm_batch(kern, params, count) == 0
                X.check()
            L.expect(TC if route == "single" else SIMT, route)
            got = back(d_c, bt.buf_c)
            for t in range(count):
                one = Batch(m, n, k, ta, tb, F32, beta0, count=1, br=1, vnni=4, ldc=m + 2, tile_gap=32, guard=0)
                one.buf_a[:] = bt.buf_a[t * bt.sta:(t + 1) * bt.sta]; one.buf_b[:] = bt.buf_b[t * bt.stb:(t + 1) * bt.stb]
                one.buf_c[:] = bt.buf_c[t * bt.stc // 4:(t + 1) * bt.stc // 4]
                expect_int8(one, got[t * bt.stc // 4:(t + 1) * bt.stc // 4].copy(), scf=scales[t])
            expect_untouched(bt, got)


# ---- BCSC ----------------------------------------------------------------------------------------------------------------------
def bcsc_case(rng, ta, mblocks, M, K, N, bk, bn, beta0, out_of_range=True, empty_cols=(1,)):
    """pattern with unsorted row indices per column, block-rows >= K/bk (to be ignored) and empty block-columns"""
    nbr, nbc = K // bk, N // bn
    colptr = [0]; rows = []
    for j in range(nbc):
        r = [] if j in empty_cols else list(rng.permutation(nbr)[:max(1, nbr // 2 + j % 3)])
        if out_of_range and r:
            r.insert(len(r) // 2, nbr + j % 3)
        rows += r; colptr.append(len(rows))
    colptr = np.array(colptr, np.uint32); rowidx = np.array(rows or [0], np.uint32)
    nnzb = max(int(colptr[-1]), 1)
    if ta == BF16:
        a = grid_ints(rng, (mblocks, K, M), 15) / 4.0                          # [mb][k][m] logical
        bv = grid_ints(rng, (nnzb, bn, bk), 15) / 4.0                          # [z][n][k]
        c0 = grid_ints(rng, (mblocks, N, M), 255) / 16.0
        a_bits = encode(a.reshape(mblocks, K // 2, 2, M).transpose(0, 1, 3, 2), BF16)   # VNNI2: [mb][K/2][M][2]
        return colptr, rowidx, a, bv, c0, a_bits, encode(bv, BF16), encode(c0, BF16)
    lo, hi = (-128, 127) if ta == I8 else (0, 255)
    a = rng.integers(lo, hi + 1, size=(mblocks, K, M)); bv = rng.integers(-128, 128, size=(nnzb, bn, bk)) if ta == U8 else rng.integers(0, 256, size=(nnzb, bn, bk))
    c0 = rng.integers(-(1 << 31), 1 << 31, size=(mblocks, N, M))
    a_bits = encode(a.reshape(mblocks, K // 4, 4, M).transpose(0, 1, 3, 2), ta)    # VNNI4: [mb][K/4][M][4]
    return colptr, rowidx, a, bv, c0, a_bits, encode(bv, I8 if ta == U8 else U8), encode(c0, I32)


def bcsc_reference(colptr, rowidx, a, bv, c0, K, bk, bn, beta0):
    mblocks, _, M = a.shape
    N = (len(colptr) - 1) * bn
    acc = np.zeros((mblocks, N, M), dtype=a.dtype); mag = np.zeros_like(acc)
    for j in range(len(colptr) - 1):
        for z in range(colptr[j], colptr[j + 1]):
            kb = int(rowidx[z])
            if kb >= K // bk:
                continue
            blk = a[:, kb * bk:(kb + 1) * bk, :]                              # [mb][bk][M]
            acc[:, j * bn:(j + 1) * bn, :] += np.einsum("nk,bkm->bnm", bv[z], blk)
            mag[:, j * bn:(j + 1) * bn, :] += np.einsum("nk,bkm->bnm", np.abs(bv[z]), np.abs(blk))
    return acc, mag, (acc if beta0 else acc + c0)


def run_bcsc(ta, tb, tc, mblocks, M, K, N, bk, bn, beta0, a_bits, b_bits, c_bits, colptr, rowidx, backend):
    flags = (BETA_0 if beta0 else 0) | VNNI_A
    kern = X.libxsmm_create_packed_spgemm_bcsc(X.libxsmm_create_gemm_shape(mblocks, 0, K, K, 0, N, ta, tb, tc, F32 if tc == BF16 else I32), flags, 0,
                                               X.SpgemmConfig(M, bk, bn))
    assert kern
    if beta0 and tc == BF16:
        c_bits = np.full_like(c_bits, NAN_C[BF16])              # beta = 0 must not read C
    cbuf = np.concatenate([c_bits.ravel(), np.full(128 // ES[tc], int.from_bytes(bytes([SENTINEL]) * ES[tc], "little"), UINT[ES[tc]])])
    d_a, d_b, d_c, d_cp, d_ri = dev(a_bits), dev(b_bits), dev(cbuf), dev(colptr), dev(rowidx)
    with Launches() as L:
        X.call_gemm(kern, d_a, d_b, d_c, colptr=d_cp, rowidx=d_ri, nblocks=N // bn)
        X.check()
    L.expect(backend, ("bcsc", ta, M, K, N, bk, bn))
    X.libxsmm_release_kernel(kern)
    got = back(d_c, cbuf)
    assert np.all(got.view(np.uint8)[c_bits.nbytes:] == SENTINEL), "guard band after C written"
    return got[:c_bits.size].reshape(c_bits.shape)


@pytest.mark.parametrize("geo", [(4, 32, 128, 96, 32, 32), (3, 16, 64, 64, 16, 16), (5, 64, 192, 128, 64, 32), (3, 128, 64, 48, 16, 48)])
def test_bcsc_wgmma_exact(geo):
    mblocks, M, K, N, bk, bn = geo
    rng = np.random.default_rng(8000 + M + bk)
    for beta0 in (0, 1):
        colptr, rowidx, a, bv, c0, a_bits, b_bits, c_bits = bcsc_case(rng, BF16, mblocks, M, K, N, bk, bn, beta0)
        got = run_bcsc(BF16, BF16, BF16, mblocks, M, K, N, bk, bn, beta0, a_bits, b_bits, c_bits, colptr, rowidx, TC)
        acc, mag, exact = bcsc_reference(colptr, rowidx, a, bv, c0, K, bk, bn, beta0)
        assert np.all((mag + (0 if beta0 else np.abs(c0))) * 16 < 2 ** 24)
        want = round_out(exact, BF16)
        assert np.array_equal(got, want), (geo, beta0, int(np.count_nonzero(got != want)))
        if not beta0:                            # an empty block-column under beta = 1 keeps C bit for bit
            assert np.array_equal(got[:, bn:2 * bn, :], c_bits[:, bn:2 * bn, :])


@pytest.mark.parametrize("ta", [U8, I8])
def test_bcsc_int8_full_range(ta):
    """the exact-order BCSC kernel over the full int8 range (mixed signedness), unsorted rows, block-rows outside A ignored"""
    rng = np.random.default_rng(8100 + ta)
    tb = I8 if ta == U8 else U8
    for (mblocks, M, K, N, bk, bn) in ((3, 32, 128, 64, 32, 16), (2, 16, 64, 96, 16, 32)):
        for beta0 in (0, 1):
            colptr, rowidx, a, bv, c0, a_bits, b_bits, c_bits = bcsc_case(rng, ta, mblocks, M, K, N, bk, bn, beta0)
            got = run_bcsc(ta, tb, I32, mblocks, M, K, N, bk, bn, beta0, a_bits, b_bits, c_bits, colptr, rowidx, SIMT)
            _, _, exact = bcsc_reference(colptr, rowidx, a, bv, c0, K, bk, bn, beta0)
            assert np.array_equal(got.view(np.int32).astype(np.int64), wrap32(exact)), ((mblocks, M, K, N, bk, bn), beta0)


# ---- fused post-ops without a per-call operand through the batch forms ---------------------------------------------------------
@pytest.mark.parametrize("op", [X.MELTW_TYPE_UNARY_RELU, X.MELTW_TYPE_UNARY_SIGMOID])
def test_relu_and_sigmoid_without_mask_batch_equals_single_calls(op):
    """ReLU without a bit mask and sigmoid need nothing beyond A, B and C, so the batch forms run them: bit-identical to one call per tile"""
    rng = np.random.default_rng(9000 + op)
    m, n, k, count = 48, 24, 32, 7
    bt = Batch(m, n, k, F32, F32, F32, 0, count=count, br=2, ldc=m + 3, tile_gap=16)
    bt.fill(encode(rng.standard_normal(bt.idx_a.shape).astype(np.float32), F32), encode(rng.standard_normal(bt.idx_b.shape).astype(np.float32), F32),
            encode(rng.standard_normal(bt.idx_c.shape).astype(np.float32), F32))
    argops = X.libxsmm_create_gemm_ext_unary_argops(0, 0, 0, 0, 0, 0, 0, 0, m + 3, op, 0, 0)
    postops = X.libxsmm_create_gemm_ext_binary_postops(0, 0, 0, 0)
    kern = X.libxsmm_dispatch_brgemm_ext(X.libxsmm_create_gemm_shape(m, n, k, m, k, m + 3, F32, F32, F32, F32), 0, 0,
                                         X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, bt.bsa, bt.bsb, 0), argops, postops)
    assert kern
    d_a, d_b = dev(bt.buf_a), dev(bt.buf_b)
    d_c1, d_c2 = dev(bt.buf_c), dev(bt.buf_c)
    assert X.libxsmm_b200_gemm_batch_strided(kern, d_a.data_ptr(), d_b.data_ptr(), d_c1.data_ptr(), bt.sta, bt.stb, bt.stc, 2, count) == 0
    X.check()
    brv = C.c_ulonglong(2)
    for t in range(count):
        p = X.GemmExtParam(); p.op.tertiary = C.addressof(brv)
        p.a.primary, p.b.primary, p.c.primary = d_a.data_ptr() + t * bt.sta, d_b.data_ptr() + t * bt.stb, d_c2.data_ptr() + t * bt.stc
        X.GEMMFUNCTION_EXT(kern)(C.byref(p))
    X.check()
    got1, got2 = back(d_c1, bt.buf_c), back(d_c2, bt.buf_c)
    assert np.array_equal(got1, got2)
    expect_untouched(bt, got1)
    assert not np.array_equal(got1, bt.buf_c)
