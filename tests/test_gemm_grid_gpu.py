"""GPU: libxsmm_b200_gemm_batch_grid, the blocked GEMM of a BRGEMM handle over a grid of C tiles in one launch.

For each kernel family a grid can reach -- wgmma with flat bf16 / f16 A, VNNI2 bf16 A and VNNI4 int8 A, and the exact-order f32,
int8 dp4a, dequantising (BF8 x F16) and low-bit (I2 x I8) kernels -- a ragged 3 x 2 grid in the plain-matrix and the blocked C layout
must equal, byte for byte, the same tiles run one block column at a time through libxsmm_b200_gemm_batch_strided with unique copies
of the shared B block (so that those calls stay on their usual kernel), and the oracle tile by tile: bit for bit on the exact-order
kernels and int8 wgmma, within the reference's norms on bf16 / f16 wgmma. libxsmm_b200_launch_count_backend shows that a grid is one
launch of the kernel family a strided batch of the handle runs on, and that a grid whose A stride breaks the TMA rules runs on the
exact-order kernel. A 40 x 24 grid has more tiles than the wgmma kernel starts
CTAs, so every CTA walks several of them. Last, a 1024 x 768 x 2048 bf16 GEMM in plain-matrix layout, 64 x 64 blocks with K reduced by
stride batch-reduce, against a float64 product."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import gen
import libxsmm_b200 as X
from gpu_util import dev, host
from oracle_ffi import oracle, iarr

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden_gemm_batch as G  # noqa: E402  (the operand filler shared with the batch table)

pytestmark = pytest.mark.gpu

F32, BF16, F16, BF8, I32, I8, I2X4 = G.F32, G.BF16, G.F16, G.BF8, G.I32, G.I8, G.I2X4
VNNI_A, INTLV_A, BETA_0 = G.VNNI_A, G.INTLV_A, G.BETA_0
TC, SIMT = X.BACKEND_TCGEN05, X.BACKEND_SIMT

# name: (m, n, k), (A, B, comp, C), flags, br_type, oracle, backend, tolerance (None: bit for bit), force the exact-order kernel
FAMILIES = {
    "bf16_flat_f32": ((64, 64, 64), (BF16, BF16, F32, F32), 0, 3, "plain", TC, 1.2e-5, False),
    "f16_flat_f32_m128": ((128, 96, 64), (F16, F16, F32, F32), 0, 3, "plain", TC, 1.2e-5, False),
    "bf16_vnni2_bf16": ((64, 64, 64), (BF16, BF16, F32, BF16), VNNI_A, 3, "plain", TC, 5e-3, False),
    "i8_vnni4_i32": ((64, 64, 128), (I8, I8, I32, I32), VNNI_A, 3, "plain", TC, None, False),
    "f32": ((24, 20, 40), (F32, F32, F32, F32), 0, 3, "plain", SIMT, None, False),
    "i8_vnni4_i32_dp4a": ((32, 32, 64), (I8, I8, I32, I32), VNNI_A, 0, "plain", SIMT, None, True),
    "bf8f16_dq": ((32, 16, 32), (BF8, F16, F32, F32), 0, 3, "dq", SIMT, None, False),
    "i2i8_lowbit": ((32, 16, 64), (I2X4, I8, I32, I32), VNNI_A | INTLV_A, 0, "lowbit", SIMT, None, False),
}
GM, GN = 3, 2


def backend_counts():
    return X.libxsmm_b200_launch_count_backend(TC), X.libxsmm_b200_launch_count_backend(SIMT)


class Grid:
    def __init__(self, name, layout, a_skew=0, seed=11, gm=GM, gn=GN):
        (m, n, k), (ta, tb, tcomp, tc), flags, br_type, self.oracle, self.backend, self.tol, simt = FAMILIES[name]
        rng = np.random.default_rng(seed)
        self.m, self.n, self.k, self.types, self.flags, self.br_type = m, n, k, (ta, tb, tcomp, tc), flags, br_type
        self.br = 3 if br_type else 1
        self.gm, self.gn = gm, gn
        self.lda, self.ldb, self.ldc = m, k, (gm * m if layout == "plain" else m) + 8   # plain matrix: room for gm row blocks
        self.blk_a, self.blk_b = self.lda * k * G.TS[ta], self.ldb * n * G.TS[tb]
        shape = X.libxsmm_create_gemm_shape(m, n, k, self.lda, self.ldb, self.ldc, ta, tb, tc, tcomp)
        X.libxsmm_b200_set_force_simt(1 if simt else 0)
        try:
            if br_type:
                cfg = X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, self.blk_a, self.blk_b, 0)
                self.kernel = X.libxsmm_dispatch_brgemm(shape, flags, 0, cfg)
            else:
                self.kernel = X.libxsmm_dispatch_gemm(shape, flags, 0)
        finally:
            X.libxsmm_b200_set_force_simt(0)
        assert self.kernel and X.libxsmm_b200_kernel_backend(self.kernel) == self.backend, name
        self.sa, self.sb = self.blk_a * self.br + a_skew, self.blk_b * self.br
        self.A, self.B = G._fill(rng, self.sa * self.gm, ta), G._fill(rng, self.sb * self.gn, tb)
        self.esz = G.TS[tc]
        self.span = ((n - 1) * self.ldc + m) * self.esz
        self.sm, self.sn = (m * self.esz, n * self.ldc * self.esz) if layout == "plain" else (self.span, self.gm * self.span)
        self.C0 = G._fill(rng, (self.gm - 1) * self.sm + (self.gn - 1) * self.sn + self.span, tc)

    def grid(self):
        d_a, d_b, d_c = dev(self.A), dev(self.B), dev(self.C0)
        before = backend_counts()
        assert X.libxsmm_b200_gemm_batch_grid(self.kernel, d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), self.sa, self.sb, self.sm,
                                              self.sn, self.br, self.gm, self.gn) == 0
        X.check()
        after = backend_counts()
        return host(d_c, np.uint8), (after[0] - before[0], after[1] - before[1])

    def by_columns(self):
        """the same tiles, one strided batch per block column, each tile with its own copy of the column's B block"""
        d_a, d_c = dev(self.A), dev(self.C0)
        counts = []
        for j in range(self.gn):
            d_b = dev(np.tile(self.B[j * self.sb:(j + 1) * self.sb], self.gm))
            before = backend_counts()
            assert X.libxsmm_b200_gemm_batch_strided(self.kernel, d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr() + j * self.sn, self.sa,
                                                     self.sb, self.sm, self.br, self.gm) == 0
            X.check()
            after = backend_counts()
            counts.append((after[0] - before[0], after[1] - before[1]))
        return host(d_c, np.uint8), counts

    def oracle_tiles(self):
        c = self.C0.copy()
        dims, types = iarr(self.m, self.n, self.k, self.lda, self.ldb, self.ldc), iarr(*self.types)
        for j in range(self.gn):
            for i in range(self.gm):
                a, b = self.A.ctypes.data + i * self.sa, self.B.ctypes.data + j * self.sb
                cp = c.ctypes.data + i * self.sm + j * self.sn
                args = (dims, types, self.flags, self.br_type, self.blk_a, self.blk_b, self.br, a, b, cp, None, None)
                if self.oracle == "plain":
                    rc = oracle["gemm"](*args, 0.0, 0)
                elif self.oracle == "dq":
                    import dq_ffi
                    rc = dq_ffi.oracle_gemm_dq(*args, None, None)
                else:
                    import lowbit_ffi
                    rc = lowbit_ffi.oracle_gemm_lowbit(*args, None, None)
                assert rc == 0
        return c

    def c_values(self, raw):
        """the C elements of every tile, as float64"""
        tc = self.types[3]
        out = []
        for j in range(self.gn):
            for i in range(self.gm):
                for col in range(self.n):
                    off = i * self.sm + j * self.sn + col * self.ldc * self.esz
                    seg = raw[off:off + self.m * self.esz]
                    out.append(gen.to_f64(seg.view(gen.NP_OF[tc]), tc))
        return np.concatenate(out)


@pytest.mark.parametrize("layout", ["plain", "blocked"])
@pytest.mark.parametrize("name", list(FAMILIES))
def test_grid_equals_strided_columns_and_the_oracle(name, layout):
    g = Grid(name, layout)
    got, counts = g.grid()
    want, col_counts = g.by_columns()
    assert np.array_equal(got, want), name
    one = (1, 0) if g.backend == TC else (0, 1)
    assert counts == one and col_counts == [one] * g.gn, (counts, col_counts)
    ref = g.oracle_tiles()
    if g.tol is None:
        assert np.array_equal(got, ref)
    else:
        assert gen.normf_rel(g.c_values(ref), g.c_values(got)) <= g.tol
        # bytes outside the tiles are untouched
        mask = np.ones(got.size, bool)
        for j in range(g.gn):
            for i in range(g.gm):
                for col in range(g.n):
                    off = i * g.sm + j * g.sn + col * g.ldc * g.esz
                    mask[off:off + g.m * g.esz] = False
        assert np.array_equal(got[mask], g.C0[mask])


@pytest.mark.parametrize("name", ["bf16_flat_f32", "bf16_vnni2_bf16", "i8_vnni4_i32"])
def test_misaligned_grid_runs_on_the_exact_order_kernel(name):
    g = Grid(name, "blocked", a_skew=8)                 # row blocks of A 8 bytes off a 16-byte multiple: no tensor map
    got, counts = g.grid()
    want, col_counts = g.by_columns()
    assert counts == (0, 1) and col_counts == [(0, 1)] * g.gn
    assert np.array_equal(got, want)
    ref = g.oracle_tiles()
    assert np.array_equal(got, ref)                   # the exact-order kernel restates the reference's order


@pytest.mark.parametrize("name", ["bf16_flat_f32", "f16_flat_f32_m128", "bf16_vnni2_bf16", "i8_vnni4_i32"])
def test_every_cta_walks_several_grid_tiles(name):
    # 40 x 24 = 960 tiles, more than the 132 SMs x up to 3 CTAs the wgmma kernel starts: each CTA takes tiles b, b + G, ... and
    # recovers (i, j) from each of them
    g = Grid(name, "blocked", gm=40, gn=24)
    got, counts = g.grid()
    want, col_counts = g.by_columns()
    assert counts == (1, 0) and col_counts == [(1, 0)] * g.gn
    assert np.array_equal(got, want)
    assert not np.array_equal(got, g.C0)


def test_large_gemm_in_plain_matrix_layout():
    M, N, K, b = 1024, 768, 2048, 64
    rng = np.random.default_rng(3)
    a = gen.values(rng, M * K, gen.BF16)              # column-major M x K, lda = M
    bm = gen.values(rng, K * N, gen.BF16)             # column-major K x N, ldb = K
    shape = X.libxsmm_create_gemm_shape(b, b, b, M, K, M, BF16, BF16, F32, F32)
    cfg = X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, b * M * 2, b * 2, 0)
    kernel = X.libxsmm_dispatch_brgemm(shape, BETA_0, 0, cfg)
    assert kernel and X.libxsmm_b200_kernel_backend(kernel) == TC
    d_a, d_b = dev(a), dev(bm)
    d_c = torch.zeros(M * N * 4, dtype=torch.uint8, device="cuda")
    before = backend_counts()
    assert X.libxsmm_b200_gemm_batch_grid(kernel, d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), b * 2, b * K * 2, b * 4, b * M * 4,
                                          K // b, M // b, N // b) == 0
    X.check()
    after = backend_counts()
    assert (after[0] - before[0], after[1] - before[1]) == (1, 0)
    A = gen.to_f64(a, gen.BF16).reshape(K, M).T
    B = gen.to_f64(bm, gen.BF16).reshape(N, K).T
    want = (A @ B).T.reshape(-1)                      # column-major M x N
    got = host(d_c, np.float32).astype(np.float64)
    assert gen.normf_rel(want, got) <= 1.2e-5
