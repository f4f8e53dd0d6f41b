"""CPU-only: the grid batch form (libxsmm_b200_gemm_batch_grid) on the simulated device of tests/c/hostsim_runtime.c, where every
GEMM tile is answered by the oracle of its family and "device" memory is host memory.

What this checks is the host half and the one tile mapping every exact-order kernel and the simulation share (xb_gemm_tile): tile
(i, j) of a grid reads row block i of A, column block j of B and writes its own C tile, for grids 1x1, 1xN, Nx1 and M x N, in the
plain-matrix and both blocked C layouts, without and with stride batch-reduce, for one handle of each family the simulated device
answers (plain, dequantising, low-bit); each C is compared bit for bit with single calls of the same handle on the same tiles. Then
every return code: the handle classes the strided form refuses, foreign and fused handles, negative sizes and strides, NULL operands,
pageable operands, empty grids, and both sides of every bound of the C overlap rule, with nothing launched and C untouched on a
refusal."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_gemm_batch as G  # noqa: E402  (the simulated libraries, one per family, and the handle table)
import libxsmm_b200 as X  # noqa: E402

F32, BF16, F16, BF8, I32, I8 = G.F32, G.BF16, G.F16, G.BF8, G.I32, G.I8
I2X4, VNNI_A, INTLV_A = G.I2X4, G.VNNI_A, G.INTLV_A
P, LL, ULL = C.c_void_p, C.c_longlong, C.c_ulonglong
NOT_BATCHABLE = -6   # include/libxsmm_b200.h

# name: family, (m, n, k, lda, ldb, ldc), (A, B, comp, C), flags, br_type (0 or 3). ldc leaves room for three row blocks of C, so that
# the same handle can write a plain 3 x N matrix of tiles.
RUNS = {
    "f32": ("plain", (8, 4, 8, 10, 9, 26), (F32, F32, F32, F32), 0, 0),
    "f32_stride": ("plain", (8, 4, 8, 10, 9, 26), (F32, F32, F32, F32), 0, 3),
    "bf16_f32_stride": ("plain", (8, 4, 8, 8, 9, 26), (BF16, BF16, F32, F32), 0, 3),
    "i8_i32_vnni": ("plain", (8, 4, 8, 8, 12, 26), (I8, I8, I32, I32), VNNI_A, 0),
    "bf8f16": ("dq", (8, 4, 8, 9, 8, 26), (BF8, F16, F32, F32), 0, 0),
    "bf8f16_stride": ("dq", (8, 4, 8, 9, 8, 26), (BF8, F16, F32, F32), 0, 3),
    "i2i8": ("lowbit", (8, 4, 16, 9, 17, 26), (I2X4, I8, I32, I32), VNNI_A | INTLV_A, 0),
}
GRIDS = [(1, 1), (1, 3), (3, 1), (3, 2), (2, 3)]
LAYOUTS = ["plain", "blocked", "blocked_t"]

_LIBS = {}


def lib_of(family):
    if family not in _LIBS:
        lib = G.build(family)
        fn = lib.libxsmm_b200_gemm_batch_grid
        fn.restype, fn.argtypes = C.c_int, [P] * 4 + [LL] * 4 + [ULL, LL, LL]
        fn = lib.libxsmm_b200_launch_count_backend
        fn.restype, fn.argtypes = ULL, [C.c_int]
        _LIBS[family] = lib
    return _LIBS[family]


@pytest.fixture(autouse=True)
def device_pointers(monkeypatch):
    monkeypatch.setenv("XB_HOSTSIM_PTR_KIND", "1")


class Grid:
    """a handle of RUNS and the operands of a gm x gn grid: gm row blocks of A, gn column blocks of B, C in `layout`"""

    def __init__(self, name, gm, gn, layout, seed=7):
        family, (m, n, k, lda, ldb, ldc), (ta, tb, tcomp, tc), flags, br_type = RUNS[name]
        self.lib, self.m, self.n, self.ldc, self.tc, self.gm, self.gn = lib_of(family), m, n, ldc, tc, gm, gn
        rng = np.random.default_rng(seed)
        self.br = 2 if br_type else 1
        blk_a, blk_b = lda * k * G.TS[ta], ldb * max(n, k) * G.TS[tb]
        shape = X.GemmShape(m, n, k, lda, ldb, ldc, ta, tb, tc, tcomp)
        if br_type:
            cfg = X.BatchReduceConfig(G.BR_API[br_type], blk_a, blk_b, 0)
            self.kernel = self.lib.libxsmm_dispatch_brgemm(shape, flags, 0, cfg)
        else:
            self.kernel = self.lib.libxsmm_dispatch_gemm(shape, flags, 0)
        assert self.kernel, name
        self.sa, self.sb = blk_a * self.br + 16, blk_b * self.br + 32      # row blocks of A and column blocks of B, with gaps
        self.A, self.B = G._fill(rng, self.sa * gm, ta), G._fill(rng, self.sb * gn, tb)
        esz = G.TS[tc]
        self.esz, self.span = esz, ((n - 1) * ldc + m) * esz
        if layout == "plain":        # one column-major C, row blocks m apart, column blocks n columns apart
            self.sm, self.sn = m * esz, n * ldc * esz
        elif layout == "blocked":    # whole tiles, column-major over the grid
            self.sm, self.sn = self.span, gm * self.span
        else:                        # whole tiles, row-major over the grid
            self.sm, self.sn = gn * self.span, self.span
        if gn == 1 and layout != "blocked_t":
            self.sn = 0              # a column of tiles: the column stride is never used
        extent = (gm - 1) * self.sm + (gn - 1) * self.sn + self.span
        self.C0 = G._fill(rng, extent, tc)
        self.brv = C.c_ulonglong(self.br)

    def grid(self, cbuf, **kw):
        a = dict(a=self.A.ctypes.data, b=self.B.ctypes.data, c=cbuf.ctypes.data, sa=self.sa, sb=self.sb, sm=self.sm, sn=self.sn,
                 gm=self.gm, gn=self.gn, kernel=self.kernel)
        a.update(kw)
        return self.lib.libxsmm_b200_gemm_batch_grid(a["kernel"], a["a"], a["b"], a["c"], a["sa"], a["sb"], a["sm"], a["sn"], self.br,
                                                     a["gm"], a["gn"])

    def singles(self):
        """C after one single call of the handle per tile (the oracle, tile by tile)"""
        c = self.C0.copy()
        for j in range(self.gn):
            for i in range(self.gm):
                p = X.GemmParam()
                p.op.tertiary = C.addressof(self.brv)
                p.a.primary = self.A.ctypes.data + i * self.sa
                p.b.primary = self.B.ctypes.data + j * self.sb
                p.c.primary = c.ctypes.data + i * self.sm + j * self.sn
                X.GEMMFUNCTION(self.kernel)(C.byref(p))
        return c


# a row or a column of tiles takes the strided rule, so it has no plain-matrix layout (test_row_or_column_of_tiles_takes_the_strided_rule)
SHAPES = [(gm, gn, layout) for gm, gn in GRIDS for layout in LAYOUTS if not (layout == "plain" and (gm == 1 or gn == 1))]


@pytest.mark.parametrize("gm,gn,layout", SHAPES, ids=["%dx%d_%s" % s for s in SHAPES])
@pytest.mark.parametrize("name", sorted(RUNS))
def test_grid_equals_single_calls_tile_by_tile(name, gm, gn, layout):
    g = Grid(name, gm, gn, layout)
    want = g.singles()
    c = g.C0.copy()
    n0 = g.lib.libxsmm_b200_launch_count()
    assert g.grid(c) == 0
    assert g.lib.libxsmm_b200_launch_count() - n0 == gm * gn      # the simulation counts one launch per tile
    assert np.array_equal(c, want)
    assert not np.array_equal(c, g.C0)


def test_pinned_operands_run_in_place(monkeypatch):
    monkeypatch.setenv("XB_HOSTSIM_PTR_KIND", "3")
    g = Grid("f32_stride", 3, 2, "blocked")
    want = g.singles()
    c = g.C0.copy()
    assert g.grid(c) == 0 and np.array_equal(c, want)


def refused(g, rc_want, **kw):
    """the call returns rc_want (0: an empty grid), launches nothing and leaves C alone"""
    c = g.C0.copy()
    n0 = g.lib.libxsmm_b200_launch_count()
    rc = g.grid(c, **kw)
    assert rc == rc_want, (kw, rc)
    assert g.lib.libxsmm_b200_launch_count() == n0
    assert np.array_equal(c, g.C0)


def accepted(g, **kw):
    """the call runs; C is sized for the strides of the call"""
    sm, sn = kw.get("sm", g.sm), kw.get("sn", g.sn)
    c = np.zeros((g.gm - 1) * sm + (g.gn - 1) * sn + g.span, dtype=np.uint8)
    n0 = g.lib.libxsmm_b200_launch_count()
    assert g.grid(c, **kw) == 0, kw
    assert g.lib.libxsmm_b200_launch_count() - n0 == g.gm * g.gn


def test_argument_faults():
    g = Grid("f32", 3, 2, "blocked")
    refused(g, -1, kernel=None)
    refused(g, -1, kernel=g.A.ctypes.data)              # not a handle
    for key in ("gm", "gn", "sa", "sb", "sm", "sn"):
        refused(g, -1, **{key: -1})
    for key in ("a", "b", "c"):
        refused(g, -1, **{key: None})
    refused(g, -1, gm=1 << 31, gn=1, sm=g.span)         # more tiles than a launch addresses
    for gm, gn in ((0, 2), (3, 0), (0, 0)):
        refused(g, 0, gm=gm, gn=gn)                     # an empty grid: 0, and nothing read or written
        refused(g, 0, gm=gm, gn=gn, a=None)


def test_pageable_operands(monkeypatch):
    monkeypatch.setenv("XB_HOSTSIM_PTR_KIND", "0")
    refused(Grid("f32", 3, 2, "blocked"), -4)


def test_fused_handle_is_refused():
    lib = lib_of("plain")
    ext = [i for i, h in enumerate(G.HANDLES) if h[0] == "ext"][0]
    h = G.Handle(lib, ext)
    c = h.C0.copy()
    assert lib.libxsmm_b200_gemm_batch_grid(h.kernel, h.A.ctypes.data, h.B.ctypes.data, c.ctypes.data, 0, 0, 0, 0, 1, 1, 1) == -1
    assert np.array_equal(c, h.C0)


# every handle class of the batch table that the strided form refuses, and two it runs: the grid form answers each the same way
@pytest.mark.parametrize("hname,want", [("f32_addr", -2), ("f32_offs", -2), ("bf16_vnni_c", NOT_BATCHABLE), ("u8i8_f32", NOT_BATCHABLE),
                                        ("i4x2u8_i32", NOT_BATCHABLE), ("i8bf16", NOT_BATCHABLE), ("i4f16", NOT_BATCHABLE),
                                        ("mxhf8_f32", NOT_BATCHABLE), ("mxbf8_c", NOT_BATCHABLE), ("mxfp4i8", NOT_BATCHABLE),
                                        ("f32", 0), ("f32_stride", 0)])
def test_handle_classes_match_the_strided_form(hname, want):
    hi = [i for i, h in enumerate(G.HANDLES) if h[0] == hname][0]
    lib = lib_of(G.HANDLES[hi][1])
    h = G.Handle(lib, hi)
    c = h.C0.copy()
    rc_strided = lib.libxsmm_b200_gemm_batch_strided(h.kernel, h.A.ctypes.data, h.B.ctypes.data, c.ctypes.data, h.tile_a, h.tile_b,
                                                     h.tile_c, h.br, h.count)
    assert rc_strided == want
    c = h.C0.copy()
    n0 = lib.libxsmm_b200_launch_count()
    rc = lib.libxsmm_b200_gemm_batch_grid(h.kernel, h.A.ctypes.data, h.B.ctypes.data, c.ctypes.data, h.tile_a, 0, h.tile_c, 0, h.br, h.count, 1)
    assert rc == want
    if want != 0:
        assert lib.libxsmm_b200_launch_count() == n0 and np.array_equal(c, h.C0)
        # the handle's refusal comes before the grid's own arguments are looked at, an empty grid included
        assert lib.libxsmm_b200_gemm_batch_grid(h.kernel, None, None, None, 0, 0, 0, 0, h.br, 0, 0) == want


def test_overlap_bounds_plain_matrix():
    g = Grid("f32", 3, 2, "plain")
    m, n, ldc, esz = g.m, g.n, g.ldc, g.esz
    accepted(g)
    refused(g, -1, sm=m * esz - 1)                                  # stride_c_m >= m*esz
    top = (ldc - m) * esz // 2                                      # (grid_m - 1)*stride_c_m + m*esz <= ldc*esz, grid_m = 3
    accepted(g, sm=top)
    refused(g, -1, sm=top + 1)
    refused(g, -1, sn=n * ldc * esz - 1)                            # stride_c_n >= n*ldc*esz
    accepted(g, sn=n * ldc * esz + 4)


def test_overlap_bounds_blocked():
    g = Grid("f32", 3, 2, "blocked")
    span = g.span
    accepted(g)
    refused(g, -1, sm=span - 1)                                     # stride_c_m >= span
    refused(g, -1, sn=3 * span - 1)                                 # stride_c_n >= grid_m*stride_c_m
    accepted(g, sm=span + 4, sn=3 * (span + 4))
    refused(g, -1, sm=span + 4, sn=3 * (span + 4) - 1)
    # the roles exchanged: column blocks whole tiles apart, row blocks whole rows of grid_n tiles apart
    accepted(g, sn=span, sm=2 * span)
    refused(g, -1, sn=span - 1, sm=2 * span)
    refused(g, -1, sn=span, sm=2 * span - 1)


def test_row_or_column_of_tiles_takes_the_strided_rule():
    col = Grid("f32", 3, 1, "blocked")                              # N x 1: stride_c_m >= span, stride_c_n unused
    accepted(col, sm=col.span, sn=0)
    refused(col, -1, sm=col.span - 1, sn=0)
    refused(col, -1, sm=col.m * col.esz, sn=col.n * col.ldc * col.esz)   # as a plain matrix it would not overlap; the strided rule decides
    row = Grid("f32", 1, 3, "blocked_t")                            # 1 x N: stride_c_n >= span, stride_c_m unused
    accepted(row, sn=row.span, sm=0)
    refused(row, -1, sn=row.span - 1, sm=0)
    one = Grid("f32", 1, 1, "blocked")                              # one tile: no stride is read
    accepted(one, sm=0, sn=0, sa=0, sb=0)
