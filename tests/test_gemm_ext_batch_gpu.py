"""GPU: libxsmm_b200_gemm_ext_batch_strided / libxsmm_b200_gemm_ext_batch, the batch forms of libxsmm_dispatch_brgemm_ext handles.
Every tile of a batch must equal, byte for byte, one single call of the same handle on the same operands -- C and the ReLU bit mask,
the mask's padding bits included -- and tile 0 the oracle under the bars of test_gemm_gpu.py's fused test. The single calls run on the
same fused kernel, which test_gemm_gpu.py, test_tc_exact_gpu.py and test_oracle_vs_ref.py pin against the reference."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import cases
import gen
import libxsmm_b200 as X
from gpu_util import dev, host, shape_of

pytestmark = pytest.mark.gpu

TYPES = [(gen.F32, gen.F32, gen.F32, gen.F32), (gen.BF16, gen.BF16, gen.F32, gen.BF16), (gen.BF16, gen.BF16, gen.F32, gen.F32),
         (gen.F16, gen.F16, gen.F32, gen.F16), (gen.U8, gen.I8, gen.I32, gen.F32)]
R, S = cases.RELU, cases.SIGMOID
FUSIONS = {"bias": (1, 0, 0, 0), "relu": (0, R, 0, 0), "relu_mask": (0, R, 1, 0), "sigmoid": (0, S, 0, 0), "bias_relu_mask": (1, R, 1, 0),
           "vnni_c": (0, 0, 0, 1), "bias_relu_vnni_c": (1, R, 0, 1)}
# the fused kernel's CTA block is 64 x 16 (32 x 32 for m <= 32). m % 32 != 0, m % 8 != 0, ldc > m, k past one 32-k chunk and not a
# multiple of it in the first two; 100 x 70 spans two row blocks (the second one partial) and five column blocks, 40 x 70 one row
# block; and a tile smaller than one block
SHAPES = [(100, 70, 72, 3), (40, 70, 72, 3), (13, 6, 8, 1)]
BR_MODES = [(0, 1), (3, 3), (2, 3)]


class Batch:
    """`count` tiles of one fused handle: device operands, the bias columns and the masks of every tile"""

    def __init__(self, types, fuse, beta0, br_type, br, shape, count, seed, alloc=dev, layout=None):
        ta, tb, tcomp, tc = types
        m, n, k, pad = shape
        rng = np.random.default_rng(seed)
        vnni_a = ta in (gen.I8, gen.U8) or (ta != gen.F32 and k % 2 == 0 and m % 2 == 0)
        flags = (cases.FLAG_BETA_0 if beta0 else 0) | ((cases.FLAG_VNNI_A if vnni_a else 0) if layout is None else layout)
        self.case = case = cases.GemmCase(m, n, k, ta, tb, tcomp, tc, flags=flags, br_type=br_type, br=br, pad=pad)
        self.ops = ops = cases.Operands(case, seed=int(rng.integers(1 << 30)), count=count)
        self.fuse, self.count, self.tc = fuse, count, tc
        self.mask_bytes = (case.ldc + 15) // 16 * 16 // 8 * n
        self.bias = gen.values(rng, m * count, tc)
        self.mask0 = rng.integers(0, 256, size=self.mask_bytes * count, dtype=np.uint8)
        argops = X.libxsmm_create_gemm_ext_unary_argops(0, 0, 0, 0, 0, 0, 0, 0, case.ldc, fuse[1], X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT if fuse[2] else 0, 0)
        postops = X.libxsmm_create_gemm_ext_binary_postops(case.ldc, tc, X.MELTW_TYPE_BINARY_ADD if fuse[0] else 0, X.MELTW_FLAG_BINARY_BCAST_COL_IN_0 if fuse[0] else 0)
        brt = {0: X.GEMM_BATCH_REDUCE_NONE, 1: X.GEMM_BATCH_REDUCE_ADDRESS, 2: X.GEMM_BATCH_REDUCE_OFFSET, 3: X.GEMM_BATCH_REDUCE_STRIDE}[br_type]
        cfg = X.libxsmm_create_gemm_batch_reduce_config(brt, ops.stride_a, ops.stride_b, 0)
        self.k = X.libxsmm_dispatch_brgemm_ext(shape_of(case), flags | (cases.FLAG_VNNI_C if fuse[3] else 0), 0, cfg, argops, postops)
        assert self.k, (case, fuse)
        self.alloc = alloc
        self.a, self.b, self.d = alloc(ops.a), alloc(ops.b), alloc(self.bias)
        self.keep = []

    def fresh(self):
        return self.alloc(self.ops.c0), self.alloc(self.mask0)

    def param(self, t, c, mk, scf=None):
        o, case = self.ops, self.case
        p = X.GemmExtParam(); brv = C.c_ulonglong(case.br); s = C.c_float(o.scf if scf is None else scf); self.keep += [brv, s]
        p.op.tertiary = C.addressof(brv); p.c.tertiary = C.addressof(s)
        if case.br_type == 1:
            o.case_br = case.br
            aa, ab = o.addr_arrays(self.a.data_ptr(), self.b.data_ptr(), t); self.keep += [aa, ab]
            p.a.primary, p.b.primary = C.addressof(aa), C.addressof(ab)
        else:
            p.a.primary, p.b.primary = self.a.data_ptr() + t * o.tile_a, self.b.data_ptr() + t * o.tile_b
        if o.offs_a is not None:
            p.a.secondary, p.b.secondary = o.offs_a.ctypes.data, o.offs_b.ctypes.data
        p.c.primary = c.data_ptr() + t * o.tile_c
        if self.fuse[0]:
            p.d.primary = self.d.data_ptr() + t * self.case.m * gen.TS[self.tc]
        if self.fuse[2]:
            p.c.secondary = mk.data_ptr() + t * self.mask_bytes
        return p

    def singles(self):
        c, mk = self.fresh()
        for t in range(self.count):
            X.GEMMFUNCTION_EXT(self.k)(C.byref(self.param(t, c, mk)))
        X.check()
        return c, mk

    def strided(self):
        c, mk = self.fresh()
        o = self.ops
        s = X.GemmExtStrides(o.tile_a, o.tile_b, o.tile_c, self.case.m * gen.TS[self.tc], self.mask_bytes)
        rc = X.libxsmm_b200_gemm_ext_batch_strided(self.k, C.byref(self.param(0, c, mk)), C.byref(s), self.count)
        assert rc == 0, (rc, X.libxsmm_b200_last_error_string())
        X.check()
        return c, mk

    def records(self, scales=None):
        c, mk = self.fresh()
        ps = (X.GemmExtParam * self.count)(*[self.param(t, c, mk, None if scales is None else scales[t]) for t in range(self.count)])
        rc = X.libxsmm_b200_gemm_ext_batch(self.k, ps, self.count)
        assert rc == 0, (rc, X.libxsmm_b200_last_error_string())
        X.check()
        return c, mk

    def oracle_tile0(self):
        from oracle_ffi import oracle
        want, wmask = self.ops.c0[:self.case.size_c].copy(), self.mask0[:self.mask_bytes].copy()
        assert cases.run_gemm_ext(oracle, self.case, self.ops, self.fuse, self.bias[:self.case.m] if self.fuse[0] else None,
                                  wmask if self.fuse[2] else None, want) == 0
        return want, wmask


def same(x, y):
    return np.array_equal(host(x, np.uint8), host(y, np.uint8))


def check_oracle(b, c, mk):
    want, wmask = b.oracle_tile0()
    got = host(c, gen.NP_OF[b.tc])[:b.case.size_c]
    if b.fuse[1] == S:
        tol = {gen.F32: 3e-7, gen.BF16: 8e-3, gen.F16: 1e-3}[b.tc]
        assert np.allclose(gen.to_f64(got, b.tc), gen.to_f64(want, b.tc), rtol=tol, atol=tol)
    else:
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
    if b.fuse[2]:
        assert np.array_equal(host(mk, np.uint8)[:b.mask_bytes], wmask)


@pytest.mark.parametrize("types", TYPES, ids=lambda t: "-".join(map(str, t)))
@pytest.mark.parametrize("fusion", sorted(FUSIONS))
def test_batches_equal_single_calls(types, fusion):
    fuse = FUSIONS[fusion]
    for shape in SHAPES:
        if fuse[3] and (types[3] == gen.F32 or shape[1] % 2):
            continue
        for beta0 in (1, 0):
            for br_type, br in BR_MODES + [(1, 3)]:
                b = Batch(types, fuse, beta0, br_type, br, shape, count=5, seed=zlib.crc32(repr((types, fusion, shape, beta0, br_type)).encode()))
                sc, sm = b.singles()
                if br_type != 1:
                    c, mk = b.strided()
                    assert same(c, sc) and same(mk, sm), (b.case, fusion, "strided")
                c, mk = b.records()
                assert same(c, sc) and same(mk, sm), (b.case, fusion, "records")
                if br_type in (0, 3):
                    check_oracle(b, sc, sm)


TA, TB, VA, VB = cases.FLAG_TRANS_A, cases.FLAG_TRANS_B, cases.FLAG_VNNI_A, cases.FLAG_VNNI_B
# every layout flag the fused dispatch serves, by how the kernel stages the operand: A p-major (TRANS_A), B packed (TRANS_B, VNNI-T B),
# and the operands the reference reads as zero (TRANS_A with VNNI_A, VNNI_B without TRANS_B for bf16)
LAYOUTS = [(TYPES[0], TA), (TYPES[0], TB), (TYPES[0], TA | TB),
           (TYPES[1], TA), (TYPES[1], TA | VA), (TYPES[1], TB | VA), (TYPES[1], TB | VB | VA), (TYPES[1], VB | VA),
           (TYPES[2], TA | TB), (TYPES[2], TB | VB | VA), (TYPES[3], TB | VA), (TYPES[3], TB)]


@pytest.mark.parametrize("types,layout", LAYOUTS, ids=lambda v: str(v))
def test_transposed_and_packed_layouts(types, layout):
    for fusion in ("bias_relu_mask", "sigmoid"):
        for beta0 in (1, 0):
            for shape in ((100, 70, 72, 3), (13, 6, 8, 1)):
                b = Batch(types, FUSIONS[fusion], beta0, 3, 2, shape, count=3, seed=zlib.crc32(repr((types, layout, fusion, beta0, shape)).encode()),
                          layout=layout)
                sc, sm = b.singles()
                c, mk = b.strided()
                assert same(c, sc) and same(mk, sm), (b.case, fusion, "strided")
                c, mk = b.records()
                assert same(c, sc) and same(mk, sm), (b.case, fusion, "records")
                check_oracle(b, sc, sm)


def test_one_simt_launch_per_batch_and_one_stream_pass_for_vnni_c():
    for fusion in ("bias_relu_mask", "vnni_c", "bias_relu_vnni_c"):
        b = Batch(TYPES[1], FUSIONS[fusion], 0, 3, 3, SHAPES[0], count=9, seed=5)
        for run in (b.strided, b.records):
            simt, stream = (X.libxsmm_b200_launch_count_backend(x) for x in (X.BACKEND_SIMT, X.BACKEND_STREAM))
            run()
            assert X.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT) - simt == 1, (fusion, run)
            assert X.libxsmm_b200_launch_count_backend(X.BACKEND_STREAM) - stream == (1 if "vnni_c" in fusion else 0), (fusion, run)


def test_unfused_bf16_ext_handle_stays_on_wgmma():
    b = Batch(TYPES[2], (0, 0, 0, 0), 1, 3, 4, (64, 64, 64, 0), count=6, seed=6)
    assert X.libxsmm_b200_kernel_backend(b.k) == X.BACKEND_TCGEN05
    sc, _ = b.singles()
    tc = X.libxsmm_b200_launch_count_backend(X.BACKEND_TCGEN05)
    c, _ = b.strided()
    assert X.libxsmm_b200_launch_count_backend(X.BACKEND_TCGEN05) - tc == 1
    assert same(c, sc)


def test_count_above_the_grid_cap():
    """more CTA blocks than the fused kernel's grid (4096 CTAs): the grid-stride loop covers them"""
    b = Batch(TYPES[1], FUSIONS["bias_relu_mask"], 0, 3, 2, (40, 40, 16, 0), count=1500, seed=7)   # 1500 tiles x 3 blocks
    sc, sm = b.singles()
    c, mk = b.strided()
    assert same(c, sc) and same(mk, sm)


def test_full_range_int8_with_per_tile_scales_in_the_record_form():
    b = Batch(TYPES[4], FUSIONS["bias_relu_mask"], 0, 3, 3, SHAPES[0], count=4, seed=8)
    rng = np.random.default_rng(9)
    full = rng.integers(0, 256, size=b.ops.a.size, dtype=np.uint8)
    b.a = dev(full.view(b.ops.a.dtype)); b.b = dev(rng.integers(0, 256, size=b.ops.b.size, dtype=np.uint8).view(b.ops.b.dtype))
    scales = [2.0 ** -(t + 3) for t in range(4)]
    c, mk = b.records(scales)
    sc, sm = b.fresh()
    for t in range(4):
        X.GEMMFUNCTION_EXT(b.k)(C.byref(b.param(t, sc, sm, scales[t])))
    X.check()
    assert same(c, sc) and same(mk, sm)


@pytest.mark.parametrize("kind", ["managed", "pinned"])
def test_managed_and_pinned_operands(kind):
    def managed(arr):
        raw = np.ascontiguousarray(arr).view(np.uint8)
        p = X.libxsmm_aligned_malloc(raw.size, 64)
        C.memmove(p, raw.ctypes.data, raw.size)
        return type("M", (), {"data_ptr": lambda self: p, "cpu": lambda self: torch.from_numpy(np.ctypeslib.as_array((C.c_ubyte * raw.size).from_address(p)).copy())})()

    def pinned(arr):
        return torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).copy()).pin_memory()
    alloc = managed if kind == "managed" else pinned
    b = Batch(TYPES[1], FUSIONS["bias_relu_mask"], 0, 3, 3, SHAPES[0], count=4, seed=10, alloc=alloc)
    sc, sm = b.singles()
    c, mk = b.strided()
    assert same(c, sc) and same(mk, sm)
    c, mk = b.records()
    assert same(c, sc) and same(mk, sm)
