"""Fused BRGEMM batches (libxsmm_b200_gemm_ext_batch_strided / libxsmm_b200_gemm_ext_batch) through the host half of the library on the
simulated device of test_meltw_batch_hostsim.py, where every fused tile is answered by the oracle and a batched mateltwise launch call by
call. What this checks is the host code: the per-tile bias / mask / C pointers handed to the launcher, a shared bias column, the -1 / -2
/ -4 rules with C and the mask untouched, count == 0, the VNNI_C chunks with a ragged last one -- each batch against single calls of the
same handle on the same tiles, bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gen
import libxsmm_b200 as X
from test_hostsim import CSRC, HOST_C, ORACLE, ROOT

OUT = os.path.join(ROOT, "tests", "c", "_hostsim", "gemm_ext_batch")


def build_sim():
    """the simulated device with a batched mateltwise launch answered call by call, and every exact-order GEMM launch counted once"""
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, "libxsmm.so")
    srcs = [os.path.join(CSRC, f) for f in HOST_C] + \
        [os.path.join(ROOT, "tests", "c", f) for f in ("hostsim_runtime.c", "hostsim_meltw_batch.c", "hostsim_gemm_launches.c")]
    if not (os.path.exists(so) and all(os.path.getmtime(f) < os.path.getmtime(so) for f in srcs + [os.path.join(CSRC, "xb_internal.h")])):
        cmd = ["gcc", "-O1", "-std=gnu99", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-Wl,--wrap=xb_meltw_launch",
               "-Wl,--wrap=xb_gemm_simt_launch", "-o", so] + srcs + ["-L" + ORACLE, "-loracle", "-Wl,-rpath," + ORACLE, "-lpthread", "-ldl", "-lm"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-3000:]
    lib = C.CDLL(so)
    for name in ("hostsim_batch_launches", "hostsim_gemm_launches"):
        fn = getattr(lib, name); fn.restype, fn.argtypes = C.c_ulonglong, []
    return lib

F32, BF16 = gen.F32, gen.BF16
I, U, P, LL, ULL, UB = C.c_int, C.c_uint, C.c_void_p, C.c_longlong, C.c_ulonglong, C.c_ubyte
RELU, BITMASK = X.MELTW_TYPE_UNARY_RELU, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT


@pytest.fixture(scope="module")
def sim():
    lib = build_sim()
    for name, res, args in (("libxsmm_create_gemm_shape", X.GemmShape, [I] * 10), ("libxsmm_create_gemm_batch_reduce_config", X.BatchReduceConfig, [I, I, I, UB]),
                            ("libxsmm_create_gemm_ext_unary_argops", X.GemmExtUnaryArgops, [I, I, U, I, I, I, U, I, I, I, U, I]),
                            ("libxsmm_create_gemm_ext_binary_postops", X.GemmExtBinaryPostops, [I, I, I, U]),
                            ("libxsmm_dispatch_gemm", P, [X.GemmShape, U, U]),
                            ("libxsmm_dispatch_brgemm_ext", P, [X.GemmShape, U, U, X.BatchReduceConfig, X.GemmExtUnaryArgops, X.GemmExtBinaryPostops]),
                            ("libxsmm_b200_gemm_ext_batch_strided", I, [P, C.POINTER(X.GemmExtParam), C.POINTER(X.GemmExtStrides), LL]),
                            ("libxsmm_b200_gemm_ext_batch", I, [P, C.POINTER(X.GemmExtParam), LL]),
                            ("libxsmm_b200_launch_count_backend", ULL, [I])):
        fn = getattr(lib, name); fn.restype, fn.argtypes = res, args
    return lib


@pytest.fixture(autouse=True)
def device_pointers(monkeypatch):
    monkeypatch.setenv("XB_HOSTSIM_PTR_KIND", "1")


class Tiles:
    def __init__(self, sim, tc, bias, relu, mask, beta0, br_type, count, m=13, n=6, k=8, pad=3, vnni_c=False, c_stride=None, seed=1):
        rng = np.random.default_rng(seed)
        self.sim, self.tc, self.count, self.m, self.n, self.k, self.br = sim, tc, count, m, n, k, (3 if br_type else 1)
        self.ldc, lda, ldb = m + pad, m + pad, k + pad
        self.bias_on, self.mask_on, self.br_type = bias, mask, br_type
        shape = sim.libxsmm_create_gemm_shape(m, n, k, lda, ldb, self.ldc, tc, tc, tc, F32)
        self.blk_a, self.blk_b = k * lda * gen.TS[tc], n * ldb * gen.TS[tc]
        brt = {0: X.GEMM_BATCH_REDUCE_NONE, 1: X.GEMM_BATCH_REDUCE_ADDRESS, 2: X.GEMM_BATCH_REDUCE_OFFSET, 3: X.GEMM_BATCH_REDUCE_STRIDE}[br_type]
        cfg = sim.libxsmm_create_gemm_batch_reduce_config(brt, self.blk_a, self.blk_b, 0)
        argops = sim.libxsmm_create_gemm_ext_unary_argops(0, 0, 0, 0, 0, 0, 0, 0, self.ldc, RELU if relu else 0, BITMASK if mask else 0, 0)
        postops = sim.libxsmm_create_gemm_ext_binary_postops(self.ldc, tc, X.MELTW_TYPE_BINARY_ADD if bias else 0, X.MELTW_FLAG_BINARY_BCAST_COL_IN_0 if bias else 0)
        flags = (X.GEMM_FLAG_BETA_0 if beta0 else 0) | (X.GEMM_FLAG_VNNI_A if tc == BF16 else 0) | (X.GEMM_FLAG_VNNI_C if vnni_c else 0)
        self.k_ext = sim.libxsmm_dispatch_brgemm_ext(shape, flags, 0, cfg, argops, postops)
        assert self.k_ext
        self.tile_a, self.tile_b = self.blk_a * self.br, self.blk_b * self.br
        c_bytes = n * self.ldc * gen.TS[tc]
        self.tile_c = c_stride or c_bytes
        self.mask_bytes = (self.ldc + 15) // 16 * 16 // 8 * n
        self.a = gen.values(rng, self.tile_a * count // gen.TS[tc], tc)
        self.b = gen.values(rng, self.tile_b * count // gen.TS[tc], tc)
        self.bias = gen.values(rng, m * count, tc)
        self.c0 = np.zeros(self.tile_c * (count - 1) + c_bytes, dtype=np.uint8)
        for t in range(count):
            self.c0[t * self.tile_c:t * self.tile_c + c_bytes] = gen.values(rng, c_bytes // gen.TS[tc], tc).view(np.uint8)
        self.mask0 = rng.integers(0, 256, size=self.mask_bytes * count, dtype=np.uint8)
        self.offs_a = (rng.permutation(self.br) * self.blk_a).astype(np.int64); self.offs_b = (rng.permutation(self.br) * self.blk_b).astype(np.int64)
        self.keep = []

    def param(self, t, c, mk, bias_stride=None):
        p = X.GemmExtParam(); brv = C.c_ulonglong(self.br); s = C.c_float(0.5); self.keep += [brv, s]
        p.op.tertiary = C.addressof(brv); p.c.tertiary = C.addressof(s)
        if self.br_type == 1:
            aa = (C.c_void_p * self.br)(*[self.a.ctypes.data + t * self.tile_a + r * self.blk_a for r in range(self.br)])
            ab = (C.c_void_p * self.br)(*[self.b.ctypes.data + t * self.tile_b + r * self.blk_b for r in range(self.br)])
            self.keep += [aa, ab]; p.a.primary, p.b.primary = C.addressof(aa), C.addressof(ab)
        else:
            p.a.primary, p.b.primary = self.a.ctypes.data + t * self.tile_a, self.b.ctypes.data + t * self.tile_b
        if self.br_type == 2:
            p.a.secondary, p.b.secondary = self.offs_a.ctypes.data, self.offs_b.ctypes.data
        p.c.primary = c.ctypes.data + t * self.tile_c
        if self.bias_on:
            p.d.primary = self.bias.ctypes.data + t * (self.m * gen.TS[self.tc] if bias_stride is None else bias_stride)
        if self.mask_on:
            p.c.secondary = mk.ctypes.data + t * self.mask_bytes
        return p

    def strides(self, bias_stride=None):
        return X.GemmExtStrides(self.tile_a, self.tile_b, self.tile_c, self.m * gen.TS[self.tc] if bias_stride is None else bias_stride, self.mask_bytes)

    def singles(self, bias_stride=None):
        c, mk = self.c0.copy(), self.mask0.copy()
        for t in range(self.count):
            X.GEMMFUNCTION_EXT(self.k_ext)(C.byref(self.param(t, c, mk, bias_stride)))
        return c, mk

    def strided(self, bias_stride=None, strides=None, count=None):
        c, mk = self.c0.copy(), self.mask0.copy()
        rc = self.sim.libxsmm_b200_gemm_ext_batch_strided(self.k_ext, C.byref(self.param(0, c, mk, bias_stride)), C.byref(strides or self.strides(bias_stride)),
                                                          self.count if count is None else count)
        return rc, c, mk

    def records(self):
        c, mk = self.c0.copy(), self.mask0.copy()
        ps = (X.GemmExtParam * self.count)(*[self.param(t, c, mk) for t in range(self.count)])
        return self.sim.libxsmm_b200_gemm_ext_batch(self.k_ext, ps, self.count), c, mk


@pytest.mark.parametrize("tc", [F32, BF16])
@pytest.mark.parametrize("br_type", [0, 2, 3])
def test_batches_equal_single_calls(sim, tc, br_type):
    for beta0 in (0, 1):
        for bias, relu, mask in ((1, 1, 1), (1, 0, 0), (0, 1, 1), (0, 1, 0)):
            tl = Tiles(sim, tc, bias, relu, mask, beta0, br_type, count=4, seed=beta0 * 7 + br_type)
            sc, sm = tl.singles()
            for run in (tl.strided, tl.records):
                launches = sim.hostsim_gemm_launches()
                rc, c, mk = run()
                assert rc == 0 and np.array_equal(c, sc) and np.array_equal(mk, sm), (tc, br_type, beta0, bias, relu, mask, run.__name__)
                assert sim.hostsim_gemm_launches() - launches == 1, "one launch per batch"


def test_stride_zero_shares_one_bias_column(sim):
    tl = Tiles(sim, F32, 1, 1, 1, 1, 3, count=5, seed=3)
    sc, sm = tl.singles(bias_stride=0)
    rc, c, mk = tl.strided(bias_stride=0)
    assert rc == 0 and np.array_equal(c, sc) and np.array_equal(mk, sm)
    assert not np.array_equal(sc, tl.singles()[0]), "the shared column is not every tile's own"


def test_address_mode_in_the_record_form_and_minus_2_in_the_strided_form(sim):
    tl = Tiles(sim, BF16, 1, 1, 1, 0, 1, count=3, seed=4)
    sc, sm = tl.singles()
    rc, c, mk = tl.records()
    assert rc == 0 and np.array_equal(c, sc) and np.array_equal(mk, sm)
    rc, c, mk = tl.strided()
    assert rc == -2 and np.array_equal(c, tl.c0) and np.array_equal(mk, tl.mask0)


def test_refusals_leave_c_and_the_mask_untouched(sim, monkeypatch):
    tl = Tiles(sim, F32, 1, 1, 1, 0, 3, count=3, seed=5)
    plain = sim.libxsmm_dispatch_gemm(sim.libxsmm_create_gemm_shape(13, 6, 8, 16, 11, 16, F32, F32, F32, F32), 0, 0)
    s = tl.strides

    def refused(want, **kw):
        before = sim.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT)
        rc, c, mk = tl.strided(**kw)
        assert rc == want, (kw, rc)
        assert np.array_equal(c, tl.c0) and np.array_equal(mk, tl.mask0), kw
        assert sim.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT) == before, kw
    refused(-1, count=-1)
    for field in ("a", "b", "c", "bias", "mask"):
        st = s(); setattr(st, field, -1); refused(-1, strides=st)
    st = s(); st.c = ((tl.n - 1) * tl.ldc + tl.m) * 4 - 1; refused(-1, strides=st)   # C of tile t reaches into tile t + 1
    st = s(); st.mask = tl.mask_bytes - 1; refused(-1, strides=st)               # so does its mask
    c, mk = tl.c0.copy(), tl.mask0.copy()
    for field in ("d", "c"):                                                     # a NULL bias / mask the handle needs
        p = tl.param(0, c, mk)
        setattr(getattr(p, field), "primary" if field == "d" else "secondary", None)
        assert sim.libxsmm_b200_gemm_ext_batch_strided(tl.k_ext, C.byref(p), C.byref(s()), 3) == -1
        ps = (X.GemmExtParam * 3)(*[tl.param(t, c, mk) for t in range(3)]); ps[2] = p
        assert sim.libxsmm_b200_gemm_ext_batch(tl.k_ext, ps, 3) == -1
    assert np.array_equal(c, tl.c0) and np.array_equal(mk, tl.mask0)
    assert sim.libxsmm_b200_gemm_ext_batch_strided(plain, C.byref(tl.param(0, c, mk)), C.byref(s()), 3) == -1
    assert sim.libxsmm_b200_gemm_ext_batch(plain, (X.GemmExtParam * 1)(tl.param(0, c, mk)), 1) == -1
    assert sim.libxsmm_b200_gemm_ext_batch_strided(None, C.byref(tl.param(0, c, mk)), C.byref(s()), 3) == -1
    monkeypatch.setenv("XB_HOSTSIM_PTR_KIND", "0")                               # pageable host memory
    refused(-4)
    rc, c, mk = tl.records()
    assert rc == -4 and np.array_equal(c, tl.c0) and np.array_equal(mk, tl.mask0)


def test_count_zero_does_nothing(sim):
    tl = Tiles(sim, F32, 1, 1, 1, 0, 3, count=2, seed=6)
    before = sim.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT)
    rc, c, mk = tl.strided(count=0)
    assert rc == 0 and np.array_equal(c, tl.c0) and np.array_equal(mk, tl.mask0)
    assert sim.libxsmm_b200_gemm_ext_batch(tl.k_ext, None, 0) == 0
    assert sim.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT) == before


def test_vnni_c_runs_in_chunks_with_a_ragged_last_one(sim):
    """C tiles 8 MiB apart: the 64 MiB scratch budget holds 8 tiles' span, so 20 tiles run as 8 + 8 + 4, each chunk one batched
    re-pack; every tile's packed C equals its single call's"""
    stride = 8 << 20
    tl = Tiles(sim, BF16, 1, 1, 0, 0, 3, count=20, m=6, n=4, k=8, pad=2, vnni_c=True, c_stride=stride, seed=7)
    sc, _ = tl.singles()
    passes, launches = sim.hostsim_batch_launches(), sim.hostsim_gemm_launches()
    rc, c, _ = tl.strided()
    assert rc == 0 and np.array_equal(c, sc)
    assert sim.hostsim_batch_launches() - passes == 3, "one batched re-pack per chunk"
    assert sim.hostsim_gemm_launches() - launches == 3, "one product launch per chunk"
    rc, c, _ = tl.records()
    assert rc == 0 and np.array_equal(c, sc)
    assert sim.hostsim_batch_launches() - passes == 6
    assert sim.hostsim_gemm_launches() - launches == 6


def test_record_form_under_vnni_c_refuses_unevenly_spaced_c(sim):
    """the re-pack after a VNNI_C batch is one strided pass: C tiles of the record form must sit at one distance from each other, at
    least one C apart; otherwise -1, with nothing launched and C untouched"""
    tl = Tiles(sim, BF16, 1, 1, 0, 0, 3, count=4, m=6, n=4, k=8, pad=2, vnni_c=True, seed=8)
    c_bytes = tl.n * tl.ldc * 2
    for gaps in ((1, 1, 2), (1, 0, 1)):          # tile 3 one C further; tiles 1 and 2 on top of each other
        c = np.zeros(c_bytes * 6, dtype=np.uint8); c0 = c.copy(); mk = tl.mask0.copy()
        offs = np.concatenate([[0], np.cumsum(gaps)]) * c_bytes
        ps = (X.GemmExtParam * 4)(*[tl.param(t, c, mk) for t in range(4)])
        for t in range(4):
            ps[t].c.primary = c.ctypes.data + int(offs[t])
        launches = sim.hostsim_gemm_launches()
        assert sim.libxsmm_b200_gemm_ext_batch(tl.k_ext, ps, 4) == -1, gaps
        assert np.array_equal(c, c0) and sim.hostsim_gemm_launches() == launches, gaps
