"""CPU-only: the C-ABI library loads, exports every symbol the headers declare, and its host-side logic
(dispatch identity, registry, descriptor validation, kernel info, conversions, thread safety) behaves like the
reference's (SURVEY.md 8b). No kernel is launched here."""
import ctypes as C
import glob
import os
import re
import threading

import numpy as np

import gen
import libxsmm_b200 as X
from oracle_ffi import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    names = set()
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        txt = open(h).read()
        txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
        for m in re.finditer(r"LIBXSMM_API(?:VAR)?\s+[^;{(]*?\b(libxsmm_\w+)\s*\(", txt):
            names.add(m.group(1))
    return sorted(names)


def test_every_declared_symbol_is_exported():
    names = declared_symbols()
    assert len(names) >= 70, names
    missing = [n for n in names if not hasattr(X.lib, n)]
    assert not missing, missing
    for g in ("libxsmm_ninit", "libxsmm_verbosity", "libxsmm_target_archid"):      # data symbols read by the LIBXSMM_INIT macro
        C.c_int.in_dll(X.lib, g)
    assert C.c_int.in_dll(X.lib, "libxsmm_ninit").value >= 1                        # the library constructor ran libxsmm_init
    assert set(X.EXPORTED) <= set(names) | {"libxsmm_aligned_malloc", "libxsmm_malloc", "libxsmm_free"}


def test_typesize_typename_and_arch():
    for t, sz in ((gen.F64, 8), (gen.F32, 4), (gen.BF16, 2), (gen.F16, 2), (gen.I32, 4), (gen.I16, 2), (gen.I8, 1), (gen.U8, 1)):
        assert X.libxsmm_typesize(t) == sz
    assert X.libxsmm_get_typename(gen.F32) == b"f32" and X.libxsmm_get_typename(gen.BF16) == b"bf16"
    assert X.libxsmm_get_target_arch() == b"sm_90a"
    v = X.libxsmm_get_verbosity(); X.libxsmm_set_verbosity(v)


def test_host_conversions_match_the_oracle():
    rng = np.random.default_rng(5)
    bits = np.concatenate([rng.integers(0, 2**32, size=5000, dtype=np.uint64).astype(np.uint32),
                           np.array([0, 0x80000000, 0x7f800000, 0xff800000, 0x7fc00000, 0x7f800001, 1, 0x007fffff, 0x38800000, 0x387fffff,
                                     0x33000000, 0x33000001, 0x477fe000, 0x477ff000, 0x47800000], dtype=np.uint32)])
    for u in bits:
        f = float(np.array([u], dtype=np.uint32).view(np.float32)[0])
        assert X.libxsmm_convert_f32_to_bf16_rne(f) == oracle["f32_to_bf16"](f), hex(u)
        assert X.libxsmm_convert_f32_to_f16(f) == oracle["f32_to_f16"](f), hex(u)
    for h in range(0, 65536, 13):
        g, w = X.libxsmm_convert_bf16_to_f32(h), oracle["bf16_to_f32"](h)
        assert g == w or (g != g and w != w), h
        g, w = X.libxsmm_convert_f16_to_f32(h), oracle["f16_to_f32"](h)
        assert g == w or (g != g and w != w), h


def _shape(m, n, k, t=gen.F32):
    return X.libxsmm_create_gemm_shape(m, n, k, m, k, m, t, t, t, t)


def test_dispatch_identity_registry_and_kernel_info():
    reg0 = X.RegistryInfo(); assert X.libxsmm_get_registry_info(C.byref(reg0)) == 0
    assert reg0.capacity >= 4096                                             # tests/threadsafety.c dispatches ~800 shapes at once
    k1 = X.libxsmm_dispatch_gemm(_shape(13, 5, 7), 0, 0)
    k2 = X.libxsmm_dispatch_gemm(_shape(13, 5, 7), 0, 0)
    k3 = X.libxsmm_dispatch_gemm(_shape(13, 5, 7), X.GEMM_FLAG_BETA_0, 0)
    k4 = X.libxsmm_dispatch_gemm(_shape(13, 5, 8), 0, 0)
    assert k1 and k1 == k2 and len({k1, k3, k4}) == 3                         # same descriptor -> same pointer
    reg1 = X.RegistryInfo(); X.libxsmm_get_registry_info(C.byref(reg1))
    assert reg1.size >= reg0.size + 1 and reg1.capacity == reg0.capacity
    info = X.KernelInfo(); assert X.libxsmm_get_kernel_info(k1, C.byref(info)) == 0
    assert info.nflops == 2 * 13 * 5 * 7 and info.is_reference_kernel == 0   # nflops is not multiplied by br (libxsmm_main.c:2184)
    mm = X.MMKernelInfo(); assert X.libxsmm_get_mmkernel_info(k3, C.byref(mm)) == 0
    assert (mm.m, mm.n, mm.k, mm.lda, mm.ldb, mm.ldc) == (13, 5, 7, 13, 7, 13) and (mm.flags & X.GEMM_FLAG_BETA_0)
    assert X.libxsmm_get_kernel_info(0, C.byref(info)) != 0                  # not one of our handles
    X.libxsmm_release_kernel(k1)                                             # registry-owned: must stay valid (libxsmm_main.c:3916-3921)
    assert X.libxsmm_dispatch_gemm(_shape(13, 5, 7), 0, 0) == k1
    # batch-reduce variants are distinct kernels
    cfg = X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, 13 * 7 * 4, 7 * 5 * 4, 0)
    kb = X.libxsmm_dispatch_brgemm(_shape(13, 5, 7), 0, 0, cfg)
    assert kb and kb != k1
    assert X.libxsmm_b200_kernel_backend(k1) == X.BACKEND_SIMT
    bf = X.libxsmm_create_gemm_shape(64, 64, 64, 64, 64, 64, gen.BF16, gen.BF16, gen.F32, gen.F32)
    cfgb = X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, 8192, 8192, 0)
    assert X.libxsmm_b200_kernel_backend(X.libxsmm_dispatch_brgemm(bf, X.GEMM_FLAG_BETA_0, 0, cfgb)) == X.BACKEND_TCGEN05


def test_unsupported_descriptors_return_null():
    BF8, HF8 = 4, 5
    assert X.libxsmm_dispatch_gemm(X.libxsmm_create_gemm_shape(16, 16, 16, 16, 16, 16, BF8, BF8, gen.F32, gen.F32), 0, 0)       # 8-bit float tuples are served (exact-order kernel)
    assert not X.libxsmm_dispatch_gemm(X.libxsmm_create_gemm_shape(16, 16, 16, 16, 16, 16, BF8, HF8, gen.F32, gen.F32), 0, 0)   # mixed 8-bit operands: no reference branch
    assert not X.libxsmm_dispatch_gemm(X.libxsmm_create_gemm_shape(16, 16, 16, 16, 16, 16, 20, gen.BF16, gen.F32, gen.F32), 0, 0)  # MXFP4 A: SURVEY 8f-2, not built
    assert not X.libxsmm_dispatch_gemm(X.libxsmm_create_gemm_shape(16, 16, 16, 8, 16, 16, gen.F32, gen.F32, gen.F32, gen.F32), 0, 0)   # lda < m
    assert not X.libxsmm_dispatch_gemm(X.libxsmm_create_gemm_shape(0, 16, 16, 16, 16, 16, gen.F32, gen.F32, gen.F32, gen.F32), 0, 0)
    # inconsistent tile-config flags (libxsmm_generator.c:154-157)
    both = X.GEMM_FLAG_NO_RESET_TILECONFIG | X.GEMM_FLAG_NO_SETUP_TILECONFIG
    assert X.libxsmm_dispatch_tilecfg_gemm(_shape(16, 16, 16), X.GEMM_FLAG_NO_RESET_TILECONFIG)
    assert not X.libxsmm_dispatch_tilecfg_gemm(_shape(16, 16, 16), both)


def test_fsspmdm_variant_of_no_handle():
    """libxsmm_b200_fsspmdm_variant answers -1 without a handle (0 / 1..3 name the direct and the staged kernel)"""
    b = np.zeros(64, dtype=np.float32)
    assert X.libxsmm_b200_fsspmdm_variant(None, None, None) == -1
    assert X.libxsmm_b200_fsspmdm_variant(None, b.ctypes.data, b.ctypes.data) == -1


def test_meltw_dispatch_host_logic():
    sh = X.libxsmm_create_meltw_unary_shape(10, 7, 10, 10, gen.F32, gen.F32, gen.F32)
    k = X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_RELU, sh, 0)
    assert k and k == X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_RELU, sh, 0)
    assert k != X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_TANH, sh, 0)
    assert X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_DROPOUT, sh, 0)                          # 16-lane generator like the reference's 512-bit targets
    assert not X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_STOCHASTIC_ROUND, sh, 0)             # not built
    bs = X.libxsmm_create_meltw_binary_shape(10, 7, 10, 10, 10, gen.F32, gen.F32, gen.F32, gen.F32)
    assert X.libxsmm_dispatch_meltw_binary(X.MELTW_TYPE_BINARY_ADD, bs, 0)
    info = X.KernelInfo(); assert X.libxsmm_get_kernel_info(k, C.byref(info)) == 0


def test_concurrent_dispatch_is_consistent():
    """tests/threadsafety.c in miniature: many threads dispatch an overlapping set of shapes"""
    shapes = [(m, n, k) for m in range(1, 9) for n in range(1, 9) for k in (4, 8, 12)]
    results = [dict() for _ in range(8)]

    def work(tid):
        rng = np.random.default_rng(tid)
        for i in rng.permutation(len(shapes)):
            m, n, k = shapes[i]
            results[tid][shapes[i]] = X.libxsmm_dispatch_gemm(_shape(m + 40, n + 40, k), 0, 0)
    th = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    [t.start() for t in th]; [t.join() for t in th]
    for s in shapes:
        ptrs = {r[s] for r in results}
        assert len(ptrs) == 1 and None not in ptrs and 0 not in ptrs, s
    assert len({results[0][s] for s in shapes}) == len(shapes)
