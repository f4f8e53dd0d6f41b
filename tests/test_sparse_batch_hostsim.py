"""Batched packed-sparse, packed-dense and BCSC calls (libxsmm_b200_spgemm_batch_strided) through the host half of the library on the
simulated device: the host_*.c objects, tests/c/hostsim_runtime.c and tests/c/hostsim_sparse_batch.c (every packed / BCSC launch
answered call by call by the oracle) linked into tests/c/_hostsim/sparse_batch/libxsmm.so. What this checks is the host code: the
strides handed to the launchers, the C extent behind the overlap rule, the -1 / -4 / NOT_BATCHABLE rules and that the BCSC pattern
is read once, from call 0 -- each batch against single calls of the same handle on the same operands."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gen
import libxsmm_b200 as X
from sparse_batch_cases import PACKED_KINDS, POISON, BcscCase, PackedCase, param
from test_hostsim import CSRC, HOST_C, ORACLE, ROOT

OUT = os.path.join(ROOT, "tests", "c", "_hostsim", "sparse_batch")
NOT_BATCHABLE = -6
BCSC_TYPES = {"f32": (gen.F32, gen.F32, gen.F32, gen.F32), "bf16": (gen.BF16, gen.BF16, gen.F32, gen.BF16),
              "u8i8": (gen.U8, gen.I8, gen.I32, gen.I32)}


def build_sim():
    os.makedirs(OUT, exist_ok=True)
    if not os.path.exists(os.path.join(ORACLE, "liboracle.so")):
        subprocess.check_call(["make", "-C", ROOT, "oracle"])
    so = os.path.join(OUT, "libxsmm.so")
    srcs = [os.path.join(CSRC, f) for f in HOST_C] + [os.path.join(ROOT, "tests", "c", f) for f in ("hostsim_runtime.c", "hostsim_sparse_batch.c")]
    deps = srcs + [os.path.join(CSRC, "xb_internal.h"), os.path.join(ROOT, "include", "libxsmm_b200.h")]
    if not (os.path.exists(so) and all(os.path.getmtime(s) < os.path.getmtime(so) for s in deps)):
        wrap = "-Wl,--wrap=xb_packed_sp_launch,--wrap=xb_bcsc_launch,--wrap=xb_rt_ptr_kind"
        cmd = ["gcc", "-O1", "-std=gnu99", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), wrap, "-o", so] + \
            srcs + ["-L" + ORACLE, "-loracle", "-Wl,-rpath," + ORACLE, "-lpthread", "-ldl", "-lm"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-3000:]
    lib = C.CDLL(so)
    P, LL, I = C.c_void_p, C.c_longlong, C.c_int
    sp = [X.GemmShape, C.c_uint, C.c_uint, I, P, P, P]
    for name, res, args in (("libxsmm_create_packed_spgemm_csr", P, sp), ("libxsmm_create_packed_spgemm_csc", P, sp),
                            ("libxsmm_create_packed_gemm", P, [X.GemmShape, C.c_uint, C.c_uint, I]),
                            ("libxsmm_create_packed_gemm_ac_rm", P, [X.GemmShape, C.c_uint, C.c_uint, I]),
                            ("libxsmm_create_packed_gemm_bc_rm", P, [X.GemmShape, C.c_uint, C.c_uint, I]),
                            ("libxsmm_create_packed_spgemm_bcsc", P, [X.GemmShape, C.c_uint, C.c_uint, X.SpgemmConfig]),
                            ("libxsmm_create_spgemm_csr_areg", P, [X.GemmShape, C.c_uint, C.c_uint, I, P, P, P]),
                            ("libxsmm_dispatch_gemm", P, [X.GemmShape, C.c_uint, C.c_uint]),
                            ("libxsmm_b200_spgemm_batch_strided", I, [P, C.POINTER(X.GemmParam), C.POINTER(X.SpgemmStrides), LL]),
                            ("hostsim_sparse_launches", C.c_ulonglong, []), ("hostsim_sparse_calls", C.c_ulonglong, []),
                            ("hostsim_sparse_last_bcsc", None, [C.POINTER(P), C.POINTER(P), C.POINTER(C.c_ulonglong), C.POINTER(C.c_uint)]),
                            ("hostsim_sparse_mark_pageable", None, [P, C.c_size_t]), ("hostsim_sparse_clear_pageable", None, [])):
        fn = getattr(lib, name); fn.restype, fn.argtypes = res, args
    return lib


@pytest.fixture(scope="module")
def sim():
    return build_sim()


@pytest.fixture(autouse=True)
def device_pointers(monkeypatch, sim):
    monkeypatch.setenv("XB_HOSTSIM_PTR_KIND", "1")      # every pointer is "device memory" unless a test marks it pageable
    sim.hostsim_sparse_clear_pageable()
    yield
    sim.hostsim_sparse_clear_pageable()


def run_batch(sim, k, case, count, extra=None):
    """the batch on copies of the case's images; returns (rc, C image, launches)"""
    a, b, c = case.a.copy(), case.b.copy(), case.c.copy()
    extra = extra or {}
    p = param(a.ctypes.data, b.ctypes.data, c.ctypes.data, case.strides, 0, **extra)
    before = sim.hostsim_sparse_launches()
    rc = sim.libxsmm_b200_spgemm_batch_strided(k, C.byref(p), C.byref(X.SpgemmStrides(*case.strides)), count)
    return rc, c, sim.hostsim_sparse_launches() - before


def run_singles(k, case, count, extra=None):
    a, b, c = case.a.copy(), case.b.copy(), case.c.copy()
    for t in range(count):
        X.GEMMFUNCTION(k)(C.byref(param(a.ctypes.data, b.ctypes.data, c.ctypes.data, case.strides, t, **(extra or {}))))
    return c


@pytest.mark.parametrize("kind,dtype", [(k, t) for k in PACKED_KINDS for t in (gen.F32, gen.F64) if not (k == "c_csc" and t == gen.F64)])
def test_packed_batch_equals_single_calls(sim, kind, dtype):
    """every packed kind (C-sparse CSC exists for f32 only), padded leading dimensions and per-call strides with gaps, then A and B
    shared (stride 0)"""
    rng = np.random.default_rng(7)
    for pads, beta0 in (((8, 16, 24), 0), ((None, 8, 8), 1), ((8, None, 0), 0)):
        case = PackedCase(rng, kind, dtype, 5, P=16, pads=pads, beta0=beta0)
        k = case.create(sim)
        assert k, kind
        rc, c, launches = run_batch(sim, k, case, 5)
        assert rc == 0 and launches == 1
        assert np.array_equal(c, run_singles(k, case, 5)), (kind, pads)
        gaps = c.reshape(5, case.strides[2])[:, case.nbytes[2]:]
        assert np.all(gaps == POISON)


@pytest.mark.parametrize("types", sorted(BCSC_TYPES))
def test_bcsc_batch_reads_the_pattern_once(sim, types):
    """a device-resident pattern reaches the launch as given (block count unknown on the host); a pageable one is staged once and
    its block count read; either way one launch runs every call on call 0's pattern and equals the single calls"""
    rng = np.random.default_rng(11)
    case = BcscCase(rng, BCSC_TYPES[types], 4)
    k = case.create(sim)
    assert k
    nbc = C.c_ulonglong(case.nbc)
    pat = dict(colptr=case.colptr.ctypes.data, rowidx=case.rowidx.ctypes.data, nbc=nbc)
    want = run_singles(k, case, 4, pat)
    for pageable in (False, True):
        if pageable:
            sim.hostsim_sparse_mark_pageable(case.colptr.ctypes.data, case.colptr.nbytes)
            sim.hostsim_sparse_mark_pageable(case.rowidx.ctypes.data, case.rowidx.nbytes)
        calls = sim.hostsim_sparse_calls()
        rc, c, launches = run_batch(sim, k, case, 4, pat)
        assert rc == 0 and launches == 1 and sim.hostsim_sparse_calls() - calls == 4
        assert np.array_equal(c, want), (types, pageable)
        cp, ri, n, nnzb = C.c_void_p(), C.c_void_p(), C.c_ulonglong(), C.c_uint()
        sim.hostsim_sparse_last_bcsc(C.byref(cp), C.byref(ri), C.byref(n), C.byref(nnzb))
        assert n.value == case.nbc
        if pageable:
            assert cp.value != case.colptr.ctypes.data and nnzb.value == int(case.colptr[-1])
        else:
            assert cp.value == case.colptr.ctypes.data and ri.value == case.rowidx.ctypes.data and nnzb.value == 0


def test_return_codes(sim):
    rng = np.random.default_rng(3)
    f = sim.libxsmm_b200_spgemm_batch_strided
    case = PackedCase(rng, "a_csr", gen.F32, 3, pads=(8, 8, 0))
    k = case.create(sim)
    a, b, c = case.a.copy(), case.b.copy(), case.c.copy()
    p = param(a.ctypes.data, b.ctypes.data, c.ctypes.data, case.strides, 0)
    cb = case.nbytes[2]
    S = lambda sa, sb, sc: C.byref(X.SpgemmStrides(sa, sb, sc))
    ok = S(*case.strides)
    assert f(None, C.byref(p), ok, 2) == -1
    assert f(sim.libxsmm_dispatch_gemm(X.libxsmm_create_gemm_shape(8, 8, 8, 8, 8, 8, gen.F32, gen.F32, gen.F32, gen.F32), 0, 0),
             C.byref(p), ok, 2) == -1                                                           # a dense GEMM handle is foreign here
    assert f(k, None, ok, 2) == -1 and f(k, C.byref(p), None, 2) == -1
    assert f(k, C.byref(p), ok, -1) == -1
    before = sim.hostsim_sparse_launches()
    assert f(k, C.byref(p), ok, 0) == 0 and sim.hostsim_sparse_launches() == before and np.array_equal(c, case.c)
    for bad in ((-4, case.strides[1], cb), (case.strides[0], -4, cb), (case.strides[0], case.strides[1], -4),
                (case.strides[0] + 2, case.strides[1], cb), (case.strides[0], case.strides[1], cb + 2),   # not a multiple of 4 bytes
                (case.strides[0], case.strides[1], cb - 4), (case.strides[0], case.strides[1], 0)):      # C of consecutive calls overlaps
        assert f(k, C.byref(p), S(*bad), 2) == -1, bad
    assert f(k, C.byref(p), S(case.strides[0], case.strides[1], cb), 3) == 0                      # outputs may touch, not overlap
    assert f(k, C.byref(p), S(case.strides[0], case.strides[1], 0), 1) == 0                       # one call cannot overlap itself
    for field in ("a", "b", "c"):
        q = param(a.ctypes.data, b.ctypes.data, c.ctypes.data, case.strides, 0)
        setattr(getattr(q, field), "primary", None)
        assert f(k, C.byref(q), ok, 2) == -1, field
    for buf in (a, b, c):                                                                            # pageable operands are not staged
        sim.hostsim_sparse_mark_pageable(buf.ctypes.data, buf.nbytes)
        assert f(k, C.byref(p), ok, 2) == -4
        sim.hostsim_sparse_clear_pageable()
    # fsspmdm handles (sparse A in the kernel) have no batch form
    ptr, idx, vals = np.array([0, 1, 2], dtype=np.uint32), np.array([0, 1], dtype=np.uint32), np.ones(2)
    areg = sim.libxsmm_create_spgemm_csr_areg(X.libxsmm_create_gemm_shape(2, 16, 2, 0, 16, 16, gen.F32, gen.F32, gen.F32, gen.F32), 0, 0, 16,
                                              ptr.ctypes.data, idx.ctypes.data, vals.ctypes.data)
    assert areg and f(areg, C.byref(p), ok, 2) == NOT_BATCHABLE
    # BCSC: the pattern must be given; C extent from the block-column count
    bc = BcscCase(rng, BCSC_TYPES["f32"], 2)
    kb = bc.create(sim)
    nbc = C.c_ulonglong(bc.nbc)
    ba, bb, bcc = bc.a.copy(), bc.b.copy(), bc.c.copy()
    q = param(ba.ctypes.data, bb.ctypes.data, bcc.ctypes.data, bc.strides, 0, colptr=bc.colptr.ctypes.data, rowidx=bc.rowidx.ctypes.data, nbc=nbc)
    assert f(kb, C.byref(q), S(*bc.strides), 2) == 0
    assert f(kb, C.byref(q), S(bc.strides[0], bc.strides[1], bc.nbytes[2]), 2) == 0
    assert f(kb, C.byref(q), S(bc.strides[0], bc.strides[1], bc.nbytes[2] - 4), 2) == -1
    q.b.tertiary = None
    assert f(kb, C.byref(q), S(*bc.strides), 2) == -1
