"""Batched matrix-eltwise and equation calls through the host half of the library on the simulated device: the host_*.c objects,
tests/c/hostsim_runtime.c and tests/c/hostsim_meltw_batch.c (a batch launch answered call by call by the oracle) linked into
tests/c/_hostsim/meltw_batch/libxsmm.so. What this checks is the host code: the stride arithmetic handed to the launcher, the extents
behind the overlap rule, the -1 / -4 / NOT_BATCHABLE rules, equation chunking and the DUMP wiring -- each batch against single calls
of the same handle on the same tiles."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import libxsmm_b200 as X
from test_hostsim import CSRC, HOST_C, ORACLE, ROOT

OUT = os.path.join(ROOT, "tests", "c", "_hostsim", "meltw_batch")
NOT_BATCHABLE = -6
F32 = X.DATATYPE_F32
M, N, LDI, LDO = 24, 10, 28, 30


def build_sim():
    os.makedirs(OUT, exist_ok=True)
    so = os.path.join(OUT, "libxsmm.so")
    srcs = [os.path.join(CSRC, f) for f in HOST_C] + [os.path.join(ROOT, "tests", "c", f) for f in ("hostsim_runtime.c", "hostsim_meltw_batch.c")]
    deps = srcs + [os.path.join(CSRC, "xb_internal.h")]
    if not (os.path.exists(so) and all(os.path.getmtime(s) < os.path.getmtime(so) for s in deps)):
        cmd = ["gcc", "-O1", "-std=gnu99", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-Wl,--wrap=xb_meltw_launch", "-o", so] + \
            srcs + ["-L" + ORACLE, "-loracle", "-Wl,-rpath," + ORACLE, "-lpthread", "-ldl", "-lm"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-3000:]
    lib = C.CDLL(so)
    P, LL = C.c_void_p, C.c_longlong
    for name, res, args in (("libxsmm_dispatch_meltw_unary", P, [C.c_int, X.MeltwUnaryShape, C.c_uint]),
                            ("libxsmm_dispatch_meltw_binary", P, [C.c_int, X.MeltwBinaryShape, C.c_uint]),
                            ("libxsmm_dispatch_meltw_ternary", P, [C.c_int, X.MeltwTernaryShape, C.c_uint]),
                            ("libxsmm_b200_meltw_batch_strided", C.c_int, [P, P, C.POINTER(X.MeltwStrides), LL]),
                            ("libxsmm_b200_meqn_batch_strided", C.c_int, [P, C.POINTER(X.MeqnParam), C.POINTER(LL), LL, LL, C.POINTER(LL), LL]),
                            ("libxsmm_meqn_create", C.c_int, []),
                            ("libxsmm_meqn_push_back_arg", C.c_int, [X.MeqnMetadata, X.MeqnArgShape, X.MatrixArgAttributes]),
                            ("libxsmm_meqn_push_back_unary_op", C.c_int, [X.MeqnMetadata, C.c_int, C.c_int, C.c_uint]),
                            ("libxsmm_meqn_push_back_binary_op", C.c_int, [X.MeqnMetadata, C.c_int, C.c_int, C.c_uint]),
                            ("libxsmm_dispatch_meqn", P, [C.c_int, X.MeqnArgShape]),
                            ("hostsim_batch_launches", C.c_ulonglong, [])):
        fn = getattr(lib, name); fn.restype, fn.argtypes = res, args
    return lib


@pytest.fixture(scope="module")
def sim():
    return build_sim()


@pytest.fixture(autouse=True)
def device_pointers(monkeypatch):
    monkeypatch.setenv("XB_HOSTSIM_PTR_KIND", "1")      # every pointer is "device memory" unless a test says otherwise


def rand(rng, nbytes):
    return rng.standard_normal(nbytes // 4).astype(np.float32).view(np.uint8).copy()


def poison(nbytes):
    return np.full(nbytes, 0xA5, dtype=np.uint8)


def addr(a, off=0):
    return a.ctypes.data + off


def unary(sim, op, flags=0, m=M, n=N, ldi=LDI, ldo=LDO):
    k = sim.libxsmm_dispatch_meltw_unary(op, X.MeltwUnaryShape(m, n, ldi, ldo, F32, F32, F32), flags)
    assert k
    return k


def test_unary_strides_and_secondaries(sim):
    """RELU with a bit mask and RELU_INV reading one: in.primary, in.secondary, out.primary and out.secondary all strided, gaps kept"""
    rng = np.random.default_rng(1)
    count, sx, so, sm = 5, LDO * N * 4 + 12, LDO * N * 4 + 8, LDO // 8 * N + 24   # sx covers both handles' inputs (ldi 28 and 30)
    fwd = unary(sim, X.MELTW_TYPE_UNARY_RELU, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT)
    inv = unary(sim, X.MELTW_TYPE_UNARY_RELU_INV, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT, ldi=LDO)
    x = rand(rng, count * sx)
    for k, s, mask_in in ((fwd, X.MeltwStrides(in0=sx, out=so, out_aux=sm), False), (inv, X.MeltwStrides(in0=sx, in_aux=sm, out=so), True)):
        mask = rand(rng, count * sm)
        o, a = poison(count * so), (mask.copy() if mask_in else poison(count * sm))
        o1, a1 = o.copy(), a.copy()

        def param(t, out, aux):
            p = X.MeltwUnaryParam(); p.inp.primary = addr(x, t * sx); p.out.primary = addr(out, t * so)
            if mask_in:
                p.inp.secondary = addr(aux, t * sm)
            else:
                p.out.secondary = addr(aux, t * sm)
            return p
        before = sim.hostsim_batch_launches()
        assert sim.libxsmm_b200_meltw_batch_strided(k, C.addressof(param(0, o, a)), C.byref(s), count) == 0
        assert sim.hostsim_batch_launches() == before + 1
        for t in range(count):
            X.MELTW_UNARY_FN(k)(C.byref(param(t, o1, a1)))
        assert np.array_equal(o, o1) and np.array_equal(a, a1)
        assert np.all(o.reshape(count, so)[:, (N - 1) * LDO * 4 + M * 4:] == 0xA5)


def test_binary_and_ternary_strides(sim):
    """ADD with a per-call in1 and a shared (stride 0) BCAST_COL in1; MULADD with three strided inputs"""
    rng = np.random.default_rng(2)
    count, sx, so = 4, LDI * N * 4, LDO * N * 4 + 16
    for flags, s1 in ((0, LDI * N * 4 + 4), (X.MELTW_FLAG_BINARY_BCAST_COL_IN_1, 0)):
        k = sim.libxsmm_dispatch_meltw_binary(X.MELTW_TYPE_BINARY_ADD, X.MeltwBinaryShape(M, N, LDI, LDI, LDO, F32, F32, F32, F32), flags)
        x, y, o = rand(rng, count * sx), rand(rng, max(count * s1, LDI * N * 4)), poison(count * so)
        o1 = o.copy()

        def param(t, out):
            p = X.MeltwBinaryParam(); p.in0.primary, p.in1.primary, p.out.primary = addr(x, t * sx), addr(y, t * s1), addr(out, t * so)
            return p
        s = X.MeltwStrides(in0=sx, in1=s1, out=so)
        assert sim.libxsmm_b200_meltw_batch_strided(k, C.addressof(param(0, o)), C.byref(s), count) == 0
        for t in range(count):
            X.MELTW_BINARY_FN(k)(C.byref(param(t, o1)))
        assert np.array_equal(o, o1)
    k = sim.libxsmm_dispatch_meltw_ternary(X.MELTW_TYPE_TERNARY_MULADD, X.MeltwTernaryShape(M, N, LDI, LDI, LDI, LDO, F32, F32, F32, F32, F32), 0)
    assert k
    ins = [rand(rng, count * sx) for _ in range(3)]
    o = poison(count * so); o1 = o.copy()

    def tparam(t, out):
        p = X.MeltwTernaryParam()
        p.in0.primary, p.in1.primary, p.in2.primary, p.out.primary = addr(ins[0], t * sx), addr(ins[1], t * sx), addr(ins[2], t * sx), addr(out, t * so)
        return p
    s = X.MeltwStrides(in0=sx, in1=sx, in2=sx, out=so)
    assert sim.libxsmm_b200_meltw_batch_strided(k, C.addressof(tparam(0, o)), C.byref(s), count) == 0
    for t in range(count):
        X.MELTW_TERNARY_FN(k)(C.byref(tparam(t, o1)))
    assert np.array_equal(o, o1)


def test_meltw_return_codes(sim, monkeypatch):
    k = unary(sim, X.MELTW_TYPE_UNARY_RELU, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT)
    sx, so, sm = LDI * N * 4, LDO * N * 4, 32 // 8 * N          # a bit-mask column is ldo rounded up to 16 bits
    x, o, a = rand(np.random.default_rng(3), 3 * sx), poison(3 * so), poison(3 * sm)
    p = X.MeltwUnaryParam(); p.inp.primary, p.out.primary, p.out.secondary = addr(x), addr(o), addr(a)
    f = sim.libxsmm_b200_meltw_batch_strided
    ok = X.MeltwStrides(in0=sx, out=so, out_aux=sm)
    assert f(None, C.addressof(p), C.byref(ok), 2) == -1
    assert f(k, C.addressof(p), C.byref(ok), -1) == -1
    assert f(k, C.addressof(p), C.byref(ok), 0) == 0 and np.all(o == 0xA5)
    for field, v in (("in0", -4), ("out", -4), ("out_aux", -1), ("out", (N - 1) * LDO * 4 + M * 4 - 1), ("out_aux", sm - 1)):
        bad = X.MeltwStrides(in0=sx, out=so, out_aux=sm); setattr(bad, field, v)
        assert f(k, C.addressof(p), C.byref(bad), 2) == -1, (field, v)
    exact = X.MeltwStrides(in0=sx, out=(N - 1) * LDO * 4 + M * 4, out_aux=sm)      # outputs may touch, not overlap
    assert f(k, C.addressof(p), C.byref(exact), 2) == 0
    monkeypatch.setenv("XB_HOSTSIM_PTR_KIND", "0")
    assert f(k, C.addressof(p), C.byref(ok), 2) == -4
    monkeypatch.setenv("XB_HOSTSIM_PTR_KIND", "3")                                  # pinned memory is device-accessible
    assert f(k, C.addressof(p), C.byref(ok), 2) == 0
    refused = [unary(sim, op) for op in (X.MELTW_TYPE_UNARY_DROPOUT, X.MELTW_TYPE_UNARY_REPLICATE_COL_VAR, X.MELTW_TYPE_UNARY_GATHER,
                                         X.MELTW_TYPE_UNARY_SCATTER, X.MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_ADD, X.MELTW_TYPE_UNARY_UNZIP,
                                         X.MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X2)]
    refused.append(unary(sim, X.MELTW_TYPE_UNARY_IDENTITY, X.MELTW_FLAG_UNARY_STOCHASTIC_ROUND))
    refused.append(sim.libxsmm_dispatch_meltw_binary(X.MELTW_TYPE_BINARY_ADD, X.MeltwBinaryShape(M, N, LDI, LDI, LDO, F32, F32, F32, F32),
                                                     X.MELTW_FLAG_BINARY_STOCHASTIC_ROUND))
    for h in refused:
        assert h and f(h, C.addressof(p), C.byref(ok), 2) == NOT_BATCHABLE


# ---- equations ---------------------------------------------------------------------------------------------------------------------
def build_eqn(sim, nodes):
    eq = sim.libxsmm_meqn_create()
    for nd in nodes:
        if nd[0] == "arg":
            rc = sim.libxsmm_meqn_push_back_arg(X.MeqnMetadata(eq, nd[1]), X.MeqnArgShape(*nd[2:]), X.MatrixArgAttributes(0, 0, 0, 0))
        else:
            fn = {"u": sim.libxsmm_meqn_push_back_unary_op, "b": sim.libxsmm_meqn_push_back_binary_op}[nd[0]]
            rc = fn(X.MeqnMetadata(eq, nd[4]), nd[1], F32, nd[2])
        assert rc == 0, nd
    k = sim.libxsmm_dispatch_meqn(eq, X.MeqnArgShape(M, N, LDO, F32))
    assert k
    return k


# (x - colsum(x)) * gamma, gamma shared by every call
LN = [("b", X.MELTW_TYPE_BINARY_MUL, X.MELTW_FLAG_BINARY_BCAST_COL_IN_1, 0, -1), ("b", X.MELTW_TYPE_BINARY_SUB, X.MELTW_FLAG_BINARY_BCAST_COL_IN_1, 0, -1),
      ("arg", 0, M, N, LDI, F32), ("u", X.MELTW_TYPE_UNARY_REDUCE_X_OP_ADD, X.MELTW_FLAG_UNARY_REDUCE_COLS, 0, -1), ("arg", 0, M, N, LDI, F32),
      ("arg", 1, M, 1, M, F32)]
# exp(x) dumped into ops_args[0] = inputs[1], then read back as an argument: exp(x) + inputs[1] (the softmax pattern)
DUMP = [("b", X.MELTW_TYPE_BINARY_ADD, 0, 0, -1), ("u", X.MELTW_TYPE_UNARY_DUMP, 0, 0, 0), ("u", X.MELTW_TYPE_UNARY_EXP, 0, 0, -1),
        ("arg", 0, M, N, LDI, F32), ("arg", 1, M, N, M, F32)]


def run_eqn(sim, nodes, count, in1_stride, ops_stride=None, out_stride=LDO * N * 4 + 4, rng_seed=5):
    k = build_eqn(sim, nodes)
    rng = np.random.default_rng(rng_seed)
    sx, n = LDI * N * 4, max(count, 1)
    x0 = rand(rng, n * sx)
    x1 = rand(rng, max(n * in1_stride, LDI * N * 4))
    o = poison(n * out_stride)
    x1b, ob = x1.copy(), o.copy()
    dump = ops_stride is not None

    def param(t, xa, xb, out, keep):
        ins = (X.MatrixArg * 2)(); ins[0].primary, ins[1].primary = addr(xa, t * sx), addr(xb, t * in1_stride)
        ops = (X.MatrixOpArg * 1)(); ops[0].primary = addr(xb, t * in1_stride)
        p = X.MeqnParam(); p.inputs = C.addressof(ins); p.output.primary = addr(out, t * out_stride)
        if dump:
            p.ops_args = C.addressof(ops)
        keep += [ins, ops]
        return p
    keep = []
    strides = (C.c_longlong * 2)(sx, in1_stride)
    ops_s = (C.c_longlong * 1)(ops_stride) if dump else None
    before = sim.hostsim_batch_launches()
    rc = sim.libxsmm_b200_meqn_batch_strided(k, C.byref(param(0, x0, x1, o, keep)), strides, out_stride, 0, ops_s, count)
    return k, rc, sim.hostsim_batch_launches() - before, (x0, x1, o, x1b, ob, param, keep)


def check_against_single_calls(k, count, state, tiles):
    x0, x1, o, x1b, ob, param, keep = state
    for t in tiles:
        X.MEQN_FN(k)(C.byref(param(t, x0, x1b, ob, keep)))
    for t in tiles:
        assert np.array_equal(o.reshape(count, -1)[t], ob.reshape(count, -1)[t]), t
        if x1.size == count * (x1.size // count):                        # per-call second input (the DUMP target)
            assert np.array_equal(x1.reshape(count, -1)[t], x1b.reshape(count, -1)[t]), t


def test_layernorm_equation_batch(sim):
    k, rc, launches, st = run_eqn(sim, LN, 6, 0)
    assert rc == 0 and launches == 3
    check_against_single_calls(k, 6, st, range(6))


def test_dump_feeding_an_argument(sim):
    s1 = M * N * 4 + 8
    k, rc, launches, st = run_eqn(sim, DUMP, 5, s1, ops_stride=s1)
    assert rc == 0 and launches == 3
    check_against_single_calls(k, 5, st, range(5))
    assert run_eqn(sim, DUMP, 5, s1, ops_stride=s1 + 4)[1] == -1             # the DUMP's and the argument's strides disagree
    assert run_eqn(sim, DUMP, 5, s1, ops_stride=M * N * 4 - 4)[1] == -1      # DUMP copies would overlap


def test_equation_chunks(sim):
    """temporaries: SUB 24 x 10 f32 (960 B -> 1024 at 256-byte strides) and the reduction (96 B -> 256): 64 MiB hold 52,428 calls,
    so 60,000 run in two chunks, each one launch per node"""
    count = 60000
    k, rc, launches, st = run_eqn(sim, LN, count, 0)
    assert rc == 0 and launches == 3 * 2
    check_against_single_calls(k, count, st, [0, 52427, 52428, count - 1])


def test_equation_return_codes(sim, monkeypatch):
    k, rc, _, _ = run_eqn(sim, LN, 3, 0, out_stride=LDO * (N - 1) * 4 + M * 4 - 4)
    assert rc == -1                                                            # overlapping outputs
    assert run_eqn(sim, LN, 0, 0)[1] == 0
    assert run_eqn(sim, LN, -1, 0)[1] == -1
    assert run_eqn(sim, DUMP, 3, M * N * 4)[1] == -1                          # DUMP without ops_strides
    monkeypatch.setenv("XB_HOSTSIM_PTR_KIND", "0")
    assert run_eqn(sim, LN, 3, 0)[1] == -4
