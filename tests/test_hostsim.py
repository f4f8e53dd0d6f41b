"""Host logic of the matrix equations (libxsmm_b200/csrc/host_meqn.c) exercised WITHOUT a GPU.

The host_*.c sources are linked with tests/c/hostsim_runtime.c -- a stand-in for runtime.cu and the kernel launchers in which
"device" memory is host memory and every elementwise launch is answered by the oracle -- into tests/c/_hostsim/libxsmm.so (test
infrastructure, never shipped). What this checks is the part of an equation that is not a kernel: the order nodes run in, the
shape / leading dimension / type each node is launched with, where secondary outputs land (reference
src/generator_matequation_reference_impl.c:16-61: the bit mask of a relu at the head -> output.secondary, a DUMP node ->
ops_args[pos].primary) and that an argument is read when its consumer runs (a DUMP below may have written it: the softmax sample).
Kernels are validated on the GPU in test_meqn.py / test_meltw_gpu.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import gen
import libxsmm_b200 as X          # constants and struct layouts only: every call below goes to the simulation library
from test_meqn import EQUATIONS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "libxsmm_b200", "csrc")
OUT = os.path.join(ROOT, "tests", "c", "_hostsim")
DRV = os.path.join(ROOT, "oracle", "_ref", "drivers")
ORACLE = os.path.join(ROOT, "oracle")
F32, BF16 = gen.F32, gen.BF16
HOST_C = ["host_core.c", "host_thunks.c", "host_sparse.c", "host_meltw.c", "host_utils.c", "host_meqn.c"]


def build_sim():
    os.makedirs(OUT, exist_ok=True)
    if not os.path.exists(os.path.join(ORACLE, "liboracle.so")):
        subprocess.check_call(["make", "-C", ROOT, "oracle"])
    so = os.path.join(OUT, "libxsmm.so")
    srcs = [os.path.join(CSRC, f) for f in HOST_C] + [os.path.join(ROOT, "tests", "c", "hostsim_runtime.c")]
    if os.path.exists(so) and all(os.path.getmtime(s) < os.path.getmtime(so) for s in srcs + [os.path.join(CSRC, "xb_internal.h")]):
        return so
    cmd = ["gcc", "-O1", "-std=gnu99", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-o", so] + srcs + \
          ["-L" + ORACLE, "-loracle", "-Wl,-rpath," + ORACLE, "-lpthread", "-ldl", "-lm"]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    return so


class Sim:
    def __init__(self):
        self.lib = C.CDLL(build_sim())
        I, U, P = C.c_int, C.c_uint, C.c_void_p
        for name, res, args in (
                ("libxsmm_meqn_create", I, []), ("libxsmm_create_meqn_arg_shape", X.MeqnArgShape, [I] * 4),
                ("libxsmm_create_matrix_arg_attributes", X.MatrixArgAttributes, [I] * 4),
                ("libxsmm_create_meqn_arg_metadata", X.MeqnMetadata, [I, I]), ("libxsmm_create_meqn_op_metadata", X.MeqnMetadata, [I, I]),
                ("libxsmm_meqn_push_back_arg", I, [X.MeqnMetadata, X.MeqnArgShape, X.MatrixArgAttributes]),
                ("libxsmm_meqn_push_back_unary_op", I, [X.MeqnMetadata, I, I, U]), ("libxsmm_meqn_push_back_binary_op", I, [X.MeqnMetadata, I, I, U]),
                ("libxsmm_meqn_push_back_ternary_op", I, [X.MeqnMetadata, I, I, U]), ("libxsmm_dispatch_meqn", P, [I, X.MeqnArgShape])):
            fn = getattr(self.lib, name); fn.restype = res; fn.argtypes = args
            setattr(self, name[len("libxsmm_"):], fn)

    def build(self, nodes):
        """nodes in pre-order: ('arg', pos, m, n, ld, dtype) | ('u'|'b'|'t', op, dtype, flags[, op_arg_pos])"""
        eq = self.meqn_create()
        for nd in nodes:
            if nd[0] == "arg":
                rc = self.meqn_push_back_arg(self.create_meqn_arg_metadata(eq, nd[1]), self.create_meqn_arg_shape(*nd[2:6]), self.create_matrix_arg_attributes(0, 0, 0, 0))
            else:
                fn = {"u": self.meqn_push_back_unary_op, "b": self.meqn_push_back_binary_op, "t": self.meqn_push_back_ternary_op}[nd[0]]
                rc = fn(self.create_meqn_op_metadata(eq, nd[4] if len(nd) > 4 else -1), nd[1], nd[2], nd[3])
            assert rc == 0, nd
        return eq

    def run(self, fn, ins, out, out_secondary=None, ops=None):
        args = (X.MatrixArg * max(1, len(ins)))()
        for i, x in enumerate(ins):
            args[i].primary = x.ctypes.data
        opa = (X.MatrixOpArg * 32)()
        for pos, buf in (ops or {}).items():
            opa[pos].primary = buf.ctypes.data
        p = X.MeqnParam(); p.inputs = C.addressof(args); p.ops_args = C.addressof(opa); p.output.primary = out.ctypes.data
        if out_secondary is not None:
            p.output.secondary = out_secondary.ctypes.data
        X.MEQN_FN(fn)(C.byref(p))


@pytest.fixture(scope="module")
def sim():
    return Sim()


@pytest.mark.parametrize("name", sorted(EQUATIONS))
def test_equation_patterns_on_the_simulated_device(sim, name):
    """the four trees of test_meqn.py (chain, broadcasts, reduction, ternary) from host buffers"""
    rng = np.random.default_rng(97)
    for (m, n) in ((32, 16), (13, 7)):
        nodes, in_shapes, (om, on) = EQUATIONS[name](m, n)
        ins = [(rng.standard_normal(a * b) * 0.5).astype(np.float32) for (a, b) in in_shapes]
        A = [x.reshape(sh[1], sh[0]).T for x, sh in zip(ins, in_shapes)]
        exact = {"chain": lambda: np.tanh(A[0] + A[1]) * A[2], "bcast": lambda: np.maximum(A[0] * A[1] + A[2], 0),
                 "reduce": lambda: (A[0] * A[0]).sum(1, keepdims=True, dtype=np.float32), "ternary": lambda: A[0] - np.exp(A[1]) * A[2]}[name]()
        want = np.ascontiguousarray(exact.T.astype(np.float32)).ravel()
        fn = sim.dispatch_meqn(sim.build(nodes), sim.create_meqn_arg_shape(om, on, om, F32))
        assert fn, name
        out = np.zeros(om * on, dtype=np.float32)
        sim.run(fn, ins, out)
        assert np.allclose(out, want, rtol=2e-5, atol=2e-5), (name, m, n, np.abs(out - want).max())


def test_relu_at_the_head_writes_its_bit_mask_to_the_secondary_output(sim):
    """samples/equation/equation_relu.c: relu(bitmask) over (a + b + 1) - c; mask rows are padded to 16 bits"""
    rng = np.random.default_rng(98)
    for (m, n, ld, odt) in ((64, 32, 64, F32), (37, 5, 40, F32), (48, 7, 48, BF16)):
        nodes = [("u", X.MELTW_TYPE_UNARY_RELU, F32, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT)] + \
                ([("u", X.MELTW_TYPE_UNARY_IDENTITY, odt, 0)] if odt != F32 else []) + \
                [("b", X.MELTW_TYPE_BINARY_SUB, F32, 0), ("u", X.MELTW_TYPE_UNARY_INC, F32, 0), ("b", X.MELTW_TYPE_BINARY_ADD, F32, 0),
                 ("arg", 0, m, n, ld, F32), ("arg", 1, m, n, ld, F32), ("arg", 2, m, n, ld, F32)]
        ins = [rng.standard_normal(ld * n).astype(np.float32) for _ in range(3)]
        fn = sim.dispatch_meqn(sim.build(nodes), sim.create_meqn_arg_shape(m, n, ld, odt))
        assert fn
        mask_ld = (ld + 15) // 16 * 2
        out = np.full(ld * n, 7, dtype=gen.NP_OF[odt]); mask = np.zeros(mask_ld * n, dtype=np.uint8)
        sim.run(fn, ins, out, out_secondary=mask)
        v = [x.reshape(n, ld)[:, :m] for x in ins]
        pre = ((v[0] + v[1]) + np.float32(1.0)) - v[2]
        if odt == BF16:
            u = pre.view(np.uint32).astype(np.uint64)          # the IDENTITY below the head rounds to bf16, nearest even
            pre = (((u + 0x7fff + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32).view(np.float32)
        got = gen.to_f64(out, odt).reshape(n, ld)
        assert np.array_equal(got[:, :m], np.maximum(pre, 0).astype(np.float64)), (m, n, ld, odt)
        assert np.all(out.reshape(n, ld)[:, m:] == 7), "the padding between columns is not written"
        bits = np.unpackbits(mask.reshape(n, mask_ld), axis=1, bitorder="little")[:, :m]
        assert np.array_equal(bits.astype(bool), pre > 0), (m, n, ld, odt)


def test_a_bit_mask_below_the_head_is_refused(sim):
    nodes = [("u", X.MELTW_TYPE_UNARY_INC, F32, 0), ("u", X.MELTW_TYPE_UNARY_RELU, F32, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT), ("arg", 0, 16, 4, 16, F32)]
    assert not sim.dispatch_meqn(sim.build(nodes), sim.create_meqn_arg_shape(16, 4, 16, F32))


def test_dump_feeds_an_argument_of_the_same_equation(sim):
    """samples/equation/equation_softmax.c:527-538: out = tmp * (1 / sum(DUMP->tmp(exp(x - max(x))))) where tmp is BOTH the DUMP
    destination (ops_args[31]) and argument 0 of the head: the argument has to be read after the subtree below ran"""
    rng = np.random.default_rng(99)
    m, n, ld = 24, 6, 60
    R, Cc = X.MELTW_FLAG_UNARY_REDUCE_ROWS, X.MELTW_FLAG_UNARY_REDUCE_COLS
    S1 = X.MELTW_FLAG_BINARY_BCAST_SCALAR_IN_1
    nodes = [("b", X.MELTW_TYPE_BINARY_MUL, F32, S1), ("arg", 0, m, n, m, F32), ("u", X.MELTW_TYPE_UNARY_RECIPROCAL, F32, 0),
             ("u", X.MELTW_TYPE_UNARY_REDUCE_X_OP_ADD, F32, R), ("u", X.MELTW_TYPE_UNARY_REDUCE_X_OP_ADD, F32, Cc), ("u", X.MELTW_TYPE_UNARY_DUMP, F32, 0, 31),
             ("u", X.MELTW_TYPE_UNARY_EXP, F32, 0), ("b", X.MELTW_TYPE_BINARY_SUB, F32, S1), ("arg", 1, m, n, ld, F32),
             ("u", X.MELTW_TYPE_UNARY_REDUCE_X_OP_MAX, F32, R), ("u", X.MELTW_TYPE_UNARY_REDUCE_X_OP_MAX, F32, Cc), ("arg", 1, m, n, ld, F32)]
    fn = sim.dispatch_meqn(sim.build(nodes), sim.create_meqn_arg_shape(m, n, ld, F32))
    assert fn
    x = rng.standard_normal(ld * n).astype(np.float32)
    tmp = np.full(m * n, np.nan, dtype=np.float32)           # stale on entry: must not be what the head multiplies
    out = np.zeros(ld * n, dtype=np.float32)
    sim.run(fn, [tmp, x], out, ops={31: tmp})
    xv = x.reshape(n, ld)[:, :m].astype(np.float64)
    e = np.exp(xv - xv.max())
    assert np.allclose(tmp.reshape(n, m), e, rtol=1e-5, atol=1e-6)
    assert np.allclose(out.reshape(n, ld)[:, :m], e / e.sum(), rtol=1e-5, atol=1e-7)
    assert np.all(out.reshape(n, ld)[:, m:] == 0)


# valid argument sets of samples/eltwise/eltwise_ternary_simple.c (SELECT with the implicit bit mask as third input; :399-417)
TERNARY_RUNS = [("eltwise_ternary_simple", (1, 0, "F32", "F32", "IMPLICIT", "F32", "F32", 64, 16, 64, 64)),
                ("eltwise_ternary_simple", (1, 0, "F32", "F32", "IMPLICIT", "F32", "F32", 37, 11, 48, 40)),
                ("eltwise_ternary_simple", (1, 0, "BF16", "BF16", "IMPLICIT", "F32", "BF16", 64, 16, 64, 64)),
                ("eltwise_ternary_simple", (1, 1, "F32", "F32", "IMPLICIT", "F32", "F32", 64, 16, 64, 64)),
                ("eltwise_ternary_simple", (1, 5, "F32", "F32", "IMPLICIT", "F32", "F32", 64, 16, 64, 64)),
                ("eltwise_ternary_simple", (1, 0, "F32", "BF8", "IMPLICIT", "F32", "BF8", 64, 16, 64, 64)),
                ("eltwise_ternary_simple", (1, 0, "F32", "F32", "IMPLICIT", "F32", "BF8", 64, 16, 64, 64, 1))]

# samples/xgemm/gemm_kernel*.c: A B Comp C  M N K LDA LDB LDC  alpha beta  alignA alignC  trA trB  vnniA vnniB vnniC  prefetch  br-kind br-count
# br-unroll  reps  tilecfg [binary-postop unary-postop]
def _gk(types, m, n, k, lda, ldb, ldc, beta, tra=0, trb=0, va=0, vb=0, vc=0, br="nobr", brn=1, post=()):
    return tuple(types.split()) + (m, n, k, lda, ldb, ldc, 1, beta, 0, 0, tra, trb, va, vb, vc, "nopf", br, brn, 0, 3, 0) + tuple(post)


GEMM_RUNS = [("hello", ())] + [("gemm_kernel", a) for a in (
    _gk("F32 F32 F32 F32", 64, 64, 64, 64, 64, 64, 0), _gk("F32 F32 F32 F32", 37, 21, 45, 40, 48, 40, 1, trb=1, br="strdbr", brn=4),
    _gk("F32 F32 F32 F32", 32, 32, 32, 32, 32, 32, 1, br="addrbr", brn=3), _gk("F32 F32 F32 F32", 32, 32, 32, 32, 32, 32, 0, br="offsbr", brn=3),
    _gk("F32 F32 F32 F32", 64, 64, 64, 64, 64, 64, 0, tra=1), _gk("F64 F64 F64 F64", 13, 5, 7, 13, 7, 13, 1),
    _gk("BF16 BF16 F32 F32", 64, 64, 64, 64, 64, 64, 1, va=1), _gk("BF16 BF16 F32 BF16", 64, 64, 64, 64, 64, 64, 0, va=1, br="strdbr", brn=2),
    _gk("BF16 BF16 F32 BF16", 64, 64, 64, 64, 64, 64, 0, va=1, vc=1), _gk("F16 F16 F32 F32", 64, 64, 64, 64, 64, 64, 1, va=1),
    _gk("I8 I8 I32 I32", 64, 64, 64, 64, 64, 64, 0, va=1), _gk("U8 I8 I32 I32", 64, 64, 64, 64, 64, 64, 1, va=1),
    _gk("BF8 BF8 F32 F32", 64, 64, 64, 64, 64, 64, 1, va=1), _gk("HF8 HF8 F32 HF8", 64, 64, 64, 64, 64, 64, 0, va=1),
    _gk("F32 F32 F32 F32", 64, 64, 64, 64, 64, 64, 0, br="spmm", brn=4), _gk("BF16 BF16 F32 BF16", 64, 64, 64, 64, 64, 64, 0, va=1, br="spmm", brn=2))] + \
    [("gemm_kernel_fused", _gk("F32 F32 F32 F32", 64, 48, 32, 64, 32, 64, 1, post=(b, u))) for b in (0, 1) for u in (0, 1, 2, 3)] + \
    [("gemm_kernel_fused", _gk("BF16 BF16 F32 BF16", 64, 64, 64, 64, 64, 64, 0, va=1, br="strdbr", brn=2, post=(1, 2))),
     ("gemm_kernel_fused", _gk("BF16 BF16 F32 BF16", 64, 64, 64, 64, 64, 64, 0, va=1, vc=1, post=(1, 1))),
     ("gemm_kernel_parallel", _gk("F32 F32 F32 F32", 64, 64, 64, 64, 64, 64, 1)),
     ("gemm_kernel_parallel", _gk("BF16 BF16 F32 BF16", 64, 64, 64, 64, 64, 64, 0, va=1, br="strdbr", brn=2))]

# samples/eltwise/eltwise_unary_relu.c [D/L/E] [F/B] [bitmask] in comp out M N ldi ldo ; eltwise_unary_transform.c op type M N ldi ldo
MORE_ELTWISE_RUNS = [("eltwise_unary_relu", (t, fb, bm, "F32", "F32", "F32", 37, 11, 48, 40)) for t in "DLE" for fb in "FB" for bm in (0, 1)
                     if not (fb == "B" and bm == 0 and t != "E")] + [("eltwise_unary_relu", ("D", "F", 1, "BF16", "F32", "BF16", 64, 16, 64, 64))] + \
    [("eltwise_unary_transform", (op, "BF16", 32, 16, 32, 32)) for op in "TRSVWQFGHIXYZBCD"] + \
    [("eltwise_unary_transform", ("T", "F32", 37, 11, 40, 16)), ("eltwise_unary_transform", ("N", "I8", 32, 16, 32, 32)), ("eltwise_unary_transform", ("M", "I8", 32, 16, 32, 32))]

def test_the_more_demanding_operand_subtree_runs_first(sim):
    """out = (a - tmp) - (a*a + DUMP->tmp(a + 1)): the right operand of the head needs two temporaries, the left one, so the reference runs
    the right one first (src/libxsmm_matrixeqn.c:323-400, 745-790) and the left branch sees the tmp this very call produced"""
    m, n = 20, 6
    nodes = [("b", X.MELTW_TYPE_BINARY_SUB, F32, 0),
             ("b", X.MELTW_TYPE_BINARY_SUB, F32, 0), ("arg", 0, m, n, m, F32), ("arg", 1, m, n, m, F32),
             ("b", X.MELTW_TYPE_BINARY_ADD, F32, 0), ("u", X.MELTW_TYPE_UNARY_X2, F32, 0), ("arg", 0, m, n, m, F32),
             ("u", X.MELTW_TYPE_UNARY_DUMP, F32, 0, 3), ("u", X.MELTW_TYPE_UNARY_INC, F32, 0), ("arg", 0, m, n, m, F32)]
    fn = sim.dispatch_meqn(sim.build(nodes), sim.create_meqn_arg_shape(m, n, m, F32))
    assert fn
    a = np.random.default_rng(5).standard_normal(m * n).astype(np.float32)
    tmp = np.full(m * n, 1e30, dtype=np.float32); out = np.zeros(m * n, dtype=np.float32)
    sim.run(fn, [a, tmp], out, ops={3: tmp})
    assert np.array_equal(tmp, a + np.float32(1))
    assert np.allclose(out, (a - tmp) - (a * a + tmp), rtol=1e-6, atol=1e-6)


def test_trees_with_unwired_operands_are_declined(sim):
    """nodes without a storage type (zip / unzip trees of equation_splitSGD.c) and operations that read index arrays, masks, generator state
    or scales through operands the evaluator does not wire (equation_gather_*.c) must not dispatch"""
    bad = [[("u", X.MELTW_TYPE_UNARY_UNZIP, X.DATATYPE_IMPLICIT, 0), ("arg", 0, 16, 4, 16, F32)],
           [("u", X.MELTW_TYPE_UNARY_INC, F32, 0), ("b", X.MELTW_TYPE_BINARY_ADD, X.DATATYPE_IMPLICIT, 0), ("arg", 0, 16, 4, 16, F32), ("arg", 1, 16, 4, 16, F32)],
           [("u", X.MELTW_TYPE_UNARY_GATHER, F32, 0), ("arg", 0, 16, 4, 16, F32)],
           [("u", X.MELTW_TYPE_UNARY_RELU_INV, F32, 0), ("arg", 0, 16, 4, 16, F32)],
           [("u", X.MELTW_TYPE_UNARY_DROPOUT, F32, 0), ("arg", 0, 16, 4, 16, F32)],
           [("u", X.MELTW_TYPE_UNARY_INC, F32, 0), ("u", X.MELTW_TYPE_UNARY_QUANT, gen.I8, 0), ("arg", 0, 16, 4, 16, F32)]]
    for nodes in bad:
        assert not sim.dispatch_meqn(sim.build(nodes), sim.create_meqn_arg_shape(16, 4, 16, F32)), nodes


DRIVER_RUNS = [("equation_simple", (64, 32)), ("equation_relu", (64, 32)), ("equation_relu", (64, 32, 64, 1)), ("equation_relu", (37, 9, 48, 0)),
               ("equation_softmax", (64, 32)), ("equation_simple_layernorm", ()),
               # two DUMP nodes, one of them feeding an argument of a SHALLOWER branch: passes only with the reference's visiting order
               # (the operand subtree that needs more temporaries first). Without arguments the driver overruns its own buffers.
               ("equation_bf16_x3_split_f32", (32, 16, 40)), ("equation_bf16_x3_split_f32", (64, 7, 64))]


@pytest.mark.parametrize("name,args", DRIVER_RUNS)
def test_reference_equation_drivers_against_the_simulated_device(name, args):
    """the reference's unmodified samples/equation/*.c (built by oracle/ref_drivers.py) with the simulation library
    first on the loader's path: each driver checks itself and returns EXIT_FAILURE on a mismatch"""
    exe = os.path.join(DRV, name)
    if not os.path.exists(exe):
        pytest.skip("%s was not prebuilt (no reference tree in the build container?)" % name)
    build_sim()
    env = dict(os.environ, LD_LIBRARY_PATH=OUT + ":" + ORACLE + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="2")
    p = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=120, env=env, cwd=DRV)
    assert p.returncode == 0, (name, args, p.stdout[-1200:], p.stderr[-600:])
    assert "FAILURE" not in p.stdout.upper(), (name, args, p.stdout[-1200:])


def test_reference_eltwise_drivers_against_the_simulated_device():
    """every (driver, arguments) pair of test_ref_drivers.ELTWISE_RUNS (the GPU pass list) plus the ternary driver, with host operands:
    the staging rules of host_meltw.c (extents per operation, secondary operands, generator state in and out, padding kept) against
    the oracle's answers. Gather / scatter insist on device-accessible operands, so those runs declare the memory pinned."""
    from test_ref_drivers import ELTWISE_RUNS
    build_sim()
    ran = 0
    for name, args in ELTWISE_RUNS + TERNARY_RUNS + MORE_ELTWISE_RUNS:
        exe = os.path.join(DRV, name)
        if not os.path.exists(exe):
            continue
        env = dict(os.environ, LD_LIBRARY_PATH=OUT + ":" + ORACLE + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="2",
                   XB_HOSTSIM_PTR_KIND="3" if "gather" in name else "0")
        p = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=120, env=env, cwd=DRV)
        assert p.returncode == 0, (name, args, p.stdout[-1200:], p.stderr[-600:])
        assert "FAILURE" not in p.stdout.upper(), (name, args, p.stdout[-1200:])
        ran += 1
    if ran == 0:
        pytest.skip("no prebuilt drivers (no reference tree in the build container?)")


def test_reference_gemm_drivers_against_the_simulated_device():
    """samples/hello/hello.c and samples/xgemm/gemm_kernel.c / gemm_kernel_fused.c / gemm_kernel_parallel.c: dispatch, leading-dimension rules,
    the four batch-reduce calling conventions, staging of host A / B / C (what survives in C's padding, the relu bit mask, the bias column),
    bitmap-compressed A ("spmm") and concurrent callers (OpenMP threads sharing one kernel) -- the GEMM half of host_core.c, with every
    tile answered by the oracle; the drivers compare with their own gold and return EXIT_FAILURE on a mismatch"""
    build_sim()
    ran = 0
    for name, args in GEMM_RUNS:
        exe = os.path.join(DRV, name)
        if not os.path.exists(exe):
            continue
        env = dict(os.environ, LD_LIBRARY_PATH=OUT + ":" + ORACLE + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="4")
        p = subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=120, env=env, cwd=DRV)
        assert p.returncode == 0, (name, args, p.stdout[-1200:], p.stderr[-600:])
        assert "hostsim:" not in p.stderr, (name, args, p.stderr[-600:])
        if name != "hello":
            assert "Total Max Error 0.0000" in p.stdout, (name, args, p.stdout[-600:])
        ran += 1
    if ran == 0:
        pytest.skip("no prebuilt drivers (no reference tree in the build container?)")


@pytest.mark.parametrize("mtx", ["pyfr_p1_tet_m6-sp.mtx", "pyfr_p3_hex_m6-sp.mtx"])
def test_pyfr_driver_concurrent_column_blocks_from_pageable_memory(mtx):
    """samples/xgemm_sparse_Ainregs/pyfr_driver_asp_reg.c runs the 48-column blocks of one C under `omp parallel for`. In the simulation
    every pointer counts as pageable host memory, so each call stages its operands: only the m x max_N block of C may travel (a contiguous
    span would carry the neighbours' columns back stale -- the fault this test found). The sparse product itself is the library's direct
    loop restated in tests/c/hostsim_runtime.c."""
    exe = os.path.join(DRV, "pyfr_driver_asp_reg")
    if not os.path.exists(exe):
        pytest.skip("pyfr_driver_asp_reg was not prebuilt (no reference tree in the build container?)")
    build_sim()
    env = dict(os.environ, LD_LIBRARY_PATH=OUT + ":" + ORACLE + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="4")
    p = subprocess.run([exe, os.path.join(ROOT, "tests", "golden", "mtx", mtx), "480", "2"], capture_output=True, text=True, timeout=180, env=env, cwd=DRV)
    assert p.returncode == 0, (p.stdout[-1500:], p.stderr[-600:])
    lines = [ln for ln in p.stdout.splitlines() if "(libxsmm vs. gold)" in ln]
    assert len(lines) == 2 and all(float(ln.split("abs=")[1].split()[0]) < 1e-6 for ln in lines), p.stdout[-1500:]


def test_host_resident_strided_batch_through_the_chunked_pipeline(sim):
    """libxsmm_b200_gemm_batch_strided on HOST buffers -- the call bench.py's `e2e` leg makes: host_core.c cuts the batch into chunks (A, B, C
    extents per chunk, C copied in only when it is read, the last chunk shorter) and a three-stage pipeline moves them. Here the pipeline is
    serial and its staging buffers are poisoned between chunks; the chunk budget is forced to its minimum (1 MB) so that three chunks with a ragged tail
    occur. Stride batch-reduce (br = 3), beta = 1 and beta = 0, padded leading dimensions."""
    lib = sim.lib
    I, U, P, LL, ULL = C.c_int, C.c_uint, C.c_void_p, C.c_longlong, C.c_ulonglong
    lib.libxsmm_create_gemm_shape.restype = X.GemmShape; lib.libxsmm_create_gemm_shape.argtypes = [I] * 10
    lib.libxsmm_create_gemm_batch_reduce_config.restype = X.BatchReduceConfig; lib.libxsmm_create_gemm_batch_reduce_config.argtypes = [I, I, I, C.c_ubyte]
    lib.libxsmm_dispatch_brgemm.restype = P; lib.libxsmm_dispatch_brgemm.argtypes = [X.GemmShape, U, U, X.BatchReduceConfig]
    lib.libxsmm_b200_gemm_batch_strided.restype = I; lib.libxsmm_b200_gemm_batch_strided.argtypes = [P, P, P, P, LL, LL, LL, ULL, LL]
    rng = np.random.default_rng(11)
    m, n, k, lda, ldb, ldc, br, count = 12, 7, 9, 16, 10, 14, 3, 800      # 2960 bytes per tile: 354 tiles per 1 MB chunk -> 354 + 354 + 92
    for beta0 in (0, 1):
        a = rng.standard_normal((count, br, k, lda)).astype(np.float32)      # column-major tiles: [k][lda], rows 0..m-1 used
        b = rng.standard_normal((count, br, n, ldb)).astype(np.float32)
        c = rng.standard_normal((count, n, ldc)).astype(np.float32); c0 = c.copy()
        shape = lib.libxsmm_create_gemm_shape(m, n, k, lda, ldb, ldc, F32, F32, F32, F32)
        cfg = lib.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, k * lda * 4, n * ldb * 4, 0)
        fn = lib.libxsmm_dispatch_brgemm(shape, X.GEMM_FLAG_BETA_0 if beta0 else 0, 0, cfg)
        assert fn
        os.environ["LIBXSMM_B200_CHUNK_MB"] = "1"
        try:
            rc = lib.libxsmm_b200_gemm_batch_strided(fn, a.ctypes.data, b.ctypes.data, c.ctypes.data, a[0].nbytes, b[0].nbytes, c[0].nbytes, br, count)
        finally:
            os.environ.pop("LIBXSMM_B200_CHUNK_MB", None)
        assert rc == 0, rc
        for t in range(count):
            acc = np.zeros((n, m), dtype=np.float64) if beta0 else c0[t, :, :m].astype(np.float64)
            for r in range(br):
                acc += b[t, r, :, :k].astype(np.float64) @ a[t, r, :, :m].astype(np.float64)        # C^T[n][m] = B^T[n][k] A^T[k][m]
            assert np.allclose(c[t, :, :m], acc, rtol=1e-5, atol=1e-5), (beta0, t)
            assert np.array_equal(c[t, :, m:], c0[t, :, m:]), "padding rows of C survive"


def test_batch_entry_points_refuse_handles_they_cannot_run_like_a_single_call(sim):
    """A fused handle's bias column and ReLU bit mask are operands of one call (libxsmm_gemm_ext_param), VNNI-packed C is re-packed after a
    single call only, and the strided forms have no place for the int8 -> f32 scale of c.tertiary. Every batch form refuses such a handle with
    LIBXSMM_B200_ERROR_NOT_BATCHABLE before anything runs: C keeps its bytes and no kernel is counted. The int8 -> f32 handle stays usable
    through libxsmm_b200_gemm_batch, whose argument structs carry one scale per tile."""
    lib = sim.lib
    I, U, P, LL, ULL, UB = C.c_int, C.c_uint, C.c_void_p, C.c_longlong, C.c_ulonglong, C.c_ubyte
    for name, res, args in (("libxsmm_create_gemm_shape", X.GemmShape, [I] * 10), ("libxsmm_create_gemm_batch_reduce_config", X.BatchReduceConfig, [I, I, I, UB]),
                            ("libxsmm_create_gemm_ext_unary_argops", X.GemmExtUnaryArgops, [I, I, U, I, I, I, U, I, I, I, U, I]),
                            ("libxsmm_create_gemm_ext_binary_postops", X.GemmExtBinaryPostops, [I, I, I, U]),
                            ("libxsmm_dispatch_gemm", P, [X.GemmShape, U, U]),
                            ("libxsmm_dispatch_brgemm_ext", P, [X.GemmShape, U, U, X.BatchReduceConfig, X.GemmExtUnaryArgops, X.GemmExtBinaryPostops]),
                            ("libxsmm_b200_gemm_batch_strided", I, [P, P, P, P, LL, LL, LL, ULL, LL]),
                            ("libxsmm_b200_gemm_batch_strided_multi", I, [P, P, P, P, LL, LL, LL, ULL, LL, I]),
                            ("libxsmm_b200_gemm_batch", I, [P, C.POINTER(X.GemmParam), LL]), ("libxsmm_b200_gemm_plan_create", P, [P, C.POINTER(X.GemmParam), LL]),
                            ("libxsmm_b200_launch_count", ULL, []), ("libxsmm_b200_launch_count_backend", ULL, [I])):
        fn = getattr(lib, name); fn.restype = res; fn.argtypes = args
    NOT_BATCHABLE = -6          # include/libxsmm_b200.h
    m, n, k, count = 16, 8, 16, 3
    nobr = lib.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_NONE, 0, 0, 0)
    no_post = lib.libxsmm_create_gemm_ext_binary_postops(0, 0, 0, 0)
    no_arg = lib.libxsmm_create_gemm_ext_unary_argops(0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0)
    f32 = lib.libxsmm_create_gemm_shape(m, n, k, m, k, m, F32, F32, F32, F32)
    handles = {
        "column bias": lib.libxsmm_dispatch_brgemm_ext(f32, 0, 0, nobr, no_arg,
                                                       lib.libxsmm_create_gemm_ext_binary_postops(m, F32, X.MELTW_TYPE_BINARY_ADD, X.MELTW_FLAG_BINARY_BCAST_COL_IN_0)),
        "relu bit mask": lib.libxsmm_dispatch_brgemm_ext(f32, 0, 0, nobr, lib.libxsmm_create_gemm_ext_unary_argops(
            0, 0, 0, 0, 0, 0, 0, 0, m, X.MELTW_TYPE_UNARY_RELU, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT, 0), no_post),
        "vnni c": lib.libxsmm_dispatch_gemm(lib.libxsmm_create_gemm_shape(m, n, k, m, k, m, BF16, BF16, BF16, F32), X.GEMM_FLAG_VNNI_A | X.GEMM_FLAG_VNNI_C, 0),
        "int8 to f32": lib.libxsmm_dispatch_gemm(lib.libxsmm_create_gemm_shape(m, n, k, m, k, m, gen.U8, gen.I8, F32, gen.I32), X.GEMM_FLAG_VNNI_A, 0),
    }
    rng = np.random.default_rng(12)
    a = rng.integers(0, 256, size=count * m * k * 4, dtype=np.uint8); b = rng.integers(0, 256, size=count * k * n * 4, dtype=np.uint8)
    sa, sb, sc = m * k * 4, k * n * 4, m * n * 4
    scales = [C.c_float(2.0 ** -(t + 1)) for t in range(count)]
    for what, fn in handles.items():
        assert fn, what
        c = rng.integers(0, 256, size=count * sc, dtype=np.uint8); c0 = c.copy()
        params = (X.GemmParam * count)()
        for t in range(count):
            params[t].a.primary, params[t].b.primary, params[t].c.primary = a.ctypes.data + t * sa, b.ctypes.data + t * sb, c.ctypes.data + t * sc
            params[t].c.tertiary = C.addressof(scales[t])
        before = [lib.libxsmm_b200_launch_count()] + [lib.libxsmm_b200_launch_count_backend(x) for x in (X.BACKEND_SIMT, X.BACKEND_TCGEN05, X.BACKEND_STREAM)]
        assert lib.libxsmm_b200_gemm_batch_strided(fn, a.ctypes.data, b.ctypes.data, c.ctypes.data, sa, sb, sc, 1, count) == NOT_BATCHABLE, what
        assert lib.libxsmm_b200_gemm_batch_strided_multi(fn, a.ctypes.data, b.ctypes.data, c.ctypes.data, sa, sb, sc, 1, count, 1) == NOT_BATCHABLE, what
        if what != "int8 to f32":
            assert lib.libxsmm_b200_gemm_batch(fn, params, count) == NOT_BATCHABLE, what
            assert not lib.libxsmm_b200_gemm_plan_create(fn, params, count), what
        after = [lib.libxsmm_b200_launch_count()] + [lib.libxsmm_b200_launch_count_backend(x) for x in (X.BACKEND_SIMT, X.BACKEND_TCGEN05, X.BACKEND_STREAM)]
        assert after == before, (what, before, after)
        assert np.array_equal(c, c0), what
        if what == "int8 to f32":     # one scale per argument struct: this form runs, one exact-order tile per struct
            assert lib.libxsmm_b200_gemm_batch(fn, params, count) == 0
            assert lib.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT) == before[1] + count
            want = c0.copy()
            for t in range(count):
                p = X.GemmParam()
                p.a.primary, p.b.primary, p.c.primary, p.c.tertiary = a.ctypes.data + t * sa, b.ctypes.data + t * sb, want.ctypes.data + t * sc, C.addressof(scales[t])
                X.GEMMFUNCTION(fn)(C.byref(p))
            assert np.array_equal(c, want)
            assert not np.array_equal(c, c0)


def test_int4_zero_points_travel_per_tile_in_the_batch_form(sim):
    """An I4X2 x U8 -> I32 handle reads zero points from a.quaternary, one byte per row and reduce step. libxsmm_b200_gemm_batch carries
    each tile's pointer into its record, so the batch gives what one call per tile gives; a tile without zero points is refused (-1) before
    anything runs. The strided forms have no place for them (LIBXSMM_B200_ERROR_NOT_BATCHABLE) and a plan, which is replayed, gets none."""
    from test_oracle_vs_ref import FLAG_INTLV_A, FLAG_MXK_ZPT, I4X2, int4_case
    lib = sim.lib
    I, U, P, LL, ULL, UB = C.c_int, C.c_uint, C.c_void_p, C.c_longlong, C.c_ulonglong, C.c_ubyte
    for name, res, args in (("libxsmm_create_gemm_shape", X.GemmShape, [I] * 10), ("libxsmm_create_gemm_batch_reduce_config", X.BatchReduceConfig, [I, I, I, UB]),
                            ("libxsmm_dispatch_brgemm", P, [X.GemmShape, U, U, X.BatchReduceConfig]),
                            ("libxsmm_b200_gemm_batch_strided", I, [P, P, P, P, LL, LL, LL, ULL, LL]),
                            ("libxsmm_b200_gemm_batch_strided_multi", I, [P, P, P, P, LL, LL, LL, ULL, LL, I]),
                            ("libxsmm_b200_gemm_batch", I, [P, C.POINTER(X.GemmParam), LL]), ("libxsmm_b200_gemm_plan_create", P, [P, C.POINTER(X.GemmParam), LL]),
                            ("libxsmm_b200_launch_count", ULL, [])):
        fn = getattr(lib, name); fn.restype = res; fn.argtypes = args
    NOT_BATCHABLE = -6          # include/libxsmm_b200.h
    rng = np.random.default_rng(13)
    count, br = 3, 4
    tiles = [int4_case(rng, 13, 6, 16, br, 3) for _ in range(count)]
    dims, _, _, _, _, blk_a, blk_b = tiles[0]
    fn = lib.libxsmm_dispatch_brgemm(lib.libxsmm_create_gemm_shape(*dims, I4X2, gen.U8, gen.I32, gen.I32), X.GEMM_FLAG_VNNI_A | FLAG_INTLV_A | FLAG_MXK_ZPT, 0,
                                     lib.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, blk_a, blk_b, 0))
    assert fn
    brv = C.c_ulonglong(br)
    c = [t[4].copy() for t in tiles]
    params = (X.GemmParam * count)()
    for t, (_, a, b, zpt, _, _, _) in enumerate(tiles):
        params[t].op.tertiary = C.addressof(brv)
        params[t].a.primary, params[t].b.primary, params[t].c.primary, params[t].a.quaternary = a.ctypes.data, b.ctypes.data, c[t].ctypes.data, zpt.ctypes.data
    # a tile without zero points: nothing runs
    params[1].a.quaternary = None
    n0 = lib.libxsmm_b200_launch_count()
    assert lib.libxsmm_b200_gemm_batch(fn, params, count) == -1
    assert lib.libxsmm_b200_launch_count() == n0
    assert all(np.array_equal(c[t], tiles[t][4]) for t in range(count))
    params[1].a.quaternary = tiles[1][3].ctypes.data
    # strided forms and plans
    a0, b0, c0 = tiles[0][1], tiles[0][2], c[0]
    assert lib.libxsmm_b200_gemm_batch_strided(fn, a0.ctypes.data, b0.ctypes.data, c0.ctypes.data, 0, 0, 0, br, count) == NOT_BATCHABLE
    assert lib.libxsmm_b200_gemm_batch_strided_multi(fn, a0.ctypes.data, b0.ctypes.data, c0.ctypes.data, 0, 0, 0, br, count, 1) == NOT_BATCHABLE
    assert not lib.libxsmm_b200_gemm_plan_create(fn, params, count)
    assert lib.libxsmm_b200_launch_count() == n0
    assert all(np.array_equal(c[t], tiles[t][4]) for t in range(count))
    # the batch equals one call per tile
    assert lib.libxsmm_b200_gemm_batch(fn, params, count) == 0
    assert lib.libxsmm_b200_launch_count() == n0 + count
    for t, (_, a, b, zpt, c_init, _, _) in enumerate(tiles):
        want = c_init.copy()
        p = X.GemmParam(); p.op.tertiary = C.addressof(brv)
        p.a.primary, p.b.primary, p.c.primary, p.a.quaternary = a.ctypes.data, b.ctypes.data, want.ctypes.data, zpt.ctypes.data
        X.GEMMFUNCTION(fn)(C.byref(p))
        assert np.array_equal(c[t], want), t
        assert not np.array_equal(want, c_init), t
