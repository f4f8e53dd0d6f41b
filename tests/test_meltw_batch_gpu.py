"""GPU: libxsmm_b200_meltw_batch_strided / libxsmm_b200_meqn_batch_strided. Every call of a batch must equal, byte for byte, the
single call of the same handle on the same tile (the single calls are pinned to the reference elsewhere), the bytes between tiles
must keep their poison, a batch must launch what one single call launches, and every return code of the header is exercised."""
import ctypes as C

import numpy as np
import pytest
import torch

import gen
import libxsmm_b200 as X
from test_meqn import build

pytestmark = [pytest.mark.gpu]

POISON = 0xA5
NOT_BATCHABLE = -6      # LIBXSMM_B200_ERROR_NOT_BATCHABLE
F32, BF16 = gen.F32, gen.BF16


def buf(nbytes, rng=None, dtype=None):
    """a device byte buffer: random values of `dtype` (finite, both signs), or the poison"""
    if rng is None:
        return torch.full((nbytes,), POISON, dtype=torch.uint8, device="cuda")
    if dtype == BF16:
        v = (rng.standard_normal(nbytes // 2).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
    else:
        v = rng.standard_normal(nbytes // 4).astype(np.float32)
    return torch.from_numpy(v.view(np.uint8).copy()).cuda()


def ptr_at(t, off):
    return None if t is None else t.data_ptr() + off


class Unary:
    """one unary handle on tiles of `sx` input bytes, `so` output bytes and `sa` out.secondary bytes (0: none) per call"""

    def __init__(self, op, m, n, ldi, ldo, tin, tout, flags, sx, so, sa=0, sia=0, alpha=None):
        comp = gen.F64 if tin == gen.F64 else F32
        self.k = X.libxsmm_dispatch_meltw_unary(op, X.libxsmm_create_meltw_unary_shape(m, n, ldi, ldo, tin, tout, comp), flags)
        assert self.k, (op, tin, tout, flags)
        self.tin, self.sx, self.so, self.sa, self.sia = tin, sx, so, sa, sia
        self.alpha = None if alpha is None else C.c_float(alpha)    # op.primary: read once, from call 0

    def param(self, x, o, a, ia, t, strides):
        p = X.MeltwUnaryParam()
        p.inp.primary = ptr_at(x, t * strides.in0)
        p.out.primary = ptr_at(o, t * strides.out)
        if a is not None:
            p.out.secondary = ptr_at(a, t * strides.out_aux)
        if ia is not None:
            p.inp.secondary = ptr_at(ia, t * strides.in_aux)
        if self.alpha is not None:
            p.op.primary = C.addressof(self.alpha)
        return p

    def run(self, count, rng, check_tiles=None):
        s = X.MeltwStrides(in0=self.sx, out=self.so, out_aux=self.sa, in_aux=self.sia)
        x = buf(count * self.sx, rng, self.tin)
        ia = buf(count * self.sia, rng, None) if self.sia else None
        o, a = buf(count * self.so), (buf(count * self.sa) if self.sa else None)
        before = X.libxsmm_b200_launch_count()
        assert X.libxsmm_b200_meltw_batch_strided(self.k, C.addressof(self.param(x, o, a, ia, 0, s)), C.byref(s), count) == 0
        X.check()
        launched = X.libxsmm_b200_launch_count() - before
        o1, a1 = buf(count * self.so), (buf(count * self.sa) if self.sa else None)
        tiles = range(count) if check_tiles is None else check_tiles
        before = X.libxsmm_b200_launch_count()
        for t in tiles:
            X.MELTW_UNARY_FN(self.k)(C.byref(self.param(x, o1, a1, ia, t, s)))
        X.check()
        single = (X.libxsmm_b200_launch_count() - before) // len(tiles)
        assert launched == single, (launched, single)
        for t in tiles:
            assert torch.equal(o[t * self.so:(t + 1) * self.so], o1[t * self.so:(t + 1) * self.so]), t
            if a is not None:
                assert torch.equal(a[t * self.sa:(t + 1) * self.sa], a1[t * self.sa:(t + 1) * self.sa]), t
        if check_tiles is None:                                  # every byte, gaps included
            assert torch.equal(o, o1) and (a is None or torch.equal(a, a1))
        return o


M, N, LDI, LDO = 64, 64, 72, 80
UNARY_CASES = {
    "relu_mask_f32": (X.MELTW_TYPE_UNARY_RELU, M, N, LDI, LDO, F32, F32, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT, LDI * N * 4 + 64, LDO * N * 4 + 32, 80 // 8 * N + 16),
    "tanh_bf16": (X.MELTW_TYPE_UNARY_TANH, M, N, LDI, LDO, BF16, BF16, 0, LDI * N * 2, LDO * N * 2),
    "vnni2_bf16": (X.MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2, M, N, LDI, LDO, BF16, BF16, 0, LDI * N * 2, LDO * N * 2),
    "vnni2_bf16_unaligned": (X.MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2, M, N, LDI, LDO, BF16, BF16, 0, LDI * N * 2 + 2, LDO * N * 2 + 2),
    "normt_f32": (X.MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT, M, N, LDI, LDO, F32, F32, 0, LDI * N * 4, LDO * M * 4),
    "normt_small_f32": (X.MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT, 24, 20, 24, 24, F32, F32, 0, 24 * 20 * 4, 24 * 24 * 4),
    "rows_x_x2_f32": (X.MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD, M, N, LDI, N, F32, F32, X.MELTW_FLAG_UNARY_REDUCE_ROWS, LDI * N * 4, 2 * N * 4 + 8),
    "cols_x_f32": (X.MELTW_TYPE_UNARY_REDUCE_X_OP_ADD, M, N, LDI, M, F32, F32, X.MELTW_FLAG_UNARY_REDUCE_COLS, LDI * N * 4, M * 4),
    "cols_max_argop": (X.MELTW_TYPE_UNARY_REDUCE_X_OP_MAX, M, N, LDI, M, F32, F32,
                       X.MELTW_FLAG_UNARY_REDUCE_COLS | X.MELTW_FLAG_UNARY_REDUCE_RECORD_ARGOP | X.MELTW_FLAG_UNARY_IDX_SIZE_4BYTES, LDI * N * 4, M * 4, M * 4),
    "to_scalar_f32": (X.MELTW_TYPE_UNARY_REDUCE_TO_SCALAR_OP_ADD, M, N, LDI, LDO, F32, F32, 0, LDI * N * 4, 16),
    "mxfp4": (X.MELTW_TYPE_UNARY_QUANT, M, N, LDI, LDO, BF16, X.DATATYPE_MXFP4X2, 0, LDI * N * 2, LDO // 2 * N, LDO // 32 * N),
    "nvfp4": (X.MELTW_TYPE_UNARY_QUANT, M, N, LDI, LDO, BF16, X.DATATYPE_NVFP4X2, 0, LDI * N * 2, LDO // 2 * N, LDO // 16 * N),
    "mxbf8": (X.MELTW_TYPE_UNARY_QUANT, M, N, LDI, LDO, BF16, X.DATATYPE_MXBF8, 0, LDI * N * 2, LDO * N, LDO // 32 * N),
    "quant_i8": (X.MELTW_TYPE_UNARY_QUANT, M, N, LDI, LDO, F32, X.DATATYPE_I8, 0, LDI * N * 4, LDO * N),
    "dequant_i8": (X.MELTW_TYPE_UNARY_DEQUANT, M, N, LDI, LDO, X.DATATYPE_I8, F32, 0, LDI * N, LDO * N * 4),
    "vnni4_i8": (X.MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI4, M, N, LDI, LDO, X.DATATYPE_I8, X.DATATYPE_I8, 0, LDI * N, LDO * N),
    "x2_f64": (X.MELTW_TYPE_UNARY_X2, M, N, LDI, LDO, gen.F64, gen.F64, 0, LDI * N * 8, LDO * N * 8),
    "tanh_f16": (X.MELTW_TYPE_UNARY_TANH, M, N, LDI, LDO, X.DATATYPE_F16, X.DATATYPE_F16, 0, LDI * N * 2, LDO * N * 2),
    # per-call in.secondary: a bit mask (mask ld = ldi rounded up to 16 bits), or the forward output of ELU
    "relu_inv_mask": (X.MELTW_TYPE_UNARY_RELU_INV, M, N, LDI, LDO, F32, F32, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT, LDI * N * 4, LDO * N * 4, 0, 80 // 8 * N + 8),
    "leaky_relu_inv_mask": (X.MELTW_TYPE_UNARY_LEAKY_RELU_INV, M, N, LDI, LDO, F32, F32, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT, LDI * N * 4, LDO * N * 4, 0, 80 // 8 * N + 8, 0.25),
    "elu_inv": (X.MELTW_TYPE_UNARY_ELU_INV, M, N, LDI, LDO, F32, F32, 0, LDI * N * 4, LDO * N * 4, 0, LDI * N * 4 + 4, 0.5),
    "dropout_inv_mask": (X.MELTW_TYPE_UNARY_DROPOUT_INV, M, N, LDI, LDO, F32, F32, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT, LDI * N * 4, LDO * N * 4, 0, 80 // 8 * N + 8, 0.3),
}


@pytest.mark.parametrize("count", [1, 7])
@pytest.mark.parametrize("name", sorted(UNARY_CASES))
def test_unary_batch_equals_single_calls(name, count):
    Unary(*UNARY_CASES[name]).run(count, np.random.default_rng(sum(name.encode())))


@pytest.mark.parametrize("name", ["relu_mask_f32", "vnni2_bf16", "normt_f32", "rows_x_x2_f32", "cols_max_argop", "mxfp4"])
def test_unary_large_batch_wraps_every_grid_loop(name):
    count = 20000
    Unary(*UNARY_CASES[name]).run(count, np.random.default_rng(3), check_tiles=[0, 1, count // 2, count - 2, count - 1])


@pytest.mark.parametrize("m,n", [(255, 1024), (256, 1024), (256, 2048)])
def test_column_sums_across_the_two_phase_threshold(m, n):
    """single calls at m >= 256, m*n >= 2^18 take the two-phase kernel, a batch the warp reduction: within (len + 2) u sum|x| of
    the float64 sum; bit-identical where the single call runs the warp reduction"""
    k = Unary(X.MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD, m, n, m, m, F32, F32, X.MELTW_FLAG_UNARY_REDUCE_COLS, m * n * 4, m * 4)
    two_phase = X.libxsmm_b200_meltw_variant(k.k, None) in (5, 6)
    if not two_phase:
        k.run(3, np.random.default_rng(m))
        return
    rng = np.random.default_rng(m + n)
    count = 3
    xs = rng.standard_normal((count, n, m)).astype(np.float32)
    x = torch.from_numpy(xs.reshape(-1).view(np.uint8).copy()).cuda()
    o = buf(count * m * 4)
    s = X.MeltwStrides(in0=m * n * 4, out=m * 4)
    assert X.libxsmm_b200_meltw_batch_strided(k.k, C.addressof(k.param(x, o, None, None, 0, s)), C.byref(s), count) == 0
    X.check()
    got = o.cpu().numpy().view(np.float32).reshape(count, m)
    sq = xs.astype(np.float64) ** 2
    exact = sq.sum(axis=1)
    bound = (n + 2) * 2.0 ** -24 * sq.sum(axis=1)
    assert np.all(np.abs(got - exact) <= bound)


def test_binary_bias_shared_by_stride_zero():
    """BCAST_COL bias with stride 0: one bias column for every call"""
    sh = X.libxsmm_create_meltw_binary_shape(M, N, LDI, M, LDO, F32, F32, F32, F32)
    k = X.libxsmm_dispatch_meltw_binary(X.MELTW_TYPE_BINARY_ADD, sh, X.MELTW_FLAG_BINARY_BCAST_COL_IN_1)
    assert k
    rng = np.random.default_rng(11)
    count, sx, so = 9, LDI * N * 4, LDO * N * 4
    x, bias, o, o1 = buf(count * sx, rng), buf(M * 4, rng), buf(count * so), buf(count * so)
    s = X.MeltwStrides(in0=sx, in1=0, out=so)

    def param(t, out):
        p = X.MeltwBinaryParam(); p.in0.primary = x.data_ptr() + t * sx; p.in1.primary = bias.data_ptr(); p.out.primary = out.data_ptr() + t * so
        return p
    assert X.libxsmm_b200_meltw_batch_strided(k, C.addressof(param(0, o)), C.byref(s), count) == 0
    for t in range(count):
        X.MELTW_BINARY_FN(k)(C.byref(param(t, o1)))
    X.check()
    assert torch.equal(o, o1)


def test_return_codes():
    k = Unary(*UNARY_CASES["relu_mask_f32"])
    rng = np.random.default_rng(1)
    x, o, a = buf(4 * k.sx, rng), buf(4 * k.so), buf(4 * k.sa)
    s = X.MeltwStrides(in0=k.sx, out=k.so, out_aux=k.sa)
    p = k.param(x, o, a, None, 0, s)
    f = X.libxsmm_b200_meltw_batch_strided
    assert f(None, C.addressof(p), C.byref(s), 2) == -1
    assert f(k.k, C.addressof(p), C.byref(s), -1) == -1
    assert f(k.k, C.addressof(p), C.byref(s), 0) == 0
    for field in ("in0", "out", "out_aux"):
        bad = X.MeltwStrides(in0=k.sx, out=k.so, out_aux=k.sa); setattr(bad, field, -8)
        assert f(k.k, C.addressof(p), C.byref(bad), 2) == -1, field
    for field, v in (("out", (N - 1) * LDO * 4 + M * 4 - 4), ("out_aux", 80 // 8 * N - 1)):
        bad = X.MeltwStrides(in0=k.sx, out=k.so, out_aux=k.sa); setattr(bad, field, v)
        assert f(k.k, C.addressof(p), C.byref(bad), 2) == -1, field
        assert f(k.k, C.addressof(p), C.byref(bad), 1) == 0, field        # one call cannot overlap itself
    host = np.zeros(k.sx, dtype=np.uint8)
    ph = k.param(x, o, a, None, 0, s); ph.inp.primary = host.ctypes.data
    assert f(k.k, C.addressof(ph), C.byref(s), 2) == -4
    drop = X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_DROPOUT, X.libxsmm_create_meltw_unary_shape(M, N, LDI, LDO, F32, F32, F32), 0)
    sr = X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_IDENTITY, X.libxsmm_create_meltw_unary_shape(M, N, LDI, LDO, F32, gen.BF8, F32),
                                        X.MELTW_FLAG_UNARY_STOCHASTIC_ROUND)
    rep = X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_REPLICATE_COL_VAR, X.libxsmm_create_meltw_unary_shape(M, N, LDI, LDO, F32, F32, F32), 0)
    gat = X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_GATHER, X.libxsmm_create_meltw_unary_shape(M, N, LDI, LDO, F32, F32, F32), X.MELTW_FLAG_UNARY_GS_COLS)
    idx = X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_ADD, X.libxsmm_create_meltw_unary_shape(M, N, LDI, M, F32, F32, F32), 0)
    unz = X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_DECOMP_FP32_TO_BF16X2, X.libxsmm_create_meltw_unary_shape(M, N, LDI, LDO, F32, BF16, F32), 0)
    for h in (drop, sr, rep, gat, idx, unz):
        assert h
        assert f(h, C.addressof(p), C.byref(s), 2) == NOT_BATCHABLE
    assert X.libxsmm_b200_meqn_batch_strided(None, None, None, 0, 0, None, 1) == -1


# ---- equations ------------------------------------------------------------------------------------------------------------------
LN_NODES = [("b", X.MELTW_TYPE_BINARY_MUL, F32, X.MELTW_FLAG_BINARY_BCAST_COL_IN_1),
            ("b", X.MELTW_TYPE_BINARY_SUB, F32, X.MELTW_FLAG_BINARY_BCAST_COL_IN_1),
            ("arg", 0, M, N, LDI, F32),
            ("u", X.MELTW_TYPE_UNARY_REDUCE_X_OP_ADD, F32, X.MELTW_FLAG_UNARY_REDUCE_COLS),
            ("arg", 0, M, N, LDI, F32),
            ("arg", 1, M, 1, M, F32)]
RELU_NODES = [("u", X.MELTW_TYPE_UNARY_RELU, F32, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT),
              ("b", X.MELTW_TYPE_BINARY_ADD, F32, 0),
              ("arg", 0, M, N, LDI, F32),
              ("arg", 1, M, N, LDI, F32)]


def run_eqn(nodes, count, tiles, mask=False):
    eq = build(nodes)
    k = X.libxsmm_dispatch_meqn(eq, X.MeqnArgShape(M, N, LDO, F32))
    assert k
    rng = np.random.default_rng(count)
    sx, so, sm = LDI * N * 4, LDO * N * 4, 80 // 8 * N
    is_ln = nodes is LN_NODES
    x0 = buf(count * sx, rng)
    x1 = buf(M * 4, rng) if is_ln else buf(count * sx, rng)
    strides = (C.c_longlong * 2)(sx, 0 if is_ln else sx)
    o, o1 = buf(count * so), buf(count * so)
    am, am1 = buf(count * sm), buf(count * sm)

    def param(t, out, aux):
        ins = (X.MatrixArg * 2)()
        ins[0].primary = x0.data_ptr() + t * sx
        ins[1].primary = x1.data_ptr() + t * strides[1]
        p = X.MeqnParam(); p.inputs = C.addressof(ins); p.output.primary = out.data_ptr() + t * so
        if mask:
            p.output.secondary = aux.data_ptr() + t * sm
        return p, ins
    p, keep = param(0, o, am)
    before = X.libxsmm_b200_launch_count()
    assert X.libxsmm_b200_meqn_batch_strided(k, C.byref(p), strides, so, sm, None, count) == 0
    X.check()
    launched = X.libxsmm_b200_launch_count() - before
    for t in tiles:
        p1, keep1 = param(t, o1, am1)
        X.MEQN_FN(k)(C.byref(p1))
    X.check()
    for t in tiles:
        assert torch.equal(o[t * so:(t + 1) * so], o1[t * so:(t + 1) * so]), t
        if mask:
            assert torch.equal(am[t * sm:(t + 1) * sm], am1[t * sm:(t + 1) * sm]), t
    return launched


@pytest.mark.parametrize("count", [1, 7])
def test_layernorm_style_equation(count):
    nodes = sum(1 for nd in LN_NODES if nd[0] != "arg")
    assert run_eqn(LN_NODES, count, range(count)) == nodes


def test_relu_bitmask_head_equation():
    assert run_eqn(RELU_NODES, 7, range(7), mask=True) == 2


def test_equation_batch_crosses_the_chunk_bound():
    """temporaries of 64 x 64 f32 (16 KiB + the reduction's 256 B per call): 64 MiB hold 4,032 calls, so 5,000 run in two chunks"""
    count = 5000
    assert run_eqn(LN_NODES, count, [0, 4031, 4032, count - 1]) == 3 * 2


def _binary_or_ternary(op, arity, flags, tin=F32, tout=F32, so=LDO * N * 4, ldo=LDO, ldi3=LDI, in2_bytes=None):
    if arity == 2:
        k = X.libxsmm_dispatch_meltw_binary(op, X.libxsmm_create_meltw_binary_shape(M, N, LDI, LDI, ldo, tin, tin, tout, F32), flags)
    else:
        k = X.libxsmm_dispatch_meltw_ternary(op, X.libxsmm_create_meltw_ternary_shape(M, N, LDI, LDI, ldi3, ldo, tin, tin, tin, tout, F32), flags)
    assert k
    rng = np.random.default_rng(op + 17 * arity)
    count, sx = 7, LDI * N * 4 + 4
    s2 = in2_bytes if in2_bytes is not None else sx
    ins = [buf(count * sx, rng), buf(count * sx, rng), buf(count * s2, rng)]
    o, o1 = buf(count * so), buf(count * so)
    s = X.MeltwStrides(in0=sx, in1=sx, in2=s2, out=so)

    def param(t, out):
        p = X.MeltwBinaryParam() if arity == 2 else X.MeltwTernaryParam()
        p.in0.primary, p.in1.primary, p.out.primary = ins[0].data_ptr() + t * sx, ins[1].data_ptr() + t * sx, out.data_ptr() + t * so
        if arity == 3:
            p.in2.primary = ins[2].data_ptr() + t * s2
        return p
    fn = X.MELTW_BINARY_FN if arity == 2 else X.MELTW_TERNARY_FN
    assert X.libxsmm_b200_meltw_batch_strided(k, C.addressof(param(0, o)), C.byref(s), count) == 0
    for t in range(count):
        fn(k)(C.byref(param(t, o1)))
    X.check()
    assert torch.equal(o, o1)


@pytest.mark.parametrize("case", ["mul", "cmp_gt", "mul_reduce_scalar", "muladd3", "select"])
def test_binary_and_ternary_per_call_operands(case):
    """in1 and in2 advance with the call as in0 does"""
    if case == "mul":
        _binary_or_ternary(X.MELTW_TYPE_BINARY_MUL, 2, 0)
    elif case == "cmp_gt":     # the result is a bit mask: ldo rounded up to 16 bits per column
        _binary_or_ternary(X.MELTW_TYPE_BINARY_CMP_OP_GT, 2, 0, so=80 // 8 * N + 8)
    elif case == "mul_reduce_scalar":
        _binary_or_ternary(X.MELTW_TYPE_BINARY_MUL_AND_REDUCE_TO_SCALAR_OP_ADD, 2, 0, so=16)
    elif case == "muladd3":
        _binary_or_ternary(X.MELTW_TYPE_TERNARY_MULADD, 3, 0)
    else:                      # in2: a per-call bit mask
        _binary_or_ternary(X.MELTW_TYPE_TERNARY_SELECT, 3, 0, in2_bytes=80 // 8 * N + 8)


def test_softmax_style_dump_feeding_an_argument():
    """exp(x) is dumped into ops_args[0], which is also inputs[1]: the ADD reads back what the DUMP wrote, call by call"""
    nodes = [("b", X.MELTW_TYPE_BINARY_ADD, F32, 0), ("u", X.MELTW_TYPE_UNARY_DUMP, F32, 0), ("u", X.MELTW_TYPE_UNARY_EXP, F32, 0),
             ("arg", 0, M, N, LDI, F32), ("arg", 1, M, N, M, F32)]
    eq = X.libxsmm_meqn_create()
    for i, nd in enumerate(nodes):
        if nd[0] == "arg":
            rc = X.libxsmm_meqn_push_back_arg(X.libxsmm_create_meqn_arg_metadata(eq, nd[1]), X.libxsmm_create_meqn_arg_shape(nd[2], nd[3], nd[4], nd[5]),
                                              X.libxsmm_create_matrix_arg_attributes(0, 0, 0, 0))
        else:
            fn = {"u": X.libxsmm_meqn_push_back_unary_op, "b": X.libxsmm_meqn_push_back_binary_op}[nd[0]]
            rc = fn(X.libxsmm_create_meqn_op_metadata(eq, 0 if nd[1] == X.MELTW_TYPE_UNARY_DUMP and nd[0] == "u" else -1), nd[1], nd[2], nd[3])
        assert rc == 0
    k = X.libxsmm_dispatch_meqn(eq, X.MeqnArgShape(M, N, LDO, F32))
    assert k
    rng = np.random.default_rng(21)
    count, sx, sd, so = 7, LDI * N * 4, M * N * 4 + 64, LDO * N * 4
    x, o, o1 = buf(count * sx, rng), buf(count * so), buf(count * so)
    dmp, dmp1 = buf(count * sd), buf(count * sd)

    def param(t, out, d, keep):
        ins = (X.MatrixArg * 2)(); ins[0].primary, ins[1].primary = x.data_ptr() + t * sx, d.data_ptr() + t * sd
        ops = (X.MatrixOpArg * 1)(); ops[0].primary = d.data_ptr() + t * sd
        p = X.MeqnParam(); p.inputs, p.ops_args, p.output.primary = C.addressof(ins), C.addressof(ops), out.data_ptr() + t * so
        keep += [ins, ops]
        return p
    keep = []
    st, ops_s = (C.c_longlong * 2)(sx, sd), (C.c_longlong * 1)(sd)
    assert X.libxsmm_b200_meqn_batch_strided(k, C.byref(param(0, o, dmp, keep)), st, so, 0, ops_s, count) == 0
    for t in range(count):
        X.MEQN_FN(k)(C.byref(param(t, o1, dmp1, keep)))
    X.check()
    assert torch.equal(o, o1) and torch.equal(dmp, dmp1)
    bad = (C.c_longlong * 1)(sd + 4)
    assert X.libxsmm_b200_meqn_batch_strided(k, C.byref(param(0, o, dmp, keep)), st, so, 0, bad, count) == -1
    assert X.libxsmm_b200_meqn_batch_strided(k, C.byref(param(0, o, dmp, keep)), st, (N - 1) * LDO * 4 + M * 4 - 4, 0, ops_s, count) == -1   # overlapping outputs
    assert X.libxsmm_b200_meqn_batch_strided(k, C.byref(param(0, o, dmp, keep)), st, so, 0, ops_s, 0) == 0
    host = np.zeros(count * so, dtype=np.uint8)
    ph = param(0, o, dmp, keep); ph.output.primary = host.ctypes.data
    assert X.libxsmm_b200_meqn_batch_strided(k, C.byref(ph), st, so, 0, ops_s, count) == -4
