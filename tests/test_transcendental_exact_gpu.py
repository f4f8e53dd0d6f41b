"""GPU: the transcendental elementwise ops (TANH, TANH_INV, SIGMOID, SIGMOID_INV, GELU, GELU_INV, EXP and ELU) element by element
against the 2-ulp window model of tests/ulp_window.py: every output element must be one of the bit patterns the model allows for its
input (each libm call within 2 ulp, the rest of the formula exactly in the kernel's f32 operation order, RNE into the output type).

Inputs: all 65,536 bf16 and f16 bit patterns, and an f32 sweep of every binade, zeros, infinities, quiet and signalling NaNs and dense
samples around each op's thresholds (saturation, overflow, subnormal results). Layouts: ld padding whose sentinel must survive, the
ROW / COL / SCALAR broadcast flags, m not a multiple of the kernel's 32-row chunk, device and pageable operands, and the same tiles once
more through libxsmm_b200_meltw_batch_strided, bit-identical to the single calls. ELU's bit mask is compared bit for bit.

Also the fused SIGMOID post-op of the fused GEMM on an exact pre-activation (single calls and both batch forms), and matrix equations
with TANH, EXP and GELU nodes whose arguments are exact (device and host pointers, and libxsmm_b200_meqn_batch_strided)."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import gen
import libxsmm_b200 as X
import ulp_window as U
from oracle_ffi import oracle

pytestmark = [pytest.mark.gpu]

PAIRS, OPS, TNAME, split, sweep_bits = U.PAIRS, U.OPS, U.TNAME, U.split, U.sweep_bits
M, PAD_I, PAD_O = 203, 5, 7          # 203 rows: six full 32-row chunks and a partial one
SENT = {np.uint32: 0x7FBADBAD, np.uint16: 0xBEEF, np.uint8: 0xA5}
REPORT = {}


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()


def host(t, dt):
    return t.cpu().numpy().view(dt).copy()


def what(opname, tin, tout, layout):
    return "%s %s->%s %s" % (opname, TNAME[tin], TNAME[tout], layout)


def assert_in(allowed, got, x, label):
    ok = allowed.ok(got)
    if ok.all():
        return
    i = int(np.nonzero(~ok)[0][0])
    xi = np.float32(x[i])
    raise AssertionError("%s: %d of %d elements outside the 2-ulp window; first input %r (0x%08x) gave 0x%x, allowed %s" % (
        label, int((~ok).sum()), ok.size, float(xi), int(np.array([xi]).view(np.uint32)[0]), int(np.asarray(got).reshape(-1)[i]),
        sorted({hex(int(b)) for b in allowed.bits[i]}) + (["any NaN"] if allowed.any_nan[i] else [])))


class Tile:
    """the sweep laid out as an M x n column-major tile with ld padding; the padding of the input holds junk, that of the output a
    sentinel"""

    def __init__(self, bits, tin, tout):
        self.tin, self.tout = tin, tout
        self.ti, self.to = U.BITS[tin], U.BITS[tout]
        self.N = bits.size
        self.n = -(-self.N // M)
        self.ldi, self.ldo = M + PAD_I, M + PAD_O
        full = np.resize(bits.astype(self.ti), M * self.n)                  # the tail repeats the start
        self.idx = np.resize(np.arange(self.N), M * self.n)
        xin = np.full((self.n, self.ldi), 0x7F, self.ti)
        xin[:, :M] = full.reshape(self.n, M)
        self.xin = xin.reshape(-1)
        self.out0 = np.full(self.n * self.ldo, SENT[self.to], self.to)

    def valid(self, out):
        return out.reshape(self.n, self.ldo)[:, :M].reshape(-1)

    def padding_kept(self, out):
        return bool((out.reshape(self.n, self.ldo)[:, M:] == SENT[self.to]).all())

    def mask_ld(self):
        return (self.ldo + 15) // 16 * 16


def dispatch(op, m, n, ldi, ldo, tin, tout, flags):
    k = X.libxsmm_dispatch_meltw_unary(getattr(X, "MELTW_TYPE_UNARY_" + op), X.libxsmm_create_meltw_unary_shape(m, n, ldi, ldo, tin, tout, gen.F32), flags)
    assert k, (op, tin, tout, flags)
    return k


def call(k, x_ptr, o_ptr, alpha, mask_ptr=None):
    a = C.c_float(alpha if alpha is not None else 0.0)
    p = X.MeltwUnaryParam(); p.inp.primary, p.out.primary = x_ptr, o_ptr
    p.op.primary = C.addressof(a)
    if mask_ptr is not None:
        p.out.secondary = mask_ptr
    X.MELTW_UNARY_FN(k)(C.byref(p))
    X.check()


def expected_mask(x_valid, n, mask_ld, mask0):
    """bit i of column j is !(x <= 0) for i < M; the bits past M keep their bytes"""
    m = mask0.reshape(n, mask_ld // 8).copy()
    bits = ~(x_valid.reshape(n, M) <= 0)
    full = np.zeros((n, mask_ld), bool)
    full[:, :M] = bits
    packed = np.packbits(full, axis=1, bitorder="little")
    keep = np.packbits(np.arange(mask_ld)[None, :].repeat(n, 0) >= M, axis=1, bitorder="little")
    return ((m & keep) | (packed & ~keep)).reshape(-1)


def sm_ordinal(b, t):
    """ordinal of sign-magnitude bits of any of the float formats"""
    b = np.asarray(b).astype(np.int64)
    top = {gen.F32: 31, gen.BF16: 15, gen.F16: 15, gen.BF8: 7, gen.HF8: 7}[t]
    mag = b & ((1 << top) - 1)
    return np.where((b >> top) & 1 != 0, -mag, mag)


def record(opname, tin, tout, got, bits, x, alpha):
    op = split(opname)[0]
    g = U.cpu_unary(oracle, op, alpha, bits, tin, tout)
    cr = U.store(U.correctly_rounded(op, x, alpha), tout)
    real = ~U.is_nan_bits(got, tout) & ~U.is_nan_bits(cr, tout)
    nan_ok = U.is_nan_bits(got, tout) & U.is_nan_bits(g, tout)
    same = (got == g) | nan_ok
    dist = np.abs(sm_ordinal(got, tout) - sm_ordinal(cr, tout))[real]
    REPORT[(opname, TNAME[tin], TNAME[tout])] = (float(same.mean()), int(dist.max(initial=0)), got.size)


@pytest.mark.parametrize("tin,tout", PAIRS, ids=lambda t: TNAME[t])
@pytest.mark.parametrize("opname", OPS)
def test_unary_every_input(opname, tin, tout):
    """the whole sweep in one padded tile, device operands; then pageable host operands and a strided batch of the same tiles, both
    bit-identical to the device call. ELU once more with its bit mask."""
    op, alpha = split(opname)
    bits = sweep_bits(tin)
    x = U.load(bits, tin)
    allowed = U.allowed(op, x, tout, alpha)
    t = Tile(bits, tin, tout)
    k = dispatch(op, M, t.n, t.ldi, t.ldo, tin, tout, 0)
    d_x, d_o = dev(t.xin), dev(t.out0)
    call(k, d_x.data_ptr(), d_o.data_ptr(), alpha)
    out = host(d_o, t.to)
    label = what(opname, tin, tout, "m=%d n=%d ldi=%d ldo=%d" % (M, t.n, t.ldi, t.ldo))
    assert t.padding_kept(out), label + ": the output's ld padding was written"
    got = t.valid(out)
    assert_in(allowed.take(t.idx), got, x[t.idx], label)
    record(opname, tin, tout, got[:t.N], bits, x, alpha)

    # pageable host operands
    hx, ho = t.xin.copy(), t.out0.copy()
    call(k, hx.ctypes.data, ho.ctypes.data, alpha)
    assert np.array_equal(ho, out), label + ": pageable operands differ from device operands"

    # the same tile as a strided batch of column blocks, one launch
    nb = 4
    cols = t.n // nb
    kb = dispatch(op, M, cols, t.ldi, t.ldo, tin, tout, 0)
    d_ob = dev(t.out0)
    s = X.MeltwStrides(in0=cols * t.ldi * np.dtype(t.ti).itemsize, out=cols * t.ldo * np.dtype(t.to).itemsize)
    a = C.c_float(alpha if alpha is not None else 0.0)
    p = X.MeltwUnaryParam(); p.inp.primary, p.out.primary = d_x.data_ptr(), d_ob.data_ptr(); p.op.primary = C.addressof(a)
    assert X.libxsmm_b200_meltw_batch_strided(kb, C.addressof(p), C.byref(s), nb) == 0
    X.check()
    ob = host(d_ob, t.to)
    span = nb * cols * t.ldo
    assert np.array_equal(ob[:span], out[:span]), label + ": batch_strided differs from the single call"
    assert (ob[span:] == SENT[t.to]).all(), label + ": batch_strided wrote past its tiles"

    if op == "ELU":
        km = dispatch(op, M, t.n, t.ldi, t.ldo, tin, tout, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT)
        mask0 = np.random.default_rng(7).integers(0, 256, t.mask_ld() // 8 * t.n, dtype=np.uint8)
        d_o2, d_m = dev(t.out0), dev(mask0)
        call(km, d_x.data_ptr(), d_o2.data_ptr(), alpha, d_m.data_ptr())
        assert np.array_equal(host(d_o2, t.to), out), label + ": ELU with bit mask differs from ELU without"
        xv = x[t.idx]
        assert np.array_equal(host(d_m, np.uint8), expected_mask(xv, t.n, t.mask_ld(), mask0)), label + ": ELU bit mask"


BCAST = [("ROW", "MELTW_FLAG_UNARY_BCAST_ROW"), ("COL", "MELTW_FLAG_UNARY_BCAST_COL"), ("SCALAR", "MELTW_FLAG_UNARY_BCAST_SCALAR")]


@pytest.mark.parametrize("tin,tout", [(gen.F32, gen.F32), (gen.BF16, gen.BF16), (gen.F16, gen.F32)], ids=lambda t: TNAME[t])
@pytest.mark.parametrize("bc", [b[0] for b in BCAST])
@pytest.mark.parametrize("opname", OPS)
def test_unary_broadcast(opname, bc, tin, tout):
    """ROW: column j reads in[j*ldi]; COL: row i reads in[i]; SCALAR: every element reads in[0]. A sample of the sweep with every
    special value, m = 37 (a partial chunk)"""
    op, alpha = split(opname)
    flag = getattr(X, dict(BCAST)[bc])
    bits = sweep_bits(tin)
    x_all = U.load(bits, tin)
    rng = np.random.default_rng(11)
    pick = np.unique(np.concatenate([np.nonzero(~np.isfinite(x_all) | (x_all == 0))[0], rng.choice(bits.size, 3000, replace=False)]))
    ti, to = U.BITS[tin], U.BITS[tout]
    m = 37
    if bc == "SCALAR":
        pick = pick[:: max(1, pick.size // 24)]
    sel_bits = bits[pick].astype(ti)
    x = x_all[pick]
    allowed = U.allowed(op, x, tout, alpha)
    for start in range(0, x.size, 1 if bc == "SCALAR" else x.size):
        if bc == "ROW":
            n, ldi, ldo = x.size, 3, m + 2
            xin = np.full(n * ldi, 0x7F, ti); xin[::ldi] = sel_bits
            src = np.broadcast_to(np.arange(n)[:, None], (n, m))
        elif bc == "COL":
            n, ldi, ldo = 5, x.size, x.size + 3
            m = x.size
            xin = sel_bits.copy()
            src = np.broadcast_to(np.arange(m)[None, :], (n, m))
        else:
            n, ldi, ldo = 3, m, m + 1
            xin = np.full(ldi * n, 0x7F, ti); xin[0] = sel_bits[start]
            src = np.full((n, m), start)
        k = dispatch(op, m, n, ldi, ldo, tin, tout, flag)
        d_x, d_o = dev(xin), dev(np.full(n * ldo, SENT[to], to))
        call(k, d_x.data_ptr(), d_o.data_ptr(), alpha)
        out = host(d_o, to).reshape(n, ldo)
        label = what(opname, tin, tout, "BCAST_%s m=%d n=%d" % (bc, m, n))
        assert (out[:, m:] == SENT[to]).all(), label + ": padding written"
        s = src.reshape(-1)
        assert_in(allowed.take(s), out[:, :m].reshape(-1), x[s], label)
        if bc != "SCALAR":
            break


# ---- the fused SIGMOID post-op of the fused GEMM (gemm_simt.cu: (tanhf(a / 2.0f) + 1.0f) / 2.0f on the f32 pre-activation a) -----
# A(i, kk) = v_i for every kk, B(0, j) = w_j and B(kk > 0, j) = 0, so a = v_i * w_j (* scale) + seed, seed = bias_i, C_ij, both or 0.
# v_i = s * 2^e (|s| < 256, e in [-8, -1]; U8: s alone), w_j = 2^f (f in [-2, 3]; I8: small integers), bias and C on the grid 2^-4 with
# |value| < 8: every value is exact in its type (bf16 and f16 included) and every partial sum is an f32 value, so a is known exactly; it
# runs from 0 to about +-1000, far past saturation.
FUSED_TYPES = [(gen.F32, gen.F32, gen.F32, gen.F32), (gen.BF16, gen.BF16, gen.F32, gen.F32), (gen.BF16, gen.BF16, gen.F32, gen.BF16),
               (gen.F16, gen.F16, gen.F32, gen.F16), (gen.U8, gen.I8, gen.I32, gen.F32)]


def fused_operands(b, rng):
    """dyadic A, B, bias and old C for every tile of a test_gemm_ext_batch_gpu.Batch; returns the exact pre-activation per tile"""
    case, ops = b.case, b.ops
    m, n, k, count = case.m, case.n, case.k, b.count
    i8 = case.ta == gen.U8
    if i8:
        v = rng.integers(0, 256, (count, m)).astype(np.float64); v[:, 0] = 0
        w = rng.integers(-127, 128, (count, n)).astype(np.float64)
    else:
        v = rng.integers(-255, 256, (count, m)) * 2.0 ** rng.integers(-8, 0, (count, m)); v[:, 0] = 0
        w = 2.0 ** rng.integers(-2, 4, (count, n))
    bias = rng.integers(-127, 128, (count, m)) * 2.0 ** -4
    c_old = rng.integers(-127, 128, (count, n, case.ldc)) * 2.0 ** -4
    vnni = bool(case.flags & cases_mod().FLAG_VNNI_A)
    a_arr, b_arr = [], []
    for t in range(count):
        if vnni:
            f = 4 if i8 else 2
            at = np.broadcast_to(v[t][None, :, None], (k // f, m, f))
        else:
            at = np.zeros((k, case.lda)); at[:, :m] = v[t][None, :]
        bt = np.zeros((n, case.ldb)); bt[:, 0] = w[t]
        a_arr.append(at.reshape(-1)); b_arr.append(bt.reshape(-1))

    def enc(x, t):
        x = np.asarray(x, np.float64)
        if t == gen.F32:
            return x.astype(np.float32)
        if t == gen.BF16:
            return (x.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
        if t == gen.F16:
            return x.astype(np.float16).view(np.uint16)
        return x.astype(np.uint8 if t == gen.U8 else np.int8)
    b.a, b.b = dev(enc(np.concatenate(a_arr), case.ta)), dev(enc(np.concatenate(b_arr), case.tb))
    b.bias = enc(bias.reshape(-1), case.tc); b.d = dev(b.bias)
    ops.c0 = enc(c_old.reshape(-1), case.tc)
    scale = ops.scf if i8 else 1.0
    pre = v[:, :, None] * w[:, None, :] * scale                       # (count, m, n)
    seed = np.zeros_like(pre)
    beta0 = bool(case.flags & cases_mod().FLAG_BETA_0)
    if b.fuse[0]:
        seed += bias[:, :, None]
    if not beta0:
        seed += c_old[:, :, :m].transpose(0, 2, 1)
    return pre + seed, c_old


def cases_mod():
    import cases
    return cases


@pytest.mark.parametrize("types", FUSED_TYPES, ids=lambda t: "-".join(TNAME.get(x, str(x)) for x in t))
@pytest.mark.parametrize("bias", [0, 1], ids=["nobias", "bias"])
@pytest.mark.parametrize("beta0", [1, 0], ids=["beta0", "beta1"])
def test_fused_sigmoid(types, bias, beta0):
    """single calls, libxsmm_b200_gemm_ext_batch_strided and libxsmm_b200_gemm_ext_batch: every element of C within SIGMOID's window
    at its exact pre-activation, C's padding untouched, and the batch forms bit-identical to the single calls"""
    from test_gemm_ext_batch_gpu import Batch
    shape = (100, 37, 8, 0) if types[0] == gen.U8 else (101, 37, 8, 3)      # odd m: flat A for bf16 / f16; U8 takes VNNI4 A
    b = Batch(types, (bias, cases_mod().SIGMOID, 0, 0), beta0, 0, 1, shape, count=3, seed=17)
    a_exact, _ = fused_operands(b, np.random.default_rng(23 + 2 * bias + beta0))
    case, tc = b.case, types[3]
    m, n = case.m, case.n
    a32 = a_exact.astype(np.float32)
    assert np.array_equal(a32.astype(np.float64), a_exact)
    allowed = U.allowed("SIGMOID", a32.reshape(-1), tc)
    sc, _ = b.singles()
    got = host(sc, U.BITS[tc]).reshape(b.count, n, case.ldc)
    c0 = b.ops.c0.view(U.BITS[tc]).reshape(b.count, n, case.ldc)
    label = "fused SIGMOID %s bias=%d beta0=%d m=%d n=%d" % ("-".join(TNAME.get(x, str(x)) for x in types), bias, beta0, m, n)
    assert np.array_equal(got[:, :, m:], c0[:, :, m:]), label + ": C's ld padding was written"
    assert_in(allowed, got[:, :, :m].transpose(0, 2, 1).reshape(-1), a32.reshape(-1), label)
    for name, run in (("gemm_ext_batch_strided", b.strided), ("gemm_ext_batch", b.records)):
        c, _ = run()
        assert np.array_equal(host(c, np.uint8), host(sc, np.uint8)), label + ": " + name + " differs from the single calls"


# ---- matrix equations with transcendental nodes ----------------------------------------------------------------------------------
# Inputs on grids that make every value before the transcendental exact: a, b multiples of 2^-8 below 2^8 in magnitude (exact in f32;
# for bf16 arguments 8 significant bits), so a + b and x - rowmax(x) are exact. Ops compute in f32, the head stores the output type.
EM, EN = 45, 19                  # 45 rows: one full 32-row chunk and a partial one


def _grid(rng, shape, t):
    s = rng.integers(-255, 256, shape) * 2.0 ** rng.integers(-8, 1, shape)
    if t == gen.F32:
        s = s + rng.integers(-3, 4, shape) * 2.0 ** 4
    return s.astype(np.float32)


def _enc(x32, t):
    return x32 if t == gen.F32 else (x32.view(np.uint32) >> 16).astype(np.uint16)


def _eq_nodes(name, t):
    F32 = gen.F32
    if name == "chain":         # tanh(a + b) * c
        return ([("b", X.MELTW_TYPE_BINARY_MUL, F32, 0), ("u", X.MELTW_TYPE_UNARY_TANH, F32, 0), ("b", X.MELTW_TYPE_BINARY_ADD, F32, 0),
                 ("arg", 0, EM, EN, EM, t), ("arg", 1, EM, EN, EM, t), ("arg", 2, EM, EN, EM, t)], [(EM, EN)] * 3)
    if name == "ternary":       # a - exp(b) * c
        return ([("t", X.MELTW_TYPE_TERNARY_NMULADD, F32, 0), ("u", X.MELTW_TYPE_UNARY_EXP, F32, 0), ("arg", 1, EM, EN, EM, t),
                 ("arg", 0, EM, EN, EM, t), ("arg", 2, EM, EN, EM, t)], [(EM, EN)] * 3)
    if name == "gelu_bias":     # gelu(a + column broadcast)
        return ([("u", X.MELTW_TYPE_UNARY_GELU, F32, 0), ("b", X.MELTW_TYPE_BINARY_ADD, F32, X.MELTW_FLAG_BINARY_BCAST_COL_IN_1),
                 ("arg", 0, EM, EN, EM, t), ("arg", 1, EM, 1, EM, t)], [(EM, EN), (EM, 1)])
    # softmax numerator: exp(x - rowmax(x)), rowmax over the columns of each row
    return ([("u", X.MELTW_TYPE_UNARY_EXP, F32, 0), ("b", X.MELTW_TYPE_BINARY_SUB, F32, X.MELTW_FLAG_BINARY_BCAST_COL_IN_1),
             ("arg", 0, EM, EN, EM, t), ("u", X.MELTW_TYPE_UNARY_REDUCE_X_OP_MAX, F32, X.MELTW_FLAG_UNARY_REDUCE_COLS),
             ("arg", 0, EM, EN, EM, t)], [(EM, EN)])


def _eq_allowed(name, ins, tout):
    """candidates in the equation's f32 order; ins are the loaded f32 inputs as (rows, cols) arrays"""
    F = np.float32
    with np.errstate(all="ignore"):
        if name == "chain":
            x = (ins[0] + ins[1]).T.reshape(-1)
            c = U.libm_candidates("tanh", x) * ins[2].T.reshape(-1)[:, None]
        elif name == "ternary":
            x = ins[1].T.reshape(-1)
            c = ins[0].T.reshape(-1)[:, None] - U.libm_candidates("exp", x) * ins[2].T.reshape(-1)[:, None]
        elif name == "gelu_bias":
            x = (ins[0] + ins[1]).T.reshape(-1)
            c, nan = U.result_candidates("GELU", x)
            return U.Allowed(c, nan, tout), x
        else:
            x = (ins[0] - ins[0].max(axis=1, keepdims=True)).T.reshape(-1)
            c = U.libm_candidates("exp", x)
    return U.Allowed(c.astype(F), np.isnan(c).any(axis=1), tout), x


@pytest.mark.parametrize("t", [gen.F32, gen.BF16], ids=lambda t: TNAME[t])
@pytest.mark.parametrize("name", ["chain", "ternary", "gelu_bias", "softmax_numerator"])
def test_equation(name, t):
    """device pointers, host pointers and libxsmm_b200_meqn_batch_strided (bit-identical to the single calls)"""
    from test_meqn import build
    nodes, shapes = _eq_nodes(name, t)
    rng = np.random.default_rng(zlib.crc32(repr((name, t)).encode()))
    count = 3
    raw = [[_grid(rng, (c, r), t) for (r, c) in shapes] for _ in range(count)]           # stored column-major: (cols, rows)
    enc = [[_enc(x.reshape(-1), t) for x in tile] for tile in raw]
    loaded = [[U.load(e.view(U.BITS[t]) if t != gen.F32 else e.view(np.uint32), t).reshape(x.shape).T for e, x in zip(tile_e, tile_r)]
              for tile_e, tile_r in zip(enc, raw)]
    eq = build(nodes)
    k = X.libxsmm_dispatch_meqn(eq, X.MeqnArgShape(EM, EN, EM, t))
    assert k, name
    ot = U.BITS[t]
    label = "equation %s %s m=%d n=%d" % (name, TNAME[t], EM, EN)
    outs = []
    for tile in range(count):
        allowed, x = _eq_allowed(name, loaded[tile], t)
        for resident in (1, 0):
            args = (X.MatrixArg * len(shapes))()
            if resident:
                keep = [dev(e) for e in enc[tile]]
                d_out = dev(np.zeros(EM * EN, ot)); out_ptr = d_out.data_ptr()
                for i, d in enumerate(keep):
                    args[i].primary = d.data_ptr()
            else:
                keep = [np.ascontiguousarray(e) for e in enc[tile]]
                hout = np.zeros(EM * EN, ot); out_ptr = hout.ctypes.data
                for i, h in enumerate(keep):
                    args[i].primary = h.ctypes.data
            p = X.MeqnParam(); p.inputs = C.addressof(args); p.output.primary = out_ptr
            X.MEQN_FN(k)(C.byref(p)); X.check()
            got = host(d_out, ot) if resident else hout
            assert_in(allowed, got, x, label + (" device" if resident else " host"))
            if resident:
                outs.append(got)
    # the same tiles as one strided batch
    sizes = [e.nbytes for e in enc[0]]
    packed = [dev(np.concatenate([enc[tl][i] for tl in range(count)])) for i in range(len(shapes))]
    d_o = dev(np.zeros(count * EM * EN, ot))
    args = (X.MatrixArg * len(shapes))()
    for i, d in enumerate(packed):
        args[i].primary = d.data_ptr()
    p = X.MeqnParam(); p.inputs = C.addressof(args); p.output.primary = d_o.data_ptr()
    strides = (C.c_longlong * len(shapes))(*sizes)
    assert X.libxsmm_b200_meqn_batch_strided(k, C.byref(p), strides, EM * EN * np.dtype(ot).itemsize, 0, None, count) == 0
    X.check()
    assert np.array_equal(host(d_o, ot), np.concatenate(outs)), label + ": meqn_batch_strided differs from the single calls"



def test_zz_report():
    """per op and type pair: the share of elements equal to the glibc restatement's value, and the largest ordinal distance (in the
    output type) from the result with every libm call correctly rounded. The distance includes what the formula does to a one-ulp
    difference of a call: GELU at large negative x computes erf(x / sqrt 2) + 1 and ELU near zero expf(x) - 1; both cancel, so one
    ulp of the call there moves the output by many of its own ulps while staying inside the set."""
    if not REPORT:
        pytest.skip("no unary sweep ran in this session")
    print("\nop           in->out    elements  equal to glibc  max ordinal distance from correctly rounded")
    for (op, ti, to), (same, dist, n) in sorted(REPORT.items()):
        print("%-12s %-4s->%-4s %8d  %13.4f%%  %d" % (op, ti, to, n, 100.0 * same, dist))
