"""GPU: the matrix-eltwise kernels pinned element by element, and which kernel ran.

* Sums on exact operands: integers times 2^-e on one grid, chosen so that every partial sum -- squares included -- is exact in
  f32 (largest |partial| / grid < 2^24). Every element must equal the float64 value rounded once to the output type AND the CPU
  restatement (oracle/oracle_meltw.c, pinned to the reference in tests/test_oracle_meltw*.py), bit for bit.
* Sums on full-mantissa operands: |got - exact| <= (len + 2) 2^-24 sum|x| (sum x^2 for squares, |INIT_ACC value| included), plus one
  output rounding for BF16 / F16 outputs; doubled with 2^-53 for F64.
* Max / min / absmax and argop on the edge lines of meltw_edges.py: values and indices bit for bit against an independent Python
  fold with the reference's macros and against the restatement, NaN payloads included.
* Ops with no other GPU test (ZIP, REPLICATE_COL_VAR, every broadcast flag, compare with a broadcast input, F16 and mixed types):
  bit for bit, once on device buffers and once on pageable ones (the staging path), with the same bits from both.
* Every size- or alignment-dependent kernel choice is asserted through libxsmm_b200_meltw_variant on both sides of its threshold."""
import ctypes as C

import numpy as np
import pytest
import torch

import gen
import libxsmm_b200 as X
import meltw_edges as E
from gpu_util import dev, host
from oracle_ffi import iarr, oracle, ref

pytestmark = [pytest.mark.gpu]

UNS = gen.F64 + 26
U16, I16 = 11, 10
GENERIC, TRANSPOSE, VNNI, VNNI_VEC, WARP_REDUCE, COLS2, COLS2_VEC, OTHER = range(8)
IDX_FLAG = {4: X.MELTW_FLAG_UNARY_IDX_SIZE_4BYTES, 8: X.MELTW_FLAG_UNARY_IDX_SIZE_8BYTES}
SENT = 0xA5


def checker():
    """the reference where it travelled with the tree, else the pinned restatement"""
    return ref if ref is not None else oracle


def same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def unary_param(x, out, aux=None, idx=None, count=None, nrt=None, keep=None):
    p = X.MeltwUnaryParam(); p.inp.primary, p.out.primary = x, out
    if aux is not None:
        p.out.secondary = aux
    if idx is not None:
        c = C.c_ulonglong(count); keep.append(c); p.inp.secondary, p.inp.tertiary = idx, C.addressof(c)
    if nrt is not None:
        c = C.c_ulonglong(nrt); keep.append(c); p.op.primary = C.addressof(c)
    return p


def cpu_unary(side, desc, x, out0, aux0=None, idx=None, count=None, nrt=None):
    out = out0.copy(); aux = None if aux0 is None else aux0.copy(); keep = []
    p = unary_param(x.ctypes.data, out.ctypes.data, None if aux is None else aux.ctypes.data, None if idx is None else idx.ctypes.data, count, nrt, keep)
    assert side["meltw"](iarr(*desc), C.addressof(p), 0) == 0, desc
    return out, aux


def gpu_unary(k, x, out0, aux0=None, idx=None, count=None, nrt=None, x_offset=0, variant=None, pageable=False):
    """run handle k once; x / out0 / aux0 numpy arrays (copied to the device unless pageable); returns (out, aux) as numpy"""
    keep = []
    if pageable:
        out = out0.copy(); aux = None if aux0 is None else aux0.copy()
        p = unary_param(x.ctypes.data + x_offset, out.ctypes.data, None if aux is None else aux.ctypes.data,
                        None if idx is None else idx.ctypes.data, count, nrt, keep)
    else:
        d_x, d_o = dev(x), dev(out0); d_a = None if aux0 is None else dev(aux0); d_i = None if idx is None else dev(idx)
        keep += [d_x, d_o, d_a, d_i]
        p = unary_param(d_x.data_ptr() + x_offset, d_o.data_ptr(), None if d_a is None else d_a.data_ptr(),
                        None if d_i is None else d_i.data_ptr(), count, nrt, keep)
    if variant is not None:
        assert X.libxsmm_b200_meltw_variant(k, C.addressof(p)) == variant, (X.libxsmm_b200_meltw_variant(k, C.addressof(p)), variant)
    X.MELTW_UNARY_FN(k)(C.byref(p)); X.check()
    if pageable:
        return out, aux
    return host(d_o, out0.dtype), (None if d_a is None else host(d_a, aux0.dtype))


def rne_out(v32, t):
    """f32 values -> output bits of type t (one rounding)"""
    v32 = np.asarray(v32, dtype=np.float32)
    if t == gen.F32:
        return v32.copy()
    if t == gen.BF16:
        return np.array([oracle["f32_to_bf16"](float(v)) for v in v32], dtype=np.uint16)
    return np.array([oracle["f32_to_f16"](float(v)) for v in v32], dtype=np.uint16)


# ---------------------------------------------------------------------------------------------------------------------------------
# sums
def grid_ints(rng, size, t, len_):
    """integers k with len_ * k^2 < 2^22 (so x and x^2 sums stay exact in f32 with room for INIT_ACC), representable in type t"""
    lim = max(1, int(np.sqrt((1 << 22) / max(len_, 1))))
    lim = min(lim, {gen.BF16: 255, gen.F16: 2047}.get(t, 1 << 11))
    return rng.integers(-lim, lim + 1, size=size).astype(np.float64)


def to_type(v64, t):
    if t == gen.F64:
        return v64.astype(np.float64)
    if t == gen.F32:
        return v64.astype(np.float32)
    if t == gen.BF16:
        return gen.f32_to_bf16_bits(v64.astype(np.float32))
    return v64.astype(np.float16).view(np.uint16)


SUM_OPS = ("X_OP_ADD", "X2_OP_ADD", "X_X2_OP_ADD")
# (m, n, ldi pad, x offset in elements, rows?, expected variant for an F32 input)
SUM_SHAPES = [
    (33, 17, 0, 0, 1, WARP_REDUCE), (33, 17, 2, 0, 0, WARP_REDUCE), (1, 70, 0, 0, 0, WARP_REDUCE), (70, 1, 1, 0, 1, WARP_REDUCE),
    (255, 1100, 0, 0, 0, WARP_REDUCE),                      # m = 255: below the two-phase threshold though m*n >= 2^18
    (256, 1100, 0, 0, 0, COLS2_VEC),                        # m = 256
    (513, 511, 3, 0, 0, WARP_REDUCE),                       # m*n = 2^18 - 1
    (512, 512, 0, 0, 0, COLS2_VEC),                         # m*n = 2^18
    (16384, 16, 0, 0, 0, COLS2_VEC),                        # n < 32: one slice
    (256, 8192, 0, 0, 0, COLS2_VEC),                        # 256 slices of 32 columns
    (256, 8000, 0, 0, 0, COLS2_VEC),                        # 256 slices, ragged last ones
    (258, 1024, 2, 0, 0, COLS2),                            # m % 4 != 0: scalar partial pass
    (256, 1024, 2, 0, 0, COLS2),                            # ldi % 4 != 0
    (256, 1024, 0, 1, 0, COLS2),                            # in0 4 bytes off 16-byte alignment
    (300, 2000, 5, 0, 1, WARP_REDUCE),                      # rows
]


def exact_sum_case(rng, t_in, t_out, op, m, n, pad, xoff, rows, init, want_variant):
    ldi = m + pad
    ldo = n if rows else m + 3                            # ldo > m: the x^2 plane of a column reduction sits at ldo
    len_ = m if rows else n
    e = 6
    xv = grid_ints(rng, ldi * n + xoff, t_in, len_) * 2.0 ** -e
    x = to_type(xv, t_in)
    xm = gen.to_f64(x, t_in)[xoff:].reshape(n, ldi)[:, :m]
    nres = n if rows else m
    res_size = n if rows else ldo
    planes = 2 if op == "X_X2_OP_ADD" else 1
    o64 = (rng.integers(-64, 65, size=res_size * planes) * 2.0 ** (-2 * e)) if init else np.zeros(res_size * planes)
    out0 = to_type(o64, t_out)
    if not init:
        out0 = np.frombuffer(np.full(out0.nbytes, SENT, dtype=np.uint8).tobytes(), dtype=out0.dtype).copy()
    o0 = gen.to_f64(out0, t_out)
    ax = 1 if rows else 0                                 # xm[j, i]: rows collapse i, columns collapse j
    sx, sq = xm.sum(axis=ax), (xm * xm).sum(axis=ax)
    want = out0.copy()
    plane_x = 0 if op != "X2_OP_ADD" else None
    plane_q = res_size if op == "X_X2_OP_ADD" else (0 if op == "X2_OP_ADD" else None)
    for base, s in ((plane_x, sx), (plane_q, sq)):
        if base is None:
            continue
        v = s + (o0[base:base + nres] if init else 0.0)
        assert np.all(np.abs(v) < 2.0 ** (24 - 2 * e)), "operands not exact"
        want[base:base + nres] = v.astype(np.float64) if t_out == gen.F64 else rne_out(v, t_out)
    flags = (X.MELTW_FLAG_UNARY_REDUCE_ROWS if rows else X.MELTW_FLAG_UNARY_REDUCE_COLS) | (X.MELTW_FLAG_UNARY_REDUCE_INIT_ACC if init else 0)
    opc = getattr(X, "MELTW_TYPE_UNARY_REDUCE_" + op)
    tcomp = gen.F64 if t_in == gen.F64 else gen.F32
    k = X.libxsmm_dispatch_meltw_unary(opc, X.libxsmm_create_meltw_unary_shape(m, n, ldi, ldo, t_in, t_out, tcomp), flags)
    assert k
    got, _ = gpu_unary(k, x, out0, x_offset=xoff * gen.TS[t_in], variant=want_variant)
    what = (op, t_in, t_out, m, n, pad, xoff, rows, init)
    assert same(got, want), what
    # the restatement on the same operands (result rows only: the reference also stores its scratch for rows m..ldo-1)
    cpu, _ = cpu_unary(oracle, (1, opc, flags, m, n, ldi, 0, 0, ldo, t_in, UNS, UNS, t_out, tcomp), np.ascontiguousarray(x[xoff:]), out0)
    for base in (b for b in (plane_x, plane_q) if b is not None):
        assert same(got[base:base + nres], cpu[base:base + nres]), what + ("oracle",)
    return got


def sum_variant(t_in, want):
    """the variant the shape table names for F32 input, for another input type"""
    if t_in == gen.F32:
        return want
    if want in (COLS2, COLS2_VEC):
        return WARP_REDUCE if t_in == gen.F64 else COLS2
    return want


@pytest.mark.parametrize("t_in,t_out", [(gen.F32, gen.F32), (gen.F32, gen.BF16), (gen.BF16, gen.BF16), (gen.F16, gen.F32), (gen.F64, gen.F64)])
def test_exact_sums_every_reduction_kernel(t_in, t_out):
    rng = np.random.default_rng(101)
    seen = set()
    for (m, n, pad, xoff, rows, var) in SUM_SHAPES:
        if t_in != gen.F32 and (m * n > 600000 or xoff):
            continue
        for op in SUM_OPS:
            if t_in == gen.F64 and "X2" in op:
                continue       # the reference's F64 path never stores the sums of squares (:1150-1153, :1291): no contract
            for init in (0, 1):
                if m * n > 600000 and (init or op != "X_X2_OP_ADD"):
                    continue
                v = sum_variant(t_in, var)
                exact_sum_case(rng, t_in, t_out, op, m, n, pad, xoff, rows, init, v)
                seen.add(v)
    if t_in == gen.F32:
        assert seen == {WARP_REDUCE, COLS2, COLS2_VEC}, seen


@pytest.mark.parametrize("t_in,t_out", [(gen.F32, gen.F32), (gen.F32, gen.BF16), (gen.BF16, gen.F32), (gen.F16, gen.F16), (gen.F64, gen.F64)])
def test_full_mantissa_sums_within_bound(t_in, t_out):
    rng = np.random.default_rng(102)
    u = 2.0 ** -53 if t_in == gen.F64 else 2.0 ** -24
    out_u = {gen.BF16: 2.0 ** -8, gen.F16: 2.0 ** -11}.get(t_out, 0.0)
    worst = 0.0
    for (m, n, pad, xoff, rows, var) in SUM_SHAPES:
        if m * n > 600000 or (xoff and t_in != gen.F32):
            continue
        ldi, ldo = m + pad, (n if rows else m + 3)
        res_size = n if rows else ldo
        nres, len_ = (n, m) if rows else (m, n)
        x = to_type(rng.standard_normal(ldi * n + xoff) * np.exp2(rng.integers(-3, 4, size=ldi * n + xoff)), t_in)
        xm = gen.to_f64(x, t_in)[xoff:].reshape(n, ldi)[:, :m]
        for op in SUM_OPS:
            if t_in == gen.F64 and "X2" in op:
                continue
            for init in (0, 1):
                out0 = to_type(rng.standard_normal(2 * res_size), t_out)
                o0 = gen.to_f64(out0, t_out)
                flags = (X.MELTW_FLAG_UNARY_REDUCE_ROWS if rows else X.MELTW_FLAG_UNARY_REDUCE_COLS) | (X.MELTW_FLAG_UNARY_REDUCE_INIT_ACC if init else 0)
                k = X.libxsmm_dispatch_meltw_unary(getattr(X, "MELTW_TYPE_UNARY_REDUCE_" + op),
                                                   X.libxsmm_create_meltw_unary_shape(m, n, ldi, ldo, t_in, t_out, gen.F64 if t_in == gen.F64 else gen.F32), flags)
                got, _ = gpu_unary(k, x, out0, x_offset=xoff * gen.TS[t_in], variant=sum_variant(t_in, var))
                g = gen.to_f64(got, t_out)
                planes = []
                if op != "X2_OP_ADD":
                    planes.append((0, xm))
                if op != "X_OP_ADD":
                    planes.append((res_size if op == "X_X2_OP_ADD" else 0, xm * xm))
                for base, vals in planes:
                    ax = 1 if rows else 0
                    ex = vals.sum(axis=ax) + (o0[base:base + nres] if init else 0.0)
                    mag = np.abs(vals).sum(axis=ax) + (np.abs(o0[base:base + nres]) if init else 0.0)
                    bsum = (len_ + 2 + init) * u * mag * (2.0 if t_in == gen.F64 else 1.0)
                    bound = bsum + out_u * (np.abs(ex) + bsum)
                    err = np.abs(g[base:base + nres] - ex)
                    assert np.all(err <= bound), (op, m, n, rows, init, float(np.max(err / np.maximum(bound, 1e-300))))
                    worst = max(worst, float(np.max(err / np.maximum(bound, 1e-300))))
    print("largest err / bound: %.3f" % worst)


@pytest.mark.parametrize("t", [gen.F32, gen.BF16, gen.F64])
def test_exact_reduce_to_scalar_and_dot(t):
    rng = np.random.default_rng(103)
    tcomp = gen.F64 if t == gen.F64 else gen.F32
    for (m, n, ld) in ((37, 11, 40), (1, 1, 1), (1000, 300, 1001)):
        a64 = rng.integers(-5, 6, size=ld * n) * 2.0 ** -4      # sum |a b| / 2^-8 < 2^24: every partial sum of the dot is exact
        b64 = rng.integers(-5, 6, size=ld * n) * 2.0 ** -4
        a, b = to_type(a64, t), to_type(b64, t)
        am, bm = gen.to_f64(a, t).reshape(n, ld)[:, :m], gen.to_f64(b, t).reshape(n, ld)[:, :m]
        for name, exact in (("unary", am.sum()), ("dot", (am * bm).sum())):
            want = np.array([exact]) if t == gen.F64 else rne_out([exact], t)
            assert abs(exact) < 2.0 ** 16
            y0 = to_type(np.array([7.0]), t)
            if name == "unary":
                k = X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_REDUCE_TO_SCALAR_OP_ADD, X.libxsmm_create_meltw_unary_shape(m, n, ld, ld, t, t, tcomp), 0)
                got, _ = gpu_unary(k, a, y0, variant=OTHER)
                cpu, _ = cpu_unary(oracle, (1, X.MELTW_TYPE_UNARY_REDUCE_TO_SCALAR_OP_ADD, 0, m, n, ld, 0, 0, ld, t, UNS, UNS, t, tcomp), a, y0)
            else:
                k = X.libxsmm_dispatch_meltw_binary(X.MELTW_TYPE_BINARY_MUL_AND_REDUCE_TO_SCALAR_OP_ADD, X.libxsmm_create_meltw_binary_shape(m, n, ld, ld, ld, t, t, t, tcomp), 0)
                d_a, d_b, d_y = dev(a), dev(b), dev(y0)
                p = X.MeltwBinaryParam(); p.in0.primary, p.in1.primary, p.out.primary = d_a.data_ptr(), d_b.data_ptr(), d_y.data_ptr()
                X.MELTW_BINARY_FN(k)(C.byref(p)); X.check()
                got = host(d_y, y0.dtype)
                cpu = y0.copy(); q = X.MeltwBinaryParam(); q.in0.primary, q.in1.primary, q.out.primary = a.ctypes.data, b.ctypes.data, cpu.ctypes.data
                assert oracle["meltw"](iarr(2, X.MELTW_TYPE_BINARY_MUL_AND_REDUCE_TO_SCALAR_OP_ADD, 0, m, n, ld, ld, 0, ld, t, t, UNS, t, tcomp), C.addressof(q), 0) == 0
            assert same(got, want), (name, t, m, n)
            assert same(got, cpu), (name, t, m, n, "oracle")


# ---------------------------------------------------------------------------------------------------------------------------------
# max / min / absmax / argop
def load32(bits, t):
    if t == gen.F64:
        return bits.view(np.float64)
    if t == gen.F32:
        return bits.view(np.float32)
    if t == gen.BF16:
        return (bits.astype(np.uint32) << 16).view(np.float32)
    return bits.view(np.float16).astype(np.float32)    # f16 -> f32 keeps NaN-ness; payload checked against the restatement below


def fold_line(vals, kind, rows, argop, is64):
    """the reference's loop (:1215-1428) with LIBXSMM_MAX / MIN / ABS, on numpy scalars; returns (value, index or None)"""
    MAX = lambda a, b: b if a < b else a          # noqa: E731
    MIN = lambda a, b: a if a < b else b          # noqa: E731
    ABS = lambda a: a if 0 <= a else -a           # noqa: E731
    ft = np.float64 if is64 else np.float32
    if rows:
        tmp = vals[0]
        for v in vals:
            tmp = MAX(tmp, v) if kind == "MAX" else (MAX(ABS(tmp), ABS(v)) if kind == "ABSMAX" else MIN(tmp, v))
        return tmp, None
    tmp = ft(-E.FLT_MAX) if kind == "MAX" else (ft(0) if kind == "ABSMAX" else ft(E.FLT_MAX))
    arg = None
    for j, v in enumerate(vals):
        if kind == "ABSMAX":
            v = ABS(v)
        if argop:
            if (v <= tmp) if kind == "MIN" else (v >= tmp):
                tmp, arg = v, j
        else:
            tmp = MIN(v, tmp) if kind == "MIN" else MAX(v, tmp)
    return tmp, arg


def out_bits(vals, t_out, t_in):
    if t_out == gen.F64:
        return np.asarray(vals, dtype=np.float64)
    v = np.asarray(vals, dtype=np.float32)
    return v.copy() if t_out == gen.F32 else rne_out(v, t_out)


@pytest.mark.parametrize("t_in,t_out", [(gen.F32, gen.F32), (gen.F32, gen.BF16), (gen.BF16, gen.BF16), (gen.F16, gen.F16), (gen.F16, gen.F32), (gen.F64, gen.F64)])
def test_max_min_absmax_argop_bit_exact(t_in, t_out):
    rng = np.random.default_rng(104)
    tcomp = gen.F64 if t_in == gen.F64 else gen.F32
    np_out = E.BITS_OF[t_out] if t_out != gen.F32 else np.uint32
    with np.errstate(invalid="ignore", over="ignore"):
        for L in (1, 3, 37, 70, 129):
            bits = E.encode(E.sequences(rng, L), t_in)
            for rows in (1, 0):
                x, m, n, ldi = E.layout(bits, rows, 3, E.NAN_BITS[t_in][2])
                nres = n if rows else m
                for kind in ("MAX", "MIN", "ABSMAX"):
                    for isz in ((0,) if rows else (0, 4, 8)):
                        flags = (X.MELTW_FLAG_UNARY_REDUCE_ROWS if rows else X.MELTW_FLAG_UNARY_REDUCE_COLS)
                        if isz:
                            flags |= X.MELTW_FLAG_UNARY_REDUCE_RECORD_ARGOP | IDX_FLAG[isz]
                        op = getattr(X, "MELTW_TYPE_UNARY_REDUCE_X_OP_" + kind)
                        k = X.libxsmm_dispatch_meltw_unary(op, X.libxsmm_create_meltw_unary_shape(m, n, ldi, nres, t_in, t_out, tcomp), flags)
                        assert k
                        out0 = np.full(nres, 0, dtype=np_out); out0.view(np.uint8)[:] = SENT
                        aux0 = np.full(nres * max(isz, 1), SENT, dtype=np.uint8)
                        got, gaux = gpu_unary(k, x, out0, aux0 if isz else None, variant=WARP_REDUCE)
                        # independent fold
                        lines = load32(bits, t_in)
                        want_v, want_i = zip(*(fold_line(list(lines[r]), kind, rows, isz, t_in == gen.F64) for r in range(nres)))
                        want = out_bits(want_v, t_out, t_in).view(np_out)
                        what = (kind, rows, isz, L, t_in, t_out)
                        if t_in in (gen.F32, gen.F64) and t_out == t_in:
                            assert same(got, want), what
                        else:     # through a conversion: NaN <-> NaN, everything else bit for bit
                            gw = gen.to_f64(got.view(gen.NP_OF[t_out]), t_out); ww = gen.to_f64(want.view(gen.NP_OF[t_out]), t_out)
                            nan = np.isnan(ww)
                            assert np.array_equal(np.isnan(gw), nan) and same(got[~nan], want[~nan]), what
                        cpu, caux = cpu_unary(checker(), (1, op, flags, m, n, ldi, 0, 0, nres, t_in, UNS, UNS, t_out, tcomp), x, out0, aux0 if isz else None)
                        assert same(got, cpu), what + ("restatement",)
                        if isz:
                            idx = gaux.view(np.uint32 if isz == 4 else np.uint64)
                            untouched = np.frombuffer(bytes([SENT]) * isz, dtype=idx.dtype)[0]
                            want_idx = np.array([untouched if i is None else i for i in want_i], dtype=idx.dtype)
                            assert np.array_equal(idx, want_idx), what + ("argop",)
                            assert same(gaux, caux), what + ("argop restatement",)


@pytest.mark.parametrize("t_in,t_out", [(gen.F32, gen.F32), (gen.BF16, gen.F32), (gen.F64, gen.F64)])
def test_cols_idx_reductions_and_pageable_argop(t_in, t_out):
    """REDUCE_COLS_IDX_OP_{ADD,MAX,MIN} with duplicated / unsorted lists and a list of one; the argop buffer of MAX / MIN also as
    pageable memory (staged in and out) -- in and out of the data stay device-resident, as the indexed ops require"""
    rng = np.random.default_rng(105)
    tcomp = gen.F64 if t_in == gen.F64 else gen.F32
    L = 45
    bits = E.encode(E.sequences(rng, L), t_in)
    x, m, n, ldi = E.layout(bits, 0, 2, E.NAN_BITS[t_in][0])
    np_out = np.uint64 if t_out == gen.F64 else np.uint32
    lists = [rng.integers(0, n, size=80), np.array([L - 1]), np.array([5, 5, 5]), rng.permutation(n)[:19]]
    d_x = dev(x)
    for name in ("ADD", "MAX", "MIN"):
        op = getattr(X, "MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_" + name)
        for cols in lists:
            for isz in (4, 8):
                for argop in ((0, 1) if name != "ADD" else (0,)):
                    if name == "ADD":       # sums: finite exact operands
                        xa = to_type(rng.integers(-40, 41, size=ldi * n) * 0.25, t_in); d_xa = dev(xa)
                    else:
                        xa, d_xa = x, d_x
                    idx = cols.astype(np.uint32 if isz == 4 else np.uint64)
                    flags = X.MELTW_FLAG_UNARY_REDUCE_COLS | IDX_FLAG[isz] | (X.MELTW_FLAG_UNARY_REDUCE_RECORD_ARGOP if argop else 0)
                    k = X.libxsmm_dispatch_meltw_unary(op, X.libxsmm_create_meltw_unary_shape(m, n, ldi, m, t_in, t_out, tcomp), flags)
                    assert k
                    out0 = np.zeros(m, dtype=np_out); out0.view(np.uint8)[:] = SENT
                    aux0 = np.full(m * isz, SENT, dtype=np.uint8)
                    cpu, caux = cpu_unary(checker(), (1, op, flags, m, n, ldi, 0, 0, m, t_in, UNS, UNS, t_out, tcomp), xa, out0, aux0, idx=idx, count=len(idx))
                    for pageable_aux in ((0, 1) if argop else (0,)):
                        d_o, d_i = dev(out0), dev(idx)
                        aux = aux0.copy(); d_aux = dev(aux0)
                        keep = []
                        p = unary_param(d_xa.data_ptr(), d_o.data_ptr(), aux.ctypes.data if pageable_aux else d_aux.data_ptr(), idx.ctypes.data if pageable_aux else d_i.data_ptr(), len(idx), None, keep)
                        assert X.libxsmm_b200_meltw_variant(k, C.addressof(p)) == WARP_REDUCE
                        X.MELTW_UNARY_FN(k)(C.byref(p)); X.check()
                        got = host(d_o, np_out)
                        gaux = aux if pageable_aux else host(d_aux, np.uint8)
                        what = (name, len(idx), isz, argop, pageable_aux)
                        assert same(got, cpu), what
                        if argop:
                            assert same(gaux, caux), what + ("argop",)
                    if name == "ADD":
                        xm = gen.to_f64(xa, t_in).reshape(n, ldi)[:, :m]
                        ex = xm[cols, :].sum(axis=0)
                        assert same(got, ex.astype(np.float64) if t_out == gen.F64 else ex.astype(np.float32)), what


# ---------------------------------------------------------------------------------------------------------------------------------
# element-wise ops with no other GPU test
def run_binary_both(k, desc, ins, out0, t_out):
    """device run, pageable run and the CPU checker; all three must give the same bits"""
    results = []
    for pageable in (0, 1):
        keep = []
        if pageable:
            bufs = [np.ascontiguousarray(a) for a in ins]; out = out0.copy(); ptrs = [b.ctypes.data for b in bufs]; optr = out.ctypes.data
        else:
            bufs = [dev(a) for a in ins]; d_o = dev(out0); ptrs = [b.data_ptr() for b in bufs]; optr = d_o.data_ptr()
        keep += bufs
        if len(ins) == 2:
            p = X.MeltwBinaryParam(); p.in0.primary, p.in1.primary, p.out.primary = ptrs[0], ptrs[1], optr
            X.MELTW_BINARY_FN(k)(C.byref(p))
        else:
            p = X.MeltwTernaryParam(); p.in0.primary, p.in1.primary, p.in2.primary, p.out.primary = ptrs[0], ptrs[1], ptrs[2], optr
            X.MELTW_TERNARY_FN(k)(C.byref(p))
        X.check()
        results.append(out if pageable else host(d_o, out0.dtype))
    want = out0.copy()
    if len(ins) == 2:
        q = X.MeltwBinaryParam(); q.in0.primary, q.in1.primary, q.out.primary = ins[0].ctypes.data, ins[1].ctypes.data, want.ctypes.data
    else:
        q = X.MeltwTernaryParam(); q.in0.primary, q.in1.primary, q.in2.primary, q.out.primary = ins[0].ctypes.data, ins[1].ctypes.data, ins[2].ctypes.data, want.ctypes.data
    assert checker()["meltw"](iarr(*desc), C.addressof(q), 0) == 0, desc
    assert same(results[0], results[1]), (desc, "device vs pageable")
    assert same(results[0], want), desc
    return results[0]


def operand(rng, t, size):
    if t in (U16, I16):
        return rng.integers(0, 1 << 16, size=size, dtype=np.uint16)
    return to_type(rng.integers(1, 64, size=size) * rng.choice([-1.0, 1.0], size=size) / 16, t)     # no zero: DIV stays finite


BIN_BCAST = {"ROW_IN_0": X.MELTW_FLAG_BINARY_BCAST_ROW_IN_0, "ROW_IN_1": X.MELTW_FLAG_BINARY_BCAST_ROW_IN_1,
             "COL_IN_0": X.MELTW_FLAG_BINARY_BCAST_COL_IN_0, "COL_IN_1": X.MELTW_FLAG_BINARY_BCAST_COL_IN_1,
             "SCALAR_IN_0": X.MELTW_FLAG_BINARY_BCAST_SCALAR_IN_0, "SCALAR_IN_1": X.MELTW_FLAG_BINARY_BCAST_SCALAR_IN_1}


def test_zip_broadcasts_compares_and_mixed_types():
    rng = np.random.default_rng(106)
    m, n, pad = 37, 13, 3
    ld = m + pad
    # ZIP: two 16-bit planes into one 32-bit word, in1 the high half
    for t in (U16, gen.BF16, I16):
        for fl in (0,) + tuple(BIN_BCAST.values()):
            a, b = operand(rng, t, ld * n), operand(rng, t, ld * n)
            out0 = np.full((ld * n), 0xDEADBEEF, dtype=np.uint32)
            k = X.libxsmm_dispatch_meltw_binary(X.MELTW_TYPE_BINARY_ZIP, X.libxsmm_create_meltw_binary_shape(m, n, ld, ld, ld, t, t, gen.F32, gen.F32), fl)
            assert k, t
            got = run_binary_both(k, (2, X.MELTW_TYPE_BINARY_ZIP, fl, m, n, ld, ld, 0, ld, t, t, UNS, gen.F32, gen.F32), [a, b], out0, gen.F32)
            if fl == 0:
                am, bm = a.reshape(n, ld)[:, :m].astype(np.uint32), b.reshape(n, ld)[:, :m].astype(np.uint32)
                assert np.array_equal(got.reshape(n, ld)[:, :m], am | (bm << 16))
    # every binary broadcast flag, arithmetic and compares, in f32 / f16 / mixed types
    for (t0, t1, to) in ((gen.F32, gen.F32, gen.F32), (gen.F16, gen.F16, gen.F16), (gen.BF16, gen.F32, gen.F16), (gen.F32, gen.BF16, gen.BF16), (gen.F16, gen.BF16, gen.F32)):
        for fname, fl in (("NONE", 0),) + tuple(BIN_BCAST.items()):
            a, b = operand(rng, t0, ld * n), operand(rng, t1, ld * n)
            for name in ("ADD", "SUB", "MUL", "DIV", "MULADD", "MAX", "MIN", "CMP_OP_GT", "CMP_OP_GE", "CMP_OP_LT", "CMP_OP_LE", "CMP_OP_EQ", "CMP_OP_NE"):
                op = getattr(X, "MELTW_TYPE_BINARY_" + name)
                cmp_ = name.startswith("CMP")
                if cmp_ and fname == "NONE" and to != t0:
                    continue
                out0 = (np.full((ld + 15) // 16 * 2 * n, SENT, dtype=np.uint8) if cmp_ else operand(rng, to, ld * n))
                flags = fl | (X.MELTW_FLAG_BINARY_BITMASK_2BYTEMULT if cmp_ else 0)
                k = X.libxsmm_dispatch_meltw_binary(op, X.libxsmm_create_meltw_binary_shape(m, n, ld, ld, ld, t0, t1, to, gen.F32), flags)
                assert k, (name, fname, t0, t1, to)
                got = run_binary_both(k, (2, op, flags, m, n, ld, ld, 0, ld, t0, t1, UNS, to, gen.F32), [a, b], out0, to)
                if name in ("ADD", "MUL") and to == gen.F32 and fname == "NONE":   # independent: one IEEE f32 operation per element
                    x0 = load32(a, t0).reshape(n, ld)[:, :m]; x1 = load32(b, t1).reshape(n, ld)[:, :m]
                    ex = (x0 + x1) if name == "ADD" else (x0 * x1)
                    assert same(got.reshape(n, ld)[:, :m], ex.astype(np.float32)), (name, t0, t1)


TER_BCAST = {"%s_IN_%d" % (kind, w): getattr(X, "MELTW_FLAG_TERNARY_BCAST_%s_IN_%d" % (kind, w)) for kind in ("ROW", "COL", "SCALAR") for w in (0, 1, 2)}


def test_ternary_every_broadcast_and_mixed_types():
    rng = np.random.default_rng(107)
    m, n, pad = 37, 11, 2
    ld = m + pad
    for (t0, t1, t2, to) in ((gen.F32, gen.F32, gen.F32, gen.F32), (gen.F16, gen.F16, gen.F16, gen.F16), (gen.BF16, gen.F32, gen.F16, gen.F32),
                             (gen.F32, gen.BF16, gen.F32, gen.BF16)):
        for fname, fl in (("NONE", 0),) + tuple(TER_BCAST.items()):
            for name in ("MULADD", "NMULADD", "SELECT"):
                if name == "SELECT" and fname.endswith("_2"):
                    continue        # in2 of SELECT is the bit mask, addressed by its own pitch (:2620)
                op = getattr(X, "MELTW_TYPE_TERNARY_" + name)
                a, b = operand(rng, t0, ld * n), operand(rng, t1, ld * n)
                c3 = rng.integers(0, 256, size=(ld + 15) // 16 * 2 * n, dtype=np.uint8) if name == "SELECT" else operand(rng, t2, ld * n)
                tt2 = t0 if name == "SELECT" else t2
                flags = fl | (X.MELTW_FLAG_TERNARY_BITMASK_2BYTEMULT if name == "SELECT" else 0)
                out0 = operand(rng, to, ld * n)
                k = X.libxsmm_dispatch_meltw_ternary(op, X.libxsmm_create_meltw_ternary_shape(m, n, ld, ld, ld, ld, t0, t1, tt2, to, gen.F32), flags)
                assert k, (name, fname)
                got = run_binary_both(k, (3, op, flags, m, n, ld, ld, ld, ld, t0, t1, tt2, to, gen.F32), [a, b, c3], out0, to)
                if name == "MULADD" and fname == "NONE" and to == gen.F32:      # in2 + in0*in1, two f32 roundings
                    x, y, z = (load32(v, t).reshape(n, ld)[:, :m] for v, t in ((a, t0), (b, t1), (c3, t2)))
                    assert same(got.reshape(n, ld)[:, :m], (z + (x * y).astype(np.float32)).astype(np.float32))


def test_replicate_col_var():
    rng = np.random.default_rng(108)
    for (tin, tout) in ((gen.F32, gen.F32), (gen.BF16, gen.F32), (gen.F32, gen.BF16), (gen.F16, gen.F16)):
        for (m, nrt, ldo) in ((1, 1, 1), (37, 5, 40), (64, 200, 64)):
            x = operand(rng, tin, m)
            out0 = operand(rng, tout, ldo * nrt + 8)
            k = X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_REPLICATE_COL_VAR, X.libxsmm_create_meltw_unary_shape(m, 1, m, ldo, tin, tout, gen.F32), 0)
            assert k
            want, _ = cpu_unary(checker(), (1, X.MELTW_TYPE_UNARY_REPLICATE_COL_VAR, 0, m, 1, m, 0, 0, ldo, tin, UNS, UNS, tout, gen.F32), x, out0, nrt=nrt)
            for pageable in (0, 1):
                got, _ = gpu_unary(k, x, out0, nrt=nrt, pageable=pageable, variant=OTHER)
                assert same(got, want), (tin, tout, m, nrt, pageable)
            if tin == tout:
                col = got[: ldo * nrt].reshape(nrt, ldo)[:, :m]
                assert np.array_equal(col, np.broadcast_to(x, (nrt, m)))


# ---------------------------------------------------------------------------------------------------------------------------------
# data movement: the kernel choice on both sides of every threshold
def test_transpose_boundaries():
    rng = np.random.default_rng(109)
    for (m, n, var) in ((63, 65, GENERIC), (64, 64, TRANSPOSE), (1, 5000, TRANSPOSE), (5000, 1, TRANSPOSE), (128, 192, TRANSPOSE), (1, 4095, GENERIC), (4096, 1, TRANSPOSE)):
        for t, npdt in ((gen.F32, np.uint32), (gen.BF16, np.uint16), (gen.F64, np.uint64), (gen.I8, np.uint8)):
            ldi, ldo = m + 1, n + 2
            x = rng.integers(0, np.iinfo(npdt).max, size=ldi * n, dtype=npdt)
            out0 = np.full(ldo * m, 7, dtype=npdt)
            k = X.libxsmm_dispatch_meltw_unary(X.MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT, X.libxsmm_create_meltw_unary_shape(m, n, ldi, ldo, t, t, t), 0)
            got, _ = gpu_unary(k, x, out0, variant=var)
            want = out0.copy().reshape(m, ldo); want[:, :n] = x.reshape(n, ldi)[:, :m].T
            assert np.array_equal(got, want.reshape(-1)), (m, n, t)


def test_vnni_pack_boundaries():
    rng = np.random.default_rng(110)
    cases_ = [  # (op, t, npdt, m, n, ldi, ldo, x byte offset, variant)
        ("NORM_TO_VNNI2", gen.BF16, np.uint16, 64, 67, 64, 72, 0, VNNI_VEC),       # odd n, ldo > m
        ("NORM_TO_VNNI2_PAD", gen.BF16, np.uint16, 64, 67, 64, 72, 0, VNNI_VEC),
        ("NORM_TO_VNNI2", gen.BF16, np.uint16, 64, 67, 64, 72, 2, VNNI),           # misaligned base: scalar packer
        ("NORM_TO_VNNI2", gen.BF16, np.uint16, 60, 70, 60, 64, 0, VNNI),           # m % 8 != 0
        ("NORM_TO_VNNI2", gen.BF16, np.uint16, 48, 63, 48, 64, 0, GENERIC),        # ldo * n = 4032 < 4096
        ("NORM_TO_VNNI2", gen.BF16, np.uint16, 64, 64, 64, 64, 0, VNNI_VEC),       # ldo * n = 4096
        ("NORM_TO_VNNI4", gen.I8, np.uint8, 64, 65, 80, 80, 0, VNNI_VEC),
        ("NORM_TO_VNNI4_PAD", gen.I8, np.uint8, 64, 66, 64, 80, 1, VNNI),
    ]
    for name, t, npdt, m, n, ldi, ldo, off, var in cases_:
        v = 2 if "VNNI2" in name else 4
        nn = (n + v - 1) // v * v
        x = rng.integers(1, np.iinfo(npdt).max, size=ldi * n + 16, dtype=npdt)
        out0 = np.full(ldo * nn, 3, dtype=npdt)
        op = getattr(X, "MELTW_TYPE_UNARY_TRANSFORM_" + name)
        k = X.libxsmm_dispatch_meltw_unary(op, X.libxsmm_create_meltw_unary_shape(m, n, ldi, ldo, t, t, t), 0)
        got, _ = gpu_unary(k, x, out0, x_offset=off * gen.TS[t], variant=var)
        src = x[off:off + ldi * n].reshape(n, ldi)
        want = np.zeros((nn // v, ldo, v), dtype=npdt)
        for j in range(n):
            want[j // v, :m, j % v] = src[j, :m]
        assert np.array_equal(got, want.reshape(-1)), (name, m, n, off)
        cpu, _ = cpu_unary(oracle, (1, op, 0, m, n, ldi, 0, 0, ldo, t, UNS, UNS, t, t), np.ascontiguousarray(x[off:]), out0)
        assert np.array_equal(got, cpu), (name, "oracle")
