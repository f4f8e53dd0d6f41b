"""CPU-only: the max / min / absmax / argop reductions, the column-index reductions and REPLICATE_COL_VAR of the restatement
(oracle/oracle_meltw.c) on edge inputs -- +-0 in both orders, +-inf, +-FLT_MAX, f64 values beyond FLT_MAX, NaNs first / middle /
last, runs of equal extrema -- pinned bit for bit against the unmodified reference (oracle/_ref), output values AND argop indices.

The first test needs no reference: it states, from the reference's folds (src/generator_mateltwise_reference_impl.c:1215-1428 with
LIBXSMM_MAX / MIN / ABS of include/libxsmm_macros.h:635-637), what a few short lines must give."""
import ctypes as C

import numpy as np
import pytest

import gen
import libxsmm_b200 as X     # only for the enumerators and argument structs (no kernel is launched)
import meltw_edges as E
from oracle_ffi import iarr, oracle, ref

UNS = gen.F64 + 26
need_ref = pytest.mark.skipif(ref is None, reason="oracle/_ref/libxsmm_ref.so not built (no /root/reference here)")
OPS = {"MAX": X.MELTW_TYPE_UNARY_REDUCE_X_OP_MAX, "MIN": X.MELTW_TYPE_UNARY_REDUCE_X_OP_MIN, "ABSMAX": X.MELTW_TYPE_UNARY_REDUCE_X_OP_ABSMAX}
IDX_FLAG = {4: X.MELTW_FLAG_UNARY_IDX_SIZE_4BYTES, 8: X.MELTW_FLAG_UNARY_IDX_SIZE_8BYTES}
SENTINEL = 0xEE


def run(side, desc, x, out0, aux0=None, idx=None, count=None, op_primary=None):
    out, aux = out0.copy(), (None if aux0 is None else aux0.copy())
    keep = []
    p = X.MeltwUnaryParam(); p.inp.primary, p.out.primary = x.ctypes.data, out.ctypes.data
    if aux is not None:
        p.out.secondary = aux.ctypes.data
    if idx is not None:
        cnt = C.c_ulonglong(count); keep.append(cnt)
        p.inp.secondary, p.inp.tertiary = idx.ctypes.data, C.addressof(cnt)
    if op_primary is not None:
        nrt = C.c_ulonglong(op_primary); keep.append(nrt)
        p.op.primary = C.addressof(nrt)
    rc = side["meltw"](iarr(*desc), C.addressof(p), 0)
    assert rc == 0, (desc, rc)
    return out, aux


def same(a, b):
    return np.array_equal(a.view(np.uint8), b.view(np.uint8))


def reduce_line(op, rows, t, vals, argop=0):
    """oracle result of one line (m = 1 under REDUCE_COLS, n = 1 under REDUCE_ROWS) as (output bits, argop index or None)"""
    bits = E.encode([(np.asarray(vals, dtype=np.float64), np.asarray([2 if v != v else 0 for v in vals]))], t)
    L = len(vals)
    m, n = (L, 1) if rows else (1, L)
    x = bits.reshape(-1).copy()
    flags = (X.MELTW_FLAG_UNARY_REDUCE_ROWS if rows else X.MELTW_FLAG_UNARY_REDUCE_COLS) | (X.MELTW_FLAG_UNARY_REDUCE_RECORD_ARGOP | IDX_FLAG[4] if argop else 0)
    out0 = np.zeros(1, dtype=E.BITS_OF[t]); aux0 = np.full(1, 0xEEEEEEEE, dtype=np.uint32)
    out, aux = run(oracle, (1, OPS[op], flags, m, n, m, 0, 0, 1, t, UNS, UNS, t, gen.F64 if t == gen.F64 else gen.F32), x, out0, aux0)
    return int(out[0]), (None if aux[0] == 0xEEEEEEEE else int(aux[0]))


F32_BITS = lambda v: int(np.float32(v).view(np.uint32))   # noqa: E731
NEG0, POS0 = 0x80000000, 0
QNAN_NEG = E.NAN_BITS[gen.F32][1]


def test_reference_fold_rules_by_hand():
    """cases traced by hand through the reference's loops; the restatement must give exactly these bits"""
    nan = float("nan")
    # cols MAX: tmp = MAX(x, tmp) = x < tmp ? tmp : x from -FLT_MAX -> ties take the later value, a NaN is taken and is dropped again
    assert reduce_line("MAX", 0, gen.F32, [0.0, -0.0])[0] == NEG0
    assert reduce_line("MAX", 0, gen.F32, [-np.inf, -np.inf])[0] == F32_BITS(-E.FLT_MAX)
    assert reduce_line("MAX", 0, gen.F32, [1.0, nan])[0] == QNAN_NEG
    assert reduce_line("MAX", 0, gen.F32, [nan, -np.inf])[0] == F32_BITS(-np.inf)           # after a NaN the -FLT_MAX start is gone
    # cols MIN: x < tmp ? x : tmp from FLT_MAX -> ties keep the earlier value, NaN ignored, +inf never taken
    assert reduce_line("MIN", 0, gen.F32, [0.0, -0.0])[0] == POS0
    assert reduce_line("MIN", 0, gen.F32, [np.inf])[0] == F32_BITS(E.FLT_MAX)
    assert reduce_line("MIN", 0, gen.F32, [nan, 2.0, nan])[0] == F32_BITS(2.0)
    # cols ABSMAX from +0 with ABS(-0) = -0: [-0] gives -0; ABS flips a NaN's sign
    assert reduce_line("ABSMAX", 0, gen.F32, [-0.0])[0] == NEG0
    assert reduce_line("ABSMAX", 0, gen.F32, [3.0, nan])[0] == QNAN_NEG ^ 0x80000000
    # rows MAX: tmp = MAX(tmp, x) from the first element -> ties keep the earlier value, NaN ignored unless first (then sticky)
    assert reduce_line("MAX", 1, gen.F32, [0.0, -0.0])[0] == POS0
    assert reduce_line("MAX", 1, gen.F32, [-0.0, 0.0])[0] == NEG0
    assert reduce_line("MAX", 1, gen.F32, [1.0, nan, 0.5])[0] == F32_BITS(1.0)
    assert reduce_line("MAX", 1, gen.F32, [nan, 5.0])[0] == QNAN_NEG
    # rows MIN: tmp = MIN(tmp, x) -> ties take the later value; a NaN is taken and survives only if last
    assert reduce_line("MIN", 1, gen.F32, [0.0, -0.0])[0] == NEG0
    assert reduce_line("MIN", 1, gen.F32, [1.0, nan])[0] == QNAN_NEG
    assert reduce_line("MIN", 1, gen.F32, [nan, 4.0, 7.0])[0] == F32_BITS(4.0)
    # rows ABSMAX: MAX(ABS(tmp), ABS(x)); a NaN first element flips sign once per element folded (the first one included)
    assert reduce_line("ABSMAX", 1, gen.F32, [nan, 1.0])[0] == QNAN_NEG
    assert reduce_line("ABSMAX", 1, gen.F32, [nan, 1.0, 2.0])[0] == QNAN_NEG ^ 0x80000000
    assert reduce_line("ABSMAX", 1, gen.F32, [-3.0, 3.0])[0] == F32_BITS(3.0)
    # argop (cols only): x >= tmp / x <= tmp -> the LAST extremum wins, NaN never taken, an index never taken is not written
    assert reduce_line("MAX", 0, gen.F32, [2.0, 1.0, 2.0], argop=1) == (F32_BITS(2.0), 2)
    assert reduce_line("MIN", 0, gen.F32, [-0.0, 0.0, 5.0], argop=1) == (POS0, 1)
    assert reduce_line("ABSMAX", 0, gen.F32, [-0.0], argop=1) == (NEG0, 0)
    assert reduce_line("MAX", 0, gen.F32, [-np.inf, nan], argop=1) == (F32_BITS(-E.FLT_MAX), None)
    assert reduce_line("MIN", 0, gen.F32, [np.inf], argop=1) == (F32_BITS(E.FLT_MAX), None)
    # f64: the column folds start from (double)FLT_MAX too, so values beyond it are taken
    assert reduce_line("MAX", 0, gen.F64, [-1e300, -np.inf])[0] == int(np.float64(-E.FLT_MAX).view(np.uint64))
    assert reduce_line("MIN", 0, gen.F64, [1e300])[0] == int(np.float64(E.FLT_MAX).view(np.uint64))
    assert reduce_line("MAX", 0, gen.F64, [1e300, 3.0])[0] == int(np.float64(1e300).view(np.uint64))


# input type, output type
TYPES = [(gen.F32, gen.F32), (gen.F32, gen.BF16), (gen.BF16, gen.BF16), (gen.BF16, gen.F32), (gen.F16, gen.F16), (gen.F16, gen.F32), (gen.F64, gen.F64)]


@need_ref
@pytest.mark.parametrize("tin,tout", TYPES)
def test_max_min_absmax_argop_edges(tin, tout):
    rng = np.random.default_rng(91)
    tcomp = gen.F64 if tin == gen.F64 else gen.F32
    for L in (1, 2, 3, 37, 70):
        bits = E.encode(E.sequences(rng, L), tin)
        for rows in (1, 0):
            x, m, n, ldi = E.layout(bits, rows, 3, E.NAN_BITS[tin][0])
            nres = n if rows else m
            for name, op in OPS.items():
                for idx in ((0,) if rows else (0, 4, 8)):
                    flags = (X.MELTW_FLAG_UNARY_REDUCE_ROWS if rows else X.MELTW_FLAG_UNARY_REDUCE_COLS)
                    if idx:
                        flags |= X.MELTW_FLAG_UNARY_REDUCE_RECORD_ARGOP | IDX_FLAG[idx]
                    out0 = np.full(nres * gen.TS[tout], SENTINEL, dtype=np.uint8)
                    aux0 = np.full(nres * max(idx, 1), SENTINEL, dtype=np.uint8)
                    desc = (1, op, flags, m, n, ldi, 0, 0, nres, tin, UNS, UNS, tout, tcomp)
                    want = run(ref, desc, x, out0, aux0)
                    got = run(oracle, desc, x, out0, aux0)
                    assert same(got[0], want[0]), (name, rows, idx, L)
                    assert same(got[1], want[1]), (name, rows, idx, L, "argop")


@need_ref
@pytest.mark.parametrize("tin,tout", [(gen.F32, gen.F32), (gen.BF16, gen.F32), (gen.F16, gen.F16), (gen.F64, gen.F64)])
def test_cols_idx_reductions(tin, tout):
    """REDUCE_COLS_IDX_OP_{ADD,MAX,MIN}: duplicated and unsorted column lists, a list of one, 4- and 8-byte indices, argop"""
    rng = np.random.default_rng(92)
    tcomp = gen.F64 if tin == gen.F64 else gen.F32
    L = 41
    bits = E.encode(E.sequences(rng, L), tin)
    x, m, n, ldi = E.layout(bits, 0, 2, E.NAN_BITS[tin][1])
    lists = [rng.integers(0, n, size=60), np.array([L - 1]), np.array([3, 3, 3]), rng.permutation(n)[:17], np.array([0, n - 1, 0, n - 1])]
    for name in ("ADD", "MAX", "MIN"):
        op = getattr(X, "MELTW_TYPE_UNARY_REDUCE_COLS_IDX_OP_" + name)
        for cols in lists:
            for isz in (4, 8):
                for argop in ((0, 1) if name != "ADD" else (0,)):
                    idx = cols.astype(np.uint32 if isz == 4 else np.uint64)
                    flags = X.MELTW_FLAG_UNARY_REDUCE_COLS | IDX_FLAG[isz] | (X.MELTW_FLAG_UNARY_REDUCE_RECORD_ARGOP if argop else 0)
                    out0 = np.full(m * gen.TS[tout], SENTINEL, dtype=np.uint8); aux0 = np.full(m * isz, SENTINEL, dtype=np.uint8)
                    desc = (1, op, flags, m, n, ldi, 0, 0, m, tin, UNS, UNS, tout, tcomp)
                    want = run(ref, desc, x, out0, aux0, idx=idx, count=len(idx))
                    got = run(oracle, desc, x, out0, aux0, idx=idx, count=len(idx))
                    assert same(got[0], want[0]), (name, len(idx), isz, argop)
                    assert same(got[1], want[1]), (name, len(idx), isz, argop, "argop")


@need_ref
@pytest.mark.parametrize("tin,tout", [(gen.F32, gen.F32), (gen.BF16, gen.F32), (gen.F32, gen.BF16), (gen.F16, gen.F16)])
def test_replicate_col_var(tin, tout):
    """REPLICATE_COL_VAR: column in0[0..m) copied into N columns, N read from op.primary at call time"""
    rng = np.random.default_rng(93)
    for m, n_rt, ldo in ((1, 1, 1), (37, 5, 40), (64, 40, 64)):
        x = rng.integers(0, 2**16, size=m * 4 + 7, dtype=np.uint16).view(np.uint8) if tin != gen.F32 else rng.standard_normal(m + 3).astype(np.float32).view(np.uint8)
        out0 = np.full(ldo * n_rt * gen.TS[tout] + 16, SENTINEL, dtype=np.uint8)
        desc = (1, X.MELTW_TYPE_UNARY_REPLICATE_COL_VAR, 0, m, 1, m, 0, 0, ldo, tin, UNS, UNS, tout, gen.F32)
        want = run(ref, desc, x, out0, op_primary=n_rt)[0]
        got = run(oracle, desc, x, out0, op_primary=n_rt)[0]
        assert same(got, want), (m, n_rt)
