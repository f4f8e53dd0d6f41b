"""The 2-ulp window model of tests/ulp_window.py, without a GPU.

1. It contains an independent libm: the C restatement (glibc's expf / tanhf / erff, oracle/oracle_meltw.c), and the reference itself
   where oracle/_ref is built, lands inside the allowed set at every input of the sweep, for every op and output type.
2. It rejects wrong kernels: numpy restatements of the usual shortcuts each produce at least one element outside the set."""
import ctypes as C
import warnings

import numpy as np
import pytest
from scipy import special

import gen
import ulp_window as U
from oracle_ffi import oracle, ref

PAIRS, OPS, TNAME, split, sweep_bits, cpu_unary = U.PAIRS, U.OPS, U.TNAME, U.split, U.sweep_bits, U.cpu_unary


def first_bad(ok, x, got, allowed, what):
    bad = np.nonzero(~ok)[0]
    if bad.size == 0:
        return None
    i = bad[0]
    return "%s: %d of %d elements outside the window; first x = %r (0x%08x) got 0x%x allowed %s" % (
        what, bad.size, ok.size, float(x[i]), int(x[i:i + 1].view(np.uint32)[0]), int(got[i]),
        sorted({hex(int(b)) for b in allowed.bits[i]}) + (["any NaN"] if allowed.any_nan[i] else []))


@pytest.mark.parametrize("tin,tout", PAIRS, ids=lambda t: TNAME[t])
@pytest.mark.parametrize("opname", OPS)
def test_glibc_inside_every_window(opname, tin, tout):
    op, alpha = split(opname)
    bits = sweep_bits(tin)
    x = U.load(bits, tin)
    allowed = U.allowed(op, x, tout, alpha)
    for name, lib in (("glibc restatement", oracle), ("reference", ref)):
        if lib is None:
            continue
        got = cpu_unary(lib, op, alpha, bits, tin, tout)
        msg = first_bad(allowed.ok(got), x, got, allowed, "%s %s %s->%s" % (name, opname, TNAME[tin], TNAME[tout]))
        assert msg is None, msg


# ---- wrong kernels the model must reject ---------------------------------------------------------------------------
F = np.float32


def _cr(fn, y):
    with np.errstate(all="ignore"):
        return fn(np.asarray(y, np.float32).astype(np.float64)).astype(np.float32)


def _ulps(v, k):
    """v moved k ulps away from zero (through the f32 ordinals; saturates at Inf)"""
    o = U.ordinal(v)
    o2 = np.where(o >= 0, np.minimum(o + k, U.ORD_INF), np.maximum(o - k, -U.ORD_INF))
    return np.where(np.isfinite(v), U.from_ordinal(o2, np.signbit(v)), v)


def _expf_fast(y):
    """__expf at its documented worst case: 2 + floor(1.16 |x|) ulp"""
    with np.errstate(all="ignore"):
        return _ulps(_cr(np.exp, y), (2 + np.floor(1.16 * np.abs(np.nan_to_num(y)))).astype(np.int64))


def _expf_ftz(y):
    r = _cr(np.exp, y)
    return np.where(np.abs(r) < np.float32(2.0 ** -126), F(0.0), r)


def _gelu_tanh(x):
    with np.errstate(all="ignore"):
        x64 = x.astype(np.float64)
        return (0.5 * x64 * (1.0 + np.tanh(np.sqrt(2.0 / np.pi) * (x64 + 0.044715 * x64 ** 3)))).astype(np.float32)


MUTANTS = {
    "sigmoid as 1/(1+exp(-x))": ("SIGMOID", lambda x: F(1.0) / (F(1.0) + _cr(np.exp, -x))),
    "tanh.approx, 2^-11 relative error": ("TANH", lambda x: (_cr(np.tanh, x).astype(np.float64) * (1 - 2.0 ** -11)).astype(np.float32)),
    "__expf, 2 + floor(1.16|x|) ulp": ("EXP", _expf_fast),
    "expf flushing subnormal results": ("EXP", _expf_ftz),
    "GELU by its tanh approximation": ("GELU", _gelu_tanh),
}


@pytest.mark.parametrize("tin", [gen.F32, gen.BF16, gen.F16], ids=lambda t: TNAME[t])
@pytest.mark.parametrize("name", list(MUTANTS))
def test_model_rejects_wrong_kernel(name, tin):
    op, fn = MUTANTS[name]
    x = U.load(sweep_bits(tin), tin)
    with np.errstate(all="ignore"):
        got = fn(x)
    bad = ~U.allowed(op, x, gen.F32).ok(got.view(np.uint32))
    print("%s (%s inputs): %d of %d elements outside the window" % (name, TNAME[tin], bad.sum(), x.size))
    if tin == gen.F32 or name != "expf flushing subnormal results":
        assert bad.any(), name
    # (bf16 and f16 inputs never reach exp's subnormal range: their smallest exp results are normal, or +0 below -104)


def test_model_rejects_bf16_truncation():
    """a bf16 output formed by truncating the f32 result instead of rounding it to nearest even"""
    for tin in (gen.F32, gen.BF16):
        x = U.load(sweep_bits(tin), tin)
        for op in U.TRANSCENDENTAL:
            r = U.correctly_rounded(op, x)
            trunc = (r.view(np.uint32) >> 16).astype(np.uint16)
            bad = ~U.allowed(op, x, gen.BF16).ok(trunc)
            assert bad.any(), (op, TNAME[tin])


def test_gelu_argument_by_multiplication():
    """GELU with x * 0.70710677f in place of x / sqrtf(2.0f): the argument of erff differs by one f32 ulp at many inputs, but a one-ulp
    change of the argument moves erf by less than its own 2-ulp window, so the output stays inside the set. The test says so with a
    warning carrying the counts instead of passing silently."""
    x = U.f32_sweep()
    x = x[np.isfinite(x)]
    with np.errstate(all="ignore"):
        y_mul, y_div = x * F(0.70710677), x / U.SQRT2
        differ = (y_mul.view(np.uint32) != y_div.view(np.uint32)) & ~np.isnan(y_div)
        got = (_cr(special.erf, y_mul) + F(1.0)) * F(0.5) * x
        ref_ = (_cr(special.erf, y_div) + F(1.0)) * F(0.5) * x
    allowed = U.allowed("GELU", x, gen.F32)
    bad = ~allowed.ok(got.view(np.uint32))
    assert allowed.ok(ref_.view(np.uint32)).all()
    changed = (got.view(np.uint32) != ref_.view(np.uint32))
    print("GELU with x * 0.70710677f: the erff argument differs at %d of %d inputs, the output at %d, and %d outputs leave the set"
          % (differ.sum(), x.size, changed.sum(), bad.sum()))
    assert differ.sum() > 0
    if not bad.any():
        warnings.warn("GELU with x * 0.70710677f in place of x / sqrtf(2.0f) is not detectable through erf's 2-ulp window: it changes "
                      "erff's argument at %d of %d inputs and the output at %d, all inside the set" % (differ.sum(), x.size, changed.sum()))
