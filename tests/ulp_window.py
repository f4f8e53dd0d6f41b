"""TEST INFRASTRUCTURE: the output bit patterns a correct kernel may produce for the transcendental elementwise ops.

The kernels evaluate the reference's own formulas (src/generator_mateltwise_reference_impl.c:17-40, 76-113, ELU :2138-2167) with the
same f32 operations in the same order, no contraction and IEEE division and sqrt. The only freedom left is in the libm calls
(expf, tanhf, erff), which CUDA documents as within 2 ulp. So each output element has a small set of correct bit patterns:

  window of one call f(y)   y is the f32 argument the formula computes (x / 2.0f, x / sqrtf(2.0f), -0.5f * x * x, ...); T = f(y)
                            exactly. The window is every f32 v with |v - T| <= 2 ulp(T), ulp(T) = 2^(max(e, -126) - 23) with
                            e = floor(log2 |T|); +Inf is in it when some real within that distance rounds to +Inf (T + 2 ulp >=
                            2^128 - 2^103); it stops at zero on the side of T's sign (no libm returns a negative exp, or a tanh /
                            erf of the other sign), and a zero in it carries the sign of T. C99 Annex F cases are single values: f(+-0), f(+-Inf),
                            exp(-Inf) = +0; NaN -> any NaN (no libm promises a payload).
  through the formula       every candidate of every call (GELU_INV has two calls), evaluated in numpy float32 in the kernel's
                            operation order, then stored through the output conversion (the C restatement's, pinned elsewhere).

T comes from float64 (numpy / scipy). Where the float64 value lies too close to a point of the f32 grid (a multiple of ulp/2: grid points
of its binade and the one below, window edges, powers of two) for its own error, mpmath decides at 320 bits. Where even that cannot
separate T from the grid point, T differs from it by less than 2^-280 relative, and the side is known from the function: tanh(y)
below |y| for tiny y and below 1 in magnitude when saturated, erf below 1 in magnitude, exp(y) on the side of 1 that y is on of 0.
"""
import ctypes as C
import functools

import mpmath
import numpy as np
from scipy import special

import gen
import libxsmm_b200 as X
from oracle_ffi import iarr, oracle

F32_MAX = float(np.finfo(np.float32).max)
INF_EDGE = 2.0 ** 128 - 2.0 ** 103           # the smallest real that rounds to +Inf
ORD_INF = 0x7F800000                         # ordinal of +Inf (ordinals: f32 magnitude bits, negative below zero, both zeros 0)
SQRT2 = np.float32(np.sqrt(np.float32(2.0)))                          # sqrtf(2.0f), correctly rounded like IEEE sqrt
SQRT2PI = np.float32(np.sqrt(np.float32(2.0) * np.float32(np.pi)))    # sqrtf(2.0f * 3.14159265358979323846f)
F = np.float32
TRANSCENDENTAL = ("TANH", "TANH_INV", "SIGMOID", "SIGMOID_INV", "GELU", "GELU_INV", "EXP")
OPS = list(TRANSCENDENTAL) + ["ELU:1.0", "ELU:0.3", "ELU:-0.5"]      # ELU with its alpha
PAIRS = [(gen.F32, gen.F32), (gen.F32, gen.BF16), (gen.BF16, gen.BF16), (gen.BF16, gen.F32), (gen.F16, gen.F16), (gen.F16, gen.F32),
         (gen.F32, gen.BF8), (gen.F32, gen.HF8)]                        # in -> out types of the unary sweeps
TNAME = {gen.F32: "f32", gen.BF16: "bf16", gen.F16: "f16", gen.BF8: "bf8", gen.HF8: "hf8"}
UNS = gen.F64 + 26     # LIBXSMM_DATATYPE_UNSUPPORTED


def split(opname):
    """"ELU:0.3" -> ("ELU", 0.3); "TANH" -> ("TANH", None)"""
    op, _, a = opname.partition(":")
    return op, (float(a) if a else None)


# ---- f32 ordinals ----------------------------------------------------------------------------------------------------
def ordinal(v):
    b = np.asarray(v, np.float32).view(np.uint32).astype(np.int64)
    mag = b & 0x7FFFFFFF
    return np.where(b >> 31 != 0, -mag, mag)


def from_ordinal(o, neg_zero):
    o = np.asarray(o, np.int64)
    bits = np.where(o < 0, np.abs(o) | 0x80000000, o)
    bits = np.where((o == 0) & neg_zero, 0x80000000, bits)
    return bits.astype(np.uint32).view(np.float32)


# ---- the window of one libm call ------------------------------------------------------------------------------------
_F64 = {"tanh": np.tanh, "erf": special.erf, "exp": np.exp}
_MP = {"tanh": mpmath.tanh, "erf": mpmath.erf, "exp": mpmath.exp}
_PREC = 320


def _mp_grid(x, up):
    """smallest (up) or largest f32 grid value >= / <= x (an mpf, |x| <= 2^128), as an ordinal; beyond FLT_MAX -> +-Inf"""
    if x == 0:
        return 0
    e = int(mpmath.frexp(abs(x))[1]) - 1
    s = mpmath.ldexp(1, max(e, -126) - 23)
    q = x / s
    k = int(mpmath.ceil(q) if up else mpmath.floor(q))
    v = k * s
    if abs(v) > F32_MAX:
        return ORD_INF if v > 0 else -ORD_INF
    return int(ordinal(np.float32(float(v))))


def _window_exact(T, d):
    """(lo, hi) ordinals of the window around T + d*epsilon (T an mpf at working precision, d in {-1, 0, 1}; d = 0 means T is not on
    the grid of multiples of ulp/2)"""
    if T == 0:
        u = mpmath.ldexp(1, -149)
    else:
        e = int(mpmath.frexp(abs(T))[1]) - 1
        if d != 0 and mpmath.frexp(abs(T))[0] == 0.5 and d * mpmath.sign(T) < 0:
            e -= 1                                           # a power of two approached from below sits in the binade below
        u = mpmath.ldexp(1, max(e, -126) - 23)
    lo, hi = T - 2 * u, T + 2 * u
    # an edge that is itself a grid value is in the window unless the true value lies beyond it (d points away)
    if hi > INF_EDGE or (hi == INF_EDGE and d >= 0):
        ohi = ORD_INF
    else:
        ohi = _mp_grid(min(hi, mpmath.mpf(F32_MAX)), False)
        if d < 0 and mpmath.mpf(float(from_ordinal(ohi, False))) == hi:
            ohi -= 1
    if lo < -INF_EDGE or (lo == -INF_EDGE and d <= 0):
        olo = -ORD_INF
    else:
        olo = _mp_grid(max(lo, mpmath.mpf(-F32_MAX)), True)
        if d > 0 and mpmath.mpf(float(from_ordinal(olo, False))) == lo:
            olo += 1
    return olo, ohi


def _window_grid(g, d):
    """_window_exact for arrays of f32 grid values g (float64, finite, |g| <= 1) with sides d != 0, in float64 (every edge is exact)"""
    m, e = np.frexp(np.abs(g))
    e = e.astype(np.int64) - 1
    e = np.where((m == 0.5) & (d * np.sign(g) < 0), e - 1, e)
    u = np.where(g == 0, 2.0 ** -149, np.ldexp(1.0, np.maximum(e, -126) - 23))
    lo, hi = g - 2 * u, g + 2 * u
    f_hi = hi.astype(np.float32)
    f_hi = np.where(f_hi.astype(np.float64) > hi, np.nextafter(f_hi, np.float32(-np.inf)), f_hi)
    ohi = ordinal(f_hi) - ((d < 0) & (f_hi.astype(np.float64) == hi))
    f_lo = lo.astype(np.float32)
    f_lo = np.where(f_lo.astype(np.float64) < lo, np.nextafter(f_lo, np.float32(np.inf)), f_lo)
    olo = ordinal(f_lo) + ((d > 0) & (f_lo.astype(np.float64) == lo))
    return olo, ohi


def _near_grid(T, rel):
    """T (mpf, nonzero) within rel*|T| of a multiple of ulp(T)/2; returns (bool, that multiple)"""
    e = int(mpmath.frexp(abs(T))[1]) - 1
    h = mpmath.ldexp(1, max(e, -126) - 24)
    k = mpmath.nint(T / h)
    return abs(T - k * h) <= rel * abs(T), k * h


def _side(fname, y, g):
    """which side of the grid point g the true f(y) lies on, for the coincidences the functions have"""
    if fname == "tanh" and (g == y or abs(g) == 1):
        return -1 if y > 0 else 1                            # |tanh y| < |y| and < 1
    if fname == "erf" and abs(g) == 1:
        return -1 if y > 0 else 1
    if fname == "exp" and g == 1:
        return 1 if y > 0 else -1
    if fname == "exp" and g == 0:
        return 1
    raise AssertionError("window of %s(%r) undecidable: the true value is within 2^-280 of the f32 grid point %r" % (fname, y, g))


@functools.lru_cache(maxsize=None)
def _window_one(fname, y):
    """(lo, hi, negative) of f(y) for one finite nonzero f32 y (a Python float), decided with mpmath"""
    with mpmath.workprec(_PREC):
        T = _MP[fname](mpmath.mpf(y))
        if T == 0:
            return _window_exact(mpmath.mpf(0), _side(fname, y, 0)) + (False,)
        amb, g = _near_grid(T, mpmath.ldexp(1, -(_PREC - 40)))
        if not amb:
            return _window_exact(T, 0) + (T < 0,)
        return _window_exact(g, _side(fname, y, g)) + (g < 0 or (g == 0 and y < 0),)


def _windows(fname, y):
    """ordinal windows (lo, hi), the sign a zero takes, and the NaN mask, for f(y) over a float32 array y"""
    y = np.asarray(y, np.float32)
    with np.errstate(invalid="ignore"):
        y64 = y.astype(np.float64)
    n = y.size
    lo = np.zeros(n, np.int64); hi = np.zeros(n, np.int64); neg = np.zeros(n, bool)
    nan = np.isnan(y)
    with np.errstate(all="ignore"):
        T = _F64[fname](y64)
        e = np.frexp(np.abs(T))[1].astype(np.int64) - 1
        u = np.ldexp(1.0, np.maximum(e, -126) - 23)
        h = u / 2
        amb = np.abs(T / h - np.rint(T / h)) * h <= 2.0 ** -44 * np.abs(T)
        amb |= (T == 0) | ~np.isfinite(T)
        lo_v, hi_v = T - 2 * u, T + 2 * u
        f_lo = lo_v.astype(np.float32)
        f_lo = np.where(f_lo.astype(np.float64) < lo_v, np.nextafter(f_lo, np.float32(np.inf)), f_lo)
        f_hi = np.minimum(hi_v, F32_MAX).astype(np.float32)
        f_hi = np.where(f_hi.astype(np.float64) > hi_v, np.nextafter(f_hi, np.float32(-np.inf)), f_hi)
    lo[:] = np.where(lo_v > F32_MAX, ORD_INF, ordinal(f_lo))
    hi[:] = np.where(hi_v >= INF_EDGE, ORD_INF, ordinal(f_hi))
    neg[:] = T < 0
    special_ = nan | (y == 0) | np.isinf(y)
    # Annex F single values
    one = int(ordinal(np.float32(1.0)))
    for i in np.nonzero(special_ & ~nan)[0]:
        v = y[i]
        if v == 0:
            r, ng = ((0, np.signbit(v)) if fname != "exp" else (one, False))
        elif fname == "exp":
            r, ng = ((ORD_INF, False) if v > 0 else (0, False))
        else:
            r, ng = ((one, False) if v > 0 else (-one, True))
        lo[i] = hi[i] = r; neg[i] = ng
    # saturated and tiny arguments: the side of the grid point is known without mpmath
    ay = np.abs(y64)
    fast = np.zeros(n, bool)
    if fname == "tanh":
        fast = (ay >= 20.0) | (ay < 2.0 ** -30)
    elif fname == "erf":
        fast = ay >= 6.0
    elif fname == "exp":
        fast = (ay < 2.0 ** -40) | (y64 < -745.0) | (y64 > 89.0)
    rest = amb & ~special_
    fi = np.nonzero(rest & fast)[0]
    if fi.size:
        yf = y64[fi]
        if fname == "exp":
            g = np.where(yf < -745.0, 0.0, 1.0)
            d = np.where(yf < -745.0, 1, np.sign(yf)).astype(np.int64)
        else:
            g = np.where(np.abs(yf) < 2.0 ** -30, yf, np.sign(yf))
            d = -np.sign(yf).astype(np.int64)
        lo[fi], hi[fi] = _window_grid(g, d)
        neg[fi] = g < 0
        big = fi[yf > 89.0] if fname == "exp" else fi[:0]
        lo[big] = hi[big] = ORD_INF; neg[big] = False
    for i in np.nonzero(rest & ~fast)[0]:
        lo[i], hi[i], neg[i] = _window_one(fname, float(y[i]))
    # the window stops at zero: a result never takes the sign opposite to the true value's
    lo = np.where(neg, lo, np.maximum(lo, 0))
    hi = np.where(neg, np.minimum(hi, 0), hi)
    lo[nan] = hi[nan] = 0
    return lo, hi, neg, nan


def libm_candidates(fname, y):
    """(N, K) float32 candidates of f(y): every f32 value of each element's window (rows padded by repeating their last value);
    NaN rows for NaN arguments"""
    lo, hi, neg, nan = _windows(fname, y)
    k = int((hi - lo).max(initial=0)) + 1
    o = np.minimum(lo[:, None] + np.arange(k)[None, :], hi[:, None])
    c = from_ordinal(o, neg[:, None])
    c[nan] = np.float32(np.nan)
    return c


_cache = {}


def _lc(fname, y):
    key = (fname, np.asarray(y, np.float32).tobytes())
    if key not in _cache:
        _cache[key] = libm_candidates(fname, y)
    return _cache[key]


# ---- the formulas, in the kernel's operation order (numpy float32: IEEE, round to nearest even, subnormals kept) ------
def result_candidates(op, x, alpha=None):
    """(N, C) float32 candidates of the f32 result of `op` at the loaded inputs x, and the rows whose NaN may be any NaN. ELU's
    x > 0 and NaN branch passes x through unchanged, and a NaN there keeps its bits."""
    x = np.asarray(x, np.float32)
    xc = x[:, None]
    with np.errstate(all="ignore"):
        if op == "TANH":
            r = _lc("tanh", x)
        elif op in ("SIGMOID", "SIGMOID_INV"):
            s = (_lc("tanh", x / F(2.0)) + F(1.0)) / F(2.0)
            r = s if op == "SIGMOID" else s * (F(1.0) - s)
        elif op == "TANH_INV":
            t = _lc("tanh", x)
            r = F(1.0) - t * t
        elif op == "GELU":
            r = (_lc("erf", x / SQRT2) + F(1.0)) * F(0.5) * xc
        elif op == "GELU_INV":
            e = _lc("erf", x / SQRT2)
            ex = _lc("exp", (F(-0.5) * x) * x)
            a = (F(0.5) + F(0.5) * e)[:, :, None] + ((x / SQRT2PI)[:, None, None] * ex[:, None, :])
            r = a.reshape(x.size, -1)
        elif op == "EXP":
            r = _lc("exp", x)
        elif op == "ELU":
            y = F(alpha) * (_lc("exp", x) - F(1.0))
            r = np.where(xc <= 0, y, xc)
            return r, np.isnan(r).any(axis=1) & (x <= 0)
        else:
            raise ValueError(op)
    return r, np.isnan(r).any(axis=1)


# ---- output conversion and the membership test ---------------------------------------------------------------------
BITS = {gen.F32: np.uint32, gen.BF16: np.uint16, gen.F16: np.uint16, gen.BF8: np.uint8, gen.HF8: np.uint8}


def store(v, tout):
    """f32 values -> bits of tout, through the C restatement's RNE conversions (oracle/oracle_meltw.c stf, pinned to the reference)"""
    v = np.ascontiguousarray(v, np.float32).reshape(-1)
    if tout == gen.F32:
        return v.view(np.uint32).copy()
    out = np.zeros(v.size, BITS[tout])
    p = X.MeltwUnaryParam(); p.inp.primary, p.out.primary = v.ctypes.data, out.ctypes.data
    desc = (1, X.MELTW_TYPE_UNARY_IDENTITY, 0, v.size, 1, v.size, 0, 0, v.size, gen.F32, UNS, UNS, tout, gen.F32)
    assert oracle["meltw"](iarr(*desc), C.addressof(p), 0) == 0
    return out


def is_nan_bits(b, t):
    b = np.asarray(b).astype(np.uint32)
    if t == gen.F32:
        return (b & 0x7FFFFFFF) > 0x7F800000
    if t == gen.BF16:
        return (b & 0x7FFF) > 0x7F80
    if t == gen.F16:
        return (b & 0x7FFF) > 0x7C00
    if t == gen.BF8:
        return (b & 0x7F) > 0x7C
    return (b & 0x7F) == 0x7F


class Allowed:
    """the allowed output bit patterns of every element: rows of `bits` plus `any_nan`"""

    def __init__(self, cands, any_nan, tout):
        self.tout = tout
        self.bits = store(cands, tout).reshape(cands.shape)
        self.any_nan = any_nan

    def ok(self, got_bits):
        g = np.asarray(got_bits).reshape(-1).astype(self.bits.dtype)
        return (g[:, None] == self.bits).any(axis=1) | (self.any_nan & is_nan_bits(g, self.tout))

    def take(self, idx):
        a = Allowed.__new__(Allowed)
        a.tout, a.bits, a.any_nan = self.tout, self.bits[idx], self.any_nan[idx]
        return a


def allowed(op, x, tout, alpha=None):
    return Allowed(*result_candidates(op, x, alpha), tout)


def correctly_rounded(op, x, alpha=None):
    """the f32 result with every libm call correctly rounded: the middle of each window (for the report)"""
    x = np.asarray(x, np.float32)
    fn = {"tanh": np.tanh, "erf": special.erf, "exp": np.exp}

    def cr(f, y):
        c = _lc(f, y)
        with np.errstate(all="ignore"):
            t = fn[f](np.asarray(y, np.float32).astype(np.float64))
        r = t.astype(np.float32)
        # prefer the float64 value rounded once; where it is ambiguous the window is symmetric about the true value
        good = np.isfinite(r) | np.isnan(r)
        return np.where(good, r, c[:, (c.shape[1] - 1) // 2])
    with np.errstate(all="ignore"):
        if op == "TANH":
            return cr("tanh", x)
        if op in ("SIGMOID", "SIGMOID_INV"):
            s = (cr("tanh", x / F(2.0)) + F(1.0)) / F(2.0)
            return s if op == "SIGMOID" else s * (F(1.0) - s)
        if op == "TANH_INV":
            t = cr("tanh", x); return F(1.0) - t * t
        if op == "GELU":
            return (cr("erf", x / SQRT2) + F(1.0)) * F(0.5) * x
        if op == "GELU_INV":
            return (F(0.5) + F(0.5) * cr("erf", x / SQRT2)) + (x / SQRT2PI) * cr("exp", (F(-0.5) * x) * x)
        if op == "EXP":
            return cr("exp", x)
        return np.where(x <= 0, F(alpha) * (cr("exp", x) - F(1.0)), x)


# ---- inputs --------------------------------------------------------------------------------------------------------
def load(bits, t):
    """inputs as the kernels load them (meltw.cu ld_f32): bf16 flushes subnormals, f16 widens exactly and quiets a NaN"""
    bits = np.asarray(bits)
    if t == gen.F32:
        return bits.astype(np.uint32).view(np.float32)
    if t == gen.BF16:
        h = bits.astype(np.uint32)
        h = np.where((h & 0x7F80) == 0, h & 0x8000, h)
        return (h << 16).astype(np.uint32).view(np.float32)
    h = bits.astype(np.uint16)
    h = np.where((h & 0x7C00) == 0x7C00, np.where((h & 0x3FF) != 0, h | 0x200, h), h).astype(np.uint16)
    with np.errstate(invalid="ignore"):
        return h.view(np.float16).astype(np.float32)


def all_bits16():
    return np.arange(65536, dtype=np.uint32).astype(np.uint16)


def sweep_bits(t):
    """the input bit patterns of a sweep: the f32 sweep, or every 16-bit pattern"""
    return f32_sweep().view(np.uint32) if t == gen.F32 else all_bits16()


def cpu_unary(lib, op, alpha, bits, tin, tout):
    """one m x 1 unary call of the C restatement (oracle) or the reference (ref) over the input bit patterns; returns the output bits"""
    x = np.ascontiguousarray(bits.astype(BITS[tin]))
    out = np.zeros(x.size, BITS[tout])
    a = C.c_float(alpha if alpha is not None else 0.0)
    p = X.MeltwUnaryParam(); p.inp.primary, p.out.primary = x.ctypes.data, out.ctypes.data
    p.op.primary = C.addressof(a)
    desc = (1, getattr(X, "MELTW_TYPE_UNARY_" + op), 0, x.size, 1, x.size, 0, 0, x.size, tin, UNS, UNS, tout, gen.F32)
    assert lib["meltw"](iarr(*desc), C.addressof(p), 0) == 0
    return out


def _span(a, b, n):
    oa, ob = int(ordinal(np.float32(a))), int(ordinal(np.float32(b)))
    return from_ordinal(np.unique(np.linspace(oa, ob, n).astype(np.int64)), False)


def _around(v, k):
    o = int(ordinal(np.float32(v)))
    return from_ordinal(np.arange(o - k, o + k + 1), False)


def f32_sweep():
    """f32 inputs: a few mantissas in every binade from 2^-149 to 2^127 and both signs; zeros, infinities, quiet and signalling NaNs
    with payloads; dense samples around each threshold of the ops"""
    mants = np.array([0, 1, 0x155555, 0x2AAAAA, 0x400000, 0x5A827A, 0x7FFFFF], np.uint32)
    ex = np.arange(0, 255, dtype=np.uint32)
    grid = ((ex[:, None] << 23) | mants[None, :]).reshape(-1)
    grid = grid[grid != 0].view(np.float32)
    special_bits = np.array([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7FC00001, 0x7FFFFFFF, 0xFFFFFFFF,
                             0x7F800001, 0x7FA5A5A5, 0xFF800001, 0xFFBFFFFF], np.uint32).view(np.float32)
    parts = [grid, -grid, special_bits,
             _span(2.0 ** -14, 2.0 ** -10, 2000), _around(2.0 ** -12, 64),           # tanh(x) ~ x below 2^-12
             _span(8.0, 10.0, 3000), _around(9.01, 256),                            # tanh -> 1 near 9.01
             _span(16.0, 20.0, 3000), _around(18.02, 256),                          # x / 2 in sigmoid
             _span(3.6, 4.2, 2000), _around(3.92, 256), _span(5.2, 5.9, 2000),      # erf -> 1 near 3.92 (GELU: x / sqrt 2 near 5.54)
             _span(88.0, 89.5, 2000), _around(np.uint32(0x42B17217).view(np.float32), 64),   # exp overflow
             _span(-103.97, -87.34, 6000), _around(-87.336, 64), _around(-103.972, 64),       # exp into the subnormals
             _span(13.2, 14.4, 3000)]                                               # GELU_INV: exp(-x^2/2) underflow
    dense = np.concatenate([p.astype(np.float32) for p in parts[3:]])
    v = np.concatenate([parts[0], parts[1], parts[2], dense, -dense]).astype(np.float32)
    _, first = np.unique(v.view(np.uint32), return_index=True)
    return v[np.sort(first)]
