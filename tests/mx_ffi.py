"""TEST INFRASTRUCTURE: the MX fp8 GEMM checkers and operand generator.

  oracle_gemm_mx  oracle/liboracle_mx.so              plain-C restatement (oracle/oracle_mx.c)
  ref_gemm_mx     oracle/_ref/libxsmm_ref_mx.so       the unmodified reference's libxsmm_reference_gemm (oracle/ref_mx_shim.c),
                                                       only where build() could compile it

Both take dims {m,n,k,lda,ldb,ldc}, types {a,b,comp,c}, flags, br_type (0 / 3), br, A, B, C, A scales, B scales, C scales."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_ffi  # noqa: F401  (builds liboracle.so, which liboracle_mx.so links against)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_MX_SO = os.path.join(ROOT, "oracle", "liboracle_mx.so")
REF_MX_SO = os.path.join(ROOT, "oracle", "_ref", "libxsmm_ref_mx.so")

MXBF8, MXHF8, F32 = 14, 15, 1
TRANS_A, TRANS_B, BETA_0, VNNI_A, VNNI_B = 1, 2, 4, 256, 512
MX_FLAGS = VNNI_A | VNNI_B | TRANS_B

if not os.path.exists(ORACLE_MX_SO) or os.path.getmtime(ORACLE_MX_SO) < os.path.getmtime(os.path.join(ROOT, "oracle", "oracle_mx.c")):
    subprocess.check_call(["make", "-C", ROOT, "oracle"], stdout=subprocess.DEVNULL)

_P = C.c_void_p
_ARGS = [_P, _P, C.c_uint, C.c_int, C.c_ulonglong, _P, _P, _P, _P, _P, _P]
_oracle_lib = C.CDLL(ORACLE_MX_SO)
_oracle_lib.oracle_gemm_mx.restype, _oracle_lib.oracle_gemm_mx.argtypes = C.c_int, _ARGS
_oracle_lib.oracle_f32_to_mxbf8_block.restype, _oracle_lib.oracle_f32_to_mxbf8_block.argtypes = None, [_P, _P, _P]
_oracle_lib.oracle_e8m0_to_f32.restype, _oracle_lib.oracle_e8m0_to_f32.argtypes = C.c_float, [C.c_ubyte]
oracle_gemm_mx = _oracle_lib.oracle_gemm_mx
oracle_f32_to_mxbf8_block = _oracle_lib.oracle_f32_to_mxbf8_block
oracle_e8m0_to_f32 = _oracle_lib.oracle_e8m0_to_f32
ref_gemm_mx = None
if os.path.exists(REF_MX_SO):
    _ref_lib = C.CDLL(REF_MX_SO)
    _ref_lib.ref_gemm_mx.restype, _ref_lib.ref_gemm_mx.argtypes = C.c_int, _ARGS
    ref_gemm_mx = _ref_lib.ref_gemm_mx


class MxCase:
    """one MX GEMM call: A VNNI4 [br][k/4][lda][4], B VNNI4-T [br][k/4][ldb][4], scales [br][k/32][ld], C F32 [n][ldc] or MXBF8
    bytes [n][ldc] with scales [n][ldc/32]. Block r of A / B / the scales sits right after block r-1 (the only batch-reduce
    layout the reference defines)."""

    def __init__(self, ta, tc, m, n, k, lda=None, ldb=None, ldc=None, beta0=True, br_type=0, br=1):
        self.ta, self.tc, self.m, self.n, self.k = ta, tc, m, n, k
        self.lda, self.ldb, self.ldc = lda or m, ldb or n, ldc or m
        self.beta0, self.br_type, self.br = beta0, br_type, (br if br_type else 1)
        self.flags = MX_FLAGS | (BETA_0 if beta0 else 0)
        self.dims = (C.c_int * 6)(m, n, k, self.lda, self.ldb, self.ldc)
        self.types = (C.c_int * 4)(ta, ta, F32, tc)
        self.size_a, self.size_b = self.br * self.lda * k, self.br * self.ldb * k
        self.size_as, self.size_bs = self.br * self.lda * (k // 32), self.br * self.ldb * (k // 32)
        self.size_c = self.ldc * n                                   # elements of C's type
        self.size_cs = n * (self.ldc // 32) if tc == MXBF8 else 0

    def __repr__(self):
        return "MxCase(%s,%s,%dx%dx%d,ld %d/%d/%d,beta0=%d,br %d/%d)" % ("BF8" if self.ta == MXBF8 else "HF8", "MXBF8" if self.tc == MXBF8 else "F32",
                                                                         self.m, self.n, self.k, self.lda, self.ldb, self.ldc, self.beta0, self.br_type, self.br)

    def operands(self, rng, a=None, b=None, scales=None):
        """random A / B bytes (every pattern) and scale bytes (0, 0xFF, 127 +- 20) unless given; C: f32 values or 0 bytes"""
        def fp8(size):   # every byte pattern; Inf / NaN codes kept rare so that most results stay finite
            x = rng.integers(0, 256, size, dtype=np.uint8)
            bad = ((x & 0x7C) == 0x7C) if self.ta == MXBF8 else ((x & 0x7F) == 0x7F)
            x[bad & (rng.random(size) > min(0.02, 2.0 / (self.br * self.k)))] ^= 0x40
            return x
        A = fp8(self.size_a) if a is None else a
        B = fp8(self.size_b) if b is None else b
        if scales is None:
            rare = min(0.01, 0.05 / (self.br * self.k // 32))   # a 0xFF (+inf) scale in about one row of ten

            def sc(size):
                s = rng.integers(107, 148, size).astype(np.uint8)
                pick = rng.random(size)
                s[pick < 2 * rare] = 0
                s[(pick >= 2 * rare) & (pick < 3 * rare)] = 0xFF
                return s
            As, Bs = sc(self.size_as), sc(self.size_bs)
        else:
            As, Bs = scales
        if self.tc == F32:
            C0 = rng.standard_normal(self.size_c).astype(np.float32)
        else:
            C0 = np.zeros(self.size_c, dtype=np.uint8)
        Cs = np.zeros(max(self.size_cs, 1), dtype=np.uint8)
        return A, B, C0, As, Bs, Cs

    def run(self, fn, A, B, C0, As, Bs, Cs):
        """runs oracle_gemm_mx or ref_gemm_mx on copies; returns (rc, C, C scales)"""
        c, cs = C0.copy(), Cs.copy()
        rc = fn(self.dims, self.types, self.flags, self.br_type, self.br, A.ctypes.data, B.ctypes.data, c.ctypes.data,
                As.ctypes.data, Bs.ctypes.data, cs.ctypes.data if self.tc == MXBF8 else None)
        return rc, c, cs[:self.size_cs]


def image_nan(case, A, B, As, Bs):
    """NaN positions of the f32 image an MXBF8 C is quantised from: which NaN an x86 addition of two NaNs returns depends on the
    compiler's operand order, and the sign shows in the clamped byte (0x7B / 0xFB); there only |byte| is compared"""
    f = MxCase(case.ta, F32, case.m, case.n, case.k, case.lda, case.ldb, case.ldc, True, case.br_type, case.br)
    c = np.zeros(f.size_c, np.float32)
    _, img, _ = f.run(oracle_gemm_mx, A, B, c, As, Bs, np.zeros(1, np.uint8))
    return np.isnan(img)


def same_mxbf8(want, got, nan):
    """MXBF8 C data bytes equal, NaN positions of the image up to the sign"""
    w, g = np.asarray(want, np.uint8), np.asarray(got, np.uint8)
    return bool(np.array_equal(w[~nan], g[~nan]) and np.array_equal(w[nan] & 0x7F, g[nan] & 0x7F))


def same_bits(want, got):
    """two F32 C images equal bit for bit, NaN positions excepted (both must be NaN there)"""
    w, g = np.asarray(want, np.float32), np.asarray(got, np.float32)
    nan = np.isnan(w)
    return bool(np.array_equal(np.isnan(g), nan) and np.array_equal(w.view(np.uint32)[~nan], g.view(np.uint32)[~nan]))
