"""TEST INFRASTRUCTURE: the dequantising GEMM checkers and operand generator.

  oracle_gemm_dq  oracle/liboracle_dq.so              plain-C restatement (oracle/oracle_dq.c)
  ref_gemm_dq     oracle/_ref/libxsmm_ref_dq.so       the unmodified reference's libxsmm_reference_gemm (oracle/ref_dq_shim.c),
                                                       only where build() could compile it

Both take dims {m,n,k,lda,ldb,ldc}, types {a,b,comp,c}, flags, br_type (0 none / 1 address / 2 offset / 3 stride), stride_a,
stride_b (bytes), br, A, B, C, offs_a, offs_b (bytes), row scales, zero points."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_ffi  # noqa: F401  (builds liboracle.so, which liboracle_dq.so links against)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DQ_SO = os.path.join(ROOT, "oracle", "liboracle_dq.so")
REF_DQ_SO = os.path.join(ROOT, "oracle", "_ref", "libxsmm_ref_dq.so")

F32, BF16, F16, BF8, I8, U8, I4, U4, IMPLICIT = 1, 2, 3, 4, 12, 13, 18, 19, 25
TRANS_A, TRANS_B, BETA_0, VNNI_A, VNNI_B = 1, 2, 4, 256, 512
NAMES = {F32: "F32", BF16: "BF16", F16: "F16", BF8: "BF8", I8: "I8", U8: "U8", I4: "I4", U4: "U4", IMPLICIT: "IMPL"}

if not os.path.exists(ORACLE_DQ_SO) or os.path.getmtime(ORACLE_DQ_SO) < os.path.getmtime(os.path.join(ROOT, "oracle", "oracle_dq.c")):
    subprocess.check_call(["make", "-C", ROOT, "oracle"], stdout=subprocess.DEVNULL)

_P = C.c_void_p
_ARGS = [_P, _P, C.c_uint, C.c_int, C.c_longlong, C.c_longlong, C.c_ulonglong, _P, _P, _P, _P, _P, _P, _P]
_oracle_lib = C.CDLL(ORACLE_DQ_SO)
_oracle_lib.oracle_gemm_dq.restype, _oracle_lib.oracle_gemm_dq.argtypes = C.c_int, _ARGS
oracle_gemm_dq = _oracle_lib.oracle_gemm_dq
ref_gemm_dq = None
if os.path.exists(REF_DQ_SO):
    _ref_lib = C.CDLL(REF_DQ_SO)
    _ref_lib.ref_gemm_dq.restype, _ref_lib.ref_gemm_dq.argtypes = C.c_int, _ARGS
    ref_gemm_dq = _ref_lib.ref_gemm_dq


def _f16(x):
    return np.asarray(x, np.float32).astype(np.float16).view(np.uint16)


def _bf16(x):
    return (np.asarray(x, np.float32).view(np.uint32) >> 16).astype(np.uint16)   # truncation: any bf16 pattern will do


class DqCase:
    """one dequantising GEMM call. A (bytes): flat [br][k][lda], int4 pairs [br][k/2][lda] or bf8 VNNI2 [br][k/2][lda][2]; B (16-bit):
    [br][n][ldb] or, under TRANS_B, [br][k][ldb]; C [n][ldc]; row scales [m] (f32 next to a bf16 B, else f16); zero points [m] f16.
    Block r of A / B sits right after block r-1; offset mode visits the blocks in reverse order, address mode through an array
    of pointers to them."""

    def __init__(self, ta, tb, comp, tc, m, n, k, lda=None, ldb=None, ldc=None, beta0=True, trans_b=False, vnni_a=None, br_type=0, br=1):
        self.ta, self.tb, self.comp, self.tc, self.m, self.n, self.k = ta, tb, comp, tc, m, n, k
        self.trans_b = trans_b
        self.vnni_a = (ta in (I4, U4)) if vnni_a is None else vnni_a
        self.lda, self.ldb, self.ldc = lda or m, ldb or (n if trans_b else k), ldc or m
        self.beta0, self.br_type, self.br = beta0, br_type, (br if br_type else 1)
        self.flags = (BETA_0 if beta0 else 0) | (TRANS_B if trans_b else 0) | (VNNI_A if self.vnni_a else 0)
        self.dims = (C.c_int * 6)(m, n, k, self.lda, self.ldb, self.ldc)
        self.types = (C.c_int * 4)(ta, tb, comp, tc)
        self.block_a = self.lda * (k // 2 if ta in (I4, U4) else k)            # bytes
        self.block_b = self.ldb * (k if trans_b else n)                        # 16-bit elements
        self.size_a, self.size_b, self.size_c = self.br * self.block_a, self.br * self.block_b, self.ldc * n
        self.stride_a = self.block_a if br_type == 3 else 0
        self.stride_b = 2 * self.block_b if br_type == 3 else 0
        self.c_dtype = np.float32 if tc == F32 else np.uint16

    def __repr__(self):
        return "Dq(%s.%s.%s.%s,%dx%dx%d,ld %d/%d/%d,beta0=%d%s%s,br %d/%d)" % (
            NAMES[self.ta], NAMES[self.tb], NAMES[self.comp], NAMES[self.tc], self.m, self.n, self.k, self.lda, self.ldb, self.ldc,
            self.beta0, ",tb" if self.trans_b else "", ",vnni" if self.vnni_a else "", self.br_type, self.br)

    def needs_scales(self):
        return self.ta != BF8

    def operands(self, rng, scales=None, zpts=None):
        """A: every byte pattern (bf8 Inf / NaN codes kept rare); B, C: normal values; row scales mixing 0, negative values and values
        large enough to overflow f16 (or bf16) in a * scale; zero points non-zero, many on f16 rounding ties of an integer minus them"""
        A = rng.integers(0, 256, self.size_a, dtype=np.uint8)
        if self.ta == BF8:
            bad = (A & 0x7C) == 0x7C
            A[bad & (rng.random(self.size_a) > min(0.02, 2.0 / (self.br * self.k)))] ^= 0x40
        b = rng.standard_normal(self.size_b).astype(np.float32)
        B = _bf16(b) if self.tb == BF16 else _f16(b)
        if self.tc == F32:
            C0 = rng.standard_normal(self.size_c).astype(np.float32)
        else:
            c = rng.standard_normal(self.size_c).astype(np.float32)
            C0 = _bf16(c) if self.tc == BF16 else _f16(c)
        if scales is None:
            s = (rng.standard_normal(self.m) * 0.05).astype(np.float32)
            pick = rng.random(self.m)
            s[pick < 0.08] = 0.0
            big = 3.0e36 if self.tb == BF16 else 900.0            # 127 * 900 > 65504: inf in f16; 127 * 3e36 > FLT_MAX
            s[(pick >= 0.08) & (pick < 0.14)] = big * np.sign(rng.standard_normal(int(((pick >= 0.08) & (pick < 0.14)).sum())))
            S = s if self.tb == BF16 else _f16(s)
        else:
            S = scales
        if zpts is None:
            ties = np.array([2.0 ** -9, 3 * 2.0 ** -9, -2.0 ** -8, 0.5, -1.5, 7.5, 1.0 / 3.0, -0.1], np.float32)
            Z = _f16(np.where(rng.random(self.m) < 0.7, ties[rng.integers(0, len(ties), self.m)], rng.standard_normal(self.m) * 4.0))
        else:
            Z = zpts
        return A, B, C0, S, Z

    def run(self, fn, A, B, C0, S, Z):
        """runs oracle_gemm_dq or ref_gemm_dq on a copy of C; returns (rc, C)"""
        c = C0.copy()
        a_arg, b_arg, oa, ob, keep = A.ctypes.data, B.ctypes.data, None, None, []
        if self.br_type == 1:
            pa = (C.c_void_p * self.br)(*[A.ctypes.data + r * self.block_a for r in range(self.br)])
            pb = (C.c_void_p * self.br)(*[B.ctypes.data + 2 * r * self.block_b for r in range(self.br)])
            keep += [pa, pb]
            a_arg, b_arg = C.addressof(pa), C.addressof(pb)
        elif self.br_type == 2:
            oa_ = np.array([(self.br - 1 - r) * self.block_a for r in range(self.br)], np.int64)
            ob_ = np.array([2 * (self.br - 1 - r) * self.block_b for r in range(self.br)], np.int64)
            keep += [oa_, ob_]
            oa, ob = oa_.ctypes.data, ob_.ctypes.data
        rc = fn(self.dims, self.types, self.flags, self.br_type, self.stride_a, self.stride_b, self.br, a_arg, b_arg, c.ctypes.data,
                oa, ob, S.ctypes.data if S is not None else None, Z.ctypes.data if Z is not None else None)
        return rc, c

    def nan_mask(self, c):
        """NaN positions of a C image"""
        c = np.asarray(c)
        if self.tc == F32:
            return np.isnan(c.view(np.float32))
        h = c.view(np.uint16)
        if self.tc == BF16:
            return ((h & 0x7F80) == 0x7F80) & ((h & 0x7F) != 0)
        return ((h & 0x7C00) == 0x7C00) & ((h & 0x3FF) != 0)


def same_c(case, want, got):
    """two C images equal bit for bit, NaN positions excepted (both must be NaN there): the sign and payload of a NaN made from
    0 * inf or inf - inf is the host's choice (x86's default NaN is negative)"""
    w, g = np.asarray(want).view(case.c_dtype), np.asarray(got).view(case.c_dtype)
    nan = case.nan_mask(w)
    bits = np.uint32 if case.tc == F32 else np.uint16
    return bool(np.array_equal(case.nan_mask(g), nan) and np.array_equal(w.view(bits)[~nan], g.view(bits)[~nan]))


def case_from_meta(meta):
    """inverse of DqCase.meta(): the fixture's case descriptions"""
    v = [int(x) for x in meta]
    return DqCase(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7], v[8], v[9], bool(v[10]), bool(v[11]), bool(v[12]), v[13], v[14])


def meta(case):
    return np.array([case.ta, case.tb, case.comp, case.tc, case.m, case.n, case.k, case.lda, case.ldb, case.ldc, case.beta0, case.trans_b,
                     case.vnni_a, case.br_type, case.br], np.int64)
