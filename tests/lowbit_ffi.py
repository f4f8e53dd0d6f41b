"""TEST INFRASTRUCTURE: the low-bit weight GEMM checkers and operand generator.

  oracle_gemm_lowbit  oracle/liboracle_lowbit.so           plain-C restatement (oracle/oracle_lowbit.c)
  ref_gemm_lowbit     oracle/_ref/libxsmm_ref_lowbit.so    the unmodified reference's libxsmm_reference_gemm (oracle/ref_lowbit_shim.c),
                                                           only where build() could compile it

Both take dims {m,n,k,lda,ldb,ldc}, types {a,b,comp,c}, flags, br_type (0 none / 1 address / 2 offset / 3 stride), stride_a,
stride_b (bytes), br, A, B, C, offs_a, offs_b (bytes), A's E8M0 block scales, B's f32 block scales (address mode: arrays of br
pointers for A, B and both scales)."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle_ffi  # noqa: F401  (builds liboracle.so, which liboracle_lowbit.so links against)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_LB_SO = os.path.join(ROOT, "oracle", "liboracle_lowbit.so")
REF_LB_SO = os.path.join(ROOT, "oracle", "_ref", "libxsmm_ref_lowbit.so")

F32, BF16, I32, I8, U8, MXFP4, I2, I1 = 1, 2, 8, 12, 13, 20, 22, 23
TRANS_A, TRANS_B, BETA_0, VNNI_A, VNNI_B, VNNI_C, INTLV_A = 1, 2, 4, 256, 512, 1024, 262144
NAMES = {F32: "F32", BF16: "BF16", I32: "I32", I8: "I8", U8: "U8", MXFP4: "MXFP4", I2: "I2", I1: "I1"}
# the six tuples (A, B, C), comp I32 throughout
TUPLES = [(I2, I8, I32), (I2, U8, I32), (I1, I8, I32), (I1, U8, I32), (MXFP4, I8, F32), (MXFP4, I8, BF16)]

if not os.path.exists(ORACLE_LB_SO) or os.path.getmtime(ORACLE_LB_SO) < os.path.getmtime(os.path.join(ROOT, "oracle", "oracle_lowbit.c")):
    subprocess.check_call(["make", "-C", ROOT, "oracle"], stdout=subprocess.DEVNULL)

_P = C.c_void_p
_ARGS = [_P, _P, C.c_uint, C.c_int, C.c_longlong, C.c_longlong, C.c_ulonglong, _P, _P, _P, _P, _P, _P, _P]
_oracle_lib = C.CDLL(ORACLE_LB_SO)
_oracle_lib.oracle_gemm_lowbit.restype, _oracle_lib.oracle_gemm_lowbit.argtypes = C.c_int, _ARGS
oracle_gemm_lowbit = _oracle_lib.oracle_gemm_lowbit
ref_gemm_lowbit = None
if os.path.exists(REF_LB_SO):
    _ref_lib = C.CDLL(REF_LB_SO)
    _ref_lib.ref_gemm_lowbit.restype, _ref_lib.ref_gemm_lowbit.argtypes = C.c_int, _ARGS
    ref_gemm_lowbit = _ref_lib.ref_gemm_lowbit


def default_flags(ta):
    return VNNI_A if ta == I1 else (VNNI_A | INTLV_A)


class LbCase:
    """one low-bit GEMM call. A (bytes, per block): I2 [k/4][lda], I1 [k/4][lda/2], MXFP4 [k/8][lda][4]; B [br][n][ldb] bytes; C [n][ldc]
    (int32, f32 or bf16). MXFP4 scales: A's E8M0 bytes [br][k/32][lda], B's f32 blocks of n*ldb/32 floats each ([n][ldb/32] used).
    Block r of A / B sits right after block r-1; offset mode visits the blocks in reverse order, address mode through arrays of
    pointers to them (and to their scales)."""

    def __init__(self, ta, tb, tc, m, n, k, lda=None, ldb=None, ldc=None, beta0=True, br_type=0, br=1, flags=None):
        self.ta, self.tb, self.tc, self.m, self.n, self.k = ta, tb, tc, m, n, k
        self.lda, self.ldb, self.ldc = lda or m, ldb or k, ldc or m
        self.beta0, self.br_type, self.br = beta0, br_type, (br if br_type else 1)
        self.flags = (default_flags(ta) if flags is None else flags) | (BETA_0 if beta0 else 0)
        self.dims = (C.c_int * 6)(m, n, k, self.lda, self.ldb, self.ldc)
        self.types = (C.c_int * 4)(ta, tb, I32, tc)
        self.block_a = {I2: (k // 4) * self.lda, I1: (k // 4) * (self.lda // 2), MXFP4: (k // 8) * self.lda * 4}[ta]
        self.block_b = self.ldb * n
        self.block_sa = (k // 32) * self.lda                    # bytes: stride and offset modes move A's scales by block_a * 2 / 32
        self.block_sb = self.block_b // 32                      # floats: ... and B's by block_b / 32
        self.size_a, self.size_b, self.size_c = self.br * self.block_a, self.br * self.block_b, self.ldc * n
        self.size_sa = self.br * self.block_sa
        self.size_sb = self.br * (self.block_sb + 1) + n * (self.ldb // 32)
        self.stride_a = self.block_a if br_type == 3 else 0
        self.stride_b = self.block_b if br_type == 3 else 0
        self.c_dtype = {I32: np.int32, F32: np.float32, BF16: np.uint16}[tc]

    def __repr__(self):
        return "Lb(%s.%s.%s,%dx%dx%d,ld %d/%d/%d,beta0=%d,br %d/%d,flags %#x)" % (
            NAMES[self.ta], NAMES[self.tb], NAMES[self.tc], self.m, self.n, self.k, self.lda, self.ldb, self.ldc, self.beta0, self.br_type,
            self.br, self.flags)

    def mx(self):
        return self.ta == MXFP4

    def operands(self, rng):
        """A: every byte value (so every 2-bit code, bit pattern and table entry); B: 8-bit values with both extremes; C: any value;
        MXFP4 scales: E8M0 bytes near 127 with 0 and 254 mixed in, f32 B scales of both signs with zeros"""
        A = rng.permutation(np.resize(np.arange(256, dtype=np.uint8), self.size_a))
        B = rng.integers(0, 256, self.size_b, dtype=np.uint8)
        B[rng.random(self.size_b) < 0.05] = 0x80 if self.tb == I8 else 0xFF
        B[rng.random(self.size_b) < 0.05] = 0x7F if self.tb == I8 else 0x00
        if self.tc == I32:
            C0 = rng.integers(-2 ** 31, 2 ** 31, self.size_c, dtype=np.int64).astype(np.int32)
            C0[: min(4, self.size_c)] = [2 ** 31 - 1, -2 ** 31, -1, 0][: min(4, self.size_c)]   # wrap-around at the extremes
        elif self.tc == F32:
            C0 = rng.standard_normal(self.size_c).astype(np.float32)
        else:
            C0 = (rng.standard_normal(self.size_c).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
        SA = rng.integers(112, 140, self.size_sa, dtype=np.uint8) if self.mx() else np.zeros(1, np.uint8)
        SB = (rng.standard_normal(self.size_sb) * 0.5).astype(np.float32) if self.mx() else np.zeros(1, np.float32)
        if self.mx():
            pick = rng.random(self.size_sa)
            SA[pick < 0.04] = 0
            SA[pick > 0.97] = 254
            SB[rng.random(self.size_sb) < 0.05] = 0.0
        return A, B, C0, SA, SB

    def run(self, fn, A, B, C0, SA, SB):
        """runs oracle_gemm_lowbit or ref_gemm_lowbit on a copy of C; returns (rc, C)"""
        c = C0.copy()
        a_arg, b_arg, sa_arg, sb_arg, oa, ob, keep = A.ctypes.data, B.ctypes.data, SA.ctypes.data, SB.ctypes.data, None, None, []
        if self.br_type == 1:
            arrs = [(C.c_void_p * self.br)(*[base + r * step for r in range(self.br)])
                    for base, step in ((A.ctypes.data, self.block_a), (B.ctypes.data, self.block_b), (SA.ctypes.data, self.block_sa),
                                       (SB.ctypes.data, 4 * self.block_sb))]
            keep += arrs
            a_arg, b_arg, sa_arg, sb_arg = [C.addressof(x) for x in arrs]
        elif self.br_type == 2:
            oa_ = np.array([(self.br - 1 - r) * self.block_a for r in range(self.br)], np.int64)
            ob_ = np.array([(self.br - 1 - r) * self.block_b for r in range(self.br)], np.int64)
            keep += [oa_, ob_]
            oa, ob = oa_.ctypes.data, ob_.ctypes.data
        rc = fn(self.dims, self.types, self.flags, self.br_type, self.stride_a, self.stride_b, self.br, a_arg, b_arg, c.ctypes.data,
                oa, ob, sa_arg if self.mx() else None, sb_arg if self.mx() else None)
        return rc, c

    def nan_mask(self, c):
        c = np.asarray(c)
        if self.tc == I32:
            return np.zeros(c.shape, bool)
        if self.tc == F32:
            return np.isnan(c.view(np.float32))
        h = c.view(np.uint16)
        return ((h & 0x7F80) == 0x7F80) & ((h & 0x7F) != 0)


def same_c(case, want, got):
    """two C images equal bit for bit, NaN positions excepted (both must be NaN there): the sign and payload of a NaN made from
    inf - inf (a scale byte of 254 overflows) is the host's choice (x86's default NaN is negative)"""
    w, g = np.asarray(want).view(case.c_dtype), np.asarray(got).view(case.c_dtype)
    nan = case.nan_mask(w)
    bits = np.uint16 if case.tc == BF16 else np.uint32
    return bool(np.array_equal(case.nan_mask(g), nan) and np.array_equal(w.view(bits)[~nan], g.view(bits)[~nan]))


def meta(case):
    return np.array([case.ta, case.tb, case.tc, case.m, case.n, case.k, case.lda, case.ldb, case.ldc, case.beta0, case.br_type, case.br,
                     case.flags & ~BETA_0], np.int64)


def case_from_meta(v):
    v = [int(x) for x in v]
    return LbCase(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7], v[8], bool(v[9]), v[10], v[11], v[12])
