"""Dense GEMM/BRGEMM test-case description and seeded operand construction (host side, numpy)."""
import ctypes as C
import itertools

import numpy as np

import gen

FLAG_TRANS_A, FLAG_TRANS_B, FLAG_BETA_0, FLAG_VNNI_A, FLAG_VNNI_B, FLAG_VNNI_C = 1, 2, 4, 256, 512, 1024


class GemmCase:
    def __init__(self, m, n, k, ta, tb, tcomp, tc, flags=0, br_type=0, br=1, lda=None, ldb=None, ldc=None, pad=0):
        self.m, self.n, self.k = m, n, k
        self.ta, self.tb, self.tcomp, self.tc = ta, tb, tcomp, tc
        self.flags, self.br_type, self.br = flags, br_type, (br if br_type else 1)
        trans_a, trans_b = bool(flags & FLAG_TRANS_A), bool(flags & FLAG_TRANS_B)
        honours_a = ta in (gen.F64, gen.F32, gen.BF16, gen.BF8, gen.HF8)
        honours_b = tb in (gen.F64, gen.F32, gen.BF16, gen.F16, gen.BF8, gen.HF8)
        self.rows_a = k if (trans_a and honours_a) else m          # leading extent
        self.cols_a = m if (trans_a and honours_a) else k
        self.rows_b = n if (trans_b and honours_b) else k
        self.cols_b = k if (trans_b and honours_b) else n
        self.lda = lda if lda is not None else self.rows_a + pad
        self.ldb = ldb if ldb is not None else self.rows_b + pad
        self.ldc = ldc if ldc is not None else m + pad
        self.size_a, self.size_b, self.size_c = self.cols_a * self.lda, self.cols_b * self.ldb, n * self.ldc

    @property
    def dims(self):
        return (self.m, self.n, self.k, self.lda, self.ldb, self.ldc)

    @property
    def types(self):
        return (self.ta, self.tb, self.tcomp, self.tc)

    def __repr__(self):
        return "gemm(m%d n%d k%d ld%d/%d/%d t%s f%d br%d x%d)" % (self.m, self.n, self.k, self.lda, self.ldb, self.ldc,
                                                                 self.types, self.flags, self.br_type, self.br)


class Operands:
    """Host operands of `count` independent tiles. Stride mode lays the br blocks of a tile out back to back."""

    def __init__(self, case, seed=555, count=1):
        rng = np.random.default_rng(seed)
        c = case
        nblk = c.br if c.br_type in (2, 3) else 1
        self.blk_a, self.blk_b = c.size_a * gen.TS[c.ta], c.size_b * gen.TS[c.tb]       # bytes per block
        if c.br_type == 1:   # address mode: blocks live in a pool, per-tile pointer arrays select them
            self.pool_a = gen.values(rng, c.size_a * c.br * count, c.ta)
            self.pool_b = gen.values(rng, c.size_b * c.br * count, c.tb)
            self.a, self.b = self.pool_a, self.pool_b
        else:
            self.a = gen.values(rng, c.size_a * nblk * count, c.ta)
            self.b = gen.values(rng, c.size_b * nblk * count, c.tb)
        self.c0 = gen.values(rng, c.size_c * count, c.tc)                                 # initial C (beta=1 input)
        self.tile_a, self.tile_b = self.blk_a * (c.br if c.br_type else 1), self.blk_b * (c.br if c.br_type else 1)
        self.tile_c = c.size_c * gen.TS[c.tc]
        self.stride_a = self.blk_a if c.br_type == 3 else 0
        self.stride_b = self.blk_b if c.br_type == 3 else 0
        self.offs_a = self.offs_b = None
        if c.br_type == 2:   # shuffled block order to make the offsets non-trivial
            perm = rng.permutation(c.br)
            self.offs_a = (perm * self.blk_a).astype(np.int64)
            self.offs_b = (perm[::-1] * self.blk_b).astype(np.int64)
        self.scf = 0.125 if (c.tc == gen.F32 and c.ta in (gen.I8, gen.U8)) else 0.0
        self.count = count

    def addr_arrays(self, base_a, base_b, tile):
        """ctypes void*[br] arrays for tile `tile` given the base addresses of the pools."""
        c = self.case_br
        arr_a = (C.c_void_p * c)(*[base_a + (tile * c + r) * self.blk_a for r in range(c)])
        arr_b = (C.c_void_p * c)(*[base_b + (tile * c + (c - 1 - r)) * self.blk_b for r in range(c)])
        return arr_a, arr_b


def ref_result(side, case, ops, run_gemm):
    """C after one invocation per tile computed by `side` (oracle/ref dict); returns a numpy copy."""
    c = ops.c0.copy()
    ops.case_br = case.br
    for t in range(ops.count):
        cv = c[t * case.size_c:(t + 1) * case.size_c]
        if case.br_type == 1:
            aa, ab = ops.addr_arrays(ops.a.ctypes.data, ops.b.ctypes.data, t)
            rc = run_gemm(side, case.dims, case.types, case.flags, 1, 0, 0, case.br, aa, ab, cv, scf=ops.scf)
        else:
            av = ops.a[t * (ops.tile_a // gen.TS[case.ta]):]
            bv = ops.b[t * (ops.tile_b // gen.TS[case.tb]):]
            rc = run_gemm(side, case.dims, case.types, case.flags, case.br_type, ops.stride_a, ops.stride_b, case.br, av, bv, cv,
                          offs_a=ops.offs_a, offs_b=ops.offs_b, scf=ops.scf)
        assert rc == 0, (case, rc)
    return c


# precision tuples (A, B, COMP, C) required by the first bar (SURVEY.md appendix D, bold entries)
TUPLES = [
    (gen.F64, gen.F64, gen.F64, gen.F64), (gen.F32, gen.F32, gen.F32, gen.F32),
    (gen.BF16, gen.BF16, gen.F32, gen.F32), (gen.BF16, gen.BF16, gen.F32, gen.BF16),
    (gen.F16, gen.F16, gen.F32, gen.F16), (gen.F16, gen.F16, gen.F32, gen.F32),
    (gen.U8, gen.I8, gen.I32, gen.I32), (gen.I8, gen.U8, gen.I32, gen.I32), (gen.U8, gen.U8, gen.I32, gen.I32),
    (gen.I8, gen.I8, gen.I32, gen.I32), (gen.I8, gen.I8, gen.I32, gen.F32), (gen.U8, gen.I8, gen.I32, gen.F32),
    (gen.I16, gen.I16, gen.I32, gen.I32),
    # 8-bit float A (SURVEY.md 8f-2): B and C of the same type or f32, and the mixed form with a bf16 B
    (gen.BF8, gen.BF8, gen.F32, gen.F32), (gen.BF8, gen.BF8, gen.F32, gen.BF8), (gen.HF8, gen.HF8, gen.F32, gen.F32), (gen.HF8, gen.HF8, gen.F32, gen.HF8),
    (gen.BF8, gen.BF16, gen.F32, gen.F32), (gen.BF8, gen.BF16, gen.F32, gen.BF16), (gen.HF8, gen.BF16, gen.F32, gen.F32), (gen.HF8, gen.BF16, gen.F32, gen.BF16),
]


def flag_variants(t):
    ta = t[0]
    out = [0]
    if ta in (gen.F64, gen.F32):
        out += [FLAG_TRANS_A, FLAG_TRANS_B, FLAG_TRANS_A | FLAG_TRANS_B]
    elif ta == gen.BF16:
        out += [FLAG_VNNI_A, FLAG_TRANS_A, FLAG_TRANS_B, FLAG_VNNI_A | FLAG_TRANS_B]
    elif ta == gen.F16:
        out += [FLAG_VNNI_A, FLAG_TRANS_B]
    elif ta in (gen.I8, gen.U8):
        out = [FLAG_VNNI_A] if t[3] == gen.F32 else [FLAG_VNNI_A, 0]
    elif ta == gen.I16:
        out += [FLAG_VNNI_A]
    elif ta in (gen.BF8, gen.HF8):
        out += [FLAG_VNNI_A, FLAG_TRANS_B, FLAG_VNNI_A | FLAG_TRANS_B, FLAG_TRANS_A]
    return out


def small_cases(seed=7):
    """The reference's own test matrix in miniature (samples/xgemm/kernel_test/*.tpl): random m,n,k, eqld/gtld,
    beta 0/1, the four batch-reduce modes, per-precision layout flags."""
    rng = np.random.default_rng(seed)
    cases = []
    for t in TUPLES:
        for fl, br_type, beta0, pad in itertools.product(flag_variants(t), (0, 1, 2, 3), (0, 1), (0, 3)):
            m, n = int(rng.integers(1, 40)), int(rng.integers(1, 40))
            k = int(rng.integers(1, 10)) * 4
            flags = fl | (FLAG_BETA_0 if beta0 else 0)
            cases.append(GemmCase(m, n, k, *t, flags=flags, br_type=br_type, br=5, pad=pad))
    return cases


def packed_sp_case(rng, kind, dtype, M, N, K, P, density=0.3):
    """kind: 'a_csr' | 'b_csr' | 'b_csc' | 'c_csc' -> (is_csc, dims, ptr, idx, a, b, c0, which operand holds the values)"""
    rows, cols = {"a_csr": (M, K), "b_csr": (K, N), "b_csc": (K, N), "c_csc": (M, N)}[kind]
    dense = rng.random((rows, cols)) < density
    dense[rng.integers(rows), rng.integers(cols)] = True
    if kind.endswith("csr"):
        ptr = np.concatenate([[0], np.cumsum(dense.sum(1))]).astype(np.uint32); idx = np.nonzero(dense)[1].astype(np.uint32)
    else:
        ptr = np.concatenate([[0], np.cumsum(dense.sum(0))]).astype(np.uint32); idx = np.nonzero(dense.T)[1].astype(np.uint32)
    nnz = len(idx)
    a = gen.values(rng, nnz if kind == "a_csr" else K * max(M, K) * P if kind == "c_csc" else M * K * P, dtype)
    b = gen.values(rng, nnz if kind.startswith("b_") else K * N * P, dtype)
    c0 = gen.values(rng, nnz if kind == "c_csc" else M * N * P, dtype)     # C-sparse: one scalar per non-zero
    dims = {"a_csr": (M, N, K, 0, N, N), "b_csr": (M, N, K, K, 0, N), "b_csc": (M, N, K, K, 0, N), "c_csc": (M, N, K, max(M, K), N, 0)}[kind]
    return int(kind.endswith("csc")), dims, ptr, idx, a, b, c0


RELU, SIGMOID = 5, 9       # libxsmm_meltw_unary_type values the fused GEMM accepts as post-op


def fused_variants():
    """(colbias, cp_op, relu bitmask, vnni_c) like samples/xgemm/kernel_test/gemm_kernel_fused.tpl (BINARY_POSTOP x UNARY_POSTOP x CVNNI)"""
    return [(1, 0, 0, 0), (0, RELU, 0, 0), (0, RELU, 1, 0), (1, RELU, 1, 0), (0, SIGMOID, 0, 0), (1, SIGMOID, 0, 0), (1, RELU, 0, 1), (0, 0, 0, 1)]


def run_gemm_ext(side, case, ops, fuse, colbias, mask, c):
    """one fused call on tile 0 of `ops` (stride / plain modes); c in/out"""
    from oracle_ffi import iarr
    return side["gemm_ext"](iarr(*case.dims), iarr(*case.types), case.flags, case.br_type, ops.stride_a, ops.stride_b, case.br,
                            ops.a.ctypes.data, ops.b.ctypes.data, c.ctypes.data, None, None, ops.scf, iarr(*fuse),
                            colbias.ctypes.data if colbias is not None else None, mask.ctypes.data if mask is not None else None)


def packed_dense_case(rng, kind, dtype, M, N, K, P, pad=0):
    """kind 0: C[n][m][p] += A[k][m][p] B[n][k][p]; 1 (ac_rm): C[m][n][p] += A[m][k][p] B[k][n]; 2 (bc_rm): C[m][n][p] += A[m][k] B[k][n][p]"""
    if kind == 0:
        lda, ldb, ldc = M + pad, K + pad, M + pad
        a = gen.values(rng, K * lda * P, dtype); b = gen.values(rng, N * ldb * P, dtype); c0 = gen.values(rng, N * ldc * P, dtype)
    else:
        lda, ldb, ldc = K + pad, N + pad, N + pad
        a = gen.values(rng, M * lda * (P if kind == 1 else 1), dtype); b = gen.values(rng, K * ldb * (1 if kind == 1 else P), dtype)
        c0 = gen.values(rng, M * ldc * P, dtype)
    return (M, N, K, lda, ldb, ldc), a, b, c0


# ---- fsspmdm "family E", exact by construction: A, B and the old C are dyadic on one grid 2^-q and every element satisfies
# sum_z |v_z b| + |c0| < 2^(p - q) (p = 24 for f32, 53 for f64). Every partial sum is then a value of the type, so the result cannot
# depend on the summation order: any correct kernel equals the float64 reference bit for bit. A is +-(1..7)/8, alpha is 1, -2 or 0.75
# (the folded values stay on the grid 2^-5), B has `fb` fraction bits, |c0| <= 2 on the grid 2^-q.
FSSPMDM_EXACT = {gen.F32: (24, 9, 4), gen.F64: (53, 25, 20)}     # dtype -> (p, q, fb)
FSSPMDM_EXACT_ALPHAS = (1.0, -2.0, 0.75)


def fsspmdm_pattern(rng, M, K, density=None, row_nnz=None):
    """boolean M x K pattern: Bernoulli(density), or exactly row_nnz[i] non-zeros in row i"""
    if row_nnz is None:
        return rng.random((M, K)) < density
    mask = np.zeros((M, K), dtype=bool)
    for i, z in enumerate(row_nnz):
        mask[i, rng.choice(K, size=z, replace=False)] = True
    return mask


def fsspmdm_exact_operands(rng, dtype, mask, N, ldb, ldc, alpha, lda=None):
    """(a [M][lda], b [K][ldb], c0 [M][ldc]) of family E; columns N.. of B and C hold NaN"""
    p, q, fb = FSSPMDM_EXACT[dtype]
    npdt = gen.NP_OF[dtype]
    M, K = mask.shape
    lda = lda or K
    a = np.zeros((M, lda), dtype=npdt)
    a[:, :K] = np.where(mask, rng.integers(1, 8, size=(M, K)) * rng.choice([-1.0, 1.0], size=(M, K)), 0.0) / 8.0
    bmax = 2 ** (fb + 1) - 1
    b = np.full((K, ldb), np.nan, dtype=npdt)
    for k in range(K):                                         # row by row: N may be 10^6
        b[k, :N] = rng.integers(-bmax, bmax + 1, size=N) * 2.0 ** -fb
    c0 = np.full((M, ldc), np.nan, dtype=npdt)
    for i in range(M):
        c0[i, :N] = rng.integers(-2 ** (q + 1), 2 ** (q + 1) + 1, size=N) * 2.0 ** -q
    worst = np.abs(fsspmdm_fold(dtype, a[:, :K], alpha)).sum(axis=1).max() * bmax * 2.0 ** -fb + 2.0
    assert worst < 2.0 ** (p - q), ("family E bound", worst)
    return a, b, c0


def fsspmdm_fold(dtype, a, alpha):
    """A (M x K) with alpha folded in as libxsmm_fsspmdm_create does it (f32: float32(alpha) * a in float32), as float64"""
    if dtype == gen.F32:
        return (np.float32(alpha) * np.asarray(a, dtype=np.float32)).astype(np.float64)
    return np.float64(alpha) * np.asarray(a, dtype=np.float64)


def fsspmdm_reference(v, b, c0, N, beta, magnitude=True, chunk=1 << 16):
    """float64 beta*C0 + V B over columns 0..N-1 (V = folded A, M x K) and, if asked for, the per-element magnitude sum
    |V||B| + |beta C0|; column chunk by column chunk"""
    M, K = v.shape
    exact, mag = np.empty((M, N)), (np.empty((M, N)) if magnitude else None)
    av = np.abs(v)
    for j0 in range(0, N, chunk):
        j1 = min(N, j0 + chunk)
        bj = b[:K, j0:j1].astype(np.float64)
        cj = c0[:, j0:j1].astype(np.float64) if beta else np.zeros((M, j1 - j0))
        exact[:, j0:j1] = v @ bj + cj
        if magnitude:
            mag[:, j0:j1] = av @ np.abs(bj) + np.abs(cj)
    return exact, mag
