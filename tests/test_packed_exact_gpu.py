"""The EDGE/SeisSol packed kernels (A-sparse CSR, B-sparse CSR / CSC, C-sparse CSC, the three packed dense layouts) and the f32
BCSC exact-order kernel, pinned byte for byte to the oracle, which states the reference's JIT on an FMA host: one fused
multiply-add per product, in the reference's order (oracle/oracle.c).

CPU half (no GPU): the witnesses below are built so that a kernel that rounds the product and the sum separately, or sums in
another order, gives other bits; numpy restatements of those wrong kernels are shown to disagree with the oracle on them.
GPU half: the same witnesses, then shapes and edges (packed widths 1 to 100, M, N or K = 1, padded leading dimensions whose
sentinel must survive, beta 0 and 1, empty rows and block columns, subnormals, signed zeros, infinities), on device operands and
on host operands through the staging path, which kernel family ran, and strided batches up to 70,000 calls. NaN results compare
as "is NaN": payloads differ between x86 and CUDA."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

import cases
import gen
from oracle_ffi import iarr, oracle

F32, F64 = gen.F32, gen.F64
NP = {F32: np.float32, F64: np.float64}
SENTINEL = -6.5e29          # written into every padding element of C; must come back unchanged
KINDS = ("a_csr", "b_csr", "b_csc", "c_csc")
DENSE = ("pk_gemm", "pk_ac_rm", "pk_bc_rm")


# ---------------------------------------------------------------------------------------------------------------------------
# operands
def full_values(rng, n, dtype, specials=False):
    """values with full significands over a few binades (so most products are inexact); with specials, about 3 % are replaced by
    +-0, subnormals (and operands whose products are subnormal), +-Inf and NaN"""
    t = NP[dtype]
    v = (rng.standard_normal(n) * np.exp2(rng.integers(-3, 4, size=n))).astype(t)
    if specials and n:
        tiny = np.finfo(t).smallest_subnormal
        pool = np.array([0.0, -0.0, tiny, -tiny * 3, np.finfo(t).tiny * 0.75, -np.finfo(t).tiny / 3, np.inf, -np.inf, np.nan,
                         np.finfo(t).tiny * 1.5, 2.0 ** (-70 if dtype == F32 else -530)], dtype=t)
        pick = rng.random(n) < 0.03
        v[pick] = pool[rng.integers(len(pool), size=int(pick.sum()))]
    return v


def same(got, want):
    """byte equality, except that a NaN matches any NaN"""
    got, want = np.asarray(got), np.asarray(want)
    nan_g, nan_w = np.isnan(got), np.isnan(want)
    if not np.array_equal(nan_g, nan_w):
        return False
    keep = ~nan_w
    return np.array_equal(got[keep].view(np.uint8), want[keep].view(np.uint8))


def csr(mask):
    return np.concatenate([[0], np.cumsum(mask.sum(1))]).astype(np.uint32), np.nonzero(mask)[1].astype(np.uint32)


class Packed:
    """one packed sparse or dense call with its operands; pad elements of padding in every leading dimension"""

    def __init__(self, kind, dtype, M, N, K, P, mask=None, pad=0, beta0=0, a=None, b=None, c0=None, rng=None, specials=False):
        self.kind, self.dtype, self.P, self.flags = kind, dtype, P, (cases.FLAG_BETA_0 if beta0 else 0)
        self.M, self.N, self.K = M, N, K
        rng = rng if rng is not None else np.random.default_rng(0)
        self.ptr = self.idx = None
        if kind == "a_csr":
            self.ptr, self.idx = csr(mask)
            ldb = ldc = N + pad
            self.dims = (M, N, K, 0, ldb, ldc)
            sa, sb, sc = len(self.idx), K * ldb * P, M * ldc * P
        elif kind in ("b_csr", "b_csc"):
            self.ptr, self.idx = csr(mask if kind == "b_csr" else mask.T)
            lda, ldc = K + pad, N + pad
            self.dims = (M, N, K, lda, 0, ldc)
            sa, sb, sc = M * lda * P, len(self.idx), M * ldc * P
        elif kind == "c_csc":
            self.ptr, self.idx = csr(mask.T)
            lda, ldb = max(M, K) + pad, N + pad
            self.dims = (M, N, K, lda, ldb, 0)
            sa, sb, sc = K * lda * P, K * ldb * P, len(self.idx)
        else:
            d = DENSE.index(kind)
            if d == 0:
                lda, ldb, ldc = M + pad, K + pad, M + pad
                sa, sb, sc = K * lda * P, N * ldb * P, N * ldc * P
            else:
                lda, ldb, ldc = K + pad, N + pad, N + pad
                sa, sb, sc = M * lda * (P if d == 1 else 1), K * ldb * (1 if d == 1 else P), M * ldc * P
            self.dims = (M, N, K, lda, ldb, ldc)
        self.a = a if a is not None else full_values(rng, sa, dtype, specials)
        self.b = b if b is not None else full_values(rng, sb, dtype, specials)
        self.c0 = c0 if c0 is not None else full_values(rng, sc, dtype, specials)
        assert (self.a.size, self.b.size, self.c0.size) == (sa, sb, sc)
        self.c0 = self.c0.copy()
        pad_c = self.c_padding()
        if pad_c is not None:
            self.c0[pad_c] = SENTINEL

    def c_padding(self):
        """boolean mask of C's padding elements (None for C-sparse)"""
        M, N, P = self.M, self.N, self.P
        if self.kind == "c_csc":
            return None
        ldc = self.dims[5]
        if self.kind == "pk_gemm":
            col = np.arange(ldc)[None, :, None] >= M
            return np.broadcast_to(col, (N, ldc, P)).ravel().copy()
        col = np.arange(ldc)[None, :, None] >= N
        return np.broadcast_to(col, (M, ldc, P)).ravel().copy()

    def create(self):
        import libxsmm_b200 as X
        dt = self.dtype
        sh = X.libxsmm_create_gemm_shape(*self.dims, dt, dt, dt, dt)
        if self.kind in DENSE:
            fn = (X.libxsmm_create_packed_gemm, X.libxsmm_create_packed_gemm_ac_rm, X.libxsmm_create_packed_gemm_bc_rm)[DENSE.index(self.kind)]
            return fn(sh, self.flags, 0, self.P)
        fn = X.libxsmm_create_packed_spgemm_csc if self.kind.endswith("csc") else X.libxsmm_create_packed_spgemm_csr
        vals = self.a if self.kind == "a_csr" else self.b if self.kind.startswith("b_") else self.c0
        return fn(sh, self.flags, 0, self.P, self.ptr.ctypes.data, self.idx.ctypes.data, vals.ctypes.data)

    def oracle(self, a=None, b=None, c=None):
        a = self.a if a is None else a
        b = self.b if b is None else b
        c = self.c0.copy() if c is None else c
        if self.kind in DENSE:
            rc = oracle["packed_dense"](DENSE.index(self.kind), self.dtype, iarr(*self.dims), self.flags, self.P, a.ctypes.data, b.ctypes.data, c.ctypes.data)
        else:
            rc = oracle["packed_sp"](int(self.kind.endswith("csc")), self.dtype, iarr(*self.dims), self.flags, self.P, self.ptr.ctypes.data,
                                     self.idx.ctypes.data, None, a.ctypes.data, b.ctypes.data, c.ctypes.data)
        assert rc == 0, (self.kind, self.dims, self.P)
        return c

    def run_gpu(self):
        """device operands and host operands (staging path) -> the two C images; checks which kernel family ran"""
        import libxsmm_b200 as X
        from gpu_util import dev, host
        k = self.create()
        assert k, (self.kind, self.dims, self.P)
        assert X.libxsmm_b200_kernel_backend(k) == X.BACKEND_STREAM
        d_a, d_b, d_c = dev(self.a), dev(self.b), dev(self.c0)
        before = X.libxsmm_b200_launch_count_backend(X.BACKEND_STREAM)
        X.call_gemm(k, d_a, d_b, d_c); X.check()
        assert X.libxsmm_b200_launch_count_backend(X.BACKEND_STREAM) == before + 1
        got = host(d_c, NP[self.dtype])
        c_h = self.c0.copy()
        X.call_gemm(k, self.a.ctypes.data, self.b.ctypes.data, c_h.ctypes.data); X.check()
        X.libxsmm_release_kernel(k)
        return got, c_h

    def check_gpu(self, want=None):
        want = self.oracle() if want is None else want
        got, got_h = self.run_gpu()
        what = (self.kind, self.dtype, self.dims, self.P, self.flags)
        assert same(got, want), what
        assert same(got_h, want), what + ("host operands",)
        pad_c = self.c_padding()
        if pad_c is not None:
            assert np.all(got[pad_c] == NP[self.dtype](SENTINEL)), what + ("padding",)
        return got


class Bcsc:
    """one f32 BCSC call: keep[j][kb] says whether block (kb, j) is stored"""

    def __init__(self, mblocks, M, K, N, bk, bn, keep, beta0=0, trans_a=0, a=None, bvals=None, c0=None, rng=None, specials=False):
        rng = rng if rng is not None else np.random.default_rng(0)
        self.geo, self.flags = (mblocks, M, K, N, bk, bn), (cases.FLAG_BETA_0 if beta0 else 0) | (cases.FLAG_TRANS_A if trans_a else 0)
        self.colptr, rowidx = csr(np.asarray(keep, dtype=bool))
        self.rowidx = rowidx if rowidx.size else np.zeros(1, dtype=np.uint32)
        nnzb = int(self.colptr[-1])
        self.a = a if a is not None else full_values(rng, mblocks * K * M, F32, specials)
        self.bvals = bvals if bvals is not None else full_values(rng, max(nnzb, 1) * bk * bn, F32, specials)
        self.c0 = (c0 if c0 is not None else full_values(rng, mblocks * N * M, F32, specials)).copy()

    def oracle(self):
        c = self.c0.copy()
        assert oracle["bcsc"](iarr(F32, F32, F32, F32), iarr(*self.geo), self.flags, self.a.ctypes.data, self.bvals.ctypes.data,
                              self.colptr.ctypes.data, self.rowidx.ctypes.data, c.ctypes.data) == 0
        return c

    def check_gpu(self, want=None):
        import libxsmm_b200 as X
        from gpu_util import dev, host
        want = self.oracle() if want is None else want
        mblocks, M, K, N, bk, bn = self.geo
        k = X.libxsmm_create_packed_spgemm_bcsc(X.libxsmm_create_gemm_shape(mblocks, 0, K, K, 0, N, F32, F32, F32, F32), self.flags, 0,
                                                X.SpgemmConfig(M, bk, bn))
        assert k, self.geo
        assert X.libxsmm_b200_bcsc_variant(k, N // bn) == 0
        d_a, d_b, d_cp, d_ri, d_c = dev(self.a), dev(self.bvals), dev(self.colptr), dev(self.rowidx), dev(self.c0)
        before = X.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT)
        X.call_gemm(k, d_a, d_b, d_c, colptr=d_cp, rowidx=d_ri, nblocks=N // bn); X.check()
        assert X.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT) == before + 1
        got = host(d_c, np.float32)
        c_h = self.c0.copy()
        X.call_gemm(k, self.a.ctypes.data, self.bvals.ctypes.data, c_h.ctypes.data, colptr=self.colptr, rowidx=self.rowidx, nblocks=N // bn)
        X.check()
        X.libxsmm_release_kernel(k)
        assert same(got, want), (self.geo, self.flags)
        assert same(c_h, want), (self.geo, self.flags, "host operands")
        return got


# ---------------------------------------------------------------------------------------------------------------------------
# FMA witnesses: every element is one product a*b added to c0 = -round(a*b). With one FMA the result is the exact rounding
# residual a*b - round(a*b), which is non-zero wherever the product is inexact; multiply-then-add gives exactly 0 everywhere.
def residual(a, b, dtype):
    """exact a*b - round(a*b) per element (representable: the error of a rounded product is a value of the type)"""
    t = NP[dtype]
    prod = (a.astype(t) * b.astype(t)).astype(t)
    out = np.array([float(Fraction(float(x)) * Fraction(float(y)) - Fraction(float(p))) for x, y, p in zip(a.ravel(), b.ravel(), prod.ravel())], dtype=t)
    return out.reshape(np.shape(a)), prod


def fma_witness(kind, dtype, rng, P=8):
    """(Packed case at beta = 1, expected C from exact arithmetic, share of elements that must be non-zero)"""
    t = NP[dtype]
    M, N, K = 5, 4, 6
    if kind == "a_csr":                       # one non-zero per row: C[i][j][p] = fma(A[z], B[col][j][p], c0)
        mask = np.zeros((M, K), dtype=bool); mask[np.arange(M), rng.integers(K, size=M)] = True
        cs = Packed(kind, dtype, M, N, K, P, mask=mask, rng=rng)
        col = np.nonzero(mask)[1]
        av = np.repeat(cs.a, N * P).reshape(M, N, P)
        bv = cs.b.reshape(K, N, P)[col]
    elif kind in ("b_csr", "b_csc"):          # one non-zero per column j: C[i][j][p] = fma(A[i][row][p], b[z], c0)
        mask = np.zeros((K, N), dtype=bool); mask[rng.integers(K, size=N), np.arange(N)] = True
        cs = Packed(kind, dtype, M, N, K, P, mask=mask, rng=rng)
        row = np.nonzero(mask.T)[1]           # row of column j
        bj = cs.b if kind == "b_csc" else cs.b[np.argsort(np.nonzero(mask)[1], kind="stable")]
        av = cs.a.reshape(M, K, P)[:, row, :]
        bv = np.broadcast_to(bj[None, :, None], (M, N, P))
    else:                                     # packed dense with K = 1
        cs = Packed(kind, dtype, M, N, 1, P, rng=rng)
        if kind == "pk_gemm":                 # C[n][m][p] = A[0][m][p] * B[n][0][p]
            av = np.broadcast_to(cs.a.reshape(M, P)[None], (N, M, P))
            bv = np.broadcast_to(cs.b.reshape(N, P)[:, None], (N, M, P))
        elif kind == "pk_ac_rm":              # C[m][n][p] = A[m][0][p] * B[0][n]
            av = np.broadcast_to(cs.a.reshape(M, 1, P), (M, N, P))
            bv = np.broadcast_to(cs.b.reshape(1, N, 1), (M, N, P))
        else:                                 # C[m][n][p] = A[m][0] * B[0][n][p]
            av = np.broadcast_to(cs.a.reshape(M, 1, 1), (M, N, P))
            bv = np.broadcast_to(cs.b.reshape(1, N, P), (M, N, P))
    res, prod = residual(np.ascontiguousarray(av), np.ascontiguousarray(bv), dtype)
    cs.c0 = (-prod).astype(t).ravel().copy()
    return cs, res.ravel()


def csparse_witness(rng, P=16):
    """C-sparse, beta = 1, C0 = 0: non-zero z gets, in accumulator lane 0, 1 * (-round(x*y)) at k = 0 and x * y at k = 1: the FMA
    leaves the residual, every other lane and product is zero"""
    M, N, K = 3, 4, 2
    mask = np.zeros((M, N), dtype=bool); mask[rng.integers(M, size=N), np.arange(N)] = True
    cs = Packed("c_csc", F32, M, N, K, P, mask=mask, rng=rng)
    lda, ldb = cs.dims[3], cs.dims[4]
    a = np.zeros((K, lda, P), np.float32); b = np.zeros((K, ldb, P), np.float32)
    x = full_values(rng, M, F32); y = full_values(rng, N, F32)
    res, prod = residual(x[:, None] * np.ones((1, N), np.float32), np.ones((M, 1), np.float32) * y[None, :], F32)
    rows = np.nonzero(mask.T)[1]
    for j in range(N):
        i = rows[j]
        a[0, i, 0] = 1.0; b[0, j, 0] = -prod[i, j]
        a[1, i, 0] = x[i]; b[1, j, 0] = y[j]
    cs.a, cs.b, cs.c0 = a.ravel(), b.ravel(), np.zeros(N, np.float32)
    return cs, np.array([res[rows[j], j] for j in range(N)], np.float32)


def bcsc_witness(rng):
    """f32 BCSC, beta = 1: block (0, 0) holds y at k = 0 of every column, A holds x at k = 0; C0 = -round(x*y) in block column 0,
    other k and block columns hold zeros or are empty"""
    mblocks, M, K, N, bk, bn = 2, 16, 16, 32, 8, 16
    keep = np.zeros((N // bn, K // bk), dtype=bool); keep[0, 0] = True; keep[1, 1] = True
    a = np.zeros((mblocks, K, M), np.float32); a[:, 0, :] = full_values(rng, mblocks * M, F32).reshape(mblocks, M)
    bv = np.zeros((2, bn, bk), np.float32); bv[0, :, 0] = full_values(rng, bn, F32)
    xb = np.broadcast_to(a[:, 0, :][:, None, :], (mblocks, bn, M))               # [mb][n][i]
    yb = np.broadcast_to(bv[0, :, 0][None, :, None], (mblocks, bn, M))
    res, prod = residual(np.ascontiguousarray(xb), np.ascontiguousarray(yb), F32)
    c0 = full_values(rng, mblocks * N * M, F32).reshape(mblocks, N, M)
    c0[:, :bn, :] = -prod
    want = c0.copy(); want[:, :bn, :] = res
    cs = Bcsc(mblocks, M, K, N, bk, bn, keep, a=a.ravel(), bvals=bv.ravel(), c0=c0.ravel(), rng=rng)
    return cs, want.ravel()


WITNESS_KINDS = [(k, t) for k in ("a_csr", "b_csr", "b_csc") + DENSE for t in (F32, F64)]


@pytest.mark.parametrize("kind,dtype", WITNESS_KINDS)
def test_fma_witness_rejects_multiply_then_add(kind, dtype):
    rng = np.random.default_rng(100)
    cs, want = fma_witness(kind, dtype, rng)
    got = cs.oracle()
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), "the oracle is not one FMA per product"
    assert np.count_nonzero(want) > 0.5 * want.size
    # multiply-then-add: round(round(a*b) + c0) with c0 = -round(a*b) is exactly zero in every element
    t = NP[dtype]
    mul_add = (-cs.c0 + cs.c0).astype(t)
    assert not np.any(mul_add) and np.count_nonzero(got != mul_add) == np.count_nonzero(want)


def test_fma_witness_csparse_and_bcsc():
    rng = np.random.default_rng(101)
    cs, want = csparse_witness(rng)
    got = cs.oracle()
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8)) and np.count_nonzero(want) >= 3
    bc, want = bcsc_witness(rng)
    got = bc.oracle()
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
    assert np.count_nonzero(want.reshape(2, 32, 16)[:, :16]) > 0.5 * 2 * 16 * 16


# ---------------------------------------------------------------------------------------------------------------------------
# order witnesses: every product is exact (powers of two and small integers), so only the order of the additions matters
BIG = {F32: 2.0 ** 25, F64: 2.0 ** 54}


def order_witness_sparse(kind, dtype):
    """a row (A-CSR) or column (B-CSC / B-CSR) with products 1, BIG, -BIG in z order: ascending gives 0, descending gives 1"""
    t = NP[dtype]
    M, N, K, P = 2, 3, 3, 4
    terms = np.array([1.0, BIG[dtype], -BIG[dtype]], t)
    if kind == "a_csr":
        mask = np.ones((M, K), dtype=bool)
        a = np.tile(terms, M).astype(t)
        cs = Packed(kind, dtype, M, N, K, P, mask=mask, a=a, b=np.ones(K * N * P, t), c0=np.zeros(M * N * P, t), beta0=1)
    else:
        mask = np.ones((K, N), dtype=bool)
        b = np.tile(terms, N).astype(t)                  # CSC order = k order; CSR (rows of k) lists the same values for every column
        if kind == "b_csr":
            b = np.repeat(terms, N).astype(t)
        cs = Packed(kind, dtype, M, N, K, P, mask=mask, a=np.ones(M * K * P, t), b=b, c0=np.zeros(M * N * P, t), beta0=1)
    return cs


def order_witness_dense(kind, dtype):
    """K = 3 with products 1, BIG, -BIG in k order"""
    t = NP[dtype]
    M, N, K, P = 2, 2, 3, 4
    terms = np.array([1.0, BIG[dtype], -BIG[dtype]], t)
    cs = Packed(kind, dtype, M, N, K, P, beta0=1)
    d = DENSE.index(kind)
    if d == 0:                                           # A[k][m][p]
        cs.a = np.repeat(terms, M * P).astype(t); cs.b = np.ones(cs.b.size, t)
    elif d == 1:                                         # A[m][k][p] x B[k][n]
        cs.a = np.ones(cs.a.size, t); cs.b = np.repeat(terms, N).astype(t)
    else:                                                # A[m][k] x B[k][n][p]
        cs.a = np.tile(terms, M).astype(t); cs.b = np.ones(cs.b.size, t)
    cs.c0 = np.zeros(cs.c0.size, t)
    return cs


@pytest.mark.parametrize("kind,dtype", WITNESS_KINDS)
def test_order_witness_rejects_descending_order(kind, dtype):
    cs = order_witness_dense(kind, dtype) if kind in DENSE else order_witness_sparse(kind, dtype)
    got = cs.oracle()
    t = NP[dtype]
    asc = (t(1.0) + t(BIG[dtype])) - t(BIG[dtype])
    desc = (t(-BIG[dtype]) + t(BIG[dtype])) + t(1.0)
    assert asc == 0 and desc == 1
    assert np.all(got == asc), "the oracle does not sum in ascending order"
    assert not np.any(got == desc)


def csparse_numpy(cs, lanes=16, fold="ref"):
    """numpy restatement of C-sparse schedules with exact products: `lanes` accumulators (lane p % lanes, k outer), folded by
    'ref' (l + 8, l + 4, (0 + 2) + (1 + 3)), 'tree' (xor butterfly from lanes / 2 down), 'rtree' (butterfly 1, 2, 4, ...) or 'seq'"""
    M, N, K, lda, ldb, _ = cs.dims
    P = cs.P
    A = cs.a.reshape(K, lda, P); B = cs.b.reshape(K, ldb, P)
    rows = cs.idx; out = []
    for j in range(N):
        for z in range(cs.ptr[j], cs.ptr[j + 1]):
            lane = [np.float32(0)] * lanes
            for k in range(K):
                for p in range(P):
                    lane[p % lanes] = np.float32(lane[p % lanes] + np.float32(A[k, rows[z], p] * B[k, j, p]))
            if fold == "ref":
                for l in range(8):
                    lane[l] = np.float32(lane[l] + lane[l + 8])
                for l in range(4):
                    lane[l] = np.float32(lane[l] + lane[l + 4])
                acc = np.float32(np.float32(lane[0] + lane[2]) + np.float32(lane[1] + lane[3]))
            elif fold in ("tree", "rtree"):
                offs = [lanes >> s for s in range(1, lanes.bit_length())]
                for o in (offs if fold == "tree" else offs[::-1]):
                    lane = [np.float32(lane[l] + lane[l ^ o]) for l in range(lanes)]
                acc = lane[0]
            else:
                acc = np.float32(0)
                for v in lane:
                    acc = np.float32(acc + v)
            out.append(acc)
    return np.array(out, np.float32)


def csparse_order_witness():
    """P = 32, K = 2, one non-zero: p = 0 carries BIG, then -BIG at k = 1; p = 16 carries 1 at both k; p = 1 carries 1 and p = 8 -BIG/2
    twice. The 16-lane schedule rounds 1 away against BIG in lane 0, a 32-lane one keeps p = 0 and p = 16 apart, and the fold
    orders meet +-BIG at different points."""
    M, N, K, P = 1, 1, 2, 32
    mask = np.ones((M, N), dtype=bool)
    cs = Packed("c_csc", F32, M, N, K, P, mask=mask, beta0=1)
    lda, ldb = cs.dims[3], cs.dims[4]
    a = np.zeros((K, lda, P), np.float32); b = np.zeros((K, ldb, P), np.float32)
    big = np.float32(2.0 ** 25)
    a[:, 0, :] = 1.0
    b[0, 0, 0], b[1, 0, 0] = big, -big
    b[0, 0, 16], b[1, 0, 16] = 1.0, 1.0
    b[0, 0, 1], b[0, 0, 9] = 1.0, big
    b[1, 0, 8] = -big
    cs.a, cs.b, cs.c0 = a.ravel(), b.ravel(), np.zeros(1, np.float32)
    return cs


def test_order_witness_csparse_rejects_other_schedules():
    cs = csparse_order_witness()
    got = cs.oracle()
    ref16 = csparse_numpy(cs, 16, "ref")
    assert np.array_equal(got, ref16), (got, ref16)       # products are exact: the FMA changes nothing, the order is all
    others = {"32-lane tree": csparse_numpy(cs, 32, "tree"), "16-lane butterfly 1,2,4,8": csparse_numpy(cs, 16, "rtree"),
              "16 lanes summed in sequence": csparse_numpy(cs, 16, "seq")}
    for name, v in others.items():
        assert not np.array_equal(v, got), name


def test_csparse_butterfly_equals_reference_fold():
    """the kernel's half-warp butterfly (offsets 8, 4, 2, 1) forms exactly (l0 + l2) + (l1 + l3) after the 8 and 4 folds: checked on
    random lanes against the reference fold"""
    rng = np.random.default_rng(7)
    for _ in range(200):
        lane = list(full_values(rng, 16, F32))
        ref = [np.float32(lane[l] + lane[l + 8]) for l in range(8)]
        ref = [np.float32(ref[l] + ref[l + 4]) for l in range(4)]
        want = np.float32(np.float32(ref[0] + ref[2]) + np.float32(ref[1] + ref[3]))
        v = lane[:]
        for o in (8, 4, 2, 1):
            v = [np.float32(v[l] + v[l ^ o]) for l in range(16)]
        assert v[0].view(np.uint32) == want.view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
@pytest.mark.gpu
@pytest.mark.parametrize("kind,dtype", WITNESS_KINDS)
def test_gpu_fma_and_order_witnesses(kind, dtype):
    rng = np.random.default_rng(200)
    cs, want = fma_witness(kind, dtype, rng)
    cs.check_gpu(want)
    cs = order_witness_dense(kind, dtype) if kind in DENSE else order_witness_sparse(kind, dtype)
    cs.check_gpu()


@pytest.mark.gpu
def test_gpu_csparse_and_bcsc_witnesses():
    rng = np.random.default_rng(201)
    cs, want = csparse_witness(rng)
    cs.check_gpu(want)
    csparse_order_witness().check_gpu()
    bc, want = bcsc_witness(rng)
    bc.check_gpu(want)


SHAPES = ((5, 4, 6), (1, 7, 5), (6, 1, 5), (7, 5, 1), (20, 9, 35))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ("a_csr", "b_csr", "b_csc") + DENSE)
@pytest.mark.parametrize("dtype", [F32, F64])
def test_gpu_packed_shapes_and_edges(kind, dtype):
    """P in {1, 3, 8, 13, 16, 17, 32, 48, 100}, M, N or K = 1, leading dimensions padded (sentinel must survive), beta 0 and 1,
    special values among the operands; A-CSR with an empty row, B-CSR with columns past the last populated one"""
    rng = np.random.default_rng(300 + 7 * DENSE.index(kind) if kind in DENSE else 300 + KINDS.index(kind))
    for P in (1, 3, 8, 13, 16, 17, 32, 48, 100):
        for (M, N, K) in SHAPES:
            if P >= 32 and M * N > 30:
                continue
            for beta0 in (0, 1):
                pad = (P + M) % 3
                mask = None
                if kind == "a_csr":
                    mask = rng.random((M, K)) < 0.4
                    mask[rng.integers(M), rng.integers(K)] = True
                    if M > 1:
                        mask[M // 2] = False                      # an empty row: untouched, even under BETA_0
                elif kind in ("b_csr", "b_csc"):
                    mask = rng.random((K, N)) < 0.4
                    mask[rng.integers(K), 0] = True
                    if kind == "b_csr" and N > 2:
                        mask[:, N - 2:] = False                   # columns past the last populated one: untouched
                cs = Packed(kind, dtype, M, N, K, P, mask=mask, pad=pad, beta0=beta0, rng=rng, specials=True)
                want = cs.oracle()
                got = cs.check_gpu(want)
                c3 = got.reshape(-1, cs.dims[5], P) if kind != "pk_gemm" else None
                if kind == "a_csr" and M > 1:
                    assert same(c3[M // 2], cs.c0.reshape(-1, cs.dims[5], P)[M // 2]), "empty row written"
                if kind == "b_csr" and N > 2:
                    assert same(c3[:, N - 2:N], cs.c0.reshape(-1, cs.dims[5], P)[:, N - 2:N]), "columns past the last non-zero written"


@pytest.mark.gpu
def test_gpu_csparse_shapes_and_edges():
    """C-sparse: P in {16, 32, 48, 64, 128}, K = 1 and larger, padded lda / ldb, beta 0 and 1, special values"""
    rng = np.random.default_rng(310)
    for P in (16, 32, 48, 64, 128):
        for (M, N, K) in ((5, 4, 6), (1, 6, 3), (6, 1, 4), (7, 5, 1), (20, 9, 35)):
            for beta0 in (0, 1):
                mask = rng.random((M, N)) < 0.5
                mask[rng.integers(M), rng.integers(N)] = True
                Packed("c_csc", F32, M, N, K, P, mask=mask, pad=P % 3 + 1, beta0=beta0, rng=rng, specials=True).check_gpu()


@pytest.mark.gpu
def test_gpu_signed_zeros_and_infinities():
    """+-0 products under beta 0 and 1 (the sign of a zero sum follows the FMA rules), +-Inf operands and Inf - Inf = NaN"""
    rng = np.random.default_rng(320)
    for dtype in (F32, F64):
        t = NP[dtype]
        pool = np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, 2.0 ** -60], t)
        for kind in ("a_csr", "b_csr", "b_csc") + DENSE:
            for beta0 in (0, 1):
                mask = np.ones((3, 4), dtype=bool) if kind == "a_csr" else np.ones((4, 3), dtype=bool) if kind.startswith("b_") else None
                cs = Packed(kind, dtype, 3, 3, 4, 5, mask=mask, beta0=beta0, rng=rng)
                cs.a = pool[rng.integers(len(pool), size=cs.a.size)]
                cs.b = pool[rng.integers(len(pool), size=cs.b.size)]
                cs.c0 = pool[rng.integers(3, size=cs.c0.size)].copy()
                cs.check_gpu()
    for beta0 in (0, 1):
        mask = np.ones((3, 3), dtype=bool)
        cs = Packed("c_csc", F32, 3, 3, 2, 16, mask=mask, beta0=beta0, rng=rng)
        pool = np.array([0.0, -0.0, 1.0, np.inf, -np.inf], np.float32)
        cs.a = pool[rng.integers(len(pool), size=cs.a.size)]; cs.b = pool[rng.integers(3, size=cs.b.size)]
        cs.c0 = np.array([-0.0, 0.0, 1.0] * 3, np.float32)[:cs.c0.size].copy()
        cs.check_gpu()


@pytest.mark.gpu
def test_gpu_bcsc_f32_shapes_and_edges():
    """f32 BCSC on the exact-order kernel: empty block columns, M = 1, bk = bn = 1, TRANS_A, beta 0 and 1, special values"""
    rng = np.random.default_rng(330)
    for (mblocks, M, K, N, bk, bn, dens) in ((3, 16, 64, 48, 16, 16, 0.5), (2, 1, 32, 32, 8, 8, 0.6), (1, 13, 7, 6, 1, 1, 0.5),
                                             (2, 32, 128, 64, 32, 16, 0.3), (4, 8, 32, 32, 8, 8, 0.0), (1, 5, 48, 96, 16, 32, 1.0)):
        for beta0, trans_a in ((1, 0), (0, 0), (1, 1), (0, 1)):
            keep = rng.random((N // bn, K // bk)) < dens
            if dens > 0 and N // bn > 1:
                keep[N // bn - 1] = False                                # an empty block column
            Bcsc(mblocks, M, K, N, bk, bn, keep, beta0=beta0, trans_a=trans_a, rng=rng, specials=True).check_gpu()


BATCH_KINDS = [("a_csr", F32), ("a_csr", F64), ("b_csr", F32), ("b_csr", F64), ("b_csc", F32), ("b_csc", F64), ("c_csc", F32),
               ("pk_gemm", F32), ("pk_gemm", F64), ("pk_ac_rm", F32), ("pk_ac_rm", F64), ("pk_bc_rm", F32), ("pk_bc_rm", F64), ("bcsc", F32)]


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1, 7, 70000])
@pytest.mark.parametrize("kind,dtype", BATCH_KINDS)
def test_gpu_batch_calls_match_oracle(kind, dtype, count):
    """libxsmm_b200_spgemm_batch_strided: one launch on the expected family; spot calls (first, 65,534, 65,535, last) byte for byte
    against the oracle"""
    import torch
    import libxsmm_b200 as X
    from sparse_batch_cases import BcscCase, PackedCase, param
    rng = np.random.default_rng(400 + count)
    if kind == "bcsc":
        case = BcscCase(rng, (F32, F32, F32, F32), count, mblocks=1, M=16, K=32, N=32, bk=16, bn=16, pads=(16, None, 48), beta0=count % 2)
        family = X.BACKEND_SIMT
    else:
        case = PackedCase(rng, kind, dtype, count, M=5, N=4, K=6, P=16 if kind == "c_csc" else 8, pad=1, pads=(8, 8, 8), beta0=count % 2)
        family = X.BACKEND_STREAM
    k = case.create()
    assert k
    d_a, d_b, d_c = [torch.from_numpy(x).cuda() for x in (case.a, case.b, case.c)]
    extra = {}
    if kind == "bcsc":
        d_cp = torch.from_numpy(case.colptr.view(np.int32).copy()).cuda(); d_ri = torch.from_numpy(case.rowidx.view(np.int32).copy()).cuda()
        nbc = C.c_ulonglong(case.nbc)
        extra = dict(colptr=d_cp.data_ptr(), rowidx=d_ri.data_ptr(), nbc=nbc)
    p = param(d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), case.strides, 0, **extra)
    before = X.libxsmm_b200_launch_count_backend(family)
    assert X.libxsmm_b200_spgemm_batch_strided(k, C.byref(p), C.byref(X.SpgemmStrides(*case.strides)), count) == 0
    X.check()
    assert X.libxsmm_b200_launch_count_backend(family) == before + 1
    got = d_c.cpu().numpy()
    for t in sorted({0, count - 1} | ({65534, 65535} if count > 65535 else set())):
        a = case.a[t * case.strides[0]:][:case.nbytes[0]].copy(); b = case.b[t * case.strides[1]:][:case.nbytes[1]].copy()
        want = case.c[t * case.strides[2]:][:case.nbytes[2]].copy()
        assert case.oracle_call(oracle, a, b, want) == 0
        assert np.array_equal(got[t * case.strides[2]:][:case.nbytes[2]], want), (kind, dtype, t)
    X.libxsmm_release_kernel(k)
