"""Operands of strided batches of packed-sparse, packed-dense and BCSC calls (libxsmm_b200_spgemm_batch_strided), shared by the
simulated-device and the GPU tests. A case holds one handle's geometry and, per operand, a byte image of `count` calls at its
stride: each call's values, then poison (0xA5) up to the stride. A stride of 0 is one operand shared by every call."""
import ctypes as C

import numpy as np

import cases
import gen
import libxsmm_b200 as X

PACKED_KINDS = ("a_csr", "b_csr", "b_csc", "c_csc", "pk_gemm", "pk_ac_rm", "pk_bc_rm")
DENSE = {"pk_gemm": 0, "pk_ac_rm": 1, "pk_bc_rm": 2}
POISON = 0xA5


def values(rng, n, dtype):
    """n elements of `dtype` on the tenths grid of gen.values, drawn through int8 so that images of many calls stay cheap"""
    tenths = rng.integers(-5, 6, size=n, dtype=np.int8)
    if dtype in (gen.F32, gen.F64):
        return (tenths.astype(gen.NP_OF[dtype]) / 10).astype(gen.NP_OF[dtype])
    if dtype == gen.BF16:
        return gen.f32_to_bf16_bits(tenths.astype(np.float32) / 10)
    if dtype == gen.I32:
        return tenths.astype(np.int32) * 200
    return (tenths * 4).astype(np.int8) if dtype == gen.I8 else (np.abs(tenths) * 4).astype(np.uint8)


def pattern(rng, rows, cols, density, by_cols):
    dense = rng.random((rows, cols)) < density
    dense[rng.integers(rows), rng.integers(cols)] = True
    if by_cols:
        dense = dense.T
    ptr = np.concatenate([[0], np.cumsum(dense.sum(1))]).astype(np.uint32)
    return ptr, np.nonzero(dense)[1].astype(np.uint32)


def strided(vals, stride):
    """byte image of the calls' operands (vals: one row per call) at `stride` (0: row 0 alone, shared)"""
    rows = np.ascontiguousarray(vals).view(np.uint8).reshape(vals.shape[0], -1)
    if stride == 0:
        return rows[0].copy()
    assert rows.shape[1] <= stride
    out = np.full(rows.shape[0] * stride, POISON, dtype=np.uint8)
    out.reshape(rows.shape[0], stride)[:, :rows.shape[1]] = rows
    return out


class PackedCase:
    """kind in PACKED_KINDS; M x N x K with packed width P and leading dimensions padded by `pad` elements; values of call t drawn
    per call. pads: extra bytes between consecutive calls of A, B, C (None: that operand is shared, stride 0)"""

    def __init__(self, rng, kind, dtype, count, M=9, N=7, K=11, P=8, pad=2, pads=(8, 16, 24), beta0=0, density=0.3):
        self.kind, self.dtype, self.count, self.P = kind, dtype, count, P
        self.ts = 8 if dtype == gen.F64 else 4
        self.flags = cases.FLAG_BETA_0 if beta0 else 0
        self.ptr = self.idx = None
        n = max(count, 1)
        if kind in DENSE:
            self.dims, a0, b0, c0 = cases.packed_dense_case(rng, DENSE[kind], dtype, M, N, K, P, pad)
            sizes = (a0.size, b0.size, c0.size)
        else:
            if kind == "a_csr":
                self.ptr, self.idx = pattern(rng, M, K, density, False); self.dims = (M, N, K, 0, N + pad, N + pad)
                sizes = (len(self.idx), K * (N + pad) * P, M * (N + pad) * P)
            elif kind in ("b_csr", "b_csc"):
                self.ptr, self.idx = pattern(rng, K, N, density, kind == "b_csc"); self.dims = (M, N, K, K + pad, 0, N + pad)
                sizes = (M * (K + pad) * P, len(self.idx), M * (N + pad) * P)
            else:                                        # c_csc: A [K][lda][P], B [K][ldb][P], one C scalar per non-zero
                self.ptr, self.idx = pattern(rng, M, N, density, True); lda = max(M, K) + pad
                self.dims = (M, N, K, lda, N + pad, 0)
                sizes = (K * lda * P, K * (N + pad) * P, len(self.idx))
        self.nbytes = [s * self.ts for s in sizes]
        self.strides = [0 if pd is None else nb + pd for nb, pd in zip(self.nbytes, pads)]
        imgs = []
        for s, st in zip(sizes, self.strides):
            calls = 1 if st == 0 else n
            imgs.append(strided(values(rng, s * calls, dtype).reshape(calls, s), st))
        self.a, self.b, self.c = imgs

    def create(self, lib=None):
        sh = X.libxsmm_create_gemm_shape(*self.dims, self.dtype, self.dtype, self.dtype, self.dtype)
        if self.kind in DENSE:
            fn = (lib.libxsmm_create_packed_gemm, lib.libxsmm_create_packed_gemm_ac_rm, lib.libxsmm_create_packed_gemm_bc_rm)[DENSE[self.kind]] if lib else \
                 (X.libxsmm_create_packed_gemm, X.libxsmm_create_packed_gemm_ac_rm, X.libxsmm_create_packed_gemm_bc_rm)[DENSE[self.kind]]
            return fn(sh, self.flags, 0, self.P)
        csc = self.kind.endswith("csc")
        fn = getattr(lib or X, "libxsmm_create_packed_spgemm_csc" if csc else "libxsmm_create_packed_spgemm_csr")
        vals = np.zeros(max(len(self.idx), 1), dtype=gen.NP_OF[self.dtype])       # values travel with every call
        return fn(sh, self.flags, 0, self.P, self.ptr.ctypes.data, self.idx.ctypes.data, vals.ctypes.data)

    def oracle_call(self, oracle, a, b, c):
        """call on host byte images a, b, c (one call each), C in place"""
        from oracle_ffi import iarr
        if self.kind in DENSE:
            return oracle["packed_dense"](DENSE[self.kind], self.dtype, iarr(*self.dims), self.flags, self.P, a.ctypes.data, b.ctypes.data, c.ctypes.data)
        return oracle["packed_sp"](int(self.kind.endswith("csc")), self.dtype, iarr(*self.dims), self.flags, self.P, self.ptr.ctypes.data,
                                   self.idx.ctypes.data, None, a.ctypes.data, b.ctypes.data, c.ctypes.data)


class BcscCase:
    """BCSC handle over m_blocks of packed width M: types (a, b, comp, c); A VNNI-packed unless f32; pads as in PackedCase"""

    def __init__(self, rng, types, count, mblocks=3, M=16, K=64, N=64, bk=16, bn=16, density=0.5, pads=(16, 32, 48), beta0=0):
        self.types, self.count = types, count
        ta, tb, tcomp, tc = types
        self.geo = (mblocks, M, K, N, bk, bn)
        self.nbc = N // bn
        self.flags = (cases.FLAG_BETA_0 if beta0 else 0) | (cases.FLAG_VNNI_A if ta != gen.F32 else 0)
        self.colptr, self.rowidx = pattern(rng, K // bk, self.nbc, density, True)
        nnzb = int(self.colptr[-1])
        sizes = (mblocks * K * M, nnzb * bk * bn, mblocks * N * M)
        tsz = {gen.F32: 4, gen.BF16: 2, gen.I8: 1, gen.U8: 1, gen.I32: 4}
        self.nbytes = [s * tsz[t] for s, t in zip(sizes, (ta, tb, tc))]
        self.strides = [0 if pd is None else nb + pd for nb, pd in zip(self.nbytes, pads)]
        n = max(count, 1)
        imgs = []
        for s, st, t in zip(sizes, self.strides, (ta, tb, tc)):
            calls = 1 if st == 0 else n
            imgs.append(strided(values(rng, s * calls, t).reshape(calls, s), st))
        self.a, self.b, self.c = imgs

    def create(self, lib=None):
        ta, tb, tcomp, tc = self.types
        mblocks, M, K, N, bk, bn = self.geo
        sh = X.libxsmm_create_gemm_shape(mblocks, 0, K, K, 0, N, ta, tb, tc, tcomp)
        return (lib or X).libxsmm_create_packed_spgemm_bcsc(sh, self.flags, 0, X.SpgemmConfig(M, bk, bn))

    def oracle_call(self, oracle, a, b, c):
        from oracle_ffi import iarr
        return oracle["bcsc"](iarr(*self.types), iarr(*self.geo), self.flags, a.ctypes.data, b.ctypes.data, self.colptr.ctypes.data,
                              self.rowidx.ctypes.data, c.ctypes.data)


def param(a, b, c, strides, t, colptr=None, rowidx=None, nbc=None):
    """libxsmm_gemm_param of call t: a, b, c are base addresses; BCSC: pattern addresses and a c_ulonglong block-column count"""
    p = X.GemmParam()
    p.a.primary, p.b.primary, p.c.primary = a + t * strides[0], b + t * strides[1], c + t * strides[2]
    if colptr is not None:
        p.b.secondary, p.b.tertiary, p.b.quaternary = colptr, rowidx, C.addressof(nbc)
    return p
