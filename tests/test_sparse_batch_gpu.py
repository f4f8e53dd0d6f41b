"""GPU: libxsmm_b200_spgemm_batch_strided. Every call of a batch must equal, byte for byte, the single call of the same handle on the
same device operands (the gaps between calls included), and a batch must be one launch. The exact-order kernels (packed A-CSR,
B-CSR, B-CSC and the BCSC CUDA-core kernel) are also pinned bit for bit against the oracle; the BCSC tensor-core kernel is pinned
against its own single call. Counts 1, 7, 20,000 and 70,000: the last is past the 65,535 rows of calls one launch places side by
side, so the kernels' loop over the calls runs."""
import ctypes as C

import numpy as np
import pytest
import torch

import gen
import libxsmm_b200 as X
from oracle_ffi import oracle
from sparse_batch_cases import PACKED_KINDS, POISON, BcscCase, PackedCase, param

pytestmark = pytest.mark.gpu
NOT_BATCHABLE = -6
EXACT = ("a_csr", "b_csr", "b_csc", "c_csc", "pk_gemm", "pk_ac_rm", "pk_bc_rm")   # same order as the oracle, one FMA per product
PACKED = [(k, t) for k in PACKED_KINDS for t in (gen.F32, gen.F64) if not (k == "c_csc" and t == gen.F64)]
BCSC_TYPES = {"bf16": (gen.BF16, gen.BF16, gen.F32, gen.BF16), "f32": (gen.F32, gen.F32, gen.F32, gen.F32),
              "u8i8": (gen.U8, gen.I8, gen.I32, gen.I32)}


class Launches:
    FAMILIES = (X.BACKEND_STREAM, X.BACKEND_SIMT, X.BACKEND_TCGEN05)

    def __enter__(self):
        self.total = X.libxsmm_b200_launch_count()
        self.before = [X.libxsmm_b200_launch_count_backend(f) for f in self.FAMILIES]
        return self

    def __exit__(self, *exc):
        self.total = X.libxsmm_b200_launch_count() - self.total
        self.moved = dict(zip(self.FAMILIES, (X.libxsmm_b200_launch_count_backend(f) - b for f, b in zip(self.FAMILIES, self.before))))


def on_device(case):
    return [torch.from_numpy(x).cuda() for x in (case.a, case.b, case.c)]


def batch_vs_singles(k, case, count, extra_dev=None, expect_family=None):
    """the batch and the loop of single calls on the same device A and B, each on its own copy of C; returns both C images"""
    d_a, d_b, d_c = on_device(case)
    d_c1 = d_c.clone()
    p = param(d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), case.strides, 0, **(extra_dev or {}))
    with Launches() as L:
        rc = X.libxsmm_b200_spgemm_batch_strided(k, C.byref(p), C.byref(X.SpgemmStrides(*case.strides)), count)
        X.libxsmm_b200_sync()
    assert rc == 0
    X.check()
    assert L.total == (1 if count > 0 else 0)
    if expect_family is not None:
        assert L.moved[expect_family] == 1, L.moved
    X.libxsmm_b200_set_blocking(0)
    try:
        fn = X.GEMMFUNCTION(k)
        for t in range(count):
            fn(C.byref(param(d_a.data_ptr(), d_b.data_ptr(), d_c1.data_ptr(), case.strides, t, **(extra_dev or {}))))
        X.libxsmm_b200_sync()
    finally:
        X.libxsmm_b200_set_blocking(1)
    X.check()
    assert torch.equal(d_c, d_c1), "batch differs from its single calls"
    return d_c.cpu().numpy()


def check_oracle(case, got, calls):
    for t in calls:
        a = case.a[t * case.strides[0]:][:case.nbytes[0]].copy(); b = case.b[t * case.strides[1]:][:case.nbytes[1]].copy()
        want = case.c[t * case.strides[2]:][:case.nbytes[2]].copy()
        assert case.oracle_call(oracle, a, b, want) == 0
        assert np.array_equal(got[t * case.strides[2]:][:case.nbytes[2]], want), t


@pytest.mark.parametrize("kind,dtype", PACKED)
@pytest.mark.parametrize("count", [1, 7])
def test_packed_batch(kind, dtype, count):
    """padded leading dimensions, per-call strides with gaps; then A shared and B shared (stride 0)"""
    rng = np.random.default_rng(17)
    for pads, beta0 in (((8, 16, 24), 0), ((None, 8, 8), 1), ((8, None, 0), 0)):
        case = PackedCase(rng, kind, dtype, count, P=16, pads=pads, beta0=beta0)
        k = case.create()
        assert k
        got = batch_vs_singles(k, case, count, expect_family=X.BACKEND_STREAM)
        if case.strides[2]:
            assert np.all(got.reshape(count, -1)[:, case.nbytes[2]:] == POISON)
        if kind in EXACT:
            check_oracle(case, got, sorted({0, count - 1}))
        X.libxsmm_release_kernel(k)


# past one row of calls per CTA row (65,535): the kernels loop over the calls
@pytest.mark.parametrize("count", [20000, 70000])
@pytest.mark.parametrize("kind,dtype", [("a_csr", gen.F32), ("b_csr", gen.F64), ("b_csc", gen.F32), ("c_csc", gen.F32),
                                        ("pk_gemm", gen.F64), ("pk_ac_rm", gen.F32), ("pk_bc_rm", gen.F64)])
def test_packed_batch_many_calls(kind, dtype, count):
    rng = np.random.default_rng(23)
    case = PackedCase(rng, kind, dtype, count, M=5, N=4, K=6, P=16 if kind == "c_csc" else 8, pad=1, pads=(8, 8, 8))
    k = case.create()
    got = batch_vs_singles(k, case, count, expect_family=X.BACKEND_STREAM)
    if kind in EXACT:
        check_oracle(case, got, [0, 65534, 65535, count - 1] if count > 65535 else [0, count - 1])
    X.libxsmm_release_kernel(k)


def bcsc_run(case, count, device_pattern, expect_family):
    k = case.create()
    assert k
    nbc = C.c_ulonglong(case.nbc)
    if device_pattern:
        d_cp, d_ri = torch.from_numpy(case.colptr.view(np.int32).copy()).cuda(), torch.from_numpy(case.rowidx.view(np.int32).copy()).cuda()
        pat = dict(colptr=d_cp.data_ptr(), rowidx=d_ri.data_ptr(), nbc=nbc)
    else:
        pat = dict(colptr=case.colptr.ctypes.data, rowidx=case.rowidx.ctypes.data, nbc=nbc)
    got = batch_vs_singles(k, case, count, pat, expect_family)
    return k, got


@pytest.mark.parametrize("types", sorted(BCSC_TYPES))
@pytest.mark.parametrize("count,device_pattern", [(1, False), (1, True), (7, False), (7, True), (20000, True), (70000, True)])
def test_bcsc_batch(types, count, device_pattern):
    """bf16 on the tensor-core kernel, f32 and u8 x i8 on the exact-order kernel (pinned against the oracle); a host-resident and
    a device-resident pattern (the many-call cases with the device-resident one only: each single call would stage a host one)"""
    rng = np.random.default_rng(29)
    tc = types == "bf16"
    big = count > 7                              # many calls: one m_block, the block values shared (stride 0)
    case = BcscCase(rng, BCSC_TYPES[types], count, mblocks=1 if big else 2, M=16, K=64, N=32 if big else 48, bk=16, bn=16,
                    pads=(16, None, 48) if big else (16, 32, 48), beta0=int(count == 7))
    k, got = bcsc_run(case, count, device_pattern, X.BACKEND_TCGEN05 if tc else X.BACKEND_SIMT)
    assert X.libxsmm_b200_bcsc_variant(k, case.nbc) == int(tc)
    if not tc:
        check_oracle(case, got, sorted({0, count // 2, count - 1}))
    X.libxsmm_release_kernel(k)


def test_bcsc_shared_operands_and_unaligned_strides():
    """A or the block values shared (stride 0) keep the tensor-core kernel; a per-call stride that is not a multiple of 16 bytes
    sends a bf16 batch to the exact-order kernel, whose calls equal its own single calls"""
    rng = np.random.default_rng(31)
    T = BCSC_TYPES["bf16"]
    for pads in ((None, 32, 16), (16, None, 16)):
        k, _ = bcsc_run(BcscCase(rng, T, 7, pads=pads), 7, True, X.BACKEND_TCGEN05)
        X.libxsmm_release_kernel(k)
    case = BcscCase(rng, T, 7, pads=(2, 32, 16))
    d_a, d_b, d_c = on_device(case)
    nbc = C.c_ulonglong(case.nbc)
    p = param(d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), case.strides, 0, colptr=case.colptr.ctypes.data, rowidx=case.rowidx.ctypes.data, nbc=nbc)
    k = case.create()
    with Launches() as L:
        assert X.libxsmm_b200_spgemm_batch_strided(k, C.byref(p), C.byref(X.SpgemmStrides(*case.strides)), 7) == 0
    X.check()
    assert L.total == 1 and L.moved[X.BACKEND_SIMT] == 1 and L.moved[X.BACKEND_TCGEN05] == 0
    # each call against the exact-order single call: the same handle forced onto that kernel by an unaligned A of its own
    got = d_c.cpu().numpy()
    for t in (0, 3, 6):
        a = torch.zeros(case.nbytes[0] + 2, dtype=torch.uint8, device="cuda")
        a[2:] = d_a[t * case.strides[0]:][:case.nbytes[0]]
        c = torch.from_numpy(case.c[t * case.strides[2]:][:case.nbytes[2]].copy()).cuda()
        with Launches() as L1:
            X.GEMMFUNCTION(k)(C.byref(param(a.data_ptr() + 2, d_b.data_ptr() + t * case.strides[1], c.data_ptr(), case.strides, 0,
                                            colptr=case.colptr.ctypes.data, rowidx=case.rowidx.ctypes.data, nbc=nbc)))
        X.check()
        assert L1.moved[X.BACKEND_SIMT] == 1
        assert np.array_equal(c.cpu().numpy(), got[t * case.strides[2]:][:case.nbytes[2]]), t
    X.libxsmm_release_kernel(k)


def test_return_codes():
    rng = np.random.default_rng(37)
    case = PackedCase(rng, "b_csc", gen.F32, 3, pads=(8, 8, 0))
    k = case.create()
    d_a, d_b, d_c = on_device(case)
    c0 = d_c.clone()
    p = param(d_a.data_ptr(), d_b.data_ptr(), d_c.data_ptr(), case.strides, 0)
    f = X.libxsmm_b200_spgemm_batch_strided
    S = lambda sa, sb, sc: C.byref(X.SpgemmStrides(sa, sb, sc))
    ok, cb = S(*case.strides), case.nbytes[2]
    with Launches() as L:
        assert f(None, C.byref(p), ok, 2) == -1
        assert f(k, C.byref(p), ok, -1) == -1
        assert f(k, C.byref(p), ok, 0) == 0
        for bad in ((-8, case.strides[1], cb), (case.strides[0], case.strides[1], cb - 4), (case.strides[0], case.strides[1], cb + 2)):
            assert f(k, C.byref(p), S(*bad), 2) == -1, bad
        host_c = case.c.copy()                                               # pageable C: batches do not stage
        assert f(k, C.byref(param(d_a.data_ptr(), d_b.data_ptr(), host_c.ctypes.data, case.strides, 0)), ok, 2) == -4
        areg_vals = np.ones(2)
        ptr, idx = np.array([0, 1, 2], dtype=np.uint32), np.array([0, 1], dtype=np.uint32)
        areg = X.libxsmm_create_spgemm_csr_areg(X.libxsmm_create_gemm_shape(2, 16, 2, 0, 16, 16, gen.F32, gen.F32, gen.F32, gen.F32), 0, 0, 16,
                                                ptr.ctypes.data, idx.ctypes.data, areg_vals.ctypes.data)
        assert areg and f(areg, C.byref(p), ok, 2) == NOT_BATCHABLE
    assert L.total == 0 and torch.equal(d_c, c0)
    with Launches() as L:                                                    # outputs that touch do not overlap
        assert f(k, C.byref(p), S(case.strides[0], case.strides[1], cb), 3) == 0
    X.check()
    assert L.total == 1
    X.libxsmm_release_kernel(k)
    X.libxsmm_release_kernel(areg)
