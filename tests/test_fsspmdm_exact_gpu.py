"""The fsspmdm kernels (sparse.cu: sreg_kernel with 1, 2 or 3 TMA stages, sreg_direct_kernel) and the packed dense and C-sparse CSC
kernels, element by element against a float64 reference built from the operands handed to the library.

 * Family E (exact by construction, cases.fsspmdm_exact_operands): every partial sum is a value of the type, so the result cannot
   depend on the summation order. The kernel must equal the reference and oracle["fsspmdm"] bit for bit (zeros compare by value).
 * Family R (full mantissas, alpha = 0.1): per element |got - exact| <= (nnz_row + 2) u (sum_z |v_z||b| + |c0|), u = 2^-24 / 2^-53;
   doubled for f64, whose float64 reference rounds as well. The largest err/bound ratio seen per dtype is printed.
 * Geometry: N is chosen so that every CTA of the staged kernel walks at least 2S+1 strips (the stage ring wraps and every barrier
   parity flips) and the last strip is ragged. libxsmm_b200_fsspmdm_variant is asserted before every call, and the launch counts
   show that a streaming kernel ran and nothing else did.
 * Columns N..ldb-1 of B hold NaN; columns N..ldc-1 of C and a guard band after C hold a byte sentinel and must come back unchanged;
   beta = 0 runs over a C whose logical part is NaN. No NaN or Inf ever enters a sum."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import cases  # noqa: E402
import gen  # noqa: E402
import libxsmm_b200 as X  # noqa: E402
from golden_cases import read_mtx  # noqa: E402
from oracle_ffi import iarr, oracle  # noqa: E402

pytestmark = pytest.mark.gpu

F32, F64 = gen.F32, gen.F64
STRIP = {F32: 128, F64: 64}                     # columns of one 512-byte strip
UNIT = {F32: 2.0 ** -24, F64: 2.0 ** -53}
TS = {F32: 4, F64: 8}
SENTINEL, GUARD = 0xA5, 256
R_ALPHA = 0.1
WORST = {}                                      # dtype -> largest err/bound ratio of family R


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def wrap_n(dtype, laps=7):
    """every CTA of the staged kernel (grid = #SMs) walks `laps` strips or more (>= 2S+1 for S <= 3); the last strip is ragged"""
    return STRIP[dtype] * sms() * laps + (48 if dtype == F32 else 24)


class Launches:
    """kernels launched per family while the block runs: a streaming kernel must run, nothing else"""

    FAMILIES = (X.BACKEND_STREAM, X.BACKEND_SIMT, X.BACKEND_TCGEN05)

    def __enter__(self):
        self.before = [X.libxsmm_b200_launch_count_backend(f) for f in self.FAMILIES]
        return self

    def __exit__(self, *exc):
        self.moved = [X.libxsmm_b200_launch_count_backend(f) - b for f, b in zip(self.FAMILIES, self.before)]

    def expect_stream(self, what):
        assert self.moved[0] > 0 and self.moved[1] == 0 and self.moved[2] == 0, ("not (only) a streaming kernel ran", what, self.moved)


def r_operands(rng, dtype, mask, N, ldb, ldc, lda=None, values=None):
    """family R: standard-normal A (on `mask`, or the given dense values), B and C0; NaN in the padding columns of B and C"""
    npdt = gen.NP_OF[dtype]
    M, K = mask.shape
    lda = lda or K
    a = np.zeros((M, lda), dtype=npdt)
    a[:, :K] = values if values is not None else np.where(mask, rng.standard_normal((M, K)), 0.0)
    b = np.full((K, ldb), np.nan, dtype=npdt)
    b[:, :N] = rng.standard_normal((K, N), dtype=np.float32 if dtype == F32 else np.float64)
    c0 = np.full((M, ldc), np.nan, dtype=npdt)
    c0[:, :N] = rng.standard_normal((M, N))
    return a, b, c0


def run(dtype, a, b, c0, N, alpha, beta, variant, what, b_offset=0):
    """create a handle, lay B and C out on the device with poison around them, assert the kernel the query names, execute once and
    check that nothing outside the logical M x N block of C changed; returns that block"""
    npdt, ts = gen.NP_OF[dtype], TS[dtype]
    M, lda = a.shape
    K, ldb = b.shape
    ldc = c0.shape[1]
    al, bt = np.array([alpha], dtype=npdt), np.array([beta], dtype=npdt)
    h = X.libxsmm_fsspmdm_create(dtype, M, N, K, lda, ldb, ldc, al.ctypes.data, bt.ctypes.data, a.ctypes.data, 0, None)
    assert h, what
    b_bytes = np.ascontiguousarray(b).view(np.uint8).ravel()
    d_b = torch.empty(b_bytes.size + 16, dtype=torch.uint8, device="cuda")
    d_b[b_offset:b_offset + b_bytes.size].copy_(torch.from_numpy(b_bytes))
    nc = M * ldc * ts
    img = np.full(nc + GUARD, SENTINEL, dtype=np.uint8)
    img[:nc].view(npdt).reshape(M, ldc)[:, :N] = c0[:, :N] if beta else np.nan
    d_c = torch.from_numpy(img).cuda()
    bp, cp = d_b.data_ptr() + b_offset, d_c.data_ptr()
    assert X.libxsmm_b200_fsspmdm_variant(h, bp, cp) == variant, (what, X.libxsmm_b200_fsspmdm_variant(h, bp, cp), variant)
    with Launches() as launches:
        X.libxsmm_fsspmdm_execute(h, bp, cp)
        X.check()
    launches.expect_stream(what)
    X.libxsmm_fsspmdm_destroy(h)
    out = d_c.cpu().numpy()
    assert np.array_equal(out[nc:], img[nc:]), (what, "guard band after C written")
    assert np.array_equal(out[:nc].reshape(M, ldc * ts)[:, N * ts:], img[:nc].reshape(M, ldc * ts)[:, N * ts:]), (what, "columns N..ldc of C written")
    return out[:nc].view(npdt).reshape(M, ldc)[:, :N].copy()


def check_exact(dtype, got, a, b, c0, N, alpha, beta, what):
    """family E: every element bit for bit (zeros by value) against the float64 reference; against oracle["fsspmdm"] everywhere for
    N <= 4096, else on the first 512 columns and the last 528 (the ragged tail)"""
    npdt, ts = gen.NP_OF[dtype], TS[dtype]
    M, lda = a.shape
    K, ldb = b.shape
    ldc = c0.shape[1]
    exact, _ = cases.fsspmdm_reference(cases.fsspmdm_fold(dtype, a[:, :K], alpha), b, c0, N, beta, magnitude=False)
    want = exact.astype(npdt)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (what, "elements differing from the exact result", len(bad), bad[:5].tolist())
    al, bt = np.array([alpha], dtype=npdt), np.array([beta], dtype=npdt)
    for j0, j1 in ([(0, N)] if N <= 4096 else [(0, 512), (N - 528, N)]):
        orc = np.ascontiguousarray(c0).copy()
        assert oracle["fsspmdm"](dtype, M, j1 - j0, K, lda, ldb, ldc, al.ctypes.data, bt.ctypes.data, a.ctypes.data,
                                 b.ctypes.data + j0 * ts, orc.ctypes.data + j0 * ts) == 0
        assert np.array_equal(got[:, j0:j1], orc[:, j0:j1]), (what, "differs from the oracle", (j0, j1))


def check_bounded(dtype, got, a, b, c0, N, alpha, beta, what):
    """family R: every element within (nnz_row + 2) u (sum |v||b| + |c0|), doubled for f64"""
    K = b.shape[0]
    v = cases.fsspmdm_fold(dtype, a[:, :K], alpha)
    exact, mag = cases.fsspmdm_reference(v, b, c0, N, beta)
    nnz = (v != 0).sum(axis=1)[:, None]
    bound = (nnz + 2) * UNIT[dtype] * mag * (2.0 if dtype == F64 else 1.0)
    err = np.abs(got.astype(np.float64) - exact)
    assert np.all(np.isfinite(got)), what
    bad = np.argwhere(err > bound)
    assert bad.size == 0, (what, "elements outside the bound", len(bad), bad[:5].tolist())
    pos = bound > 0
    ratio = float((err[pos] / bound[pos]).max()) if pos.any() else 0.0
    WORST[dtype] = max(WORST.get(dtype, 0.0), ratio)
    print("family R %s %s: largest err/bound %.3g" % ("f32" if dtype == F32 else "f64", what, ratio))


ROWS = lambda M: [(3 + 7 * i) % 10 for i in range(M)]      # 0..9 non-zeros per row: the unroll by 4, its remainder, empty rows


@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("K,stages", [(128, 3), (192, 2), (256, 1)])
def test_stage_ring_wraps_at_every_depth(dtype, K, stages):
    """M = 32, 15 % non-zeros: K picks the pipeline depth S; every CTA walks >= 2S+1 strips, the last one ragged"""
    rng = np.random.default_rng(1000 + K + dtype)
    M, N = 32, wrap_n(dtype)
    for beta, alpha in ((0.0, -2.0), (1.0, 0.75)):
        mask = cases.fsspmdm_pattern(rng, M, K, density=0.15)
        a, b, c0 = cases.fsspmdm_exact_operands(rng, dtype, mask, N, N, N, alpha)
        what = ("E", K, beta)
        check_exact(dtype, run(dtype, a, b, c0, N, alpha, beta, stages, what), a, b, c0, N, alpha, beta, what)
    a, b, c0 = r_operands(rng, dtype, mask, N, N, N)
    what = ("R", K)
    check_bounded(dtype, run(dtype, a, b, c0, N, R_ALPHA, 1.0, stages, what), a, b, c0, N, R_ALPHA, 1.0, what)


# (what, dtype, M, K, density, ldb - N, B offset in bytes, N, variant)
_PLAN = (("K=300: direct", F32, 32, 300, 0.15, 0, 0, "small", 0),
         ("K=512: direct", F64, 32, 512, 0.15, 0, 0, "small", 0),
         ("ldb = N+2: unaligned rows, direct", F32, 32, 128, 0.15, 2, 0, "small", 0),
         ("B one f64 element off 16 bytes: direct", F64, 32, 128, 0.15, 0, 8, "small", 0),
         ("dense A, M=64: three stages do not fit, two do", F32, 64, 128, 1.0, 0, 0, "wrap", 2),
         ("dense A, M=64: one stage", F64, 64, 128, 1.0, 0, 0, "wrap", 1))


@pytest.mark.parametrize("case", _PLAN, ids=[c[0] for c in _PLAN])
def test_every_path_of_the_plan(case):
    what, dtype, M, K, density, ldb_pad, b_offset, size, variant = case
    rng = np.random.default_rng(2000 + K + M)
    N = wrap_n(dtype) if size == "wrap" else wrap_n(dtype, laps=1)
    ldb = N + ldb_pad
    for beta, alpha in ((0.0, 0.75), (1.0, 1.0)):
        mask = cases.fsspmdm_pattern(rng, M, K, density=density)
        a, b, c0 = cases.fsspmdm_exact_operands(rng, dtype, mask, N, ldb, N + 16, alpha)
        check_exact(dtype, run(dtype, a, b, c0, N, alpha, beta, variant, (what, beta), b_offset), a, b, c0, N, alpha, beta, (what, beta))
    a, b, c0 = r_operands(rng, dtype, mask, N, ldb, N + 16)
    check_bounded(dtype, run(dtype, a, b, c0, N, R_ALPHA, 1.0, variant, (what, "R"), b_offset), a, b, c0, N, R_ALPHA, 1.0, (what, "R"))


@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("M", [1, 3, 33, 192])
def test_rows_and_warps(dtype, M):
    """4 warps for M < 4, one row per warp for M <= 32, 32 warps taking 2 (M = 33) or 6 (M = 192) rows each; rows hold 0 to 9
    non-zeros, empty rows under both betas"""
    rng = np.random.default_rng(3000 + M + dtype)
    K, N = 128, wrap_n(dtype)
    mask = cases.fsspmdm_pattern(rng, M, K, row_nnz=ROWS(M))
    for beta, alpha in ((0.0, 1.0), (1.0, -2.0)):
        a, b, c0 = cases.fsspmdm_exact_operands(rng, dtype, mask, N, N + 8, N + 16, alpha)
        check_exact(dtype, run(dtype, a, b, c0, N, alpha, beta, 3, ("E", M, beta)), a, b, c0, N, alpha, beta, ("E", M, beta))
    a, b, c0 = r_operands(rng, dtype, mask, N, N + 8, N + 16)
    check_bounded(dtype, run(dtype, a, b, c0, N, R_ALPHA, 1.0, 3, ("R", M)), a, b, c0, N, R_ALPHA, 1.0, ("R", M))


@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("mtx,stages", [("pyfr_p3_hex_m6-sp.mtx", 3), ("pyfr_p3_hex_m132-sp.mtx", 2)])
def test_pyfr_operators(dtype, mtx, stages):
    """the PyFR operators of tests/golden/mtx (M=192, K=96 and M=64, K=192): their own values (family R) and their pattern with
    exact values (family E), at ring-wrapping N"""
    rng = np.random.default_rng(4000 + stages + dtype)
    M, K, dense = read_mtx(mtx)
    N = wrap_n(dtype)
    mask = dense != 0
    for beta in (0.0, 1.0):
        a, b, c0 = r_operands(rng, dtype, mask, N, N, N, values=dense)
        what = (mtx, "R", beta)
        check_bounded(dtype, run(dtype, a, b, c0, N, R_ALPHA, beta, stages, what), a, b, c0, N, R_ALPHA, beta, what)
    a, b, c0 = cases.fsspmdm_exact_operands(rng, dtype, mask, N, N, N, 0.75)
    what = (mtx, "E")
    check_exact(dtype, run(dtype, a, b, c0, N, 0.75, 1.0, stages, what), a, b, c0, N, 0.75, 1.0, what)


def test_bench_geometry_every_element():
    """the benchmark's fsspmdm (f32, M=32, K=128, N=10^6, 15 % non-zeros, beta = 0), exact family, every element of C"""
    rng = np.random.default_rng(5000)
    M, K, N = 32, 128, 1000000
    mask = cases.fsspmdm_pattern(rng, M, K, density=0.15)
    a, b, c0 = cases.fsspmdm_exact_operands(rng, F32, mask, N, N, N, 0.75)
    what = "bench geometry"
    check_exact(F32, run(F32, a, b, c0, N, 0.75, 0.0, 3, what), a, b, c0, N, 0.75, 0.0, what)


@pytest.mark.parametrize("memory", ["pageable", "managed"])
@pytest.mark.parametrize("dtype", [F32, F64])
def test_host_pointers_column_blocks_run_concurrently(dtype, memory):
    """the PyFR driver pattern: 4 handles with max_N = N/4 and ldb = ldc = N, run from 4 fresh threads on one C (beta = 1) in pageable
    memory (each call stages its m x N/4 block of C and nothing else) or in managed memory from libxsmm_aligned_malloc (nothing is staged,
    and the call is the first CUDA work of its thread: the staged kernel must still run there). Every block equals the device-pointer
    result bit for bit"""
    rng = np.random.default_rng(6000 + dtype)
    npdt, ts = gen.NP_OF[dtype], TS[dtype]
    M, K, nb = 32, 128, STRIP[dtype] * 40 + (48 if dtype == F32 else 24)
    N = 4 * nb
    mask = cases.fsspmdm_pattern(rng, M, K, density=0.15)
    a, b, c0 = r_operands(rng, dtype, mask, N, N, N)
    one = np.array([1.0], dtype=npdt); al = np.array([R_ALPHA], dtype=npdt)
    handles = [X.libxsmm_fsspmdm_create(dtype, M, nb, K, K, N, N, al.ctypes.data, one.ctypes.data, a.ctypes.data, 0, None) for _ in range(4)]
    assert all(handles)
    d_b, d_c = torch.from_numpy(b.view(np.uint8).ravel().copy()).cuda(), torch.from_numpy(c0.view(np.uint8).ravel().copy()).cuda()
    with Launches() as launches:
        for j, h in enumerate(handles):
            bp, cp = d_b.data_ptr() + j * nb * ts, d_c.data_ptr() + j * nb * ts
            assert X.libxsmm_b200_fsspmdm_variant(h, bp, cp) == 3
            X.libxsmm_fsspmdm_execute(h, bp, cp)
        X.check()
    launches.expect_stream("device pointers")
    want = d_c.cpu().numpy().view(npdt).reshape(M, N)
    check_bounded(dtype, want, a, b, c0, N, R_ALPHA, 1.0, "column blocks")

    if memory == "pageable":
        c_host = c0.copy()
        pb, pc = b.ctypes.data, c_host.ctypes.data
    else:
        pb, pc = X.libxsmm_aligned_malloc(b.nbytes, 256), X.libxsmm_aligned_malloc(c0.nbytes, 256)
        assert pb and pc
        C.memmove(pb, b.ctypes.data, b.nbytes); C.memmove(pc, c0.ctypes.data, c0.nbytes)
    for j, h in enumerate(handles):
        assert X.libxsmm_b200_fsspmdm_variant(h, pb + j * nb * ts, pc + j * nb * ts) == 3

    errors = []

    def worker(j):
        try:
            X.libxsmm_fsspmdm_execute(handles[j], pb + j * nb * ts, pc + j * nb * ts)
            X.check()                # errors are kept per thread
        except Exception as e:      # noqa: BLE001 -- reported by the main thread
            errors.append((j, e))

    with Launches() as launches:
        threads = [threading.Thread(target=worker, args=(j,)) for j in range(4)]
        [t.start() for t in threads]; [t.join() for t in threads]
    assert not errors, errors
    launches.expect_stream(memory)
    if memory == "managed":
        c_host = np.empty_like(c0)
        C.memmove(c_host.ctypes.data, pc, c0.nbytes)
        X.libxsmm_free(pb); X.libxsmm_free(pc)
    for j in range(4):
        blk = slice(j * nb, (j + 1) * nb)
        assert np.array_equal(c_host[:, blk], want[:, blk]), ("block differs from the device-pointer result", memory, j)
    [X.libxsmm_fsspmdm_destroy(h) for h in handles]


# ---- the other streaming sparse kernels: packed dense GEMM (FMA over k) and C-sparse CSC (shuffle tree over the packed dimension) ----
def dyadic(rng, shape, dtype, role):
    """family E values of the packed kernels: A +-(1..7)/8, B with `fb` fraction bits, C within +-2 on the grid of the products"""
    _, q, fb = cases.FSSPMDM_EXACT[dtype]
    if role == "a":
        return rng.integers(1, 8, size=shape) * rng.choice([-1.0, 1.0], size=shape) / 8.0
    if role == "b":
        bmax = 2 ** (fb + 1) - 1
        return rng.integers(-bmax, bmax + 1, size=shape) * 2.0 ** -fb
    return rng.integers(-2 ** (fb + 4), 2 ** (fb + 4) + 1, size=shape) * 2.0 ** -(fb + 3)


def packed_dense_views(kind, dims, P, a, b, c):
    """logical views (float64 einsum operands) of the three packed dense layouts and the reference product"""
    M, N, K, lda, ldb, ldc = dims
    if kind == 0:         # C[n][m][p] += A[k][m][p] B[n][k][p]
        A, B, Cv = a.reshape(K, lda, P)[:, :M], b.reshape(N, ldb, P)[:, :K], c.reshape(N, ldc, P)[:, :M]
        return A, B, Cv, "kmp,nkp->nmp"
    if kind == 1:         # C[m][n][p] += A[m][k][p] B[k][n]
        return a.reshape(M, lda, P)[:, :K], b.reshape(K, ldb)[:, :N], c.reshape(M, ldc, P)[:, :N], "mkp,kn->mnp"
    return a.reshape(M, lda)[:, :K], b.reshape(K, ldb, P)[:, :N], c.reshape(M, ldc, P)[:, :N], "mk,knp->mnp"


def run_packed(k, a, b, c0, what):
    d_a, d_b = torch.from_numpy(a.view(np.uint8).copy()).cuda(), torch.from_numpy(b.view(np.uint8).copy()).cuda()
    img = np.concatenate([c0.view(np.uint8), np.full(GUARD, SENTINEL, dtype=np.uint8)])
    d_c = torch.from_numpy(img).cuda()
    with Launches() as launches:
        X.call_gemm(k, d_a, d_b, d_c)
        X.check()
    launches.expect_stream(what)
    out = d_c.cpu().numpy()
    assert np.array_equal(out[c0.nbytes:], img[c0.nbytes:]), (what, "guard band after C written")
    return out[:c0.nbytes].view(c0.dtype).copy()


@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_packed_dense_exact_and_bounded(kind, dtype):
    """libxsmm_create_packed_gemm / _ac_rm / _bc_rm: family E bit for bit against the float64 product and the oracle, family R per
    element within (K + 2) u sum |a||b| + |c0| (doubled for f64); padding of A and B holds NaN, padding of C must survive. Packed widths
    1, 8, 16, 48; for _bc_rm also the EDGE star matrix as the unpacked A"""
    rng = np.random.default_rng(7000 + 10 * kind + dtype)
    npdt = gen.NP_OF[dtype]
    create = (X.libxsmm_create_packed_gemm, X.libxsmm_create_packed_gemm_ac_rm, X.libxsmm_create_packed_gemm_bc_rm)[kind]
    geos = [(9, 9, 9, P, 2) for P in (1, 8, 16, 48)] + [(20, 9, 35, 16, 0), (56, 9, 56, 48, 1)]
    if kind == 2:
        rows, cols, star = read_mtx("tet4_starMatrix_csr.mtx")
        geos.append((rows, 20, cols, 16, 1, star))
    for geo in geos:
        M, N, K, P, pad = geo[:5]
        for family in ("E", "R"):
            for beta0 in (0, 1):
                dims, a, b, c0 = cases.packed_dense_case(rng, kind, dtype, M, N, K, P, pad)
                a[:] = np.nan; b[:] = np.nan; c0[:] = np.nan
                A, B, Cv, spec = packed_dense_views(kind, dims, P, a, b, c0)
                if family == "E":
                    A[...], B[...], Cv[...] = dyadic(rng, A.shape, dtype, "a"), dyadic(rng, B.shape, dtype, "b"), dyadic(rng, Cv.shape, dtype, "c")
                else:
                    A[...], B[...], Cv[...] = rng.standard_normal(A.shape), rng.standard_normal(B.shape), rng.standard_normal(Cv.shape)
                if len(geo) > 5:           # the EDGE operator: its values (R) or its pattern (E)
                    A[...] = geo[5] if family == "R" else np.where(geo[5] != 0, A, 0.0)
                flags = cases.FLAG_BETA_0 if beta0 else 0
                what = (kind, dtype, dims, P, family, beta0)
                k = create(X.libxsmm_create_gemm_shape(*dims, dtype, dtype, dtype, dtype), flags, 0, P)
                assert k, what
                got = run_packed(k, a, b, c0, what)
                X.libxsmm_release_kernel(k)
                g = packed_dense_views(kind, dims, P, a, b, got)[2]
                c_old = np.zeros(Cv.shape) if beta0 else Cv.astype(np.float64)
                exact = np.einsum(spec, A.astype(np.float64), B.astype(np.float64)) + c_old
                pad_got, pad_c0 = got.copy(), c0.copy()
                packed_dense_views(kind, dims, P, a, b, pad_got)[2][...] = 0
                packed_dense_views(kind, dims, P, a, b, pad_c0)[2][...] = 0
                assert np.array_equal(pad_got.view(np.uint8), pad_c0.view(np.uint8)), (what, "padding of C written")
                if family == "E":
                    assert np.array_equal(g, exact.astype(npdt)), (what, "differs from the exact result")
                    want = c0.copy()
                    assert oracle["packed_dense"](kind, dtype, iarr(*dims), flags, P, a.ctypes.data, b.ctypes.data, want.ctypes.data) == 0
                    assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (what, "differs from the oracle")
                else:
                    mag = np.einsum(spec, np.abs(A.astype(np.float64)), np.abs(B.astype(np.float64))) + np.abs(c_old)
                    bound = (K + 2) * UNIT[dtype] * mag * (2.0 if dtype == F64 else 1.0)
                    err = np.abs(g.astype(np.float64) - exact)
                    assert np.all(err <= bound), (what, "elements outside the bound", int((err > bound).sum()))
                    WORST[dtype] = max(WORST.get(dtype, 0.0), float((err / bound).max()))


def test_c_sparse_csc_exact_and_bounded():
    """libxsmm_create_packed_spgemm_csc with C sparse (f32, P % 16 == 0): C[z] (+)= sum_k sum_p A[k][row(z)][p] B[k][col(z)][p]. Family E
    bit for bit against the float64 sum and the oracle, family R within (K P + 2) u sum |a||b| + |c0|; random patterns and the EDGE
    operator patterns of tests/golden/mtx; packed widths 16 and 48"""
    rng = np.random.default_rng(8000)
    geos = [(M, N, K, P, None) for (M, N, K) in ((9, 9, 9), (20, 9, 35), (56, 9, 56), (35, 20, 9)) for P in (16, 48)]
    for name in ("tet4_2_fluxN_0_csc.mtx", "tet4_3_stiffT_0_csc.mtx"):
        rows, cols, dense = read_mtx(name)
        geos.append((rows, cols, 9, 16, dense != 0))
    for (M, N, K, P, pattern) in geos:
        for family in ("E", "R"):
            for beta0 in (0, 1):
                is_csc, dims, ptr, idx, a, b, c0 = cases.packed_sp_case(rng, "c_csc", F32, M, N, K, P, density=0.3)
                if pattern is not None:
                    ptr = np.concatenate([[0], np.cumsum(pattern.sum(0))]).astype(np.uint32)
                    idx = np.nonzero(pattern.T)[1].astype(np.uint32)
                    c0 = np.zeros(len(idx), dtype=np.float32)
                _, _, _, lda, ldb, _ = dims
                a = np.full((K, lda, P), np.nan, dtype=np.float32); b = np.full((K, ldb, P), np.nan, dtype=np.float32)
                gen_v = (lambda s, role: dyadic(rng, s, F32, role)) if family == "E" else (lambda s, role: rng.standard_normal(s))
                a[:, :M] = gen_v((K, M, P), "a"); b[:, :N] = gen_v((K, N, P), "b"); c0[:] = gen_v(c0.shape, "c")
                a, b = a.ravel(), b.ravel()
                flags = cases.FLAG_BETA_0 if beta0 else 0
                what = ((M, N, K, P), pattern is not None, family, beta0)
                k = X.libxsmm_create_packed_spgemm_csc(X.libxsmm_create_gemm_shape(*dims, F32, F32, F32, F32), flags, 0, P, ptr.ctypes.data,
                                                       idx.ctypes.data, c0.ctypes.data)
                assert k, what
                got = run_packed(k, a, b, c0, what)
                X.libxsmm_release_kernel(k)
                col = np.repeat(np.arange(N), np.diff(ptr.astype(np.int64)))
                A3, B3 = a.reshape(K, lda, P).astype(np.float64), b.reshape(K, ldb, P).astype(np.float64)
                prod = A3[:, idx, :] * B3[:, col, :]
                c_old = np.zeros(len(idx)) if beta0 else c0.astype(np.float64)
                exact = prod.sum(axis=(0, 2)) + c_old
                if family == "E":
                    assert np.array_equal(got, exact.astype(np.float32)), (what, "differs from the exact result")
                    want = c0.copy()
                    assert oracle["packed_sp"](is_csc, F32, iarr(*dims), flags, P, ptr.ctypes.data, idx.ctypes.data, c0.ctypes.data,
                                               a.ctypes.data, b.ctypes.data, want.ctypes.data) == 0
                    assert np.array_equal(got, want), (what, "differs from the oracle")
                else:
                    bound = (K * P + 2) * UNIT[F32] * (np.abs(prod).sum(axis=(0, 2)) + np.abs(c_old))
                    err = np.abs(got.astype(np.float64) - exact)
                    assert np.all(err <= bound), (what, "elements outside the bound", int((err > bound).sum()))
                    WORST[F32] = max(WORST.get(F32, 0.0), float((err / bound).max()))


def test_zz_report_largest_ratio():
    """prints the largest family-R err/bound ratio per dtype over this file (run with -s to see it)"""
    for dtype, r in sorted(WORST.items()):
        print("largest family-R err/bound ratio, %s: %.3g" % ("f32" if dtype == F32 else "f64", r))
        assert r <= 1.0
