"""Writes tests/golden/gemm_dispatch.npz: which dense GEMM descriptors dispatch, and to which backend.

For every point of a fixed grid it records libxsmm_b200_kernel_backend of the handle that libxsmm_dispatch_gemm, _brgemm or
_brgemm_ext returns, or 0 for NULL. The grid covers:
  - every (A, B, C, comp) tuple over the types a dispatch rule names, under the flag sets that open each A form, and under the
    ext ABI with and without a fusion;
  - every combination of the flags a rule reads, for one or more tuples of every exact-order path and of their declined neighbours;
  - both sides of every leading-dimension bound and every divisibility rule (m, n, k, lda, ldc) for those tuples;
  - the four batch-reduce modes, with stride hints equal and not equal to lda*k / ldb*k.
tests/test_gemm_dispatch_table.py rebuilds the grid and compares point by point. Run from the repository root after `make lib`:
    python3 tests/golden/make_golden_dispatch.py"""
import ctypes as C
import hashlib
import multiprocessing
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import libxsmm_b200 as X  # noqa: E402

F64, F32, BF16, F16, BF8, HF8, I32, I16, I8, U8 = 0, 1, 2, 3, 4, 5, 8, 10, 12, 13
MXBF8, MXHF8, I4X2, U4X2, MXFP4X2, I2X4, I1X8, BF32, IMPLICIT = 14, 15, 18, 19, 20, 22, 23, 24, 25
TYPES = [F64, F32, BF32, BF16, F16, BF8, HF8, I32, I16, I8, U8, MXBF8, MXHF8, I4X2, U4X2, MXFP4X2, I2X4, I1X8]
COMPS = TYPES + [IMPLICIT]

TRANS_A, TRANS_B, BETA_0, VNNI_A, VNNI_B, VNNI_C = 1, 2, 4, 256, 512, 1024
USE_XGEMM_ABI, USE_XGEMM_EXT_ABI, INTLV_A, BITMAP_A = 2048, 4096, 262144, 524288
RULE_FLAGS = [TRANS_A, TRANS_B, VNNI_A, VNNI_B, VNNI_C, INTLV_A, BITMAP_A, BETA_0]

# how a point is dispatched: libxsmm_dispatch_gemm, _brgemm, or _brgemm_ext without a fusion, with a column bias, ReLU, ReLU with
# a bit mask, or sigmoid
GEMM, BRGEMM, EXT, EXT_BIAS, EXT_RELU, EXT_RELU_MASK, EXT_SIGMOID = range(7)
EXT_APIS = [EXT, EXT_BIAS, EXT_RELU, EXT_RELU_MASK, EXT_SIGMOID]
# batch-reduce modes as libxsmm_gemm_batch_reduce_type
BR_NONE, BR_ADDRESS, BR_OFFSET, BR_STRIDE = 0, 1, 2, 4

COLUMNS = ("m", "n", "k", "lda", "ldb", "ldc", "ta", "tb", "tc", "tcomp", "flags", "api", "br_type", "hint_a", "hint_b")

# one or more (A, B, C, comp) tuples of every exact-order path, and the neighbours its rule declines
TUPLES = [
    (F64, F64, F64, F64), (F32, F32, F32, F32), (BF32, F32, F32, F32), (F32, BF32, F32, F32), (BF32, BF32, F32, F32),
    (I16, I16, I32, I32), (I8, I8, I32, I32), (U8, I8, I32, I32), (I8, U8, I32, I32), (U8, U8, I32, I32), (I8, I8, F32, I32),
    (U8, U8, F32, I32), (F16, F16, F16, F16), (F16, F16, F16, IMPLICIT), (F16, F16, F32, F32), (BF16, BF16, F32, F32),
    (BF16, BF16, BF16, F32), (BF16, F16, F32, F32), (F32, BF16, F16, F64), (BF8, BF8, F32, F32), (HF8, HF8, HF8, F32),
    (BF8, BF16, BF16, F32), (HF8, BF16, F32, F32), (MXBF8, MXBF8, F32, F32), (MXBF8, MXBF8, MXBF8, F32),
    (MXHF8, MXHF8, F32, F32), (MXHF8, MXHF8, MXHF8, F32), (I8, BF16, F32, F32), (I8, BF16, BF16, F32), (I8, F16, F16, F16),
    (I8, F16, F32, IMPLICIT), (I4X2, F16, F16, F32), (U4X2, F16, F32, F16), (BF8, F16, F16, F32), (BF8, F16, F32, F32),
    (U8, F16, F16, F32), (U8, BF16, F32, F32), (I4X2, BF16, F32, F32), (I4X2, I8, I32, I32), (U4X2, U8, I32, I32),
    (I2X4, I8, I32, I32), (I2X4, U8, I32, I32), (I1X8, I8, I32, I32), (I1X8, U8, I32, I32), (MXFP4X2, I8, F32, I32),
    (MXFP4X2, I8, BF16, I32), (MXFP4X2, U8, F32, I32),
]


def base_flags(ta, tb):
    """the layout flags an A form needs before its other rules come into play"""
    if ta in (MXBF8, MXHF8):
        return VNNI_A | VNNI_B | TRANS_B
    if ta == I1X8:
        return VNNI_A
    if ta in (I2X4, MXFP4X2) or (ta in (I4X2, U4X2) and tb in (I8, U8)):
        return VNNI_A | INTLV_A
    if ta in (I4X2, U4X2):
        return VNNI_A
    return 0


def _subsets(bits):
    out = [0]
    for b in bits:
        out += [f | b for f in out]
    return out


def grid():
    """the points, one row each (COLUMNS), in a fixed order"""
    rows = []
    base = (64, 64, 64, 64, 64, 64)
    # every tuple, under the flag sets that open each A form, and under the ext ABI
    tuple_flags = [(GEMM, 0), (GEMM, VNNI_A), (GEMM, VNNI_A | INTLV_A), (GEMM, VNNI_A | VNNI_B | TRANS_B), (GEMM, BITMAP_A),
                   (GEMM, TRANS_A | TRANS_B), (GEMM, VNNI_C | BETA_0), (GEMM, VNNI_A | VNNI_B | TRANS_B | BETA_0),
                   (EXT, 0), (EXT, VNNI_A), (EXT, VNNI_A | INTLV_A), (EXT, VNNI_A | VNNI_B | TRANS_B),
                   (EXT_BIAS, 0), (EXT_RELU, 0), (EXT_RELU_MASK, 0), (EXT_SIGMOID, 0)]
    for api, flags in tuple_flags:
        for ta in TYPES:
            for tb in TYPES:
                for tc in TYPES:
                    for tcomp in COMPS:
                        rows.append(base + (ta, tb, tc, tcomp, flags, api, BR_NONE, 0, 0))
    # every combination of the flags a rule reads, plain, as a stride BRGEMM and under each ext form; and the ABI flags given by
    # the caller
    for t in TUPLES:
        for flags in _subsets(RULE_FLAGS):
            for api in [GEMM, BRGEMM] + EXT_APIS:
                rows.append(base + t + (flags, api, BR_STRIDE if api == BRGEMM else BR_NONE, 64 * 64, 64 * 64))
        for flags in (USE_XGEMM_ABI, USE_XGEMM_EXT_ABI, USE_XGEMM_ABI | USE_XGEMM_EXT_ABI):
            for api in (GEMM, EXT, EXT_RELU):
                rows.append(base + t + (base_flags(t[0], t[1]) | flags, api, BR_NONE, 0, 0))
    # both sides of every leading-dimension bound and divisibility rule; m, n, k cover the residues the rules test
    shapes = [(32, 32, 64), (34, 31, 66), (36, 32, 68), (31, 30, 72), (32, 32, 63), (64, 32, 96)]
    for t in TUPLES:
        for toggle in _subsets([TRANS_A, TRANS_B, VNNI_A, VNNI_C, BETA_0, BITMAP_A]):
            flags = base_flags(t[0], t[1]) ^ toggle
            for m, n, k in shapes:
                for lda in sorted({m - 1, m, m + 1, k - 1, k}):
                    for ldb in sorted({n - 1, n, k - 1, k}):
                        for ldc in (m, m + 1, 96):
                            rows.append((m, n, k, lda, ldb, ldc) + t + (flags, GEMM, BR_NONE, 0, 0))
    # batch-reduce modes and stride hints
    for t in TUPLES:
        for m, n, k, lda, ldb, ldc in (base, (32, 32, 64, 33, 65, 32)):
            for br_type in (BR_NONE, BR_ADDRESS, BR_OFFSET, BR_STRIDE):
                for ha, hb in ((lda * k, ldb * k), (lda * k + 64, ldb * k), (lda * k, ldb * k + 64), (0, 0)):
                    for extra in (0, BETA_0):
                        for api in (BRGEMM, EXT, EXT_RELU):
                            rows.append((m, n, k, lda, ldb, ldc) + t + (base_flags(t[0], t[1]) | extra, api, br_type, ha, hb))
    return np.array(rows, dtype=np.int64)


def digest(g):
    return hashlib.sha256(np.ascontiguousarray(g).tobytes()).hexdigest()


def _dispatch(row):
    m, n, k, lda, ldb, ldc, ta, tb, tc, tcomp, flags, api, br_type, ha, hb = (int(v) for v in row)
    shape = X.GemmShape(m, n, k, lda, ldb, ldc, ta, tb, tc, tcomp)
    if api == GEMM:
        return X.libxsmm_dispatch_gemm(shape, flags, 0)
    cfg = X.BatchReduceConfig(br_type, ha, hb, 0)
    if api == BRGEMM:
        return X.libxsmm_dispatch_brgemm(shape, flags, 0, cfg)
    cp = {EXT_RELU: X.MELTW_TYPE_UNARY_RELU, EXT_RELU_MASK: X.MELTW_TYPE_UNARY_RELU, EXT_SIGMOID: X.MELTW_TYPE_UNARY_SIGMOID}.get(api, 0)
    argops = X.GemmExtUnaryArgops(0, 0, 0, 0, 0, 0, 0, 0, ldc, cp, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT if api == EXT_RELU_MASK else 0, 0)
    postops = X.GemmExtBinaryPostops(ldc, tc, X.MELTW_TYPE_BINARY_ADD, X.MELTW_FLAG_BINARY_BCAST_COL_IN_0) if api == EXT_BIAS \
        else X.GemmExtBinaryPostops(0, 0, 0, 0)
    return X.libxsmm_dispatch_brgemm_ext(shape, flags, 0, cfg, argops, postops)


# the registry holds 8192 handles and answers NULL when full, which would read as a decline; a child dispatches at most half that
# many points, so it cannot fill up
REGISTRY_LIMIT = 8192
CHUNK = REGISTRY_LIMIT // 2


def _sweep_chunk(g):
    """in a fresh child: the backend of every point, and the number of handles the registry then holds"""
    os.environ.pop("LIBXSMM_B200_TS", None)      # the default backend choice
    X.libxsmm_b200_set_force_simt(0)
    X.libxsmm_finalize()                         # empties the registry the child inherited
    out = np.zeros(len(g), dtype=np.uint8)
    for i, row in enumerate(g):
        kern = _dispatch(row)
        out[i] = X.libxsmm_b200_kernel_backend(kern) if kern else 0
    info = X.RegistryInfo()
    assert X.libxsmm_get_registry_info(C.byref(info)) == 0
    return out, int(info.size)


def sweep(g):
    """backends of every point; each chunk runs in its own child process, and returns the registry size it reached"""
    ctx = multiprocessing.get_context("fork")     # a child only calls the library's host code
    chunks = [g[i:i + CHUNK] for i in range(0, len(g), CHUNK)]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)    # the pool forks each child from its own handler thread
        with ctx.Pool(processes=min(8, os.cpu_count() or 1), maxtasksperchild=1) as pool:
            results = pool.map(_sweep_chunk, chunks, chunksize=1)
    sizes = [size for _, size in results]
    return np.concatenate([out for out, _ in results]), max(sizes)


def main():
    g = grid()
    backend, peak = sweep(g)
    assert peak <= REGISTRY_LIMIT // 2, peak
    np.savez_compressed(os.path.join(HERE, "gemm_dispatch.npz"), backend=backend, grid_sha256=np.array(digest(g)),
                        columns=np.array(COLUMNS))
    print("%d points, %d dispatched, busiest child registered %d handles" % (len(g), int(np.count_nonzero(backend)), peak))


if __name__ == "__main__":
    main()
