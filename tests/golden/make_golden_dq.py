"""Writes tests/golden/dequant.npz: dequantising GEMM cases (I8 x BF16, I8 / I4 / U4 / BF8 x F16; every comp, C type and batch-reduce
mode, beta 0 / 1, TRANS_B) with the C bytes computed by the UNMODIFIED reference's libxsmm_reference_gemm (oracle/_ref/libxsmm_ref_dq.so,
built by `make ref`). The GPU tests compare against these bytes where the reference is absent. Run from the repository root:
    python3 tests/golden/make_golden_dq.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from dq_ffi import BF8, BF16, F16, F32, I4, I8, IMPLICIT, U4, DqCase, meta, ref_gemm_dq  # noqa: E402

# DqCase(ta, tb, comp, tc, m, n, k, lda, ldb, ldc, beta0, trans_b, vnni_a, br_type, br)
CASES = [
    DqCase(I8, BF16, F32, BF16, 24, 10, 40, 28, 44, 26, True, False, False, 0, 1),
    DqCase(I8, BF16, F32, F32, 17, 9, 33, 20, 33, 19, False, False, False, 3, 3),
    DqCase(I8, F16, F16, F16, 20, 12, 48, 24, 12, 21, False, True, False, 2, 2),
    DqCase(I8, F16, IMPLICIT, F32, 16, 8, 36, 16, 40, 18, False, False, False, 1, 3),
    DqCase(I8, F16, F32, F32, 13, 11, 30, 15, 30, 13, True, False, False, 0, 1),
    DqCase(I4, F16, F16, F16, 18, 7, 64, 20, 66, 18, False, False, True, 3, 2),
    DqCase(U4, F16, F32, F32, 21, 6, 32, 21, 8, 23, False, True, True, 0, 1),
    DqCase(I4, F16, IMPLICIT, F32, 9, 10, 40, 12, 40, 9, True, False, True, 2, 3),
    DqCase(BF8, F16, F16, F16, 15, 9, 24, 16, 9, 15, False, True, False, 3, 2),
    DqCase(BF8, F16, F32, F32, 12, 8, 32, 12, 34, 14, False, False, True, 1, 2),
]


def main():
    assert ref_gemm_dq is not None, "build the reference shim first: make ref"
    out = {"ncases": np.array(len(CASES))}
    for t, case in enumerate(CASES):
        rng = np.random.default_rng(5150 + t)
        A, B, C0, S, Z = case.operands(rng)
        rc, c = case.run(ref_gemm_dq, A, B, C0, S, Z)
        assert rc == 0
        out.update({"meta%d" % t: meta(case), "a%d" % t: A, "b%d" % t: B, "c0%d" % t: C0, "s%d" % t: S, "z%d" % t: Z, "c%d" % t: c})
    np.savez_compressed(os.path.join(HERE, "dequant.npz"), **out)


if __name__ == "__main__":
    main()
