"""Writes tests/golden/lowbit.npz: low-bit weight GEMM cases (I2 / I1 x I8 / U8 -> I32, MXFP4 x I8 -> F32 / BF16; every batch-reduce
mode, beta 0 / 1, ld > dim, m and n not multiples of 32) with the C bytes computed by the UNMODIFIED reference's libxsmm_reference_gemm
(oracle/_ref/libxsmm_ref_lowbit.so, built by `make ref`). The GPU tests compare against these bytes where the reference is absent. Run
from the repository root:
    python3 tests/golden/make_golden_lowbit.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from lowbit_ffi import BF16, F32, I1, I2, I8, I32, MXFP4, U8, LbCase, meta, ref_gemm_lowbit  # noqa: E402

# LbCase(ta, tb, tc, m, n, k, lda, ldb, ldc, beta0, br_type, br)
CASES = [
    LbCase(I2, I8, I32, 44, 21, 68, 52, 72, 47, True, 0, 1),
    LbCase(I2, U8, I32, 36, 19, 40, 36, 44, 39, False, 3, 3),
    LbCase(I2, I8, I32, 20, 37, 52, 24, 52, 21, False, 1, 2),
    LbCase(I2, U8, I32, 8, 262, 36, 12, 40, 9, True, 2, 2),
    LbCase(I1, I8, I32, 46, 23, 64, 50, 68, 47, False, 0, 1),
    LbCase(I1, U8, I32, 30, 17, 36, 32, 40, 33, True, 3, 3),
    LbCase(I1, I8, I32, 18, 33, 44, 22, 48, 20, True, 2, 2),
    LbCase(I1, U8, I32, 50, 9, 132, 54, 132, 51, False, 1, 3),
    LbCase(MXFP4, I8, F32, 45, 22, 96, 49, 104, 47, False, 0, 1),
    LbCase(MXFP4, I8, BF16, 29, 31, 64, 33, 70, 30, True, 3, 3),
    LbCase(MXFP4, I8, F32, 17, 40, 160, 17, 160, 20, True, 1, 2),
    LbCase(MXFP4, I8, BF16, 38, 13, 32, 40, 64, 41, False, 2, 3),
    LbCase(MXFP4, I8, F32, 6, 259, 32, 8, 32, 7, False, 3, 2),
]


def main():
    assert ref_gemm_lowbit is not None, "build the reference shim first: make ref"
    out = {"ncases": np.array(len(CASES))}
    for t, case in enumerate(CASES):
        rng = np.random.default_rng(7170 + t)
        A, B, C0, SA, SB = case.operands(rng)
        rc, c = case.run(ref_gemm_lowbit, A, B, C0, SA, SB)
        assert rc == 0
        out.update({"meta%d" % t: meta(case), "a%d" % t: A, "b%d" % t: B, "c0%d" % t: C0, "sa%d" % t: SA, "sb%d" % t: SB, "c%d" % t: c})
    np.savez_compressed(os.path.join(HERE, "lowbit.npz"), **out)


if __name__ == "__main__":
    main()
