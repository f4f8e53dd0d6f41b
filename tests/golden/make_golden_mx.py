"""Writes tests/golden/mxfp8.npz: MX fp8 GEMM cases (MXBF8 / MXHF8, F32 and MXBF8 C, beta 0 / 1, no batch-reduce and stride)
with the C and C-scale bytes computed by the UNMODIFIED reference's libxsmm_reference_gemm (oracle/_ref/libxsmm_ref_mx.so, built
by `make ref`). The GPU tests compare against these bytes where the reference is absent. Run from the repository root:
    python3 tests/golden/make_golden_mx.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from mx_ffi import F32, MXBF8, MXHF8, MxCase, ref_gemm_mx  # noqa: E402

# (ta, tc, m, n, k, lda, ldb, ldc, beta0, br_type, br)
CASES = [
    (MXBF8, F32, 24, 10, 64, 28, 11, 26, 1, 0, 1), (MXHF8, F32, 24, 10, 64, 28, 11, 26, 0, 0, 1),
    (MXBF8, F32, 16, 16, 96, 16, 16, 16, 0, 3, 3), (MXHF8, F32, 40, 7, 128, 41, 8, 44, 1, 3, 2),
    (MXBF8, MXBF8, 32, 6, 64, 36, 6, 64, 1, 0, 1), (MXBF8, MXBF8, 64, 5, 32, 64, 5, 96, 1, 3, 4),
]


def main():
    assert ref_gemm_mx is not None, "build the reference shim first: make ref"
    out = {"ncases": np.array(len(CASES))}
    for t, meta in enumerate(CASES):
        case = MxCase(*meta)
        rng = np.random.default_rng(4242 + t)
        a, b, c0, sa, sb, cs0 = case.operands(rng)
        rc, c, cs = case.run(ref_gemm_mx, a, b, c0, sa, sb, cs0)
        assert rc == 0
        out.update({"meta%d" % t: np.array(meta, np.int64), "a%d" % t: a, "b%d" % t: b, "c0%d" % t: c0, "as%d" % t: sa, "bs%d" % t: sb,
                    "cs0%d" % t: cs0, "c%d" % t: c, "cs%d" % t: cs})
    np.savez_compressed(os.path.join(HERE, "mxfp8.npz"), **out)


if __name__ == "__main__":
    main()
