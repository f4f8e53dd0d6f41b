"""TEST INFRASTRUCTURE: edge-case operands for the max / min / absmax / argop reductions, shared by the CPU pins
(tests/test_oracle_meltw_edges.py) and the GPU tests (tests/test_meltw_exact_gpu.py).

Every sequence is one reduced line: a column of the matrix under REDUCE_ROWS, a row of it under REDUCE_COLS. The sequences put
+0 / -0 in both orders, all -inf / all +inf, exactly +-FLT_MAX, (for f64) values beyond FLT_MAX, NaNs of both signs and distinct
payloads (one of them signalling) first, in the middle and last, runs of equal extrema at several positions and x next to -x."""
import numpy as np

import gen

FLT_MAX = float(np.finfo(np.float32).max)
# three NaNs per type: quiet positive, quiet negative with another payload, signalling positive
NAN_BITS = {
    gen.F64: (0x7FF8000000000001, 0xFFF80000000ABCDE, 0x7FF0000000000003),
    gen.F32: (0x7FC00001, 0xFFC00ABC, 0x7F800003),
    gen.BF16: (0x7FC1, 0xFFC5, 0x7F81),
    gen.F16: (0x7E01, 0xFE05, 0x7C01),
}
BITS_OF = {gen.F64: np.uint64, gen.F32: np.uint32, gen.BF16: np.uint16, gen.F16: np.uint16}


def sequences(rng, L):
    """(values, nan_code): float64 values and, per element, 0 or the 1-based index of the NaN of NAN_BITS it stands for"""
    seqs = []

    def add(v, code=None):
        v = np.asarray(v, dtype=np.float64)
        seqs.append((v, np.zeros(L, dtype=np.int64) if code is None else code))

    def nan_at(v, pos, which=1):
        code = np.zeros(L, dtype=np.int64)
        for p, w in zip(pos, which if isinstance(which, (list, tuple)) else [which] * len(pos)):
            code[p] = w
        add(v, code)

    ints = lambda: rng.integers(-3, 4, size=L).astype(np.float64)          # noqa: E731  (many ties)
    normals = lambda: np.round(rng.standard_normal(L) * 8) / 4             # noqa: E731
    add(ints())
    add(-np.abs(ints()) - 1)                                                 # all negative: the column folds' -FLT_MAX start survives nothing
    add(np.where(rng.integers(0, 2, size=L) == 1, 0.0, -0.0))               # +0 / -0 mixed
    add(np.full(L, -0.0)); add(np.full(L, 0.0))
    z = np.full(L, 0.0); z[0] = -0.0; add(z)                                 # -0 first
    z = np.full(L, -0.0); z[-1] = 0.0; add(z)                                # +0 last
    add(np.full(L, -np.inf)); add(np.full(L, np.inf))
    add(rng.choice(np.array([-FLT_MAX, FLT_MAX, -np.inf, np.inf]), size=L))
    add(rng.choice(np.array([-FLT_MAX, -np.inf]), size=L))
    add(rng.choice(np.array([FLT_MAX, np.inf]), size=L))
    add(rng.choice(np.array([-1e39, 1e39, -1e300, 1e300, -FLT_MAX, 3.0]), size=L))   # beyond FLT_MAX: inf in the 32-bit types
    x = np.abs(ints()) + 1; x[1::2] = -x[0::2][: L // 2]; add(x)            # x next to -x
    x = ints(); x[rng.permutation(L)[: max(1, L // 3)]] = x.max(); add(x)    # a run of equal maxima at several positions
    x = ints(); x[rng.permutation(L)[: max(1, L // 3)]] = x.min(); add(x)
    for pos in sorted({0, L // 2, L - 1}):
        nan_at(normals(), [pos], 1)
        nan_at(ints(), [pos], 2)
        nan_at(np.full(L, -np.inf), [pos], 3)
    if L >= 3:
        nan_at(normals(), [L // 3, (2 * L) // 3], [1, 2])
        nan_at(np.where(rng.integers(0, 2, size=L) == 1, 0.0, -0.0), [0, L - 1], [3, 1])
    nan_at(np.zeros(L), list(range(L)), [(k % 3) + 1 for k in range(L)])   # all NaN
    z = np.where(rng.integers(0, 2, size=L) == 1, 0.0, -0.0); nan_at(z, [0], 2)
    return seqs


def encode(seqs, t):
    """(K, L) array of the element bits of type t"""
    vals = np.stack([v for v, _ in seqs]); code = np.stack([c for _, c in seqs])
    if t == gen.F64:
        out = vals.view(np.uint64).copy()
    elif t == gen.F32:
        with np.errstate(over="ignore"):
            out = vals.astype(np.float32).view(np.uint32).copy()
    elif t == gen.BF16:
        with np.errstate(over="ignore"):
            out = (vals.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)      # truncation: exact for the small integers
    else:
        with np.errstate(over="ignore"):
            out = vals.astype(np.float16).view(np.uint16).copy()
    for w in (1, 2, 3):
        out[code == w] = NAN_BITS[t][w - 1]
    return out


def layout(seq_bits, rows, pad, fill):
    """matrix holding the sequences as its reduced lines: REDUCE_ROWS -> column k = sequence k (m = L, n = K), otherwise
    row k = sequence k (m = K, n = L); ldi = m + pad, the padding filled with `fill` bits. Returns (flat bits, m, n, ldi)."""
    K, L = seq_bits.shape
    m, n = (L, K) if rows else (K, L)
    ldi = m + pad
    a = np.full((n, ldi), fill, dtype=seq_bits.dtype)
    if rows:
        a[:, :m] = seq_bits
    else:
        a[:, :m] = seq_bits.T
    return a.reshape(-1).copy(), m, n, ldi
