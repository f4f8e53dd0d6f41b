"""Writes tests/golden/meltw_dispatch.npz: which matrix-eltwise (TPP) descriptors dispatch, the kernel a call of each would run, and
whether its handle runs as a strided batch.

For every point of a fixed grid it records:
  - `typed`: 1 if libxsmm_dispatch_meltw_unary / _binary / _ternary returns a handle, else 0;
  - `desc`: what libxsmm_dispatch_meltw returns for the same descriptor built by libxsmm_meltw_descriptor_init2: 0 NULL, 1 the typed
    route's handle, 2 another handle;
  - `variant`: libxsmm_b200_meltw_variant(handle, NULL), or -1 without a handle;
  - `batch`: libxsmm_b200_meltw_batch_strided(handle, zeroed param, zero strides, 0) -- 0 or LIBXSMM_B200_ERROR_NOT_BATCHABLE, decided
    on the host -- or 1 without a handle.
The grid covers:
  - every op code of each class plus unused codes, crossed with the in / out / comp types a rule names, their neighbours and 6-bit codes
    past LIBXSMM_DATATYPE_B200_COUNT;
  - every subset of the flags a rule or the operand staging reads, for every op at two type tuples;
  - shapes on both sides of every threshold of the kernel choice, and empty extents.
tests/test_meltw_dispatch_table.py rebuilds the grid and compares point by point. No kernel is launched. Run from the repository
root after `make lib`:
    python3 tests/golden/make_golden_meltw_dispatch.py"""
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

F64, F32, BF16, F16, BF8, HF8, I64, I32, U32, I16, U16, I8, U8 = 0, 1, 2, 3, 4, 5, 6, 8, 9, 10, 11, 12, 13
MXBF8, I4X2, MXFP4X2, NVFP4X2, BF32, IMPLICIT, UNSUPPORTED = 14, 18, 20, 21, 24, 25, 26
PAST = [27, 40, 63]              # 6-bit codes past LIBXSMM_DATATYPE_B200_COUNT
TYPES = [F64, F32, BF16, F16, BF8, HF8, I8, I16, I32, U16, MXFP4X2, NVFP4X2, MXBF8,
         U8, U32, I64, BF32, I4X2, IMPLICIT, UNSUPPORTED] + PAST
FEW = [F64, F32, BF16, I8, I16, U16, IMPLICIT, 40]
COMPS = [F32, F64, IMPLICIT]

UNARY, BINARY, TERNARY = 1, 2, 3
OPS = {UNARY: list(range(77)) + [77, 100, 8191], BINARY: list(range(33)) + [33, 100], TERNARY: list(range(20)) + [20, 100]}
# the ops whose family rule reads more than one input type
BINARY_RULE_OPS = [1, 2, 3, 4, 5, 7, 9, 10, 26, 27, 28, 29, 30, 31, 32]
TERNARY_RULE_OPS = [1, 3, 4]

# flags a rule or the staging reads, per class
U_BITMASK, U_BCAST_ROW, U_BCAST_COL, U_BCAST_SCALAR, U_GS_ROWS, U_REDUCE_ROWS = 1, 2, 4, 8, 16, 32
U_IDX4, U_IDX8, U_NO_SCF, U_ARGOP, U_SR = 128, 256, 1024, 2048, 4096
UNARY_FLAGS = [U_BITMASK, U_BCAST_ROW, U_BCAST_COL, U_BCAST_SCALAR, U_GS_ROWS, U_REDUCE_ROWS, U_IDX4, U_IDX8, U_NO_SCF, U_ARGOP, U_SR]
BINARY_FLAGS = [1, 2, 4, 8, 16, 32, 64, 128]                  # BCAST_{ROW,COL,SCALAR}_IN_{0,1}, STOCHASTIC_ROUND, BITMASK
TERNARY_FLAGS = [1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024, 2048]

COLUMNS = ("op_class", "op", "flags", "m", "n", "ldi", "ldi2", "ldi3", "ldo", "t_in0", "t_in1", "t_in2", "t_out", "t_comp")


def _subsets(bits):
    out = [0]
    for b in bits:
        out += [f | b for f in out]
    return out


# per class, two type tuples (in0, in1, in2, out, comp) for the flag sweep: plain f32, and one other the op's rule accepts
def _flag_tuples(cls, op):
    if cls == UNARY:
        t0, to = {42: (F32, I8), 43: (I32, F32), 51: (I16, I16), 52: (I8, I8)}.get(op, (BF16, BF8))
        if op in (54, 55, 57, 58, 59, 60, 61, 62, 71, 72, 74):       # 8-bit layout transforms
            t0, to = I8, I8
        return [(F32, UNSUPPORTED, UNSUPPORTED, F32, F32), (t0, UNSUPPORTED, UNSUPPORTED, to, F32)]
    if cls == BINARY:
        return [(F32, F32, UNSUPPORTED, F32, F32), (BF16, BF16, UNSUPPORTED, BF8, F32) if op != 26 else (BF16, BF16, UNSUPPORTED, F32, F32)]
    return [(F32, F32, F32, F32, F32), (BF16, F16, BF16, BF8, F32)]


# shapes (m, n, ldi, ldo) on both sides of every threshold of xb_meltw_variant, and empty ones
SHAPES = [(64, 64, 64, 64), (64, 63, 64, 64), (63, 65, 64, 64), (65, 63, 72, 65), (64, 32, 64, 128), (64, 32, 64, 127),
          (56, 64, 56, 64), (60, 64, 64, 64), (64, 64, 72, 64), (64, 64, 64, 72), (48, 96, 48, 48), (16, 255, 16, 16), (16, 256, 16, 16),
          (256, 1024, 256, 256), (255, 1029, 256, 256), (256, 1023, 256, 256), (260, 1009, 260, 260), (258, 1017, 260, 258),
          (260, 1009, 262, 260), (512, 512, 512, 512), (1, 1, 1, 1), (0, 4, 16, 16), (16, 0, 16, 16), (-1, 4, 16, 16)]
SHAPE_TYPES = [F64, F32, BF16, F16, HF8, I8, I16]


def grid():
    """the points, one row each (COLUMNS), in a fixed order"""
    rows = []
    m, n, ld = 32, 16, 48
    # types: every op under every in / out / comp type; binary and ternary rule ops under every in1 (and in2) as well
    for op in OPS[UNARY]:
        for t0 in TYPES:
            for to in TYPES:
                for tc in COMPS:
                    rows.append((UNARY, op, 0, m, n, ld, 0, 0, ld, t0, UNSUPPORTED, UNSUPPORTED, to, tc))
    for op in OPS[BINARY]:
        ins1 = TYPES if op in BINARY_RULE_OPS else FEW
        for t0 in TYPES:
            for t1 in ins1:
                for to in TYPES:
                    for tc in COMPS:
                        rows.append((BINARY, op, 0, m, n, ld, ld, 0, ld, t0, t1, UNSUPPORTED, to, tc))
    for op in OPS[TERNARY]:
        rule = op in TERNARY_RULE_OPS
        for t0 in TYPES if rule else FEW:
            for t1 in TYPES if rule else FEW:
                for t2 in (F32, F64, BF16, IMPLICIT) if rule else (F32, IMPLICIT):
                    for to in TYPES if rule else FEW:
                        for tc in COMPS:
                            rows.append((TERNARY, op, 0, m, n, ld, ld, ld, ld, t0, t1, t2, to, tc))
        if rule:
            for t2 in TYPES:
                for tt in (F32, F64, BF16, HF8):
                    for tc in COMPS:
                        rows.append((TERNARY, op, 0, m, n, ld, ld, ld, ld, tt, tt, t2, tt, tc))
    # flags: every subset of the flags the rules read, for every op at two type tuples
    for cls, bits in ((UNARY, UNARY_FLAGS), (BINARY, BINARY_FLAGS), (TERNARY, TERNARY_FLAGS)):
        for op in OPS[cls]:
            for t0, t1, t2, to, tc in _flag_tuples(cls, op):
                for flags in _subsets(bits):
                    rows.append((cls, op, flags, m, n, ld, ld if cls > UNARY else 0, ld if cls == TERNARY else 0, ld, t0, t1, t2, to, tc))
    # shapes: unary ops under the flags the kernel choice reads, binary / ternary plain
    for op in OPS[UNARY]:
        for tt in SHAPE_TYPES:
            for flags in (0, U_REDUCE_ROWS, U_GS_ROWS):
                for sm, sn, sldi, sldo in SHAPES:
                    rows.append((UNARY, op, flags, sm, sn, sldi, 0, 0, sldo, tt, UNSUPPORTED, UNSUPPORTED, tt, F32))
    for cls in (BINARY, TERNARY):
        for op in (1, 26) if cls == BINARY else (1, 3):
            for sm, sn, sldi, sldo in SHAPES:
                rows.append((cls, op, 0, sm, sn, sldi, sldi, sldi if cls == TERNARY else 0, sldo, BF16 if op == 26 else F32, F32 if cls == BINARY and op != 26 else BF16 if op == 26 else F32,
                             F32 if cls == TERNARY else UNSUPPORTED, F32, F32))
    return np.array(rows, dtype=np.int64)


def digest(g):
    return hashlib.sha256(np.ascontiguousarray(g).tobytes()).hexdigest()


class Blob(C.Structure):
    _fields_ = [("data", C.c_ubyte * 96)]


def _bind():
    lib = X.lib
    init2 = lib.libxsmm_meltw_descriptor_init2
    init2.restype = C.c_void_p
    init2.argtypes = [C.POINTER(Blob)] + [C.c_int] * 5 + [C.c_int] * 6 + [C.c_ushort, C.c_ushort, C.c_ubyte]
    disp = lib.libxsmm_dispatch_meltw
    disp.restype = C.c_void_p
    disp.argtypes = [C.c_void_p]
    return init2, disp


def _typed(row):
    cls, op, flags, m, n, ldi, ldi2, ldi3, ldo, t0, t1, t2, to, tc = row
    if cls == UNARY:
        return X.libxsmm_dispatch_meltw_unary(op, X.MeltwUnaryShape(m, n, ldi, ldo, t0, to, tc), flags)
    if cls == BINARY:
        return X.libxsmm_dispatch_meltw_binary(op, X.MeltwBinaryShape(m, n, ldi, ldi2, ldo, t0, t1, to, tc), flags)
    return X.libxsmm_dispatch_meltw_ternary(op, X.MeltwTernaryShape(m, n, ldi, ldi2, ldi3, ldo, t0, t1, t2, to, tc), flags)


REGISTRY_LIMIT = 8192
CHUNK = REGISTRY_LIMIT // 2
NOT_BATCHABLE = -6


def _sweep_chunk(g):
    """in a fresh child: the four answers of every point, and the number of handles the registry then holds"""
    X.libxsmm_finalize()                         # empties the registry the child inherited
    init2, disp = _bind()
    blob = Blob()
    param = (C.c_ubyte * 256)()
    strides = X.MeltwStrides()
    out = np.zeros((len(g), 4), dtype=np.int8)
    for i, r in enumerate(g):
        row = tuple(int(v) for v in r)
        cls, op, flags, m, n, ldi, ldi2, ldi3, ldo, t0, t1, t2, to, tc = row
        h = _typed(row)
        init2(C.byref(blob), t0, t1, t2, tc, to, m, n, ldi, ldo, ldi2, ldi3, flags, op, cls)
        hd = disp(C.byref(blob))
        out[i, 0] = 1 if h else 0
        out[i, 1] = 0 if not hd else (1 if hd == h else 2)
        out[i, 2] = X.libxsmm_b200_meltw_variant(h, None) if h else -1
        out[i, 3] = X.libxsmm_b200_meltw_batch_strided(h, C.addressof(param), C.byref(strides), 0) if h else 1
    info = X.RegistryInfo()
    assert X.libxsmm_get_registry_info(C.byref(info)) == 0
    return out, int(info.size)


def sweep(g):
    """the answers of every point; each chunk runs in its own child process, and returns the registry size it reached"""
    ctx = multiprocessing.get_context("fork")     # a child only calls the library's host code
    chunks = [g[i:i + CHUNK] for i in range(0, len(g), CHUNK)]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)    # the pool forks each child from its own handler thread
        with ctx.Pool(processes=min(8, os.cpu_count() or 1), maxtasksperchild=1) as pool:
            results = pool.map(_sweep_chunk, chunks, chunksize=1)
    return np.concatenate([out for out, _ in results]), max(size for _, size in results)


def main():
    g = grid()
    got, peak = sweep(g)
    assert peak <= REGISTRY_LIMIT // 2, peak
    np.savez_compressed(os.path.join(HERE, "meltw_dispatch.npz"), answers=got, grid_sha256=np.array(digest(g)), columns=np.array(COLUMNS))
    print("%d points, %d dispatched, %d batchable, busiest child registered %d handles"
          % (len(g), int(np.count_nonzero(got[:, 0])), int(np.count_nonzero((got[:, 0] == 1) & (got[:, 3] == 0))), peak))


if __name__ == "__main__":
    main()
