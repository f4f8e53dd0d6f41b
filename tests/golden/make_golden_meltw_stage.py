"""Writes tests/golden/meltw_stage.npz: what one matrix-eltwise call stages, and whether a one-node equation over its descriptor
dispatches, on the simulated device.

The host_*.c sources, tests/c/hostsim_runtime.c and tests/c/hostsim_meltw_stage.c are linked into
tests/c/_hostsim/meltw_stage/libxsmm.so with xb_rt_upload, xb_rt_memcpy_async and xb_meltw_launch wrapped: uploads and copies back
are logged, and a launch is recorded and answered with 0 without running anything.

The descriptors are those tests/golden/meltw_dispatch.npz records as dispatching, from its type and flag sweeps (every op of each
class under every type tuple and every subset of the flags the rules read), each at two small shapes. For each it makes one call
with every operand pageable; a call that is refused for that (the operations that need device-accessible memory) is made again with
every operand pinned. Every pointer slot of the argument struct points at its own buffer, whose first words are 3 (a count the ops
can read), then plane offsets. Per call it records (COLUMNS):
  - the pointer kind the call ran with (0 pageable, 3 pinned) and the number of launches;
  - per slot of the argument struct, the bytes uploaded from it and the bytes copied back to it;
  - for each pointer field of xb_meltw_args: 0 NULL, 1 + k the caller's slot k, 99 a staged or scratch buffer;
  - the bits of alpha, n_rt and off[0], off[1].
Then, per descriptor without its comp type (an equation node computes in its own type), whether libxsmm_dispatch_meqn accepts the op
at the first shape as the head of a one-node equation over arguments, and below an IDENTITY head. It is asked only where the product
(libxsmm_b200.so) dispatches the descriptor of every node as the equation builds it, so that the answer does not depend on how the
simulated device rules. A reduction's equation gets the reduced output shape.
tests/test_meltw_stage_hostsim.py recomputes and compares point by point. Run from the repository root after `make oracle`:
    python3 tests/golden/make_golden_meltw_stage.py"""
import ctypes as C
import hashlib
import multiprocessing
import os
import subprocess
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)
import libxsmm_b200 as X  # noqa: E402  (constants, struct layouts and the product's dispatch rule; calls go to the simulation library)
import make_golden_meltw_dispatch as T  # noqa: E402

CSRC = os.path.join(ROOT, "libxsmm_b200", "csrc")
ORACLE = os.path.join(ROOT, "oracle")
OUT = os.path.join(ROOT, "tests", "c", "_hostsim", "meltw_stage")
HOST_C = ["host_core.c", "host_thunks.c", "host_sparse.c", "host_meltw.c", "host_utils.c", "host_meqn.c"]

SHAPES = [(8, 4, 8, 8), (13, 5, 24, 20)]
NSLOTS = 28                                    # pointer slots of the largest argument struct (ternary: op + 4 matrix args)
FIELDS = ("in0", "in1", "in2", "out", "in_aux", "out_aux", "rng", "rnd", "rnd8")
COLUMNS = ("ptr_kind", "launches") + tuple("up%d" % i for i in range(NSLOTS)) + tuple("down%d" % i for i in range(NSLOTS)) + \
    FIELDS + ("alpha_bits", "n_rt", "off0", "off1")
EQN_COLUMNS = ("eqn_head", "eqn_below")
BUF = 1 << 16
STAGED = 99


class Copy(C.Structure):
    _fields_ = [("host", C.c_void_p), ("bytes", C.c_ulonglong)]


class Args(C.Structure):
    _fields_ = [(f, C.c_void_p) for f in ("in0", "in1", "in2", "out", "in_aux", "out_aux")] + \
        [("alpha", C.c_float), ("n_rt", C.c_ulonglong), ("off", C.c_ulonglong * 2), ("rng", C.c_void_p), ("rnd", C.c_void_p),
         ("rnd8", C.c_void_p), ("count", C.c_longlong)] + [(f, C.c_longlong) for f in ("s_in0", "s_in1", "s_in2", "s_in_aux", "s_out", "s_out_aux")]


def build_sim():
    os.makedirs(OUT, exist_ok=True)
    if not os.path.exists(os.path.join(ORACLE, "liboracle.so")):
        subprocess.check_call(["make", "-C", ROOT, "oracle"])
    so = os.path.join(OUT, "libxsmm.so")
    srcs = [os.path.join(CSRC, f) for f in HOST_C] + [os.path.join(ROOT, "tests", "c", f) for f in ("hostsim_runtime.c", "hostsim_meltw_stage.c")]
    deps = srcs + [os.path.join(CSRC, "xb_internal.h"), os.path.join(CSRC, "xb_device.cuh")]
    if not (os.path.exists(so) and all(os.path.getmtime(s) < os.path.getmtime(so) for s in deps)):
        wrap = ",".join("--wrap=" + f for f in ("xb_rt_upload", "xb_rt_memcpy_async", "xb_meltw_launch"))
        cmd = ["gcc", "-O1", "-std=gnu99", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"), "-Wl," + wrap, "-o", so] + \
            srcs + ["-L" + ORACLE, "-loracle", "-Wl,-rpath," + ORACLE, "-lpthread", "-ldl", "-lm"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-3000:]
    lib = C.CDLL(so)
    P, I = C.c_void_p, C.c_int
    for name, res, args in (("libxsmm_dispatch_meltw_unary", P, [I, X.MeltwUnaryShape, C.c_uint]),
                            ("libxsmm_dispatch_meltw_binary", P, [I, X.MeltwBinaryShape, C.c_uint]),
                            ("libxsmm_dispatch_meltw_ternary", P, [I, X.MeltwTernaryShape, C.c_uint]),
                            ("libxsmm_finalize", None, []), ("libxsmm_meqn_create", I, []),
                            ("libxsmm_meqn_push_back_arg", I, [X.MeqnMetadata, X.MeqnArgShape, X.MatrixArgAttributes]),
                            ("libxsmm_meqn_push_back_unary_op", I, [X.MeqnMetadata, I, I, C.c_uint]),
                            ("libxsmm_meqn_push_back_binary_op", I, [X.MeqnMetadata, I, I, C.c_uint]),
                            ("libxsmm_meqn_push_back_ternary_op", I, [X.MeqnMetadata, I, I, C.c_uint]),
                            ("libxsmm_dispatch_meqn", P, [I, X.MeqnArgShape]),
                            ("hostsim_stage_reset", None, []), ("hostsim_stage_uploads", I, [C.POINTER(C.POINTER(Copy))]),
                            ("hostsim_stage_copies_back", I, [C.POINTER(C.POINTER(Copy))]), ("hostsim_stage_launches", I, []),
                            ("hostsim_stage_args", C.POINTER(Args), [])):
        fn = getattr(lib, name); fn.restype, fn.argtypes = res, args
    return lib


def cases():
    """(op_class, op, flags, t_in0, t_in1, t_in2, t_out, t_comp) of every descriptor the CPU table accepts in its type and flag sweeps"""
    want = np.load(os.path.join(HERE, "meltw_dispatch.npz"))
    g = T.grid()
    assert T.digest(g) == str(want["grid_sha256"])
    c = dict((name, i) for i, name in enumerate(T.COLUMNS))
    sel = (want["answers"][:, 0] == 1) & (g[:, c["m"]] == 32) & (g[:, c["n"]] == 16)
    keys = g[sel][:, [c[k] for k in ("op_class", "op", "flags", "t_in0", "t_in1", "t_in2", "t_out", "t_comp")]]
    return np.unique(keys, axis=0)


def served(cls, op, t0, t1, t2, to, tc):
    """whether the product (libxsmm_b200.so, whose rule tests/test_meltw_dispatch_table.py pins) dispatches this descriptor"""
    m, n, ld, _ = SHAPES[0]
    return bool(T._typed((cls, op, 0, m, n, ld, ld, ld, ld, t0, t1, t2, to, tc)))


class Runner:
    def __init__(self, lib):
        self.lib = lib
        self.bufs = [np.zeros(BUF // 8, dtype=np.uint64) for _ in range(NSLOTS)]
        for b in self.bufs:
            b[0], b[1], b[2] = 3, 4096, 8192       # a count of 3, then plane offsets
        self.slots = (C.c_void_p * NSLOTS)(*[b.ctypes.data for b in self.bufs])
        self.addr = dict((b.ctypes.data, i) for i, b in enumerate(self.bufs))

    def dispatch(self, key, shape):
        cls, op, flags, t0, t1, t2, to, tc = key
        m, n, ldi, ldo = shape
        lib = self.lib
        if cls == T.UNARY:
            return lib.libxsmm_dispatch_meltw_unary(op, X.MeltwUnaryShape(m, n, ldi, ldo, t0, to, tc), flags)
        if cls == T.BINARY:
            return lib.libxsmm_dispatch_meltw_binary(op, X.MeltwBinaryShape(m, n, ldi, ldi, ldo, t0, t1, to, tc), flags)
        return lib.libxsmm_dispatch_meltw_ternary(op, X.MeltwTernaryShape(m, n, ldi, ldi, ldi, ldo, t0, t1, t2, to, tc), flags)

    def call(self, kern, kind):
        os.environ["XB_HOSTSIM_PTR_KIND"] = str(kind)
        for b in self.bufs:
            b[0], b[1], b[2] = 3, 4096, 8192
        self.lib.hostsim_stage_reset()
        C.CFUNCTYPE(None, C.c_void_p)(kern)(C.addressof(self.slots))
        return self.lib.hostsim_stage_launches()

    def code(self, p):
        return 0 if not p else (1 + self.addr[p] if p in self.addr else STAGED)

    def stage(self, key, shape):
        kern = self.dispatch(key, shape)
        assert kern, key
        kind = 0
        if self.call(kern, 0) == 0:
            kind = 3
            self.call(kern, 3)
        row = [kind, self.lib.hostsim_stage_launches()]
        up, down = [0] * NSLOTS, [0] * NSLOTS
        for get, acc in ((self.lib.hostsim_stage_uploads, up), (self.lib.hostsim_stage_copies_back, down)):
            log = C.POINTER(Copy)()
            for i in range(get(C.byref(log))):
                k = self.code(log[i].host)
                assert 1 <= k <= NSLOTS, (key, "a copy to or from memory the caller does not own")
                acc[k - 1] += log[i].bytes
        a = self.lib.hostsim_stage_args().contents
        row += up + down + [self.code(getattr(a, f)) for f in FIELDS]
        row += [int(np.float32(a.alpha).view(np.uint32)), a.n_rt, a.off[0], a.off[1]]
        return row

    def eqn(self, key, below):
        """0 / 1: whether the equation dispatches; -1: not asked, because the product declines the descriptor of a node as the
        equation builds it (its comp type is its own type, a SELECT's third input is IMPLICIT)"""
        cls, op, flags, t0, t1, t2, to = key
        m, n, ld, _ = SHAPES[0]
        if not served(cls, op, t0, t1, T.IMPLICIT if (cls, op) == (T.TERNARY, X.MELTW_TYPE_TERNARY_SELECT) else t2, to, to):
            return -1
        if below and not served(T.UNARY, X.MELTW_TYPE_UNARY_IDENTITY, to, T.UNSUPPORTED, T.UNSUPPORTED, to, to):
            return -1
        om, on = m, n
        if cls == T.UNARY and op in REDUCE_OPS:
            om, on = (n, 1) if flags & T.U_REDUCE_ROWS else (m, 1)
        elif cls == T.UNARY and op == X.MELTW_TYPE_UNARY_REDUCE_TO_SCALAR_OP_ADD:
            om, on = 1, 1
        lib = self.lib
        eq = lib.libxsmm_meqn_create()
        assert eq >= 0
        if below:
            assert lib.libxsmm_meqn_push_back_unary_op(X.MeqnMetadata(eq, -1), X.MELTW_TYPE_UNARY_IDENTITY, to, 0) == 0
        push = {T.UNARY: lib.libxsmm_meqn_push_back_unary_op, T.BINARY: lib.libxsmm_meqn_push_back_binary_op,
                T.TERNARY: lib.libxsmm_meqn_push_back_ternary_op}[cls]
        assert push(X.MeqnMetadata(eq, 0), op, to, flags) == 0
        for pos, t in enumerate((t0, t1, t2)[:cls]):
            assert lib.libxsmm_meqn_push_back_arg(X.MeqnMetadata(eq, pos), X.MeqnArgShape(m, n, ld, t), X.MatrixArgAttributes(0, 0, 0, 0)) == 0
        return 1 if lib.libxsmm_dispatch_meqn(eq, X.MeqnArgShape(om, on, om, to)) else 0


REDUCE_OPS = (X.MELTW_TYPE_UNARY_REDUCE_X_OP_ADD, X.MELTW_TYPE_UNARY_REDUCE_X2_OP_ADD, X.MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD,
              X.MELTW_TYPE_UNARY_REDUCE_X_OP_MAX, X.MELTW_TYPE_UNARY_REDUCE_X_OP_MIN, X.MELTW_TYPE_UNARY_REDUCE_X_OP_ABSMAX)
# a child makes this many calls (each dispatch takes a registry slot, of 8192), or this many equations (two each, of 256)
CHUNK, EQN_CHUNK = 2000, 120


def _stage_chunk(keys):
    r = Runner(build_sim())
    return np.array([r.stage(tuple(int(v) for v in key), shape) for key in keys for shape in SHAPES], dtype=np.int64).reshape(-1, len(COLUMNS))


def _eqn_chunk(keys):
    X.libxsmm_finalize()                           # the product's registry, for served(): empty in every child
    r = Runner(build_sim())
    return np.array([[r.eqn(tuple(int(v) for v in key), below) for below in (False, True)] for key in keys], dtype=np.int64).reshape(-1, 2)


def _pool_map(fn, keys, chunk):
    ctx = multiprocessing.get_context("fork")      # a child only calls the library's host code
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        with ctx.Pool(processes=min(8, os.cpu_count() or 1), maxtasksperchild=1) as pool:
            return np.concatenate(pool.map(fn, [keys[i:i + chunk] for i in range(0, len(keys), chunk)], chunksize=1))


def sweep(keys):
    """(the staging of every descriptor at every shape, the equation answers of every descriptor without its comp type)"""
    build_sim()                                    # once, before the children load it
    return _pool_map(_stage_chunk, keys, CHUNK), _pool_map(_eqn_chunk, np.unique(keys[:, :7], axis=0), EQN_CHUNK)


def digest(keys):
    return hashlib.sha256(np.ascontiguousarray(keys).tobytes()).hexdigest()


def save(path, keys, stage, eqn):
    """most calls stage alike: the fixture keeps each distinct staging row once, and per call the index of its row"""
    rows, call_row = np.unique(stage, axis=0, return_inverse=True)
    assert len(rows) < 1 << 16
    np.savez_compressed(path, rows=rows, call_row=call_row.reshape(-1).astype(np.uint16), eqn=eqn.astype(np.int8),
                        keys_sha256=np.array(digest(keys)), columns=np.array(COLUMNS))


def load(path):
    """(the staging row of every call, the equation answers) as main() recorded them"""
    f = np.load(path)
    return f["rows"][f["call_row"].astype(np.int64)], f["eqn"].astype(np.int64), str(f["keys_sha256"])


def main():
    keys = cases()
    stage, eqn = sweep(keys)
    save(os.path.join(HERE, "meltw_stage.npz"), keys, stage, eqn)
    print("%d descriptors, %d calls, %d equations dispatched" % (len(keys), len(stage), int(np.count_nonzero(eqn == 1))))


if __name__ == "__main__":
    main()
