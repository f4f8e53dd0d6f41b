#!/usr/bin/env python
"""tools/bench_meltw_batch.py -- one launch per batch against one launch per call: strided mateltwise and equation batches on the GPU,
one JSON line on stdout.

  python tools/bench_meltw_batch.py [--tiles T] [--loop-tiles L] [--steps K] [--warmup W]

Workloads: `tiles` (default 65,536) tiles of 64 x 64, all device-resident, each operand unique:
  F32 RELU with bit mask, BF16 NORM_TO_VNNI2, F32 NORM_TO_NORMT, F32 row REDUCE_X_X2_OP_ADD, and a layernorm-style equation
  (x - colsum(x)) * gamma with gamma shared by every call.
For each: the median kernel time of one batch call (CUDA events, after warm-up), the compulsory bytes from the shapes, GB/s and the
fraction of the data sheet's 3.35 TB/s; and the same handle through a loop of single calls in non-blocking mode over the first
`loop_tiles` tiles (default 4,096), reported per tile, which is the launch-bound way a reference caller runs them. Before timing, the
first, a middle and the last tile of every batch are compared byte for byte with single calls. The card and its power limit are read
in the same run. Nothing is written to the repository tree."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import libxsmm_b200 as X  # noqa: E402

M = N = 64
F32, BF16 = X.DATATYPE_F32, X.DATATYPE_BF16
PEAK = 3350.0


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        power = "unknown"
    return name, power


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def rand_bytes(n, seed):
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return torch.randn(n // 4, device="cuda", generator=g).view(torch.uint8)


class Workload:
    def __init__(self, name, single, batch, nbytes, tiles):
        self.name, self.single, self.batch, self.nbytes, self.tiles = name, single, batch, nbytes, tiles


def unary_workload(name, op, tin, tout, flags, ldo, so, sa, compulsory, tiles):
    ts = 4 if tin == F32 else 2
    k = X.libxsmm_dispatch_meltw_unary(op, X.libxsmm_create_meltw_unary_shape(M, N, M, ldo, tin, tout, F32), flags)
    assert k, name
    sx = M * N * ts
    x = rand_bytes(tiles * sx, 1)
    o = torch.zeros(tiles * so, dtype=torch.uint8, device="cuda")
    a = torch.zeros(tiles * sa, dtype=torch.uint8, device="cuda") if sa else None
    s = X.MeltwStrides(in0=sx, out=so, out_aux=sa)

    def param(t, out, aux):
        p = X.MeltwUnaryParam(); p.inp.primary = x.data_ptr() + t * sx; p.out.primary = out.data_ptr() + t * so
        if aux is not None:
            p.out.secondary = aux.data_ptr() + t * sa
        return p
    p0 = param(0, o, a)
    fn = X.MELTW_UNARY_FN(k)
    params = [param(t, o, a) for t in range(tiles)]

    def batch():
        assert X.libxsmm_b200_meltw_batch_strided(k, C.addressof(p0), C.byref(s), tiles) == 0

    def single(t):
        fn(C.byref(params[t]))

    def check():
        batch(); X.check()
        o1 = torch.zeros_like(o); a1 = torch.zeros_like(a) if a is not None else None
        for t in (0, tiles // 2, tiles - 1):
            fn(C.byref(param(t, o1, a1)))
        X.check()
        for t in (0, tiles // 2, tiles - 1):
            assert torch.equal(o[t * so:(t + 1) * so], o1[t * so:(t + 1) * so]), (name, t)
            if a is not None:
                assert torch.equal(a[t * sa:(t + 1) * sa], a1[t * sa:(t + 1) * sa]), (name, t)
    w = Workload(name, single, batch, compulsory * tiles, tiles)
    w.check = check
    return w


def layernorm_workload(tiles):
    eq = X.libxsmm_meqn_create()
    sing = X.libxsmm_create_matrix_arg_attributes(0, 0, 0, 0)
    md = X.libxsmm_create_meqn_op_metadata(eq, -1)
    X.libxsmm_meqn_push_back_binary_op(md, X.MELTW_TYPE_BINARY_MUL, F32, X.MELTW_FLAG_BINARY_BCAST_COL_IN_1)
    X.libxsmm_meqn_push_back_binary_op(md, X.MELTW_TYPE_BINARY_SUB, F32, X.MELTW_FLAG_BINARY_BCAST_COL_IN_1)
    X.libxsmm_meqn_push_back_arg(X.libxsmm_create_meqn_arg_metadata(eq, 0), X.libxsmm_create_meqn_arg_shape(M, N, M, F32), sing)
    X.libxsmm_meqn_push_back_unary_op(md, X.MELTW_TYPE_UNARY_REDUCE_X_OP_ADD, F32, X.MELTW_FLAG_UNARY_REDUCE_COLS)
    X.libxsmm_meqn_push_back_arg(X.libxsmm_create_meqn_arg_metadata(eq, 0), X.libxsmm_create_meqn_arg_shape(M, N, M, F32), sing)
    X.libxsmm_meqn_push_back_arg(X.libxsmm_create_meqn_arg_metadata(eq, 1), X.libxsmm_create_meqn_arg_shape(M, 1, M, F32), sing)
    k = X.libxsmm_dispatch_meqn(eq, X.MeqnArgShape(M, N, M, F32))
    assert k
    sx = M * N * 4
    x, gamma = rand_bytes(tiles * sx, 2), rand_bytes(M * 4, 3)
    o = torch.zeros(tiles * sx, dtype=torch.uint8, device="cuda")
    keep = []

    def param(t, out):
        ins = (X.MatrixArg * 2)(); ins[0].primary, ins[1].primary = x.data_ptr() + t * sx, gamma.data_ptr()
        p = X.MeqnParam(); p.inputs, p.output.primary = C.addressof(ins), out.data_ptr() + t * sx
        keep.append(ins)
        return p
    st = (C.c_longlong * 2)(sx, 0)
    p0 = param(0, o)
    fn = X.MEQN_FN(k)
    params = [param(t, o) for t in range(tiles)]

    def batch():
        assert X.libxsmm_b200_meqn_batch_strided(k, C.byref(p0), st, sx, 0, None, tiles) == 0

    def single(t):
        fn(C.byref(params[t]))

    def check():
        batch(); X.check()
        o1 = torch.zeros_like(o)
        for t in (0, tiles // 2, tiles - 1):
            fn(C.byref(param(t, o1)))
        X.check()
        for t in (0, tiles // 2, tiles - 1):
            assert torch.equal(o[t * sx:(t + 1) * sx], o1[t * sx:(t + 1) * sx]), ("layernorm", t)
    # x read by the reduction and by the subtraction (the second read may hit L2), the output written; gamma is 256 B
    w = Workload("layernorm equation f32", single, batch, 2 * sx * tiles, tiles)
    w.check = check
    return w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=65536)
    ap.add_argument("--loop-tiles", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    T = args.tiles
    f4, b2 = M * N * 4, M * N * 2
    loads = [
        unary_workload("relu f32 + bit mask", X.MELTW_TYPE_UNARY_RELU, F32, F32, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT, M, f4, M // 8 * N,
                       2 * f4 + M // 8 * N, T),
        unary_workload("norm->vnni2 bf16", X.MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_VNNI2, BF16, BF16, 0, M, b2, 0, 2 * b2, T),
        unary_workload("norm->normt f32", X.MELTW_TYPE_UNARY_TRANSFORM_NORM_TO_NORMT, F32, F32, 0, M, f4, 0, 2 * f4, T),
        unary_workload("rows reduce_x_x2 f32", X.MELTW_TYPE_UNARY_REDUCE_X_X2_OP_ADD, F32, F32, X.MELTW_FLAG_UNARY_REDUCE_ROWS, N, 2 * N * 4, 0,
                       f4 + 2 * N * 4, T),
        layernorm_workload(T),
    ]
    out = {"metric": "strided mateltwise / equation batches: one launch per batch vs a loop of single calls", "tiles": T,
           "tile": "64 x 64", "loop_tiles": args.loop_tiles, "steps": args.steps, "warmup": args.warmup, "workloads": []}
    for w in loads:
        w.check()
        ms = timed(w.batch, args.steps, args.warmup)
        X.libxsmm_b200_set_blocking(0)
        n = min(args.loop_tiles, w.tiles)

        def loop():
            for t in range(n):
                w.single(t)
        loop_ms = timed(loop, max(2, args.steps // 3), 1)
        X.libxsmm_b200_set_blocking(1)
        X.check()
        gbs = w.nbytes / (ms * 1e-3) / 1e9
        out["workloads"].append({"op": w.name, "batch_ms": ms, "compulsory_bytes": w.nbytes, "GBps": gbs, "hbm_frac": gbs / PEAK,
                                 "batch_us_per_tile": ms * 1e3 / w.tiles, "single_call_loop_us_per_tile": loop_ms * 1e3 / n,
                                 "checked_tiles": [0, w.tiles // 2, w.tiles - 1]})
    name, power = card()
    out.update({"card": name, "power_limit": power, "peak_GBps": PEAK, "peak_src": "H100 SXM data sheet"})
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
