#!/usr/bin/env python
"""tools/bench_lowbit.py -- low-bit weight GEMM on the GPU: batched strided BRGEMM for each low-bit form and, on the same shapes, the
existing I8 x I8 -> I32 handle; one JSON line per workload on stdout.

  python tools/bench_lowbit.py [--steps K] [--warmup W] [--batch B]

Workload: m = n = 64, k = 256, br = 8 (stride mode), `batch` tiles (default 4,096), beta = 0, every operand unique and device-resident,
one batch call per step:
  I2 x I8 -> I32       ternary A (2 bits per weight), libxsmm_b200_gemm_batch_strided
  I1 x I8 -> I32       binary A (1 bit per weight), libxsmm_b200_gemm_batch_strided
  MXFP4 x I8 -> F32    E8M0 A scales per (row, 32 k), f32 B scales per (column, 32 k), libxsmm_b200_gemm_batch_strided_scaled
  I8 x I8 -> I32       VNNI4 A, libxsmm_b200_gemm_batch_strided (the existing dp4a kernel)
Before timing, the first and the last tile of each low-bit form are compared with the oracle (oracle/oracle_lowbit.c) bit for bit.
Timing: CUDA events around each step, median of `steps` steps after `warmup` steps. Reported: int-op/s (2 m n k br per tile) and the
compulsory traffic (every operand byte read once, C written once) per second. The card and its power limit are read in the same run.
Nothing is written to the repository tree."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import libxsmm_b200 as X  # noqa: E402
from lowbit_ffi import F32, I1, I2, I8, I32, MXFP4, LbCase, oracle_gemm_lowbit, same_c  # noqa: E402

M = N = 64
K = 256
BR = 8


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        power = "unknown"
    return name, power


def timed(step, steps, warmup):
    for _ in range(warmup):
        step()
    times = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); step(); e1.record(); e1.synchronize()
        times.append(e0.elapsed_time(e1))
    X.check()
    return float(np.median(times)), float(np.min(times))


def rand_bytes(n, gen):
    return torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda", generator=gen)


def run_lowbit(ta, batch, steps, warmup, gen):
    case = LbCase(ta, I8, F32 if ta == MXFP4 else I32, M, N, K, beta0=True, br_type=3, br=BR)
    sa, sb, sc = case.size_a, case.size_b, 4 * case.size_c
    a, b = rand_bytes(batch * sa, gen), rand_bytes(batch * sb, gen)
    c = torch.empty(batch * sc, dtype=torch.uint8, device="cuda")
    ssa, ssb = case.size_sa, 4 * case.size_sb
    scf_a = torch.randint(120, 134, (batch * ssa,), dtype=torch.uint8, device="cuda", generator=gen) if case.mx() else None
    scf_b = (torch.randn(batch * case.size_sb, device="cuda", generator=gen) * 0.01) if case.mx() else None
    h = X.libxsmm_dispatch_brgemm(X.libxsmm_create_gemm_shape(M, N, K, M, K, M, ta, I8, case.tc, I32), case.flags, 0,
                                  X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, case.stride_a, case.stride_b, 0))
    assert h and X.libxsmm_b200_kernel_backend(h) == X.BACKEND_SIMT

    def step():
        if case.mx():
            rc = X.libxsmm_b200_gemm_batch_strided_scaled(h, a.data_ptr(), b.data_ptr(), c.data_ptr(), sa, sb, sc,
                                                          scf_a.data_ptr(), scf_b.data_ptr(), None, ssa, ssb, 0, BR, batch)
        else:
            rc = X.libxsmm_b200_gemm_batch_strided(h, a.data_ptr(), b.data_ptr(), c.data_ptr(), sa, sb, sc, BR, batch)
        assert rc == 0, rc
    launches = X.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT)
    step(); torch.cuda.synchronize(); X.check()
    assert X.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT) == launches + 1
    for t in (0, batch - 1):                     # sample check against the oracle
        ops = [a[t * sa:(t + 1) * sa].cpu().numpy(), b[t * sb:(t + 1) * sb].cpu().numpy(), np.zeros(case.size_c, case.c_dtype),
               scf_a[t * ssa:(t + 1) * ssa].cpu().numpy() if case.mx() else np.zeros(1, np.uint8),
               scf_b[t * case.size_sb:(t + 1) * case.size_sb].cpu().numpy() if case.mx() else np.zeros(1, np.float32)]
        _, want = case.run(oracle_gemm_lowbit, *ops)
        assert same_c(case, want, c[t * sc:(t + 1) * sc].cpu().numpy().view(case.c_dtype)), "tile %d differs from the oracle" % t
    ms, ms_min = timed(step, steps, warmup)
    per_tile = sa + sb + sc + (ssa + ssb if case.mx() else 0)
    name = {I2: "I2 x I8 -> I32", I1: "I1 x I8 -> I32", MXFP4: "MXFP4 x I8 -> F32, block scales"}[ta]
    return name, "gemm_lowbit_kernel (dp4a, CUDA cores)", ms, ms_min, per_tile


def run_i8(batch, steps, warmup, gen):
    flags = X.GEMM_FLAG_VNNI_A | X.GEMM_FLAG_BETA_0
    sa, sb, sc = K * M * BR, K * N * BR, 4 * M * N
    a, b = rand_bytes(batch * sa, gen), rand_bytes(batch * sb, gen)
    c = torch.empty(batch * sc, dtype=torch.uint8, device="cuda")
    h = X.libxsmm_dispatch_brgemm(X.libxsmm_create_gemm_shape(M, N, K, M, K, M, I8, I8, I32, I32), flags, 0,
                                  X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, K * M, K * N, 0))
    assert h

    def step():
        rc = X.libxsmm_b200_gemm_batch_strided(h, a.data_ptr(), b.data_ptr(), c.data_ptr(), sa, sb, sc, BR, batch)
        assert rc == 0, rc
    step(); torch.cuda.synchronize(); X.check()
    ms, ms_min = timed(step, steps, warmup)
    return "I8 x I8 -> I32 (VNNI4 A)", "gemm_i8_kernel (dp4a, CUDA cores)", ms, ms_min, sa + sb + sc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4096)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lowbit needs a GPU"
    torch.cuda.set_device(0)
    name, power = card()
    gen = torch.Generator(device="cuda").manual_seed(4321)
    steps = max(args.steps, 10)
    runs = [run_lowbit(ta, args.batch, steps, args.warmup, gen) for ta in (I2, I1, MXFP4)] + [run_i8(args.batch, steps, args.warmup, gen)]
    for workload, kernel, ms, ms_min, per_tile in runs:
        ops = 2.0 * M * N * K * BR * args.batch
        print(json.dumps({"workload": "%s, %dx%dx%d x br %d, strided batch" % (workload, M, N, K, BR), "kernel": kernel,
                          "value": ops / ms / 1e9, "unit": "Tint-op/s", "ms_per_step_median": ms, "ms_per_step_min": ms_min,
                          "compulsory_gbs": per_tile * args.batch / ms / 1e6, "compulsory_bytes_per_tile": per_tile,
                          "steps": steps, "warmup": args.warmup, "batch": args.batch, "card": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
