#!/usr/bin/env python
"""tools/bench_dq.py -- dequantising GEMM on the GPU: batched strided I8 x BF16 -> BF16 BRGEMM with per-row f32 scales, one JSON line
on stdout.

  python tools/bench_dq.py [--steps K] [--warmup W] [--batch B]

Workload: m = n = k = 64, br = 8 (stride mode), `batch` tiles (default 16,384) of int8 weights with their own row scales, bf16
activations, beta = 0, every operand unique and device-resident, one libxsmm_b200_gemm_batch_strided_scaled call per step. The tiles
run on the exact-order CUDA-core kernel (gemm_dq_kernel), which follows the reference's order bit for bit; it is the parity path, and
no speed is claimed for it. Before timing, the first and the last tile are compared with the oracle (oracle/oracle_dq.c) bit for bit.
Timing: CUDA events around each step, median of `steps` steps after `warmup` steps. The card and its power limit are reported beside
the time. Nothing is written to the repository tree."""
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
from dq_ffi import BF16, F32, I8, DqCase, oracle_gemm_dq, same_c  # noqa: E402

M = N = K = 64
BR = 8


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        power = "unknown"
    return name, power


def run(batch, steps, warmup):
    case = DqCase(I8, BF16, F32, BF16, M, N, K, beta0=True, br_type=3, br=BR)
    sa, sb, sc, ss = case.size_a, 2 * case.size_b, 2 * case.size_c, 4 * M
    gen = torch.Generator(device="cuda").manual_seed(4321)
    a = torch.randint(0, 256, (batch * sa,), dtype=torch.uint8, device="cuda", generator=gen)
    b = torch.randn(batch * case.size_b, device="cuda", generator=gen).to(torch.bfloat16).view(torch.int16)
    s = (torch.randn(batch * M, device="cuda", generator=gen) * 0.02).to(torch.float32)
    c = torch.empty(batch * case.size_c * 2, dtype=torch.uint8, device="cuda")
    h = X.libxsmm_dispatch_brgemm(X.libxsmm_create_gemm_shape(M, N, K, M, K, M, I8, BF16, BF16, F32), case.flags, 0,
                                  X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, case.stride_a, case.stride_b, 0))
    assert h and X.libxsmm_b200_kernel_backend(h) == X.BACKEND_SIMT

    def step():
        rc = X.libxsmm_b200_gemm_batch_strided_scaled(h, a.data_ptr(), b.data_ptr(), c.data_ptr(), sa, sb, sc,
                                                      s.data_ptr(), None, None, ss, 0, 0, BR, batch)
        assert rc == 0, rc
    launches = X.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT)
    step(); torch.cuda.synchronize(); X.check()
    assert X.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT) == launches + 1
    for t in (0, batch - 1):                     # sample check against the oracle
        ops = [a[t * sa:(t + 1) * sa].cpu().numpy(), b[t * case.size_b:(t + 1) * case.size_b].cpu().numpy().view(np.uint16),
               np.zeros(case.size_c, np.uint16), s[t * M:(t + 1) * M].cpu().numpy(), None]
        _, want = case.run(oracle_gemm_dq, *ops)
        got = c[t * sc:(t + 1) * sc].cpu().numpy().view(np.uint16)
        assert same_c(case, want, got), "tile %d differs from the oracle" % t
    for _ in range(warmup):
        step()
    times = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); step(); e1.record(); e1.synchronize()
        times.append(e0.elapsed_time(e1))
    X.check()
    ms = float(np.median(times))
    flop, nbytes = 2.0 * M * N * K * BR * batch, float(sa + sb + ss + sc) * batch
    return {"workload": "I8 x BF16 -> BF16, comp F32, row scales, %d^3 x br %d, strided batch" % (M, BR),
            "kernel": "gemm_dq_kernel (exact order, CUDA cores)", "value": flop / ms / 1e6, "unit": "GFLOP/s", "ms_per_step_median": ms,
            "ms_per_step_min": float(np.min(times)), "steps": steps, "warmup": warmup, "batch": batch,
            "algorithmic_bytes_per_tile": sa + sb + ss + sc, "flop_per_tile": 2 * M * N * K * BR, "achieved_gbs": nbytes / ms / 1e6,
            "checked_tiles": [0, batch - 1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16384)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dq needs a GPU"
    torch.cuda.set_device(0)
    name, power = card()
    r = run(args.batch, max(args.steps, 1), args.warmup)
    r.update({"card": name, "power_limit": power})
    print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
