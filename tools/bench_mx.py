#!/usr/bin/env python
"""tools/bench_mx.py -- MX fp8 GEMM on the GPU: batched strided MXHF8 and MXBF8 BRGEMM, F32 C, one JSON line per type on stdout.

  python tools/bench_mx.py [--steps K] [--warmup W] [--batch B]

Workload: m = n = k = 64, br = 8 (stride mode), `batch` tiles (default 65,536), every operand unique and device-resident, one
libxsmm_b200_gemm_batch_strided_scaled call per step. MX tiles run on the exact-order CUDA-core kernel (gemm_mx8_kernel); there is
no tensor-core MX kernel yet, so there is nothing to alternate with. Before timing, the first and the last tile of the batch are
compared with the oracle (oracle/oracle_mx.c) bit for bit. Timing: CUDA events around each step, median of `steps` steps after
`warmup` steps.

Arithmetic, from data-sheet figures and not measured: per tile 2*m*n*k*br = 4,194,304 flop and 83,968 algorithmic bytes (A 32,768,
B 32,768, scales 2 x 1,024, C 16,384 written): 50 flop/B. At the H100 SXM's 3.35 TB/s that is an HBM ceiling near 167 TFLOP/s, above
the 67 TFLOP/s FP32 CUDA-core peak of the data sheet, so the bound that applies to a CUDA-core kernel is compute, not memory.
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
from mx_ffi import F32, MXBF8, MXHF8, MxCase, oracle_gemm_mx, same_bits  # noqa: E402

M = N = K = 64
BR = 8
HBM_GBS, FP32_TFLOPS = 3350.0, 67.0          # H100 SXM data sheet


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        power = "unknown"
    return name, power


def run_type(ta, batch, steps, warmup):
    case = MxCase(ta, F32, M, N, K, beta0=True, br_type=3, br=BR)
    sa, sb, sc = case.size_a, case.size_b, case.size_c * 4
    ssa, ssb = case.size_as, case.size_bs
    gen = torch.Generator(device="cuda").manual_seed(1234 + ta)
    a = torch.randint(0, 256, (batch * sa,), dtype=torch.uint8, device="cuda", generator=gen)
    b = torch.randint(0, 256, (batch * sb,), dtype=torch.uint8, device="cuda", generator=gen)
    if ta == MXBF8:                              # no Inf / NaN codes: the sample check then compares every element
        a = torch.where((a & 0x7C) == 0x7C, a ^ 0x40, a); b = torch.where((b & 0x7C) == 0x7C, b ^ 0x40, b)
    else:
        a = torch.where((a & 0x7F) == 0x7F, a ^ 0x40, a); b = torch.where((b & 0x7F) == 0x7F, b ^ 0x40, b)
    as_ = torch.randint(117, 138, (batch * ssa,), dtype=torch.uint8, device="cuda", generator=gen)
    bs_ = torch.randint(117, 138, (batch * ssb,), dtype=torch.uint8, device="cuda", generator=gen)
    c = torch.empty(batch * case.size_c, dtype=torch.float32, device="cuda")
    h = X.libxsmm_dispatch_brgemm(X.libxsmm_create_gemm_shape(M, N, K, M, N, M, ta, ta, F32, F32), case.flags, 0,
                                  X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, M * K, N * K, 0))
    assert h and X.libxsmm_b200_kernel_backend(h) == X.BACKEND_SIMT

    def step():
        rc = X.libxsmm_b200_gemm_batch_strided_scaled(h, a.data_ptr(), b.data_ptr(), c.data_ptr(), sa, sb, sc,
                                                      as_.data_ptr(), bs_.data_ptr(), None, ssa, ssb, 0, BR, batch)
        assert rc == 0, rc
    step(); torch.cuda.synchronize(); X.check()
    for t in (0, batch - 1):                     # sample check against the oracle
        ops = [a[t * sa:(t + 1) * sa].cpu().numpy(), b[t * sb:(t + 1) * sb].cpu().numpy(), np.zeros(case.size_c, np.float32),
               as_[t * ssa:(t + 1) * ssa].cpu().numpy(), bs_[t * ssb:(t + 1) * ssb].cpu().numpy(), np.zeros(1, np.uint8)]
        _, want, _ = case.run(oracle_gemm_mx, *ops)
        got = c[t * case.size_c:(t + 1) * case.size_c].cpu().numpy()
        assert same_bits(want, got) and not np.isnan(got).any(), "tile %d differs from the oracle" % t
    for _ in range(warmup):
        step()
    times = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); step(); e1.record(); e1.synchronize()
        times.append(e0.elapsed_time(e1))
    X.check()
    ms = float(np.median(times))
    flop, nbytes = 2.0 * M * N * K * BR * batch, float(sa + sb + ssa + ssb + sc) * batch
    gflops = flop / ms / 1e6
    ceiling_hbm = flop / nbytes * HBM_GBS / 1e3              # TFLOP/s
    return {"type": "MXBF8" if ta == MXBF8 else "MXHF8", "kernel": "gemm_mx8_kernel (exact order, CUDA cores)",
            "value": gflops, "unit": "GFLOP/s", "ms_per_step_median": ms, "steps": steps, "warmup": warmup, "batch": batch,
            "algorithmic_bytes_per_tile": (sa + sb + ssa + ssb + sc), "flop_per_tile": 2 * M * N * K * BR,
            "roofline": {"hbm_ceiling_tflops": ceiling_hbm, "fp32_cuda_core_peak_tflops": FP32_TFLOPS,
                         "bound": "compute (FP32 CUDA cores)" if FP32_TFLOPS < ceiling_hbm else "hbm",
                         "frac_of_bound": gflops / 1e3 / min(FP32_TFLOPS, ceiling_hbm), "src": "H100 SXM data sheet"},
            "achieved_gbs": nbytes / ms / 1e6, "checked_tiles": [0, batch - 1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=65536)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mx needs a GPU"
    torch.cuda.set_device(0)
    name, power = card()
    for ta in (MXHF8, MXBF8):
        r = run_type(ta, args.batch, max(args.steps, 1), args.warmup)
        r.update({"card": name, "power_limit": power})
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
