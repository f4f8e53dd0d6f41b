"""The blocked GEMM of one BRGEMM handle on the GPU, three ways; one JSON line on stdout.

Workload: C = A * B with M = N = 8192 and K = 4096 in bf16 (f32 C), cut into 64 x 64 blocks and stored blocked: A block (mb, kb) at
(mb * Kb + kb) * 8 KiB, B block (kb, nb) at (nb * Kb + kb) * 8 KiB, C tile (mb, nb) at (nb * Mb + mb) * 16 KiB. The handle is a
64^3 BRGEMM with stride batch-reduce over the Kb = 64 blocks of K (br = 64); C tile (mb, nb) is the call with A + mb * Kb * 8 KiB
and B + nb * Kb * 8 KiB -- the loop nest a LIBXSMM caller writes for a fully connected layer or a big matrix. Timed:
  grid     one libxsmm_b200_gemm_batch_grid call over the Mb x Nb grid
  strided  Nb libxsmm_b200_gemm_batch_strided calls, one per block column of C, with B shared (stride 0)
  records  one libxsmm_b200_gemm_batch call with Mb * Nb argument structs, built and uploaded per call
Each: the median wall time of --steps calls (--slow-steps for strided and records) after one warm-up, each call ending in a device
synchronise, as TFLOP/s of 2 * M * N * K and as a share of the 989 TFLOP/s data-sheet dense bf16 rate of an H100 SXM at 700 W. The
case is tensor-bound: A, B and C are 64 + 64 + 256 MiB, 0.12 ms at 3.35 TB/s, against 0.56 ms of bf16 work at that rate. Also
reported: which kernel family each ran (libxsmm_b200_launch_count_backend), the relative Frobenius distance of the strided and records
results from the grid's (the exact-order kernel against wgmma), and the card's name, power limit and maximum SM clock."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import libxsmm_b200 as X  # noqa: E402

B = 64
M = N = 8192
K = 4096
PEAK_BF16 = 989e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return name, float(power), float(clock)
    except Exception:   # noqa: BLE001 -- the numbers are still reported, without their context
        return torch.cuda.get_device_name(0), None, None


def timed(fn, steps):
    fn()
    X.check()
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        rc = fn()
        X.check()
        times.append(time.perf_counter() - t0)
        assert rc == 0, rc
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--slow-steps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gemm_grid needs a GPU"
    torch.cuda.set_device(0)
    name, power, clock = gpu_info()
    mb, nb, kb = M // B, N // B, K // B
    blk, tile_c = B * B * 2, B * B * 4
    gen = torch.Generator(device="cuda").manual_seed(0)
    a = (torch.randint(-5, 6, (M * K,), device="cuda", generator=gen).float() / 10).to(torch.bfloat16)
    b = (torch.randint(-5, 6, (K * N,), device="cuda", generator=gen).float() / 10).to(torch.bfloat16)
    c = {w: torch.zeros(M * N, dtype=torch.float32, device="cuda") for w in ("grid", "strided", "records")}
    shape = X.libxsmm_create_gemm_shape(B, B, B, B, B, B, X.DATATYPE_BF16, X.DATATYPE_BF16, X.DATATYPE_F32, X.DATATYPE_F32)
    cfg = X.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, blk, blk, 0)
    kernel = X.libxsmm_dispatch_brgemm(shape, X.GEMM_FLAG_BETA_0, 0, cfg)
    assert kernel and X.libxsmm_b200_kernel_backend(kernel) == X.BACKEND_TCGEN05
    sa, sb, sm, sn = kb * blk, kb * blk, tile_c, mb * tile_c
    pa, pb = a.data_ptr(), b.data_ptr()

    def grid():
        return X.libxsmm_b200_gemm_batch_grid(kernel, pa, pb, c["grid"].data_ptr(), sa, sb, sm, sn, kb, mb, nb)

    def strided():
        for j in range(nb):
            rc = X.libxsmm_b200_gemm_batch_strided(kernel, pa, pb + j * sb, c["strided"].data_ptr() + j * sn, sa, 0, sm, kb, mb)
            if rc != 0:
                return rc
        return 0

    brv = C.c_ulonglong(kb)
    params = (X.GemmParam * (mb * nb))()
    for j in range(nb):
        for i in range(mb):
            p = params[j * mb + i]
            p.op.tertiary = C.addressof(brv)
            p.a.primary, p.b.primary, p.c.primary = pa + i * sa, pb + j * sb, c["records"].data_ptr() + i * sm + j * sn

    def records():
        return X.libxsmm_b200_gemm_batch(kernel, params, mb * nb)

    flops = 2.0 * M * N * K
    out = {"workload": "blocked bf16 GEMM M=%d N=%d K=%d, %d^3 blocks, br=%d, f32 C" % (M, N, K, B, kb), "gpu": name,
           "power_limit_w": power, "max_sm_clock_mhz": clock}
    for way, fn, steps in (("grid", grid, args.steps), ("strided", strided, args.slow_steps), ("records", records, args.slow_steps)):
        tc0, simt0 = X.libxsmm_b200_launch_count_backend(X.BACKEND_TCGEN05), X.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT)
        fn()
        X.check()
        fam = "wgmma" if X.libxsmm_b200_launch_count_backend(X.BACKEND_TCGEN05) > tc0 else \
            ("exact-order" if X.libxsmm_b200_launch_count_backend(X.BACKEND_SIMT) > simt0 else "none")
        s = timed(fn, steps)
        out[way] = {"ms": round(s * 1e3, 3), "tflops": round(flops / s / 1e12, 2), "share_of_bf16_peak": round(flops / s / PEAK_BF16, 4),
                    "kernel": fam}
    ref = c["grid"].double()
    for way in ("strided", "records"):
        out[way]["normf_rel_to_grid"] = float(torch.linalg.norm(c[way].double() - ref) / torch.linalg.norm(ref))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
