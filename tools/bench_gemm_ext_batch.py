"""Fused BRGEMM batches on the GPU (libxsmm_b200_gemm_ext_batch_strided), one JSON line on stdout.

Workload: bf16 64^3 x br 8 (stride batch-reduce), 65,536 device-resident tiles, column bias + ReLU with its bit mask, once with a BF16 C
and once with an F32 C -- the shape of one fused layer over a large batch. Reported per C type: the batch time (median of --steps after
--warmup), TFLOP/s, the share of the fused kernel's compute bound, the per-tile time of a non-blocking loop of single calls over the first
--single tiles, and the unfused batch of the same tiles (libxsmm_dispatch_brgemm, wgmma) for context.

The compute bound: the exact-order kernel issues a separate FMUL and FADD per term (no contraction), so an SM retires at most 128 terms
= 256 FLOP per clock: 132 SMs x 128 x the SM clock (33.4 TFLOP/s at 1.98 GHz), half the data sheet's FP32 rate. The bytes these tiles
need (A and B 8 x 16 KiB each, C and bias per tile) take well under the compute floor at HBM speed, so the bound is compute.

--lib PATH runs only the single-call loop, against another build of the library (the call uses the LIBXSMM API alone), so that the
per-tile time of an earlier build can be put beside this one's."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import libxsmm_b200 as X  # noqa: E402

M = N = K = 64
BR = 8
BF16, F32 = X.DATATYPE_BF16, X.DATATYPE_F32


def bind(lib):
    P, I, U, LL, ULL = C.c_void_p, C.c_int, C.c_uint, C.c_longlong, C.c_ulonglong
    for name, res, args in (("libxsmm_create_gemm_shape", X.GemmShape, [I] * 10),
                            ("libxsmm_create_gemm_batch_reduce_config", X.BatchReduceConfig, [I, I, I, C.c_ubyte]),
                            ("libxsmm_create_gemm_ext_unary_argops", X.GemmExtUnaryArgops, [I, I, U, I, I, I, U, I, I, I, U, I]),
                            ("libxsmm_create_gemm_ext_binary_postops", X.GemmExtBinaryPostops, [I, I, I, U]),
                            ("libxsmm_dispatch_brgemm_ext", P, [X.GemmShape, U, U, X.BatchReduceConfig, X.GemmExtUnaryArgops, X.GemmExtBinaryPostops]),
                            ("libxsmm_b200_set_blocking", None, [I]), ("libxsmm_b200_sync", I, [])):
        fn = getattr(lib, name); fn.restype, fn.argtypes = res, args
    return lib


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return name, float(power), float(clock)
    except Exception:   # noqa: BLE001 -- the numbers are still reported, without their context
        return torch.cuda.get_device_name(0), None, None


class Layer:
    def __init__(self, lib, tc, tiles):
        self.lib, self.tc, self.tiles = lib, tc, tiles
        ts = 4 if tc == F32 else 2
        self.blk_a, self.blk_b = K * M * 2, N * K * 2
        self.tile_a, self.tile_b, self.tile_c = self.blk_a * BR, self.blk_b * BR, M * N * ts
        self.mask_bytes = (M + 15) // 16 * 16 // 8 * N
        g = torch.Generator(device="cuda").manual_seed(5)
        self.a = (torch.randn(tiles * self.tile_a // 2, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
        self.b = (torch.randn(tiles * self.tile_b // 2, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
        self.c = torch.zeros(tiles * self.tile_c, dtype=torch.uint8, device="cuda")
        self.bias = torch.randn(tiles * M, device="cuda", generator=g).to(torch.float32 if tc == F32 else torch.bfloat16)
        self.mask = torch.zeros(tiles * self.mask_bytes, dtype=torch.uint8, device="cuda")
        shape = lib.libxsmm_create_gemm_shape(M, N, K, M, K, M, BF16, BF16, tc, F32)
        self.cfg = lib.libxsmm_create_gemm_batch_reduce_config(X.GEMM_BATCH_REDUCE_STRIDE, self.blk_a, self.blk_b, 0)
        argops = lib.libxsmm_create_gemm_ext_unary_argops(0, 0, 0, 0, 0, 0, 0, 0, M, X.MELTW_TYPE_UNARY_RELU, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT, 0)
        postops = lib.libxsmm_create_gemm_ext_binary_postops(M, tc, X.MELTW_TYPE_BINARY_ADD, X.MELTW_FLAG_BINARY_BCAST_COL_IN_0)
        self.k = lib.libxsmm_dispatch_brgemm_ext(shape, X.GEMM_FLAG_BETA_0 | X.GEMM_FLAG_VNNI_A, 0, self.cfg, argops, postops)
        assert self.k
        self.shape = shape
        self.brv = C.c_ulonglong(BR)

    def param(self, t):
        p = X.GemmExtParam()
        p.op.tertiary = C.addressof(self.brv)
        p.a.primary, p.b.primary = self.a.data_ptr() + t * self.tile_a, self.b.data_ptr() + t * self.tile_b
        p.c.primary = self.c.data_ptr() + t * self.tile_c
        p.d.primary = self.bias.data_ptr() + t * M * self.bias.element_size()
        p.c.secondary = self.mask.data_ptr() + t * self.mask_bytes
        return p

    def singles(self, n):
        params = [self.param(t) for t in range(n)]
        fn = X.GEMMFUNCTION_EXT(self.k)
        self.lib.libxsmm_b200_set_blocking(0)
        self.lib.libxsmm_b200_sync(); torch.cuda.synchronize()
        t0 = time.perf_counter()
        for p in params:
            fn(C.byref(p))
        assert self.lib.libxsmm_b200_sync() == 0
        return (time.perf_counter() - t0) / n


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        times.append(e0.elapsed_time(e1) * 1e-3)
    return sorted(times)[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=65536)
    ap.add_argument("--single", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--lib", default=None, help="another build of libxsmm_b200.so: single-call loop only")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    name, power, clock = gpu_info()
    out = {"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": clock, "geometry": "bf16 %dx%dx%d br %d stride, bias+relu+mask" % (M, N, K, BR)}
    lib = bind(C.CDLL(args.lib) if args.lib else X.lib)
    for tc in (BF16, F32):
        key = "c_bf16" if tc == BF16 else "c_f32"
        layer = Layer(lib, tc, args.tiles if args.lib is None else args.single)
        layer.singles(min(256, args.single))   # warm-up
        res = {"single_call_us_per_tile": layer.singles(args.single) * 1e6}
        if args.lib is None:
            X.libxsmm_b200_set_blocking(0)
            strides = X.GemmExtStrides(layer.tile_a, layer.tile_b, layer.tile_c, M * layer.bias.element_size(), layer.mask_bytes)
            p0 = layer.param(0)

            def batch():
                assert X.libxsmm_b200_gemm_ext_batch_strided(layer.k, C.byref(p0), C.byref(strides), args.tiles) == 0
            sec = timed(batch, args.steps, args.warmup)
            flops = 2.0 * M * N * K * BR * args.tiles
            res.update({"batch_ms": sec * 1e3, "batch_us_per_tile": sec * 1e6 / args.tiles, "tflops": flops / sec / 1e12})
            if clock:
                bound = 132 * 128 * clock * 1e6 / 1e12   # FLOP per clock per SM: 128 terms over their FMUL and FADD, 2 FLOP per term
                res.update({"compute_bound_tflops": bound, "share_of_compute_bound": flops / sec / 1e12 / bound})
            plain = X.libxsmm_dispatch_brgemm(layer.shape, X.GEMM_FLAG_BETA_0 | X.GEMM_FLAG_VNNI_A, 0, layer.cfg)

            def unfused():
                assert X.libxsmm_b200_gemm_batch_strided(plain, layer.a.data_ptr(), layer.b.data_ptr(), layer.c.data_ptr(),
                                                         layer.tile_a, layer.tile_b, layer.tile_c, BR, args.tiles) == 0
            usec = timed(unfused, args.steps, args.warmup)
            res.update({"unfused_backend": X.libxsmm_b200_kernel_backend(plain), "unfused_ms": usec * 1e3, "unfused_tflops": flops / usec / 1e12})
            assert X.libxsmm_b200_sync() == 0
        out[key] = res
    out["lib"] = "this build" if args.lib is None else "other build (%s)" % os.path.basename(os.path.dirname(os.path.abspath(args.lib)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
