#!/usr/bin/env python
"""tools/bench_sparse_batch.py -- one launch per batch against one launch per call: strided batches of packed-CSR and BCSC calls
(libxsmm_b200_spgemm_batch_strided) on the GPU, one JSON line on stdout.

  python tools/bench_sparse_batch.py [--elements E] [--loop-calls L] [--steps K] [--warmup W]

Workloads, all device-resident:
  * EDGE-style packed A-CSR: C[M][N][P] += A_csr * B[K][N][P] with the tet4 matrices of tests/golden/mtx (A shared by every call,
    N = 9 quantities), packed width P = 8 and 16, f32 and f64, `elements` (default 2^20) elements = elements / P calls.
  * BCSC bf16, the geometry of bench.py (M = 32, N = K = 512, 32 x 32 blocks, 50 %, 8,192 m_blocks) split into 64 calls of 128
    m_blocks (A and C per call, the block values shared); the same work as one single call over all m_blocks is timed beside it.
For each: the median time of one batch call (CUDA events, after warm-up), the compulsory bytes (every operand element a call
reads, once, and C also written; shared operands once), GB/s and the fraction of the data sheet's 3.35 TB/s, which kernel family
ran, and the same handle through a loop of single calls in non-blocking mode over the first `loop_calls` calls (default 4,096),
reported per call. Before
timing, the first, a middle and the last call of every batch are compared byte for byte with single calls. The card and its power
limit are read in the same run. Nothing is written to the repository tree."""
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

F32, F64, BF16 = X.DATATYPE_F32, X.DATATYPE_F64, X.DATATYPE_BF16
PEAK = 3350.0
MTX = ("tet4_2_fluxN_0_csr", "tet4_3_stiffT_0_csr", "tet4_4_fluxT_1_csr", "tet4_starMatrix_csr")
FAMILIES = {X.BACKEND_STREAM: "stream", X.BACKEND_SIMT: "simt", X.BACKEND_TCGEN05: "wgmma"}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        q = "unknown"
    return name, q


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


def tenths(n, dtype, seed):
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    return (torch.randint(-5, 6, (n,), device="cuda", generator=g).to(dtype) / 10).to(dtype)


def read_csr(name):
    rows = [ln.split() for ln in open(os.path.join(ROOT, "tests", "golden", "mtx", name + ".mtx")) if not ln.startswith("%")]
    m, k, nnz = map(int, rows[0])
    ent = sorted((int(r[0]) - 1, int(r[1]) - 1, float(r[2])) for r in rows[1:1 + nnz])
    ptr = np.zeros(m + 1, dtype=np.uint32)
    for i, _, _ in ent:
        ptr[i + 1] += 1
    return m, k, np.cumsum(ptr).astype(np.uint32), np.array([e[1] for e in ent], dtype=np.uint32), np.array([e[2] for e in ent])


class Run:
    """a handle with base pointers and strides; batch, single call t, and the checks"""

    def __init__(self, k, ptrs, strides, count, extra=None):
        self.k, self.ptrs, self.strides, self.count, self.extra = k, ptrs, strides, count, extra or {}
        self.fn = X.GEMMFUNCTION(k)
        self.s = X.SpgemmStrides(*strides)
        self.p0 = self.param(0)

    def param(self, t):
        p = X.GemmParam()
        p.a.primary, p.b.primary, p.c.primary = (b + t * s for b, s in zip(self.ptrs, self.strides))
        if self.extra:
            p.b.secondary, p.b.tertiary, p.b.quaternary = self.extra["colptr"], self.extra["rowidx"], C.addressof(self.extra["nbc"])
        return p

    def batch(self):
        rc = X.libxsmm_b200_spgemm_batch_strided(self.k, C.byref(self.p0), C.byref(self.s), self.count)
        assert rc == 0, rc

    def loop(self, n):
        for t in range(n):
            self.fn(C.byref(self.param(t)))

    def families(self):
        before = {f: X.libxsmm_b200_launch_count_backend(f) for f in FAMILIES}
        total = X.libxsmm_b200_launch_count()
        self.batch(); torch.cuda.synchronize(); X.check()
        assert X.libxsmm_b200_launch_count() - total == 1
        return [FAMILIES[f] for f in FAMILIES if X.libxsmm_b200_launch_count_backend(f) > before[f]]


def check(run, c, c_bytes):
    """calls 0, count / 2 and count - 1 of a batch equal single calls of the same handle, byte for byte"""
    c0 = c.clone()
    run.batch(); torch.cuda.synchronize()
    got = c.clone()
    c.copy_(c0)
    X.libxsmm_b200_set_blocking(0)
    for t in sorted({0, run.count // 2, run.count - 1}):
        run.fn(C.byref(run.param(t)))
    X.libxsmm_b200_sync(); X.libxsmm_b200_set_blocking(1); X.check()
    cb = c.view(torch.uint8)
    for t in sorted({0, run.count // 2, run.count - 1}):
        lo = t * run.strides[2]
        assert torch.equal(got.view(torch.uint8)[lo:lo + c_bytes], cb[lo:lo + c_bytes]), ("batch differs from its single call", t)
    c.copy_(c0)


def measure(run, steps, warmup, bytes_, loop_calls):
    kinds = run.families()
    ms = timed(run.batch, steps, warmup)
    n = min(loop_calls, run.count)
    X.libxsmm_b200_set_blocking(0)
    try:
        ms_loop = timed(lambda: run.loop(n), max(3, steps // 4), 1)
    finally:
        X.libxsmm_b200_set_blocking(1)
    X.check()
    gbs = bytes_ / (ms * 1e-3) / 1e9
    return {"calls": run.count, "batch_ms": ms, "batch_us_per_call": ms * 1e3 / run.count, "loop_us_per_call": ms_loop * 1e3 / n,
            "loop_calls": n, "compulsory_bytes": bytes_, "gbs": gbs, "frac_hbm": gbs / PEAK, "kernels": kinds}


def edge(args):
    out = []
    for name in MTX:
        m, kdim, ptr, idx, vals = read_csr(name)
        nq = 9
        for dtype, tdt, ts in ((F32, torch.float32, 4), (F64, torch.float64, 8)):
            for P in (8, 16):
                calls = args.elements // P
                sh = X.libxsmm_create_gemm_shape(m, nq, kdim, 0, nq, nq, dtype, dtype, dtype, dtype)
                hv = vals.astype(np.float32 if dtype == F32 else np.float64)
                k = X.libxsmm_create_packed_spgemm_csr(sh, 0, 0, P, ptr.ctypes.data, idx.ctypes.data, hv.ctypes.data)
                assert k and X.libxsmm_b200_kernel_backend(k) == X.BACKEND_STREAM
                a = torch.from_numpy(hv).cuda()
                b = tenths(calls * kdim * nq * P, tdt, 1); c = tenths(calls * m * nq * P, tdt, 2)
                sb, sc = kdim * nq * P * ts, m * nq * P * ts
                run = Run(k, (a.data_ptr(), b.data_ptr(), c.data_ptr()), (0, sb, sc), calls)
                check(run, c, sc)
                # compulsory: the B rows A references and the C rows A populates (an empty row of A leaves its C row untouched),
                # C read and written (beta = 1), A's values once
                rows_b, rows_c = len(np.unique(idx)), int(np.count_nonzero(np.diff(ptr)))
                r = measure(run, args.steps, args.warmup, len(idx) * ts + calls * nq * P * ts * (rows_b + 2 * rows_c), args.loop_calls)
                r.update({"workload": "packed A-CSR %s (%d x %d, nnz %d) N=%d P=%d %s" % (name, m, kdim, len(idx), nq, P, "f32" if dtype == F32 else "f64")})
                out.append(r)
                X.libxsmm_release_kernel(k)
                del a, b, c
                torch.cuda.empty_cache()
    return out


def bcsc(args):
    Mb, Kb, Nb, bk, bn, mblocks, ncalls = 32, 512, 512, 32, 32, 8192, 64
    rng = np.random.default_rng(555)                    # the pattern of bench.py
    nbr, nbc = Kb // bk, Nb // bn
    keep = np.zeros(nbr * nbc, dtype=bool); keep[rng.permutation(nbr * nbc)[:nbr * nbc // 2]] = True
    keep = keep.reshape(nbc, nbr)
    colptr = np.concatenate([[0], np.cumsum(keep.sum(1))]).astype(np.uint32); rowidx = np.nonzero(keep)[1].astype(np.uint32)
    nnzb = int(colptr[-1])
    per = mblocks // ncalls
    flags = 4 | X.GEMM_FLAG_VNNI_A                       # BETA_0, VNNI-packed A
    a = tenths(mblocks * Kb * Mb, torch.bfloat16, 3); bv = tenths(nnzb * bk * bn, torch.bfloat16, 4)
    c = torch.zeros(mblocks * Nb * Mb, dtype=torch.bfloat16, device="cuda")
    d_cp = torch.from_numpy(colptr.view(np.int32).copy()).cuda(); d_ri = torch.from_numpy(rowidx.view(np.int32).copy()).cuda()
    extra = {"colptr": d_cp.data_ptr(), "rowidx": d_ri.data_ptr(), "nbc": C.c_ulonglong(nbc)}
    res = []
    for label, mb, count in (("64 calls of 128 m_blocks, one batch", per, ncalls), ("one call of 8,192 m_blocks", mblocks, 1)):
        sh = X.libxsmm_create_gemm_shape(mb, 0, Kb, Kb, 0, Nb, BF16, BF16, BF16, F32)
        k = X.libxsmm_create_packed_spgemm_bcsc(sh, flags, 0, X.SpgemmConfig(Mb, bk, bn))
        assert k
        sa, sc = mb * Kb * Mb * 2, mb * Nb * Mb * 2
        run = Run(k, (a.data_ptr(), bv.data_ptr(), c.data_ptr()), (sa, 0, sc), count, extra)
        check(run, c, sc)
        r = measure(run, args.steps, args.warmup, mblocks * (Kb + Nb) * Mb * 2 + nnzb * bk * bn * 2, args.loop_calls)
        r.update({"workload": "BCSC bf16 M=32 N=K=512 32x32 50%% m_blocks=8192: %s" % label, "bcsc_variant": X.libxsmm_b200_bcsc_variant(k, nbc)})
        res.append(r)
        X.libxsmm_release_kernel(k)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elements", type=int, default=1 << 20)
    ap.add_argument("--loop-calls", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    X.libxsmm_b200_set_device(0)
    name, q = card()
    out = {"gpu": name, "power_limit_sm_clock_max_clock": q, "peak_gbs": PEAK, "edge_packed_csr": edge(args), "bcsc_bf16": bcsc(args)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
