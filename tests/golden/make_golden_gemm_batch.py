"""Writes tests/golden/gemm_batch_rules.npz: what every GEMM batch entry point does with every kind of GEMM handle.

The points run on the simulated device of tests/c/hostsim_runtime.c, where a GEMM tile is answered by an oracle and "device" memory
is host memory. One simulated library is built per family of handles, because each family's tiles go to its own oracle through its
own wrapper of xb_gemm_simt_launch: plain (tests/c/hostsim_runtime.c alone), dequantising (hostsim_dq.c), MX fp8 (hostsim_mx.c) and
low-bit (hostsim_lowbit.c). Every library also counts batched mateltwise launches (hostsim_meltw_batch.c), which is how a batch
re-packs a VNNI-packed C.

The grid crosses:
  - handles: f32 without batch-reduce and with address, offset and stride batch-reduce; bf16 with VNNI_C; U8 x I8 -> F32 (the
    int8 scale); I4X2 x U8 -> I32 (zero points); I8 x BF16 (also under address batch-reduce), I4 x F16 and BF8 x F16 dequantising;
    MXBF8 C and MXHF8 -> F32; MXFP4 x I8 (also under address batch-reduce, with arrays of scale pointers) and I2 x I8; fused (brgemm_ext) handles without a fusion, with a bias, ReLU, ReLU with a bit mask, sigmoid, VNNI_C, and a bias
    under address batch-reduce;
  - the seven batch forms: strided, multi-GPU (one device), scaled, records, plan, fused strided and fused records;
  - the pointer kind the simulated runtime reports for every pointer (XB_HOSTSIM_PTR_KIND): pageable, device and pinned;
  - argument faults: count -1 and 0 next to 3; a NULL side operand, bias or mask; a negative stride; a C or mask stride below one
    call's extent; unevenly spaced C under VNNI_C in the record form. A fault is only crossed with the forms and handles that read it;
  - two points large enough to cross the 64 MiB scratch budget of a chunked batch with a ragged last chunk: an MXBF8-C scaled batch
    and a VNNI_C fused batch.
Per point it records the return code (a plan: PLAN_NULL, or the code of running it), the change in libxsmm_b200_launch_count (the
simulation counts one per tile and per mateltwise call), the change in batched mateltwise launches, and a digest of every caller
buffer the call may write: C, the ReLU bit mask and the MXBF8 C scales.
tests/test_gemm_batch_rules_hostsim.py rebuilds the grid and compares point by point. Run from the repository root after `make lib`:
    python3 tests/golden/make_golden_gemm_batch.py"""
import ctypes as C
import hashlib
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
TESTS = os.path.join(ROOT, "tests")
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import libxsmm_b200 as X  # noqa: E402  (struct layouts and constants only: every call goes to a simulation library)
import oracle_ffi  # noqa: E402,F401  (builds the oracles the simulation libraries link)

CSRC = os.path.join(ROOT, "libxsmm_b200", "csrc")
ORACLE = os.path.join(ROOT, "oracle")
HOST_C = ["host_core.c", "host_thunks.c", "host_sparse.c", "host_meltw.c", "host_utils.c", "host_meqn.c"]

F32, BF16, F16, BF8, I32, I8, U8 = 1, 2, 3, 4, 8, 12, 13
MXBF8, MXHF8, I4X2, MXFP4X2, I2X4 = 14, 15, 18, 20, 22
TS = {F32: 4, BF16: 2, F16: 2, BF8: 1, I32: 4, I8: 1, U8: 1, MXBF8: 1, MXHF8: 1, I4X2: 1, MXFP4X2: 1, I2X4: 1}
TRANS_B, BETA_0, VNNI_A, VNNI_B, VNNI_C, INTLV_A = 2, 4, 256, 512, 1024, 262144
RELU, SIGMOID, BITMASK = X.MELTW_TYPE_UNARY_RELU, X.MELTW_TYPE_UNARY_SIGMOID, X.MELTW_FLAG_UNARY_BITMASK_2BYTEMULT
BR_API = {0: X.GEMM_BATCH_REDUCE_NONE, 1: X.GEMM_BATCH_REDUCE_ADDRESS, 2: X.GEMM_BATCH_REDUCE_OFFSET, 3: X.GEMM_BATCH_REDUCE_STRIDE}

# family -> the wrapper of xb_gemm_simt_launch and the oracle it links
FAMILIES = {"plain": (None, []), "dq": ("hostsim_dq.c", ["-loracle_dq"]), "mx": ("hostsim_mx.c", ["-loracle_mx"]),
            "lowbit": ("hostsim_lowbit.c", ["-loracle_lowbit"])}

# name: family, (m, n, k, lda, ldb, ldc), (A, B, comp, C), flags, br_type, fused ("bias" / "relu" / "mask" / "sigmoid" or ""; None:
# a plain handle), tiles. The A, B, scale and bias bytes of each handle come from its own seed.
HANDLES = [
    ("f32", "plain", (8, 4, 8, 10, 9, 11), (F32, F32, F32, F32), 0, 0, None, 3),
    ("f32_addr", "plain", (8, 4, 8, 10, 9, 11), (F32, F32, F32, F32), 0, 1, None, 3),
    ("f32_offs", "plain", (8, 4, 8, 10, 9, 11), (F32, F32, F32, F32), BETA_0, 2, None, 3),
    ("f32_stride", "plain", (8, 4, 8, 10, 9, 11), (F32, F32, F32, F32), 0, 3, None, 3),
    ("bf16_vnni_c", "plain", (8, 4, 8, 8, 9, 10), (BF16, BF16, F32, BF16), VNNI_A | VNNI_C, 0, None, 3),
    ("u8i8_f32", "plain", (8, 4, 8, 8, 9, 10), (U8, I8, I32, F32), 0, 0, None, 3),
    ("i4x2u8_i32", "plain", (8, 4, 16, 8, 17, 9), (I4X2, U8, I32, I32), VNNI_A | INTLV_A, 0, None, 3),
    ("i8bf16", "dq", (8, 4, 8, 9, 8, 10), (I8, BF16, F32, F32), 0, 0, None, 3),
    ("i8bf16_addr", "dq", (8, 4, 8, 9, 8, 10), (I8, BF16, F32, F32), 0, 1, None, 3),
    ("i4f16", "dq", (8, 4, 8, 9, 8, 10), (I4X2, F16, F32, F16), VNNI_A, 0, None, 3),
    ("bf8f16", "dq", (8, 4, 8, 9, 8, 10), (BF8, F16, F32, F32), 0, 0, None, 3),
    ("mxbf8_c", "mx", (32, 4, 32, 33, 6, 32), (MXBF8, MXBF8, F32, MXBF8), VNNI_A | VNNI_B | TRANS_B | BETA_0, 0, None, 3),
    ("mxhf8_f32", "mx", (8, 4, 32, 9, 6, 10), (MXHF8, MXHF8, F32, F32), VNNI_A | VNNI_B | TRANS_B, 0, None, 3),
    ("mxfp4i8", "lowbit", (8, 4, 32, 9, 32, 10), (MXFP4X2, I8, I32, F32), VNNI_A | INTLV_A, 0, None, 3),
    ("mxfp4i8_addr", "lowbit", (8, 4, 32, 9, 32, 10), (MXFP4X2, I8, I32, F32), VNNI_A | INTLV_A, 1, None, 3),
    ("i2i8", "lowbit", (8, 4, 16, 9, 17, 10), (I2X4, I8, I32, I32), VNNI_A | INTLV_A, 0, None, 3),
    ("ext", "plain", (8, 4, 8, 10, 9, 11), (F32, F32, F32, F32), 0, 0, "", 3),
    ("ext_bias", "plain", (8, 4, 8, 10, 9, 11), (F32, F32, F32, F32), 0, 3, "bias", 3),
    ("ext_relu", "plain", (8, 4, 8, 10, 9, 11), (F32, F32, F32, F32), BETA_0, 0, "relu", 3),
    ("ext_mask", "plain", (8, 4, 8, 10, 9, 11), (BF16, BF16, F32, BF16), VNNI_A, 2, "mask", 3),
    ("ext_sigmoid", "plain", (8, 4, 8, 10, 9, 11), (U8, I8, I32, F32), 0, 0, "sigmoid", 3),
    ("ext_vnni_c", "plain", (6, 4, 8, 8, 10, 8), (BF16, BF16, F32, BF16), VNNI_A | VNNI_C, 3, "bias", 3),
    ("ext_bias_addr", "plain", (8, 4, 8, 10, 9, 11), (F32, F32, F32, F32), 0, 1, "bias", 3),
    # past the 64 MiB scratch budget: a 25 MiB f32 image per tile runs as chunks of 2 + 1; C tiles 8 MiB apart as 8 + 8 + 4
    ("chunk_mxbf8_c", "mx", (4096, 1600, 32, 4096, 1600, 4096), (MXBF8, MXBF8, F32, MXBF8), VNNI_A | VNNI_B | TRANS_B | BETA_0, 0, None, 3),
    ("chunk_ext_vnni_c", "plain", (6, 4, 8, 8, 10, 8), (BF16, BF16, F32, BF16), VNNI_A | VNNI_C, 3, "relu", 20),
]
CHUNK_C_STRIDE = 8 << 20
FORMS = ["strided", "multi", "scaled", "records", "plan", "ext_strided", "ext_records"]
KINDS = [0, 1, 3]
FAULTS = ["none", "count_neg", "count_zero", "null_side", "null_bias", "null_mask", "neg_stride", "c_stride_small", "mask_stride_small",
          "uneven_c"]
PLAN_NULL = -100
COLUMNS = ["handle", "form", "kind", "fault"]
OUTCOMES = ["rc", "launches", "repacks", "digest"]


def sides(h):
    """the side operands a call of the handle carries, as the grid names them"""
    name = h[0]
    return {"i8bf16": ["a_s"], "i8bf16_addr": ["a_s"], "i4f16": ["a_s", "a_q"], "mxbf8_c": ["a_s", "b_s", "c_s"],
            "chunk_mxbf8_c": ["a_s", "b_s", "c_s"], "mxhf8_f32": ["a_s", "b_s"], "mxfp4i8": ["a_s", "b_s"], "mxfp4i8_addr": ["a_s", "b_s"],
            "i4x2u8_i32": ["a_q"]}.get(name, [])


def applies(h, form, kind, fault):
    """whether the form reads what the fault breaks, for this handle"""
    fused, ext_form, strided = h[6], form.startswith("ext"), form in ("strided", "multi", "scaled", "ext_strided")
    if h[0].startswith("chunk"):               # only the forms that run them, and pinned memory is device memory here
        return fault == "none" and form in ("scaled", "ext_strided", "ext_records") and kind != 3
    if fault in ("none", "count_neg", "count_zero"):
        return True
    if fault == "null_side":
        return not ext_form and form not in ("strided", "multi") and (sides(h) or h[3][0] == U8)
    if fault == "null_bias":
        return ext_form and fused == "bias"
    if fault in ("null_mask", "mask_stride_small"):
        return ext_form and fused == "mask" and (fault == "null_mask" or form == "ext_strided")
    if fault in ("neg_stride", "c_stride_small"):
        return strided
    return fault == "uneven_c" and form in ("records", "ext_records") and (h[4] & VNNI_C) != 0


def grid():
    rows = [(hi, fi, kind, qi) for hi, h in enumerate(HANDLES) for fi, form in enumerate(FORMS) for kind in KINDS
            for qi, fault in enumerate(FAULTS) if applies(h, form, kind, fault)]
    return np.array(rows, dtype=np.int32)


def digest(g):
    names = repr((HANDLES, FORMS, KINDS, FAULTS, CHUNK_C_STRIDE)).encode()
    return hashlib.sha256(names + g.tobytes()).hexdigest()


def build(family):
    wrapper, oracles = FAMILIES[family]
    out = os.path.join(ROOT, "tests", "c", "_hostsim", "batch_rules_" + family)
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libxsmm.so")
    srcs = [os.path.join(CSRC, f) for f in HOST_C] + [os.path.join(TESTS, "c", f) for f in ["hostsim_runtime.c", "hostsim_meltw_batch.c"]
                                                      + ([wrapper] if wrapper else [])]
    deps = srcs + [os.path.join(CSRC, "xb_internal.h")]
    if not (os.path.exists(so) and all(os.path.getmtime(s) < os.path.getmtime(so) for s in deps)):
        wraps = ["-Wl,--wrap=xb_meltw_launch"] + (["-Wl,--wrap=xb_gemm_simt_launch"] if wrapper else [])
        cmd = ["gcc", "-O1", "-std=gnu99", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include")] + wraps + ["-o", so] + srcs + \
            ["-L" + ORACLE] + oracles + ["-loracle", "-Wl,-rpath," + ORACLE, "-lpthread", "-ldl", "-lm"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-3000:]
    lib = C.CDLL(so)
    P, I, LL, ULL = C.c_void_p, C.c_int, C.c_longlong, C.c_ulonglong
    for name, res, args in (
            ("libxsmm_dispatch_gemm", P, [X.GemmShape, C.c_uint, C.c_uint]),
            ("libxsmm_dispatch_brgemm", P, [X.GemmShape, C.c_uint, C.c_uint, X.BatchReduceConfig]),
            ("libxsmm_dispatch_brgemm_ext", P, [X.GemmShape, C.c_uint, C.c_uint, X.BatchReduceConfig, X.GemmExtUnaryArgops, X.GemmExtBinaryPostops]),
            ("libxsmm_b200_gemm_batch_strided", I, [P] * 4 + [LL] * 3 + [ULL, LL]),
            ("libxsmm_b200_gemm_batch_strided_multi", I, [P] * 4 + [LL] * 3 + [ULL, LL, I]),
            ("libxsmm_b200_gemm_batch_strided_scaled", I, [P] * 4 + [LL] * 3 + [P] * 3 + [LL] * 3 + [ULL, LL]),
            ("libxsmm_b200_gemm_batch", I, [P, P, LL]),
            ("libxsmm_b200_gemm_plan_create", P, [P, P, LL]),
            ("libxsmm_b200_gemm_plan_run", I, [P]),
            ("libxsmm_b200_gemm_plan_destroy", None, [P]),
            ("libxsmm_b200_gemm_ext_batch_strided", I, [P, P, P, LL]),
            ("libxsmm_b200_gemm_ext_batch", I, [P, P, LL]),
            ("libxsmm_b200_launch_count", ULL, []),
            ("hostsim_batch_launches", ULL, [])):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def _fill(rng, nbytes, t):
    """bytes of type t with moderate values, so that every operand shows in the result"""
    n = max(nbytes, 1)
    if t == F32:
        return rng.uniform(-2, 2, (n + 3) // 4).astype(np.float32).view(np.uint8)[:n].copy()
    if t == BF16:
        return (rng.uniform(-2, 2, (n + 1) // 2).astype(np.float32).view(np.uint32) >> 16).astype(np.uint16).view(np.uint8)[:n].copy()
    if t == F16:
        return rng.uniform(-2, 2, (n + 1) // 2).astype(np.float16).view(np.uint8)[:n].copy()
    if t == I32:
        return rng.integers(-50, 50, (n + 3) // 4).astype(np.int32).view(np.uint8)[:n].copy()
    if t in (BF8, MXBF8):         # e5m2: the high byte of an f16
        return (rng.uniform(-2, 2, n).astype(np.float16).view(np.uint16) >> 8).astype(np.uint8)
    if t == MXHF8:                # e4m3 with exponents around 1
        return (rng.integers(0x30, 0x48, n) | (rng.integers(0, 2, n) << 7)).astype(np.uint8)
    if t == "e8m0":
        return rng.integers(120, 134, n).astype(np.uint8)
    if t == I8:
        return rng.integers(-20, 20, n).astype(np.int8).view(np.uint8)
    return rng.integers(0, 256, n).astype(np.uint8)


class Handle:
    """a handle of one row of HANDLES in one simulation library, with every buffer a call may read"""

    def __init__(self, lib, hi):
        self.lib, self.spec = lib, HANDLES[hi]
        name, _, (m, n, k, lda, ldb, ldc), (ta, tb, tcomp, tc), flags, br_type, fused, count = self.spec
        self.m, self.n, self.k, self.lda, self.ldb, self.ldc, self.tc, self.br_type, self.fused, self.count = m, n, k, lda, ldb, ldc, tc, br_type, fused, count
        self.vnni_c, self.br = (flags & VNNI_C) != 0, (2 if br_type else 1)
        rng = np.random.default_rng(1000 + hi)
        self.blk_a, self.blk_b = lda * k * TS[ta], ldb * max(n, k) * TS[tb]
        shape = X.GemmShape(m, n, k, lda, ldb, ldc, ta, tb, tc, tcomp)
        cfg = X.BatchReduceConfig(BR_API[br_type], self.blk_a, self.blk_b, 0)
        if fused is None:
            self.kernel = lib.libxsmm_dispatch_brgemm(shape, flags, 0, cfg) if br_type else lib.libxsmm_dispatch_gemm(shape, flags, 0)
        else:
            argops = X.GemmExtUnaryArgops()
            argops.ldcp = ldc
            argops.cp_unary_type = {"relu": RELU, "mask": RELU, "sigmoid": SIGMOID}.get(fused, 0)
            argops.cp_unary_flags = BITMASK if fused == "mask" else 0
            postops = X.GemmExtBinaryPostops(ldc, tc, X.MELTW_TYPE_BINARY_ADD if fused == "bias" else 0,
                                             X.MELTW_FLAG_BINARY_BCAST_COL_IN_0 if fused == "bias" else 0)
            self.kernel = lib.libxsmm_dispatch_brgemm_ext(shape, flags, 0, cfg, argops, postops)
        assert self.kernel, name
        self.tile_a, self.tile_b = self.blk_a * self.br, self.blk_b * self.br
        self.ext_c = (n * ldc if self.vnni_c else (n - 1) * ldc + m) * TS[tc]
        self.tile_c = CHUNK_C_STRIDE if name == "chunk_ext_vnni_c" else n * ldc * TS[tc]
        self.mask_bytes = (ldc + 15) // 16 * 16 // 8 * n
        self.tile_sa, self.tile_sb, self.tile_sc, self.tile_q = 4 * lda * k, 4 * ldb * max(n, k), n * ldc, 4 * m
        scale_a = "e8m0" if ta in (MXBF8, MXHF8, MXFP4X2) else (F32 if tb == BF16 else F16)
        scale_b = F32 if ta == MXFP4X2 else "e8m0"
        self.A, self.B = _fill(rng, self.tile_a * count, ta), _fill(rng, self.tile_b * count, tb)
        self.SA, self.SB = _fill(rng, self.tile_sa * count, scale_a), _fill(rng, self.tile_sb * count, scale_b)
        self.Q = _fill(rng, self.tile_q * count, F16 if tb == F16 else U8)
        self.SCF = np.array([0.5 + t for t in range(count)], np.float32)
        self.bias = _fill(rng, m * TS[tc] * count, tc)
        self.C0 = _fill(rng, self.tile_c * (count - 1) + n * ldc * TS[tc], tc)
        self.CS0, self.MASK0 = _fill(rng, self.tile_sc * count, U8), _fill(rng, self.mask_bytes * count, U8)
        self.offs = [np.array([(self.br - 1 - r) * blk for r in range(self.br)], np.int64) for blk in (self.blk_a, self.blk_b)]
        self.brv = C.c_ulonglong(self.br)

    def param(self, cls, t, c, cs, mask, keep):
        a, b = self.A.ctypes.data + t * self.tile_a, self.B.ctypes.data + t * self.tile_b
        p = cls()
        p.op.tertiary = C.addressof(self.brv)
        if self.br_type == 1:
            arrs = [(C.c_void_p * self.br)(*[base + r * blk for r in range(self.br)]) for base, blk in ((a, self.blk_a), (b, self.blk_b))]
            keep += arrs
            p.a.primary, p.b.primary = C.addressof(arrs[0]), C.addressof(arrs[1])
        else:
            p.a.primary, p.b.primary = a, b
            if self.br_type == 2:
                p.a.secondary, p.b.secondary = self.offs[0].ctypes.data, self.offs[1].ctypes.data
        p.c.primary = c.ctypes.data + t * self.tile_c
        s = sides(self.spec)
        if "a_s" in s:
            p.a.tertiary = self.SA.ctypes.data + t * self.tile_sa
        if "b_s" in s:
            p.b.tertiary = self.SB.ctypes.data + t * self.tile_sb
        if self.spec[3][0] == MXFP4X2 and self.br_type == 1:   # address mode: arrays of br pointers to each block's scales
            arrs = [(C.c_void_p * self.br)(*[base + r * blk for r in range(self.br)])
                    for base, blk in ((p.a.tertiary, self.k // 32 * self.lda), (p.b.tertiary, self.n * self.ldb // 32 * 4))]
            keep += arrs
            p.a.tertiary, p.b.tertiary = C.addressof(arrs[0]), C.addressof(arrs[1])
        if "c_s" in s:
            p.c.tertiary = cs.ctypes.data + t * self.tile_sc
        if "a_q" in s:
            p.a.quaternary = self.Q.ctypes.data + t * self.tile_q
        if self.spec[3][0] == U8:
            p.c.tertiary = self.SCF.ctypes.data + 4 * t
        if cls is X.GemmExtParam:
            if self.fused == "bias":
                p.d.primary = self.bias.ctypes.data + t * self.m * TS[self.tc]
            if self.fused == "mask":
                p.c.secondary = mask.ctypes.data + t * self.mask_bytes
        return p

    def run(self, form, fault):
        """one call of the form under the fault: (rc, C, C scales, mask)"""
        lib, keep = self.lib, []
        c, cs, mask = self.C0.copy(), self.CS0.copy(), self.MASK0.copy()
        count = {"count_neg": -1, "count_zero": 0}.get(fault, self.count)
        if form in ("strided", "multi", "scaled", "ext_strided"):
            a, sa = self.A.ctypes.data, self.tile_a
            sc, smask = self.tile_c, self.mask_bytes
            if fault == "neg_stride":                      # tile t's A at the last tile's minus t tiles: in bounds either way
                a, sa = a + (self.count - 1) * self.tile_a, -self.tile_a
            if fault == "c_stride_small":
                sc = self.ext_c - TS[self.tc]
            if fault == "mask_stride_small":
                smask = self.mask_bytes - 1
            if form == "strided":
                rc = lib.libxsmm_b200_gemm_batch_strided(self.kernel, a, self.B.ctypes.data, c.ctypes.data, sa, self.tile_b, sc, self.br, count)
            elif form == "multi":
                rc = lib.libxsmm_b200_gemm_batch_strided_multi(self.kernel, a, self.B.ctypes.data, c.ctypes.data, sa, self.tile_b, sc,
                                                               self.br, count, 1)
            elif form == "scaled":
                s = sides(self.spec)
                scf = [self.SA.ctypes.data if "a_s" in s else None, self.SB.ctypes.data if "b_s" in s else None,
                       cs.ctypes.data if "c_s" in s else None]
                if fault == "null_side":
                    scf[0] = None
                rc = lib.libxsmm_b200_gemm_batch_strided_scaled(self.kernel, a, self.B.ctypes.data, c.ctypes.data, sa, self.tile_b, sc,
                                                                scf[0], scf[1], scf[2], self.tile_sa, self.tile_sb, self.tile_sc, self.br, count)
            else:
                p = self.param(X.GemmExtParam, 0, c, cs, mask, keep)
                p.a.primary = a if self.br_type != 1 else p.a.primary
                if fault == "null_bias":
                    p.d.primary = None
                if fault == "null_mask":
                    p.c.secondary = None
                st = X.GemmExtStrides(sa, self.tile_b, sc, self.m * TS[self.tc], smask)
                rc = lib.libxsmm_b200_gemm_ext_batch_strided(self.kernel, C.byref(p), C.byref(st), count)
            return rc, c, cs, mask
        cls = X.GemmExtParam if form == "ext_records" else X.GemmParam
        ps = (cls * self.count)(*[self.param(cls, t, c, cs, mask, keep) for t in range(self.count)])
        last = ps[self.count - 1]
        if fault == "null_side":
            s = sides(self.spec)
            if "a_s" in s:
                last.a.tertiary = None
            elif "a_q" in s:
                last.a.quaternary = None
            else:
                last.c.tertiary = None
        if fault == "null_bias":
            last.d.primary = None
        if fault == "null_mask":
            last.c.secondary = None
        if fault == "uneven_c":                             # the last tile one C further than the spacing of the others
            big = np.concatenate([c, self.C0[:self.tile_c]])
            c = big
            for t in range(self.count):
                ps[t].c.primary = c.ctypes.data + (t + (t == self.count - 1)) * self.tile_c
        if form == "plan":
            plan = lib.libxsmm_b200_gemm_plan_create(self.kernel, ps, count)
            rc = PLAN_NULL
            if plan:
                rc = lib.libxsmm_b200_gemm_plan_run(plan)
                lib.libxsmm_b200_gemm_plan_destroy(plan)
        elif form == "records":
            rc = lib.libxsmm_b200_gemm_batch(self.kernel, ps, count)
        else:
            rc = lib.libxsmm_b200_gemm_ext_batch(self.kernel, ps, count)
        return rc, c, cs, mask


def sweep(g):
    """the outcomes of every point of the grid, columns as OUTCOMES"""
    out = np.zeros((len(g), len(OUTCOMES)), dtype=np.int64)
    libs, handles = {}, {}
    saved = os.environ.get("XB_HOSTSIM_PTR_KIND")
    try:
        for i, (hi, fi, kind, qi) in enumerate(g):
            fam = HANDLES[hi][1]
            if fam not in libs:
                libs[fam] = build(fam)
            if hi not in handles:
                handles.clear()                            # one handle's buffers at a time: the chunk points are large
                handles[hi] = Handle(libs[fam], hi)
            h, lib = handles[hi], libs[fam]
            os.environ["XB_HOSTSIM_PTR_KIND"] = str(kind)
            n0, r0 = lib.libxsmm_b200_launch_count(), lib.hostsim_batch_launches()
            rc, c, cs, mask = h.run(FORMS[fi], FAULTS[qi])
            n1, r1 = lib.libxsmm_b200_launch_count(), lib.hostsim_batch_launches()
            dig = hashlib.sha256(c.tobytes() + cs.tobytes() + mask.tobytes()).digest()
            out[i] = (rc, n1 - n0, r1 - r0, int.from_bytes(dig[:8], "little", signed=True))
    finally:
        if saved is None:
            os.environ.pop("XB_HOSTSIM_PTR_KIND", None)
        else:
            os.environ["XB_HOSTSIM_PTR_KIND"] = saved
    return out


def main():
    g = grid()
    out = sweep(g)
    np.savez_compressed(os.path.join(HERE, "gemm_batch_rules.npz"), grid=g, grid_sha256=np.array(digest(g)), outcome=out)
    print("%d points, %d run (rc 0), %d distinct return codes" % (len(g), int(np.sum(out[:, 0] == 0)), len(set(out[:, 0].tolist()))))


if __name__ == "__main__":
    main()
