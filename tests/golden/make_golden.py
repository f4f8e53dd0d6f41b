#!/usr/bin/env python
"""Generates tests/golden/*.npz by running the UNMODIFIED reference (oracle/_ref/libxsmm_ref.so, built from
/root/reference by `make ref`) on seeded inputs. Run here, in the build container; the fixtures travel to the GPU
box where /root/reference does not exist.

    python tests/golden/make_golden.py

Inputs are not stored: they are re-created from the seeds by tests/cases.py / tests/gen.py; a CRC of the input
bytes is stored next to every expected output so that generator drift is detected instead of mis-diagnosed."""
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE)); sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import cases  # noqa: E402
import gen  # noqa: E402
import golden_cases as G  # noqa: E402
from oracle_ffi import ref, run_gemm  # noqa: E402


def crc(*arrs):
    c = 0
    for a in arrs:
        c = zlib.crc32(np.ascontiguousarray(a).view(np.uint8).tobytes(), c)
    return np.uint32(c)


def main():
    """usage: make_golden.py [gemm] [int8] [sparse] [mtx]  (default: all). The sparse sections need a host whose ISA the reference's JIT can build
    BCSC bf16 for (AVX512-BF16 / AMX: the GPU box); the GEMM section runs on any x86-64 host."""
    import sys
    want = set(sys.argv[1:]) or {"gemm", "int8", "sparse", "mtx"}
    assert ref is not None, "oracle/_ref/libxsmm_ref.so is missing: run `make ref` where /root/reference exists"
    out = {}
    for i, (case, seed, count) in enumerate(G.gemm_cases() if "gemm" in want else []):
        ops = cases.Operands(case, seed=seed, count=count)
        out["gemm_%03d" % i] = cases.ref_result(ref, case, ops, run_gemm)
        out["gemm_%03d_crc" % i] = crc(ops.a, ops.b, ops.c0)
    if "gemm" in want:
        np.savez_compressed(os.path.join(HERE, "gemm.npz"), **out)
        print("gemm.npz: %d cases" % (len(out) // 2))
    if "int8" in want:
        case, ops = G.int8_full_range()
        np.savez_compressed(os.path.join(HERE, "int8.npz"), gemm=cases.ref_result(ref, case, ops, run_gemm), crc=crc(ops.a, ops.b, ops.c0))
        print("int8.npz: 1 case")
    if "sparse" not in want and "mtx" not in want:
        return

    out = {}
    for i, cfg in enumerate(G.bcsc_cases()):
        inp = G.bcsc_inputs(cfg)
        c = inp["c0"].copy()
        assert G.run_bcsc(ref, cfg, inp, c) == 0, cfg
        out["bcsc_%02d" % i] = c
        out["bcsc_%02d_crc" % i] = crc(inp["a"], inp["bvals"], inp["colptr"], inp["rowidx"], inp["c0"])
    for i, cfg in enumerate(G.fsspmdm_cases()):
        inp = G.fsspmdm_inputs(cfg)
        c = inp["c0"].copy()
        assert G.run_fsspmdm(ref, cfg, inp, c) in (0, None), cfg
        out["fsspmdm_%02d" % i] = c
        out["fsspmdm_%02d_crc" % i] = crc(inp["a"], inp["b"], inp["c0"])
    np.savez_compressed(os.path.join(HERE, "sparse.npz"), **out)
    print("sparse.npz: %d cases" % (len(out) // 2))

    # the reference's own operator files (tests/golden/mtx): fsspmdm on the PyFR matrices, packed CSR/CSC on the EDGE ones
    out = {}
    for i, cfg in enumerate(G.pyfr_cases()):
        inp = G.pyfr_inputs(cfg)
        c = inp["c0"].copy()
        assert G.run_pyfr(ref, cfg, inp, c) == 0, cfg
        out["pyfr_%02d" % i] = c
        out["pyfr_%02d_crc" % i] = crc(inp["a"], inp["b"], inp["c0"])
    for i, cfg in enumerate(G.edge_cases()):
        inp = G.edge_inputs(cfg)
        c = inp["c0"].copy()
        assert G.run_edge(ref, cfg, inp, c) == 0, cfg
        out["edge_%02d" % i] = c
        out["edge_%02d_crc" % i] = crc(inp["ptr"], inp["idx"], inp["a"], inp["b"], inp["c0"])
    np.savez_compressed(os.path.join(HERE, "mtx.npz"), **out)
    print("mtx.npz: %d cases" % (len(out) // 2))


if __name__ == "__main__":
    main()
