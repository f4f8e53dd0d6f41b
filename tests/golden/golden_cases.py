"""The fixed case lists behind tests/golden/*.npz (shared by the generator and the tests)."""
import numpy as np

import cases
import gen
from oracle_ffi import iarr


def gemm_cases():
    """(GemmCase, seed, count): every precision tuple x a layout flag x the four batch-reduce modes, plus the
    reference's headline tile (64^3 x 8, stride BR) and hello's 13x5x7."""
    out = []
    for i, case in enumerate(cases.small_cases(seed=2024)):
        if i % 5 == 0:
            out.append((case, 4000 + i, 2))
    for t in ((gen.BF16, gen.BF16, gen.F32, gen.F32), (gen.BF16, gen.BF16, gen.F32, gen.BF16), (gen.F16, gen.F16, gen.F32, gen.F32)):
        out.append((cases.GemmCase(64, 64, 64, *t, flags=cases.FLAG_BETA_0, br_type=3, br=8), 77, 3))
    out.append((cases.GemmCase(13, 5, 7, gen.F64, gen.F64, gen.F64, gen.F64), 78, 4))
    out.append((cases.GemmCase(13, 5, 7, gen.F32, gen.F32, gen.F32, gen.F32), 79, 4))
    return out


def int8_full_range():
    """(GemmCase, Operands): U8 in [0, 255] x I8 in [-128, 127] -> I32 over VNNI4 A with a stride batch-reduce, and an old C spread over
    the whole int32 range so that beta = 1 wraps; gen.values keeps 8-bit operands within +-20"""
    case = cases.GemmCase(48, 20, 128, gen.U8, gen.I8, gen.I32, gen.I32, flags=cases.FLAG_VNNI_A, br_type=3, br=3)
    ops = cases.Operands(case, seed=80, count=2)
    rng = np.random.default_rng(81)
    ops.a = rng.integers(0, 256, size=ops.a.size).astype(np.uint8)
    ops.b = rng.integers(-128, 128, size=ops.b.size).astype(np.int8)
    ops.c0 = rng.integers(-2 ** 31, 2 ** 31, size=ops.c0.size).astype(np.int32)
    return case, ops


# ---- BCSC (reference: x86 JIT of libxsmm_create_packed_spgemm_bcsc; gold loop samples/xgemm_sparse/spmm_kernel.c:74-217)
def bcsc_cases():
    T_BF, T_F32, T_U8I8, T_I8U8 = (gen.BF16, gen.BF16, gen.F32, gen.BF16), (gen.F32,) * 4, (gen.U8, gen.I8, gen.I32, gen.I32), (gen.I8, gen.U8, gen.I32, gen.I32)
    return [dict(types=T_BF, geo=(5, 32, 128, 64, 32, 32), dens=0.5, beta0=1, seed=11),
            dict(types=T_BF, geo=(3, 32, 512, 512, 32, 32), dens=0.5, beta0=0, seed=12),
            dict(types=T_BF, geo=(3, 16, 64, 96, 16, 32), dens=0.4, beta0=1, seed=13),
            dict(types=T_F32, geo=(3, 32, 128, 64, 16, 16), dens=0.5, beta0=1, seed=14),
            dict(types=T_U8I8, geo=(3, 32, 128, 64, 32, 16), dens=0.5, beta0=1, seed=15),
            dict(types=T_I8U8, geo=(2, 32, 128, 64, 32, 16), dens=0.6, beta0=0, seed=16)]


def bcsc_flags(cfg):
    return (cases.FLAG_BETA_0 if cfg["beta0"] else 0) | (cases.FLAG_VNNI_A if cfg["types"][0] != gen.F32 else 0)


def bcsc_inputs(cfg):
    rng = np.random.default_rng(cfg["seed"])
    ta, tb, _, tc = cfg["types"]
    mblocks, M, K, N, bk, bn = cfg["geo"]
    nbr, nbc = K // bk, N // bn
    keep = rng.random((nbc, nbr)) < cfg["dens"]
    colptr = np.zeros(nbc + 1, dtype=np.uint32); rowidx = []
    for j in range(nbc):
        rowidx.extend(np.nonzero(keep[j])[0].tolist()); colptr[j + 1] = len(rowidx)
    rowidx = np.array(rowidx if rowidx else [0], dtype=np.uint32)
    nnzb = int(colptr[-1])
    return dict(a=gen.values(rng, mblocks * K * M, ta), bvals=gen.values(rng, max(nnzb, 1) * bk * bn, tb), colptr=colptr, rowidx=rowidx,
                c0=gen.values(rng, mblocks * N * M, tc))


def run_bcsc(side, cfg, inp, c):
    return side["bcsc"](iarr(*cfg["types"]), iarr(*cfg["geo"]), bcsc_flags(cfg), inp["a"].ctypes.data, inp["bvals"].ctypes.data,
                        inp["colptr"].ctypes.data, inp["rowidx"].ctypes.data, c.ctypes.data)


# ---- fsspmdm (reference: libxsmm_fsspmdm_create/execute, src/libxsmm_fsspmdm.c:24-545)
def fsspmdm_cases():
    return [dict(dtype=gen.F32, M=24, K=40, N=96, alpha=1.5, beta=0.0, dens=0.2, seed=21),
            dict(dtype=gen.F32, M=32, K=128, N=512, alpha=1.0, beta=1.0, dens=0.15, seed=22),
            dict(dtype=gen.F64, M=24, K=40, N=96, alpha=1.0, beta=1.0, dens=0.2, seed=23),
            dict(dtype=gen.F64, M=7, K=9, N=64, alpha=-0.5, beta=0.0, dens=0.5, seed=24)]


def fsspmdm_inputs(cfg):
    rng = np.random.default_rng(cfg["seed"])
    npdt = gen.NP_OF[cfg["dtype"]]
    M, K, N = cfg["M"], cfg["K"], cfg["N"]
    a = (gen.values(rng, M * K, gen.F64) * (rng.random(M * K) < cfg["dens"])).astype(npdt)
    return dict(a=a, b=gen.values(rng, K * N, cfg["dtype"]), c0=gen.values(rng, M * N, cfg["dtype"]),
                alpha=np.array([cfg["alpha"]], dtype=npdt), beta=np.array([cfg["beta"]], dtype=npdt))


def run_fsspmdm(side, cfg, inp, c):
    M, K, N = cfg["M"], cfg["K"], cfg["N"]
    return side["fsspmdm"](cfg["dtype"], M, N, K, K, N, N, inp["alpha"].ctypes.data, inp["beta"].ctypes.data, inp["a"].ctypes.data,
                           inp["b"].ctypes.data, c.ctypes.data)


# ---- real sparsity patterns shipped with the reference's drivers (tests/golden/mtx/*.mtx, copied input DATA of
# samples/xgemm_sparse_Ainregs/mats (PyFR operators) and samples/xgemm_norm_packed/mats (EDGE/SeisSol operators)) --------
import os

MTX_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "mtx")


def read_mtx(name):
    """MatrixMarket coordinate file -> (rows, cols, dense float64 array); same reading as the drivers' CSR readers"""
    with open(os.path.join(MTX_DIR, name)) as f:
        lines = [ln for ln in f if not ln.startswith("%")]
    rows, cols, nnz = (int(x) for x in lines[0].split())
    dense = np.zeros((rows, cols))
    for ln in lines[1:1 + nnz]:
        r, c, v = ln.split()
        dense[int(r) - 1, int(c) - 1] = float(v)
    return rows, cols, dense


def pyfr_cases():
    out = []
    for i, name in enumerate(("pyfr_p1_tet_m6-sp.mtx", "pyfr_p2_quad_m132-sp.mtx", "pyfr_p3_hex_m6-sp.mtx", "pyfr_p3_hex_m132-sp.mtx")):
        for dtype in (gen.F64, gen.F32):
            for beta in (0.0, 1.0):
                out.append(dict(mtx=name, dtype=dtype, N=96, alpha=1.0, beta=beta, seed=300 + len(out)))
    return out


def pyfr_inputs(cfg):
    M, K, dense = read_mtx(cfg["mtx"])
    rng = np.random.default_rng(cfg["seed"])
    npdt = gen.NP_OF[cfg["dtype"]]
    return dict(M=M, K=K, a=dense.astype(npdt).ravel().copy(), b=gen.values(rng, K * cfg["N"], cfg["dtype"]), c0=gen.values(rng, M * cfg["N"], cfg["dtype"]),
                alpha=np.array([cfg["alpha"]], dtype=npdt), beta=np.array([cfg["beta"]], dtype=npdt))


def run_pyfr(side, cfg, inp, c):
    M, K, N = inp["M"], inp["K"], cfg["N"]
    return side["fsspmdm"](cfg["dtype"], M, N, K, K, N, N, inp["alpha"].ctypes.data, inp["beta"].ctypes.data, inp["a"].ctypes.data,
                           inp["b"].ctypes.data, c.ctypes.data)


def edge_cases():
    """(kind, file, free dimension, packed width, dtype, beta0): the sparse operand's extents come from the file"""
    return [dict(kind="a_csr", mtx="tet4_starMatrix_csr.mtx", free=20, P=16, dtype=gen.F32, beta0=0, seed=400),
            dict(kind="a_csr", mtx="tet4_starMatrix_csr.mtx", free=35, P=8, dtype=gen.F64, beta0=1, seed=401),
            dict(kind="b_csr", mtx="tet4_2_fluxN_0_csr.mtx", free=9, P=8, dtype=gen.F64, beta0=0, seed=402),
            dict(kind="b_csc", mtx="tet4_2_fluxN_0_csc.mtx", free=9, P=16, dtype=gen.F32, beta0=0, seed=403),
            dict(kind="b_csr", mtx="tet4_3_stiffT_0_csr.mtx", free=9, P=16, dtype=gen.F32, beta0=1, seed=404),
            dict(kind="b_csc", mtx="tet4_3_stiffT_0_csc.mtx", free=9, P=8, dtype=gen.F64, beta0=0, seed=405),
            dict(kind="b_csr", mtx="tet4_4_fluxT_1_csr.mtx", free=9, P=8, dtype=gen.F64, beta0=0, seed=406),
            dict(kind="b_csc", mtx="tet4_4_fluxT_1_csc.mtx", free=9, P=16, dtype=gen.F32, beta0=1, seed=407)]


def edge_inputs(cfg):
    rows, cols, dense = read_mtx(cfg["mtx"])
    rng = np.random.default_rng(cfg["seed"])
    dtype, P, kind = cfg["dtype"], cfg["P"], cfg["kind"]
    npdt = gen.NP_OF[dtype]
    mask = dense != 0
    if kind.endswith("csr"):
        ptr = np.concatenate([[0], np.cumsum(mask.sum(1))]).astype(np.uint32); idx = np.nonzero(mask)[1].astype(np.uint32)
        vals = dense[mask].astype(npdt)
    else:
        ptr = np.concatenate([[0], np.cumsum(mask.sum(0))]).astype(np.uint32); idx = np.nonzero(mask.T)[1].astype(np.uint32)
        vals = dense.T[mask.T].astype(npdt)
    if kind == "a_csr":
        M, K, N = rows, cols, cfg["free"]
        dims = (M, N, K, 0, N, N); a = vals; b = gen.values(rng, K * N * P, dtype)
    else:
        K, N, M = rows, cols, cfg["free"]
        dims = (M, N, K, K, 0, N); a = gen.values(rng, M * K * P, dtype); b = vals
    return dict(dims=dims, ptr=ptr, idx=idx, vals=vals, a=a, b=b, c0=gen.values(rng, M * N * P, dtype), is_csc=int(kind.endswith("csc")),
                flags=cases.FLAG_BETA_0 if cfg["beta0"] else 0)


def run_edge(side, cfg, inp, c):
    return side["packed_sp"](inp["is_csc"], cfg["dtype"], iarr(*inp["dims"]), inp["flags"], cfg["P"], inp["ptr"].ctypes.data, inp["idx"].ctypes.data,
                             inp["vals"].ctypes.data, inp["a"].ctypes.data, inp["b"].ctypes.data, c.ctypes.data)
