"""The reference's OWN sample drivers, unmodified, compiled against this repository's include/ and linked with -lxsmm
(libxsmm_b200/lib): the drop-in boundary of SURVEY.md 8b.

  * CPU (`-m "not gpu"`): where the reference sources exist, every driver in DRIVERS must compile and link.
    The binaries land in oracle/_ref/drivers/ (oracle/ref_drivers.py, built by __graft_entry__.build()).
  * GPU (`-m gpu`): the built binaries run on the GPU and must report success by their own criteria (each driver
    compares against its own dense/scalar gold and prints/returns the verdict).
"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
from ref_drivers import DRIVERS, LIBDIR, OUT, build_drivers, have_sources  # noqa: E402,F401
MTX = os.path.join(ROOT, "tests", "golden", "mtx")


@pytest.mark.skipif(not have_sources(), reason="the reference sources are not present here")
def test_reference_drivers_compile_and_link_unmodified():
    res = build_drivers()
    bad = {k: v[1] for k, v in res.items() if v[0] != 0}
    assert not bad, bad


def _run(name, *args, timeout=300):
    exe = os.path.join(OUT, name)
    if not os.path.exists(exe):
        pytest.skip("%s was not built: build() compiles the drivers into oracle/_ref/drivers where the reference sources exist" % name)
    env = dict(os.environ, LD_LIBRARY_PATH=LIBDIR + ":" + os.environ.get("LD_LIBRARY_PATH", ""), OMP_NUM_THREADS="4")
    return subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=timeout, env=env, cwd=OUT)


def test_gimmik_driver_runs_on_the_utility_layer():
    """samples/xgemm_sparse_Ainregs/gimmik.c times GiMMiK-generated C operators and takes from the library only the timer and the
    aligned allocator (libxsmm_timer_tick/duration, libxsmm_aligned_malloc/free): it needs no device, so it runs in both tiers.
    One CSV record per operator (60), positive rates."""
    p = _run("gimmik", 3, timeout=120)
    assert p.returncode == 0, (p.stdout[-400:], p.stderr[-800:])
    rows = [ln.split(";") for ln in p.stdout.splitlines() if ln.count(";") == 2]
    assert len(rows) == 60 and all(float(r[1]) > 0 and float(r[2]) > 0 for r in rows), p.stdout[-600:]


@pytest.mark.parametrize("name", ["ut_threadsafety", "ut_registry", "ut_gemmflags", "ut_matdiff"])
def test_reference_unit_tests_pass(name):
    """tests/threadsafety.c (800 random shapes <= 128 dispatched concurrently under OpenMP, libxsmm_get_mmkernel_info round trip, duplicates
    resolve to the same handle, release), tests/registry.c (libxsmm_xregister / xdispatch / xrelease edge cases), tests/gemmflags.c (truth
    table of LIBXSMM_GEMM_PFLAGS) and tests/matdiff.c, unmodified: dispatch is host logic, none of them launches a kernel, so they run in
    both tiers against the real library. Each returns EXIT_SUCCESS or EXIT_FAILURE."""
    p = _run(name, timeout=180)
    assert p.returncode == 0, (name, p.stdout[-800:], p.stderr[-800:])


@pytest.mark.gpu
def test_hello_runs():
    """samples/hello/hello.c: dispatches one F64 13x5x7 kernel and calls it 1000 times on malloc'ed (host) matrices, C += A_i * B_i;
    the program prints nothing and returns 0 -- what is checked here is that an unmodified caller runs to completion on this
    library (host operands staged per call) without the library reporting an error (LIBXSMM_VERBOSE=1 would print it)"""
    p = _run("hello")
    assert p.returncode == 0, (p.stdout[-400:], p.stderr[-800:])
    assert "error" not in p.stderr.lower(), p.stderr[-800:]


@pytest.mark.gpu
@pytest.mark.parametrize("mtx", ["pyfr_p1_tet_m6-sp.mtx", "pyfr_p3_hex_m6-sp.mtx"])
def test_pyfr_driver_on_the_reference_operators(mtx):
    """samples/xgemm_sparse_Ainregs/pyfr_driver_asp_reg.c <mtx> N reps: validates both beta cases against its own gold loop
    with libxsmm_matdiff and returns non-zero when the error exceeds its epsilon"""
    p = _run("pyfr_driver_asp_reg", os.path.join(MTX, mtx), 4800, 3)
    assert p.returncode == 0, (p.stdout[-1500:], p.stderr[-800:])
    lines = [ln for ln in p.stdout.splitlines() if "(libxsmm vs. gold)" in ln]
    assert len(lines) == 2, p.stdout[-1500:]
    for ln in lines:
        assert float(ln.split("abs=")[1].split()[0]) < 1e-6, ln


@pytest.mark.gpu
def test_spmm_kernel_driver_bf16_bcsc():
    """samples/xgemm_sparse/spmm_kernel.c (the BCSC driver) on a reduced configs[3] geometry: bf16, 32x32 blocks, 50 %;
    the driver checks against its dense gold and returns EXIT_FAILURE above its own bound (0.005 for bf16)"""
    # A B Comp C  M N K M_BLOCKS  sparsity BK BN  beta trA trB vnniA vnniB vnniC  reps      (spmm_kernel.c:755-786)
    p = _run("spmm_kernel", "BF16", "BF16", "F32", "BF16", 32, 512, 512, 64, 0.5, 32, 32, 0, 0, 0, 1, 0, 0, 3)
    assert p.returncode == 0, (p.stdout[-1500:], p.stderr[-800:])
    assert "Total Max Error" in p.stdout, p.stdout[-1500:]


@pytest.mark.gpu
def test_spmm_kernel_driver_f32_and_int8():
    for types, vnni in ((("F32", "F32", "F32", "F32"), 0), (("U8", "I8", "I32", "I32"), 1)):
        p = _run("spmm_kernel", *types, 32, 128, 128, 8, 0.5, 16 if types[0] == "F32" else 32, 16, 1, 0, 0, vnni, 0, 0, 2)
        assert p.returncode == 0, (types, p.stdout[-1500:], p.stderr[-800:])


# (driver, arguments) sets that the unmodified reference drivers accept and PASS by their own criteria on the GPU
ELTWISE_RUNS = [
    ("eltwise_unary_simple", (1, 0, "F32", "F32", "F32", 37, 11, 40, 40, 0)), ("eltwise_unary_simple", (2, 0, "F32", "F32", "F32", 37, 11, 40, 40, 0)),
    ("eltwise_unary_simple", (3, 0, "F32", "F32", "F32", 37, 11, 40, 40, 0)), ("eltwise_unary_simple", (11, 0, "F32", "F32", "F32", 37, 11, 40, 40, 0)),
    ("eltwise_unary_simple", (1, 0, "BF16", "F32", "BF16", 64, 16, 64, 64, 0)), ("eltwise_unary_simple", (1, 0, "F32", "F32", "BF8", 64, 16, 64, 64, 0)),
    ("eltwise_unary_simple", (1, 0, "F32", "F32", "BF8", 64, 16, 64, 64, 1)),      # rnd_mode 1: stochastic rounding with libxsmm_rng_create_extstate
    ("eltwise_unary_simple", (1, 1, "F32", "F32", "F32", 32, 32, 32, 32, 0)),
    ("eltwise_binary_simple", (1, 0, "F32", "F32", "F32", "F32", 37, 11, 40, 40)), ("eltwise_binary_simple", (2, 0, "F32", "F32", "F32", "F32", 37, 11, 40, 40)),
    ("eltwise_binary_simple", (3, 0, "F32", "F32", "F32", "F32", 37, 11, 40, 40)), ("eltwise_binary_simple", (4, 0, "F32", "F32", "F32", "F32", 37, 11, 40, 40)),
    ("eltwise_binary_simple", (1, 3, "BF16", "BF16", "F32", "BF16", 64, 16, 64, 64)),
    ("eltwise_unary_dropout", ("F", 1, "F32", "F32", 64, 16, 64, 64)), ("eltwise_unary_dropout", ("B", 1, "F32", "F32", 64, 16, 64, 64)),
    ("eltwise_unary_dropout", ("F", 0, "BF16", "BF16", 33, 7, 40, 40)),
    ("eltwise_unary_gather_scatter", (64, 32, 80, 64, 0, 0, 0, 0, 1)), ("eltwise_unary_gather_scatter", (64, 32, 64, 80, 1, 1, 1, 1, 1)),
    ("eltwise_unary_quantization", ("F32", "I8", 64, 16, 64, 64, 0, 0)), ("eltwise_unary_quantization", ("F32", "I16", 33, 7, 40, 40, 0, 1)),
    ("eltwise_unary_quantization_to_mxbf8", (64, 16, 64, 64)), ("eltwise_unary_quantization_to_mxfp4", (64, 16, 64, 64)),
    ("eltwise_unary_quantization_to_nvfp4", (64, 16, 64, 64)),
    ("eltwise_unary_reduce", (64, 32, 64, 1, 0, 0, 0, "F32", 0, 0, 0, 0, 1)), ("eltwise_unary_reduce", (64, 32, 64, 1, 1, 1, 0, "F32", 0, 0, 0, 0, 1)),
    ("eltwise_unary_reduce", (64, 32, 64, 1, 0, 0, 1, "F32", 0, 0, 1, 0, 1)),
    ("equation_simple", (64, 32)),
]


@pytest.mark.gpu
def test_eltwise_and_equation_drivers_pass_by_their_own_criteria():
    """samples/eltwise/*.c and samples/equation/equation_simple.c: each driver computes its own scalar gold, compares with libxsmm_matdiff
    or bit for bit (quantisers, masks) and returns EXIT_FAILURE on a mismatch"""
    for name, args in ELTWISE_RUNS:
        p = _run(name, *args, timeout=120)
        assert p.returncode == 0, (name, args, p.stdout[-800:], p.stderr[-400:])
        assert "FAILURE" not in p.stdout.upper(), (name, args, p.stdout[-800:])
