"""Recipe for the reference project's own sample drivers and unit tests, compiled UNMODIFIED against this repository's
include/ and linked with -lxsmm (libxsmm_b200/lib). The binaries go to oracle/_ref/drivers/ next to the reference library
(git-ignored, built by __graft_entry__.build() where the reference sources exist), so a built tree carries them to the
machine that runs the GPU tests, where the reference sources are absent.

The reference checkout is taken from LIBXSMM_REFERENCE_DIR, default: the Makefile's REFDIR.
"""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _makefile_refdir():
    """REFDIR of the Makefile (the same checkout `make ref` builds the reference library from)"""
    with open(os.path.join(ROOT, "Makefile")) as f:
        for line in f:
            if line.startswith("REFDIR") and "=" in line:
                return line.split("=", 1)[1].strip()
    return ""


REF = os.environ.get("LIBXSMM_REFERENCE_DIR") or _makefile_refdir()
OUT = os.path.join(ROOT, "oracle", "_ref", "drivers")
LIBDIR = os.path.join(ROOT, "libxsmm_b200", "lib")

# name -> source (relative to the reference tree)
DRIVERS = {
    "hello": "samples/hello/hello.c",
    "pyfr_driver_asp_reg": "samples/xgemm_sparse_Ainregs/pyfr_driver_asp_reg.c",
    "spmm_kernel": "samples/xgemm_sparse/spmm_kernel.c",
    "gemm_kernel": "samples/xgemm/gemm_kernel.c",
    "gemm_kernel_fused": "samples/xgemm/gemm_kernel_fused.c",
    "eltwise_unary_relu": "samples/eltwise/eltwise_unary_relu.c",
    "eltwise_unary_transform": "samples/eltwise/eltwise_unary_transform.c",
    "eltwise_unary_simple": "samples/eltwise/eltwise_unary_simple.c",
    "eltwise_binary_simple": "samples/eltwise/eltwise_binary_simple.c",
    "eltwise_ternary_simple": "samples/eltwise/eltwise_ternary_simple.c",
    "eltwise_unary_dropout": "samples/eltwise/eltwise_unary_dropout.c",
    "eltwise_unary_gather_scatter": "samples/eltwise/eltwise_unary_gather_scatter.c",
    "eltwise_unary_quantization": "samples/eltwise/eltwise_unary_quantization.c",
    "eltwise_unary_quantization_to_mxbf8": "samples/eltwise/eltwise_unary_quantization_to_mxbf8.c",
    "eltwise_unary_quantization_to_mxfp4": "samples/eltwise/eltwise_unary_quantization_to_mxfp4.c",
    "eltwise_unary_quantization_to_nvfp4": "samples/eltwise/eltwise_unary_quantization_to_nvfp4.c",
    "eltwise_unary_reduce": "samples/eltwise/eltwise_unary_reduce.c",
    "equation_simple": "samples/equation/equation_simple.c",
    "equation_relu": "samples/equation/equation_relu.c",
    "equation_softmax": "samples/equation/equation_softmax.c",
    "equation_simple_layernorm": "samples/equation/equation_simple_layernorm.c",
    "equation_bf16_x3_split_f32": "samples/equation/equation_bf16_x3_split_f32.c",
    "gimmik": "samples/xgemm_sparse_Ainregs/gimmik.c",
    "gemm_kernel_parallel": "samples/xgemm/gemm_kernel_parallel.c",
    # the reference's unit tests that pin dispatch-level behaviour (SURVEY.md section 4: threadsafety, registry, gemmflags) + matdiff
    "ut_threadsafety": "tests/threadsafety.c",
    "ut_registry": "tests/registry.c",
    "ut_gemmflags": "tests/gemmflags.c",
    "ut_matdiff": "tests/matdiff.c",
}


def have_sources():
    return os.path.isdir(os.path.join(REF, "samples"))


def build_drivers(names=None):
    """compile the listed reference drivers into OUT; returns {name: (rc, stderr tail)}"""
    os.makedirs(OUT, exist_ok=True)
    res = {}
    for name, src in DRIVERS.items():
        if names and name not in names:
            continue
        # the library is found relative to the binary, wherever the tree is copied
        cmd = ["gcc", "-O2", "-fopenmp", "-I" + os.path.join(ROOT, "include"), os.path.join(REF, src), "-o", os.path.join(OUT, name),
               "-L" + LIBDIR, "-lxsmm", "-lm", "-Wl,-rpath,$ORIGIN/../../../libxsmm_b200/lib"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        res[name] = (p.returncode, p.stderr[-2000:])
    return res
