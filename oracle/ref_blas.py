"""Recipe for the reference binaries behind the BLAS-style GEMM tests (tests/test_blas_gemm.py, tests/test_blas_gemm_gpu.py):

  oracle/_ref/libxsmm_ref_blas.so            the reference's own libxsmm_dgemm / libxsmm_sgemm (oracle/ref_blas_shim.c, header-only build)
  oracle/_ref/blas/magazine_xsmm             samples/magazine/magazine_xsmm.c as shipped: one dispatched kernel called per matrix
  oracle/_ref/blas/magazine_xsmm_auto        the same file built with -DAUTO, the sample's own switch: every matrix through libxsmm_dgemm

The sample is compiled UNMODIFIED against this repository's include/ and linked with -lxsmm, next to its own magazine.h; it is kept
apart from oracle/ref_drivers.py's list so that the driver tests run what they ran before. Everything lands under oracle/_ref/
(git-ignored, built by __graft_entry__.build() where the reference sources exist) and travels with the built tree.
"""
import os
import subprocess

from ref_drivers import LIBDIR, REF, ROOT

OUT = os.path.join(ROOT, "oracle", "_ref", "blas")
SHIM_SO = os.path.join(ROOT, "oracle", "_ref", "libxsmm_ref_blas.so")
MAGAZINE = {"magazine_xsmm": [], "magazine_xsmm_auto": ["-DAUTO"]}


def have_sources():
    return os.path.isdir(os.path.join(REF, "samples", "magazine")) and os.path.isdir(os.path.join(REF, "src"))


def build():
    """returns {target: (rc, stderr tail)}"""
    os.makedirs(OUT, exist_ok=True)
    res = {}
    cmd = ["gcc", "-O2", "-fPIC", "-shared", "-fvisibility=hidden", "-Wl,-Bsymbolic", "-fopenmp", "-ffp-contract=off",
           "-I" + os.path.join(REF, "include"), "-I" + os.path.join(REF, "src"), os.path.join(ROOT, "oracle", "ref_blas_shim.c"),
           "-o", SHIM_SO, "-lm", "-lpthread", "-ldl"]
    p = subprocess.run(cmd, capture_output=True, text=True)
    res["libxsmm_ref_blas.so"] = (p.returncode, p.stderr[-2000:])
    sample = os.path.join(REF, "samples", "magazine")
    for name, defs in MAGAZINE.items():
        cmd = ["gcc", "-O2", "-fopenmp"] + defs + ["-I" + os.path.join(ROOT, "include"), "-I" + sample, os.path.join(sample, "magazine_xsmm.c"),
                                                    "-o", os.path.join(OUT, name), "-L" + LIBDIR, "-lxsmm", "-lm",
                                                    "-Wl,-rpath,$ORIGIN/../../../libxsmm_b200/lib"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        res[name] = (p.returncode, p.stderr[-2000:])
    return res
