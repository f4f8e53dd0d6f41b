"""A plain C program written against include/*.h and linked with -lxsmm, like an existing LIBXSMM caller that relinks
(INTEGRATION.md section 1). CPU: it compiles, links and its host-side checks pass. GPU: it runs the kernel on host buffers
and matches a triple loop exactly."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "c", "relink_demo.c")
EXE = os.path.join(ROOT, "build", "relink_demo")
LIBDIR = os.path.join(ROOT, "libxsmm_b200", "lib")


def build():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    cmd = ["gcc", "-std=c99", "-O1", "-ffp-contract=off", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), SRC,
           "-L" + LIBDIR, "-lxsmm", "-Wl,-rpath," + LIBDIR, "-lm", "-o", EXE]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    return EXE


def test_c_caller_compiles_links_and_dispatches():
    assert os.path.exists(os.path.join(LIBDIR, "libxsmm.so")), "run `make lib` first"
    exe = build()
    out = subprocess.run([exe, "dispatch"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "dispatch ok" in out.stdout and "target sm_90a" in out.stdout


@pytest.mark.gpu
def test_c_caller_runs_on_host_buffers():
    exe = build()
    out = subprocess.run([exe, "run"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "max_abs_diff 0.000e+00" in out.stdout
