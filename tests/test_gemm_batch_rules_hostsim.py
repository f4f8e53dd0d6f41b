"""CPU-only: what every GEMM batch entry point does with every kind of GEMM handle, point by point against
tests/golden/gemm_batch_rules.npz.

The grid (tests/golden/make_golden_gemm_batch.py) crosses plain, int8-scaled, zero-point, dequantising, MX fp8, low-bit and fused
handles with the seven batch forms, the three pointer kinds and the argument faults each form checks, plus two batches that cross the
64 MiB scratch budget of a chunked launch. Each point runs on the simulated device of its handle's family and is compared by return
code, tiles launched, batched re-pack passes and a digest of C, the ReLU bit mask and the MXBF8 C scales."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_gemm_batch as G  # noqa: E402


def test_batch_rules_match_golden():
    want = np.load(os.path.join(HERE, "golden", "gemm_batch_rules.npz"))
    g = G.grid()
    assert G.digest(g) == str(want["grid_sha256"]), "the grid differs from the one the fixture was made from"
    assert np.array_equal(g, want["grid"])
    got = G.sweep(g)
    assert np.count_nonzero(want["outcome"][:, 0] == 0) > 300
    bad = np.flatnonzero(np.any(got != want["outcome"], axis=1))
    assert bad.size == 0, "%d points differ, first: %s" % (bad.size, [
        ((G.HANDLES[g[i][0]][0], G.FORMS[g[i][1]], int(g[i][2]), G.FAULTS[g[i][3]]), dict(zip(G.OUTCOMES, want["outcome"][i].tolist())),
         dict(zip(G.OUTCOMES, got[i].tolist()))) for i in bad[:5]])
