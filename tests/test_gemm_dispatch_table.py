"""CPU-only: which dense GEMM descriptors dispatch, and to which backend, point by point against tests/golden/gemm_dispatch.npz.

The grid (tests/golden/make_golden_dispatch.py) crosses every type tuple a dispatch rule names with the flags, leading dimensions,
divisibility cases, batch-reduce modes and ext-ABI fusions the rules read. No kernel is launched."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_dispatch as G  # noqa: E402


def test_dispatch_table_matches_golden():
    want = np.load(os.path.join(HERE, "golden", "gemm_dispatch.npz"))
    g = G.grid()
    assert G.digest(g) == str(want["grid_sha256"]), "the grid differs from the one the fixture was made from"
    got, peak = G.sweep(g)
    assert peak <= G.REGISTRY_LIMIT // 2, peak      # far from full: a NULL is a decline, not a full registry
    assert np.count_nonzero(want["backend"]) > 10000
    bad = np.flatnonzero(got != want["backend"])
    assert bad.size == 0, "%d points differ, first: %s" % (bad.size, [
        (dict(zip(G.COLUMNS, (int(v) for v in g[i]))), int(want["backend"][i]), int(got[i])) for i in bad[:5]])
