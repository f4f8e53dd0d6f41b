"""CPU-only: which matrix-eltwise descriptors dispatch, through both dispatch routes, which kernel a call of each would run and
whether its handle batches, point by point against tests/golden/meltw_dispatch.npz.

The grid (tests/golden/make_golden_meltw_dispatch.py) crosses every op code of each class with the types, flags and shapes the rules
read. No kernel is launched."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_meltw_dispatch as G  # noqa: E402


def test_meltw_dispatch_table_matches_golden():
    want = np.load(os.path.join(HERE, "golden", "meltw_dispatch.npz"))
    g = G.grid()
    assert G.digest(g) == str(want["grid_sha256"]), "the grid differs from the one the fixture was made from"
    got, peak = G.sweep(g)
    assert peak <= G.REGISTRY_LIMIT // 2, peak      # far from full: a NULL is a decline, not a full registry
    assert np.count_nonzero(want["answers"][:, 0]) > 10000
    bad = np.flatnonzero(np.any(got != want["answers"], axis=1))
    assert bad.size == 0, "%d points differ, first: %s" % (bad.size, [
        (dict(zip(G.COLUMNS, (int(v) for v in g[i]))), want["answers"][i].tolist(), got[i].tolist()) for i in bad[:5]])
