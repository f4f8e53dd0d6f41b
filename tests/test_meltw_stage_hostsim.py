"""What a matrix-eltwise call stages, and whether a one-node equation over its descriptor dispatches, on the simulated device, point
by point against tests/golden/meltw_stage.npz.

The host_*.c sources are linked with tests/c/hostsim_runtime.c and tests/c/hostsim_meltw_stage.c, which logs every upload and copy
back and records each launch without running it (tests/golden/make_golden_meltw_stage.py). For every descriptor that
tests/golden/meltw_dispatch.npz records as dispatching, at two small shapes, one call with pageable operands (pinned ones for the
operations that insist): the bytes staged in and copied back per slot of the argument struct, which fields reach the launcher as NULL,
the caller's pointer or a staged buffer, alpha, the run-time count and the plane offsets. No GPU is needed."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_meltw_stage as S  # noqa: E402


def test_meltw_staging_matches_golden():
    want_stage, want_eqn, keys_sha256 = S.load(os.path.join(HERE, "golden", "meltw_stage.npz"))
    keys = S.cases()
    assert S.digest(keys) == keys_sha256, "the descriptors differ from the ones the fixture was made from"
    stage, eqn = S.sweep(keys)
    assert stage.shape == want_stage.shape and eqn.shape == want_eqn.shape
    assert np.count_nonzero(want_eqn == 1) > 100
    bad = np.flatnonzero(np.any(stage != want_stage, axis=1))
    assert bad.size == 0, "%d calls differ, first: %s" % (bad.size, [
        (keys[i // len(S.SHAPES)].tolist(), S.SHAPES[i % len(S.SHAPES)],
         dict((c, (int(w), int(h))) for c, w, h in zip(S.COLUMNS, want_stage[i], stage[i]) if w != h)) for i in bad[:5]])
    bad = np.flatnonzero(np.any(eqn != want_eqn, axis=1))
    assert bad.size == 0, "%d equations differ, first: %s" % (bad.size, [
        (np.unique(keys[:, :7], axis=0)[i].tolist(), want_eqn[i].tolist(), eqn[i].tolist()) for i in bad[:5]])
