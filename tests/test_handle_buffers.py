"""One handle serves cycles, drains and placements (the Go shim keeps one per process), and kb_run_drain and
kb_tas_find each keep a grow-only device buffer on it.  Growing one must leave the other intact: a placement, a drain
(a fresh handle's first drain allocates its buffer), the same placement again and the same drain again give the same
results, and the placements equal the oracle."""
import numpy as np
import pytest

import oracle
from kueue_b200 import synth
from tests.test_gpu_tas_paths import _same, build

pytestmark = pytest.mark.gpu

DRAIN_SCALARS = ("n_cycles", "n_decisions", "n_admitted", "n_evicted", "n_finished", "n_arrived", "end_ns", "n_afs_samples")


def test_placement_and_drain_buffers_share_one_handle():
    from kueue_b200 import native
    topo, reqs, cap, _, _ = build("slices_3_levels")
    want = oracle.tas_find(topo, reqs, cap)
    snap = synth.make_snapshot(3, W=4000, Q=40)
    ev = native.Evaluator(0)
    try:
        tas_before = ev.tas_find(topo, reqs, cap)
        drain_before = ev.run_drain(snap)
        tas_after = ev.tas_find(topo, reqs, cap)
        drain_after = ev.run_drain(snap)
    finally:
        ev.close()
    _same(tas_before, want)
    _same(tas_after, want)
    for f in ("status", "asg_start", "asg_leaf", "asg_count"):
        assert np.array_equal(getattr(tas_before, f), getattr(tas_after, f)), f
    assert drain_before.n_cycles > 1 and drain_before.n_admitted > 0
    for f in DRAIN_SCALARS:
        assert getattr(drain_before, f) == getattr(drain_after, f), f
    arrays = [k for k, v in vars(drain_before).items() if isinstance(v, np.ndarray)]
    assert "trace_wl" in arrays and "cq_usage" in arrays
    for f in arrays:
        assert np.array_equal(getattr(drain_before, f), getattr(drain_after, f)), f
