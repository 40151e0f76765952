"""Every upload lays out the handle's three upload buffers (static tables, per-cycle inputs, per-cycle scratch) from
one description each and grows them only when a snapshot needs more.  One handle takes a sequence of snapshots that
grows and shrinks each buffer and switches the cycle route: every cycle equals the oracle, and a drain in the middle
equals the same drain on a fresh handle."""
import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from tests.helpers import assert_cycle_equal
from tests.test_handle_buffers import DRAIN_SCALARS

pytestmark = pytest.mark.gpu

GEN = 73  # a fixed static_generation: uploads after the first keep the static tables


def _flat(gen=0):  # flat cohorts without admitted workloads: the k_cycle_flat route
    snap = synth.make_snapshot(3, W=3000, Q=300, heads="one_per_cq")
    snap.static_generation = gen
    return snap


def _cycle(ev, snap, want_snap=None):
    want_snap = want_snap or snap
    got = ev.run_cycle(snap, abi.CycleOut(want_snap))
    assert_cycle_equal(got, oracle.run_cycle(want_snap))


def test_upload_buffers_across_routes_and_usage_modes():
    from kueue_b200 import native
    drain_snap = synth.make_snapshot(3, W=4000, Q=40)
    fresh = native.Evaluator(0)
    try:
        drain_want = fresh.run_drain(drain_snap)
    finally:
        fresh.close()
    ev = native.Evaluator(0)
    try:
        _cycle(ev, synth.make_snapshot(1))
        _cycle(ev, _flat())
        _cycle(ev, synth.make_snapshot(3, W=600, Q=60, heads="one_per_cq", preemption=True, tight=1.1))  # fair target search
        _cycle(ev, synth.make_snapshot(4, W=400, Q=40, heads="one_per_cq", tight=1.5))                   # classical target search
        _cycle(ev, _flat(GEN))
        _cycle(ev, _flat(GEN))                                    # static tables reused
        resident = _flat(GEN)
        resident.flags |= abi.F_USAGE_RESIDENT
        _cycle(ev, resident)
        usage = np.array(resident.arrays["cq_usage"]).reshape(resident.n_cq, resident.n_fr).copy()
        dirty = np.arange(0, resident.n_cq, 7, dtype=np.int32)
        usage[dirty] = usage[dirty] // 2
        full = _flat()
        full.set("cq_usage", usage)
        inc = _flat(GEN)
        inc.set("usage_delta_cq", dirty)
        inc.set("usage_delta_rows", usage[dirty])
        inc.arrays["cq_usage"] = np.zeros(0, np.int64)             # not read: the resident table is patched
        _cycle(ev, inc, full)
        drain_got = ev.run_drain(drain_snap)
        _cycle(ev, _flat())
    finally:
        ev.close()
    assert drain_want.n_cycles > 1 and drain_want.n_admitted > 0
    for f in DRAIN_SCALARS:
        assert getattr(drain_got, f) == getattr(drain_want, f), f
    arrays = [k for k, v in vars(drain_want).items() if isinstance(v, np.ndarray)]
    assert "trace_wl" in arrays and "cq_usage" in arrays
    for f in arrays:
        assert np.array_equal(getattr(drain_got, f), getattr(drain_want, f)), f
