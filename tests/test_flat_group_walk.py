"""The group walk of k_cycle_flat (kb_flat.cuh, phase 5) against the CPU oracle.

Every case runs the fused flat-cohort kernel; each one sets inputs that steer a different branch of
findFlavorForPodSets: the start index from ps_last_tried, the fungibility policies and preference, the
preempt-while-borrowing policies, several resource groups, the pods resource, and resources without a
resource group."""
import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from tests.helpers import assert_cycle_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ev():
    from kueue_b200 import native
    e = native.Evaluator(0)
    e.set_profile(True)
    yield e
    e.close()


def _base(**kw):
    return synth.make_snapshot(3, W=3000, Q=300, heads="one_per_cq", **kw)


def _last_tried(snap, seed=5):
    """Half of the workloads carry a current last-scheduling context (wl_last_gen >= cq_generation), a quarter a stale
    one; ps_last_tried starts the walk anywhere in the flavor list."""
    rng = np.random.default_rng(seed)
    Q, F, R = snap.n_cq, snap.n_flavor, snap.n_resource
    gen = rng.integers(0, 5, Q)
    snap.set("cq_generation", gen)
    wg = gen[np.asarray(snap.wl_cq)]
    u = rng.random(len(wg))
    snap.set("wl_last_gen", np.where(u < 0.5, wg + rng.integers(0, 2, len(wg)), np.where(u < 0.75, wg - 1, -1)))
    snap.set("ps_last_tried", rng.integers(-1, F - 1, (snap.n_podset, R)))
    return snap


def _policies(snap, seed=6):
    """Random whenCanBorrow / whenCanPreempt / preference and preempt-while-borrowing policies (no admitted workloads,
    so no ClusterQueue has preemption candidates)."""
    rng = np.random.default_rng(seed)
    Q = snap.n_cq
    snap.set("cq_when_can_borrow", rng.integers(0, 2, Q))
    snap.set("cq_when_can_preempt", rng.integers(0, 2, Q))
    snap.set("cq_preference", rng.integers(0, 3, Q))
    snap.set("cq_reclaim_within", rng.choice([abi.POLICY_NEVER, abi.POLICY_LOWER_PRIORITY, abi.POLICY_ANY], Q))
    snap.set("cq_borrow_within", np.where(rng.random(Q) < 0.3, abi.POLICY_LOWER_PRIORITY, abi.POLICY_NEVER))
    return snap


def _no_fungibility(snap):
    snap.flags &= ~abi.F_FLAVOR_FUNGIBILITY
    return snap


def _classical(snap):
    snap.flags &= ~abi.F_FAIR_SHARING
    return snap


def _two_groups_and_pods(snap, seed=7):
    """Two resource groups per ClusterQueue (resources {0, 1} on flavors 0-3, {2, 3} on flavors 4-7, in either order),
    resource 3 is the pods resource and only some podsets list it."""
    rng = np.random.default_rng(seed)
    Q = snap.n_cq
    swap = rng.random(Q) < 0.5
    masks = np.stack([np.where(swap, 0b1100, 0b0011), np.where(swap, 0b0011, 0b1100)], 1).reshape(-1)
    fl = np.stack([np.where(swap, 1, 0), np.where(swap, 0, 1)], 1).reshape(-1)  # which half of the flavors
    snap.set("cq_rg_start", np.arange(Q + 1) * 2)
    snap.set("rg_res_mask", masks)
    snap.set("rg_flavor_start", np.arange(2 * Q + 1) * 4)
    snap.set("rg_flavors", (fl[:, None] * 4 + np.arange(4)[None, :]).reshape(-1))
    snap.pods_resource = 3
    snap.set("ps_req_mask", np.where(rng.random(snap.n_podset) < 0.5, 0b0111, 0b1111))
    return snap


def _ungrouped_resource(snap, seed=8):
    """Resource 3 has no resource group in a third of the ClusterQueues; half of the podsets request none of it."""
    rng = np.random.default_rng(seed)
    Q = snap.n_cq
    snap.set("rg_res_mask", np.where(rng.random(Q) < 1 / 3, 0b0111, 0b1111))
    req = np.array(snap.ps_req).reshape(snap.n_podset, snap.n_resource).copy()
    req[rng.random(snap.n_podset) < 0.5, 3] = 0
    snap.set("ps_req", req)
    return snap


@pytest.mark.parametrize("make", [
    lambda: _last_tried(_base()),
    lambda: _last_tried(_policies(_base())),
    lambda: _no_fungibility(_last_tried(_policies(_base()))),
    lambda: _two_groups_and_pods(_last_tried(_policies(_base()))),
    lambda: _classical(_two_groups_and_pods(_policies(_base()))),
    lambda: _ungrouped_resource(_policies(_base())),
    lambda: _last_tried(_policies(synth.make_snapshot(3, W=400, Q=40, F=16, R=4, heads="one_per_cq"))),    # two rounds of flavors
    lambda: _last_tried(_policies(synth.make_snapshot(3, W=900, Q=90, F=3, R=3, heads="one_per_cq"))),     # R = 3
], ids=["last_tried", "policies", "no_fungibility", "two_groups_pods", "classical_groups_pods", "ungrouped_resource",
        "F16", "R3"])
def test_flat_group_walk_matches_oracle(ev, make):
    snap = make().finalize()
    got = ev.run_cycle(snap)
    st = ev.stats()
    assert st.kernel_ms[abi.KERNEL_NAMES.index("k_cycle_flat")] > 0, "the cycle must run k_cycle_flat"
    assert st.flat_group_walk[1] > 0 and st.flat_group_walk[0] == st.flat_group_walk[1], "every entry must take the group walk"
    assert_cycle_equal(got, oracle.run_cycle(snap))


def test_flat_group_walk_and_general_walk_share_a_root(ev):
    """Entries with several podsets take the general walk, single-podset entries of the same root the group walk."""
    snap = synth.make_snapshot(3, W=3000, Q=300, heads="one_per_cq", podsets_max=2)
    got = ev.run_cycle(snap)
    st = ev.stats()
    assert st.kernel_ms[abi.KERNEL_NAMES.index("k_cycle_flat")] > 0, "the cycle must run k_cycle_flat"
    assert 0 < st.flat_group_walk[0] < st.flat_group_walk[1], "the root must mix both walks"
    assert_cycle_equal(got, oracle.run_cycle(snap))
