"""k_cycle_flat (kb_flat.cuh) against the CPU oracle on the shapes its overlapped phases branch on.

The kernel stages a root's tables in two stages, copies each entry's per-cycle records while the tree pass runs, and
publishes decisions and ClusterQueue usage rows block by block (32 iterator positions) behind the ordered loop. These
cases set root sizes and entry counts around those blocks, roots without entries, odd and wide flavor-resource rows,
resource counts that are not a multiple of four, both nominate walks in one root, every decision kind, and two cycles
on one evaluator.

A root's relocated tables take at least ~280 B of shared memory per node, so the largest root k_cycle_flat can hold
(about 800 ClusterQueues at one flavor and one resource) has fewer entries than the CTA has threads; the large cases
here go close to that size instead."""
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


def _roots(snap, sizes):
    """ClusterQueues 0.. in runs of `sizes` under the flat root cohorts, in order."""
    Q, C = snap.n_cq, snap.n_cohort
    assert len(sizes) == C and sum(sizes) == Q
    snap.set("parent", np.concatenate([Q + np.repeat(np.arange(C), sizes), np.full(C, -1)]))
    return snap


def _entries_per_root(snap, counts):
    """Keeps the heads of the first counts[k] ClusterQueues (in index order) of root k that have one."""
    Q = snap.n_cq
    heads = np.asarray(snap.arrays["heads"])
    cq = np.asarray(snap.wl_cq)[heads]
    root = np.asarray(snap.arrays["parent"])[cq] - Q
    order = np.lexsort((cq, root))
    rank = np.empty(len(heads), np.int64)
    start = np.searchsorted(root[order], root[order])
    rank[order] = np.arange(len(heads)) - start
    keep = rank < np.asarray(counts)[root]
    snap.set("heads", heads[keep])
    return snap


def _last_tried(snap, seed=21):
    """Current, stale and absent last-scheduling contexts; ps_last_tried starts the walk anywhere in the list."""
    rng = np.random.default_rng(seed)
    Q, F, R = snap.n_cq, snap.n_flavor, snap.n_resource
    gen = rng.integers(0, 5, Q)
    snap.set("cq_generation", gen)
    wg = gen[np.asarray(snap.wl_cq)]
    u = rng.random(len(wg))
    snap.set("wl_last_gen", np.where(u < 0.5, wg + rng.integers(0, 2, len(wg)), np.where(u < 0.75, wg - 1, -1)))
    snap.set("ps_last_tried", rng.integers(-1, max(F - 1, 0), (snap.n_podset, R)))
    return snap


def _preempt_policies(snap, seed=22):
    """Preemption within the ClusterQueue on half of the ClusterQueues, so some entries that fit only by preempting
    reserve (no admitted workloads: no candidates)."""
    rng = np.random.default_rng(seed)
    Q = snap.n_cq
    snap.set("cq_within_cq", np.where(rng.random(Q) < 0.5, abi.POLICY_LOWER_PRIORITY, abi.POLICY_NEVER))
    return snap


def _has_qr(snap, seed=23):
    snap.set("wl_has_quota_reservation", np.random.default_rng(seed).random(snap.n_wl) < 0.5)
    return snap


def _mixed_walks(snap, seed=24):
    """Up to three podsets per head and partial admission with reducible podsets: the general walk and the group walk
    share each root."""
    rng = np.random.default_rng(seed)
    snap.flags |= abi.F_PARTIAL_ADMISSION
    count = np.array(snap.arrays["ps_count"])
    snap.set("ps_min_count", np.where((rng.random(len(count)) < 1 / 3) & (count > 1), np.maximum(1, count // 2), -1))
    return snap


def _run(ev, snap):
    got = ev.run_cycle(snap)
    st = ev.stats()
    assert st.kernel_ms[abi.KERNEL_NAMES.index("k_cycle_flat")] > 0, "the cycle must run k_cycle_flat"
    return got


CASES = {
    # FR = 2, R = 2: one root of 550 entries (18 blocks, the last partial), small roots, one root without entries
    "blocks_fr2": lambda: _entries_per_root(_last_tried(_roots(synth.make_snapshot(3, W=6000, Q=600, F=1, R=2, heads="one_per_cq"),
                                                               [550, 10, 10, 10, 10, 10])), [550, 10, 10, 0, 10, 10]),
    # FR = 1 (per-thread staging, two commit groups): 640 entries = 20 full blocks, a root without entries
    "blocks_fr1": lambda: _entries_per_root(_roots(synth.make_snapshot(3, W=7000, Q=700, F=1, R=1, heads="one_per_cq"),
                                                   [640, 10, 10, 10, 10, 10, 10]), [640, 10, 0, 10, 10, 10, 10]),
    # FR = 32: 64 entries (two full blocks), 20 entries, none
    "counts_64_20_0": lambda: _entries_per_root(synth.make_snapshot(3, W=3000, Q=300, heads="one_per_cq"), [64, 20, 0]),
    # FR = 9: odd rows, R = 3
    "fr9": lambda: _last_tried(synth.make_snapshot(3, W=900, Q=90, F=3, R=3, heads="one_per_cq")),
    # FR = 64: the two-column ordered loop, 40 entries
    "fr64": lambda: _last_tried(synth.make_snapshot(3, W=400, Q=40, F=16, R=4, heads="one_per_cq")),
    # several podsets, reducible podsets, quota-reservation flags and last-tried rows, both walks in every root
    "mixed_walks": lambda: _has_qr(_last_tried(_mixed_walks(synth.make_snapshot(3, W=3000, Q=300, heads="one_per_cq", podsets_max=3)))),
    "mixed_walks_fr9": lambda: _has_qr(_mixed_walks(synth.make_snapshot(3, W=900, Q=90, F=3, R=3, heads="one_per_cq", podsets_max=2))),
}


@pytest.mark.parametrize("name", list(CASES))
def test_flat_overlap_matches_oracle(ev, name):
    snap = CASES[name]().finalize()
    assert_cycle_equal(_run(ev, snap), oracle.run_cycle(snap))


@pytest.mark.parametrize("fair", [True, False], ids=["fair", "classical"])
def test_flat_decision_kinds_interleaved(ev, fair):
    """Fit, NoFit and reserving Preempt entries interleaved in iterator order; the usage rows carry every kind."""
    snap = _preempt_policies(synth.make_snapshot(3, W=3000, Q=300, F=2, R=2, heads="one_per_cq"))
    if not fair:
        snap.flags &= ~abi.F_FAIR_SHARING
    snap = snap.finalize()
    got = _run(ev, snap)
    want = oracle.run_cycle(snap)
    assert_cycle_equal(got, want)
    dec = np.asarray(want.decision)
    for kind in (abi.DEC_ASSUMED, abi.DEC_PREEMPT_NO_TARGETS):
        assert (dec == kind).any(), abi.DEC_NAMES[kind]
    assert np.isin(dec, [abi.DEC_NOFIT, abi.DEC_SKIPPED_NO_FIT]).any()


def test_flat_two_cycles_one_evaluator(ev):
    """The second cycle keeps the static tables staged by the first (same static_generation) and has heads in only
    some ClusterQueues: records stamped by the first cycle must not count."""
    a = synth.make_snapshot(3, W=3000, Q=300, heads="one_per_cq")
    a.static_generation = 41
    a = a.finalize()
    assert_cycle_equal(_run(ev, a), oracle.run_cycle(a))
    b = _entries_per_root(synth.make_snapshot(3, W=3000, Q=300, heads="one_per_cq"), [60, 33, 0])
    b.set("cq_usage", (np.asarray(b.arrays["cq_usage"]) * 0.9).astype(np.int64))
    b.static_generation = 41
    b = b.finalize()
    assert_cycle_equal(_run(ev, b), oracle.run_cycle(b))
