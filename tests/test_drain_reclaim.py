"""Reclaim steps in the drain's event mode (kb_snapshot.wl_rc_start, rc_*, ps_adm_*, adm_run_start_ns;
kueue_b200/drain.py).  A running workload whose pods succeed gives back the quota of the pods it no longer needs
(Status.ReclaimablePods).  CPU: the reference's cases transcribed as schedules on the oracle, hand-derived schedules, the
equivalence without steps, seeded invariants and the refusals.  GPU: kb_run_drain equals the host definition cycle by
cycle, alone and with every other event block, and refuses bad tables."""
import ctypes as C

import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from kueue_b200.drain import ReclaimUnsupported, check_reclaims, drain

N_, A_ = abi.DEC_NOFIT, abi.DEC_ASSUMED
BE, STRICT = abi.QUEUE_BEST_EFFORT_FIFO, abi.QUEUE_STRICT_FIFO
UNSET = np.iinfo(np.int64).min


def run(snap, max_cycles=100_000):
    snap.finalize()
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000
    return drain(snap, lambda s: oracle.run_cycle(s, cap), max_cycles=max_cycles)


def cq_case(pods, per_pod, nominal=10, run_ns=100, strategy=STRICT, create=None, Q=1, wl_cq=None, cohort=False):
    """records of one podset each: pods[w] pods of per_pod[w] cpu, created at create[w] (0), running run_ns; each
    ClusterQueue has `nominal` cpu (a cohort over them when `cohort`).  One cycle takes 1 ns."""
    W = len(pods)
    s = abi.FlatSnapshot(n_cq=Q, n_cohort=1 if cohort else 0, n_flavor=1, n_resource=1)
    s.set("parent", [Q] * Q + [-1] if cohort else [-1] * Q)
    s.set("nominal", [[nominal]] * Q + ([[0]] if cohort else []))
    s.set("cq_rg_start", np.arange(Q + 1)); s.set("rg_res_mask", np.ones(Q)); s.set("rg_flavor_start", np.arange(Q + 1))
    s.set("rg_flavors", np.zeros(Q)); s.set("cq_strategy", np.full(Q, strategy))
    s.set("wl_cq", np.zeros(W) if wl_cq is None else wl_cq); s.set("wl_ts", np.arange(W))
    s.set("ps_req", (np.asarray(pods) * np.asarray(per_pod))[:, None]); s.set("ps_req_mask", np.ones(W))
    s.set("ps_count", pods)
    s.set("adm_wl", np.zeros(0)); s.set("wl_run_ns", np.full(W, run_ns) if np.isscalar(run_ns) else run_ns)
    if create is not None:
        s.set("wl_create_ns", create)
    s.now_ns, s.drain_cycle_ns = 0, 1
    return s


def steps(s, table, hashes=None):
    """table: [(record, after_ns, podset row, remaining)] in record order"""
    W = len(s.arrays["wl_cq"])
    start = np.zeros(W + 1, np.int64)
    for w, _, _, _ in table:
        start[w + 1] += 1
    s.set("wl_rc_start", np.cumsum(start)); s.set("rc_after_ns", [t for _, t, _, _ in table])
    s.set("rc_ps", [p for _, _, p, _ in table]); s.set("rc_remaining", [r for _, _, _, r in table])
    if hashes is not None:
        s.set("rc_sched_hash", hashes)
    return s


def lists(x):
    return [v.tolist() for v in x]


# ---------------------------------------------------------------- the reference's cases, transcribed
def podsets_case(n_podsets, prio, create, nominal=3, run_ns=1000):
    """the reference's preemption-cq (scheduler_test.go:185-193): nominal 3 cpu, withinClusterQueue LowerPriority,
    BestEffortFIFO; record w has n_podsets[w] podsets of one 1-cpu pod, priority prio[w], created at create[w]"""
    W = len(n_podsets)
    s = cq_case([1] * W, [1] * W, nominal=nominal, run_ns=run_ns, strategy=BE, create=create)
    P = int(sum(n_podsets))
    s.set("wl_ps_start", np.concatenate([[0], np.cumsum(n_podsets)])); s.set("ps_req", np.ones((P, 1)))
    s.set("ps_req_mask", np.ones(P)); s.set("ps_count", np.ones(P))
    s.set("wl_priority", prio); s.set("cq_within_cq", [abi.POLICY_LOWER_PRIORITY])
    return s


def dynamically_reclaimed():
    """scheduler_test.go:458 "Should admit workloads when resources are dynamically reclaimed": first-wl (podsets first,
    second, third of one 1-cpu pod) is admitted and reclaims `third` (at 5); second-wl (the same shape, priority 100,
    created at 10) preempts it; first-wl is requeued asking only for its 2 remaining pods
    (totalRequestsFromPodSets / podSetsCountsAfterReclaim) and is admitted again once second-wl reclaims `first` and
    `second` (10 after its run starts at 11)."""
    s = podsets_case([3, 3], [0, 100], [0, 10])
    return steps(s, [(0, 5, 2, 0), (1, 10, 3, 0), (1, 10, 4, 0)])


def test_dynamically_reclaimed():
    r = run(dynamically_reclaimed())
    assert r.wl_evictions.tolist() == [1, 0] and lists(r.evicted)[r.cycle_start_ns.index(10)] == [0]
    assert r.wl_admit_ns.tolist() == [21, 11]  # readmitted at second-wl's reclaim, not at its finish (1011)
    assert r.n_reclaims == 3 and r.cq_generation.tolist() == [2]  # two updates; the replayed step on `third` is a no-op
    assert r.ps_remaining.tolist() == [1, 1, 0, 0, 0, 1]


def gradually_released():
    """scheduler_test.go:506 "Should admit workloads when resources are gradually released": first-wl (three 1-cpu
    podsets) is admitted, second-wl (one 1-cpu podset, created at 10) waits, first-wl reclaims `third` at 20 and
    second-wl is admitted."""
    s = podsets_case([3, 1], [0, 0], [0, 10])
    return steps(s, [(0, 20, 2, 0)])


def test_gradually_released():
    r = run(gradually_released())
    assert r.wl_admit_ns.tolist() == [0, 20] and r.wl_evictions.tolist() == [0, 0]
    assert lists(r.decisions)[r.cycle_start_ns.index(10)] == [abi.DEC_PREEMPT_NO_TARGETS]  # pending until the reclaim
    assert r.n_reclaims == 1 and r.ps_remaining.tolist() == [1, 1, 0, 1] and r.cq_generation.tolist() == [1]


def partial_row(first=3, second=None):
    """workload_test.go:215,299 TestNewInfo "admitted with reclaim" and "... and increased reclaim": a podset of spec
    Count 5 (10m a pod) whose PodSetAssignment has Count 3 and 30m.  ReclaimablePods 2 (remaining 3, at 10): the count
    goes down, the usage stays 30m (remaining >= admCount); ReclaimablePods 3 (remaining 2, at 20): 20m.  A snapshot row
    with ps_adm_* and its run started at 0, that never finishes (the drain ends after the steps)."""
    s = cq_case([5], [10], nominal=100)
    s.now_ns = 5
    s.set("adm_cq", [0]); s.set("adm_priority", [0]); s.set("adm_ts", [0]); s.set("adm_qr_ts", [0]); s.set("adm_uid", [0])
    s.set("adm_evicted", [0]); s.set("adm_use_start", [0, 1]); s.set("adm_use_fr", [0]); s.set("adm_use_qty", [30])
    s.set("cq_usage", [[30]]); s.set("adm_wl", [0]); s.set("adm_run_start_ns", [0])
    s.set("ps_adm_flavor", [[0]]); s.set("ps_adm_count", [3]); s.set("ps_adm_usage", [[30]])
    return steps(s, [(0, 10, 0, first)] + ([(0, 20, 0, second)] if second is not None else []))


def test_partial_row_reclaim():
    r = run(partial_row())  # remaining 3 = admCount: 30m stays
    assert r.n_reclaims == 1 and r.ps_remaining.tolist() == [3] and r.cq_generation.tolist() == [1]
    assert r.cq_usage.tolist() == [[30]] and r.adm["adm_use_qty"].tolist() == [30] and r.end_ns == 10
    r = run(partial_row(second=2))  # remaining 2 < admCount: 30m / 3 * 2
    assert r.n_reclaims == 2 and r.ps_remaining.tolist() == [2] and r.cq_generation.tolist() == [2]
    assert r.cq_usage.tolist() == [[20]] and r.adm["adm_use_qty"].tolist() == [20] and r.end_ns == 20
    r = run(partial_row(first=4, second=3))  # both steps at or above admCount: the counts go down, the usage stays
    assert r.n_reclaims == 2 and r.cq_usage.tolist() == [[30]] and r.ps_remaining.tolist() == [3]


# ---------------------------------------------------------------- hand-derived schedules
def shared_cell():
    """two podsets of one record on one flavor-resource cell: each step moves that one cell"""
    s = cq_case([2, 1], [3, 4])
    s.set("wl_ps_start", [0, 2, 3]); s.set("ps_req", [[6], [4], [4]]); s.set("ps_req_mask", [1, 1, 1]); s.set("ps_count", [2, 2, 1])
    s.set("wl_cq", [0, 0])
    return steps(s, [(0, 5, 0, 1), (0, 5, 1, 0)])


def test_two_podsets_share_a_cell():
    r = run(shared_cell())
    assert r.n_reclaims == 2 and r.cq_generation.tolist() == [1]  # one instant, one update
    assert lists(r.admitted) == [[0], [], [1]] and r.ps_remaining.tolist() == [1, 0, 1]


def cohort_borrower():
    """a reclaim in one ClusterQueue lets the other's borrower in"""
    s = cq_case([4, 1], [2, 14], Q=2, wl_cq=[0, 1], cohort=True, strategy=BE)
    return steps(s, [(0, 7, 0, 1)])


def test_reclaim_lets_a_cohort_borrower_in():
    r = run(cohort_borrower())
    assert lists(r.admitted)[-1] == [1] and r.cycle_start_ns[-1] == 7 and r.n_reclaims == 1


def outdated_head():
    """BestEffortFIFO: the pending head is set aside after NoFit; the generation bump and the requeue bring it back"""
    return steps(cq_case([4, 1, 1], [2, 7, 9], strategy=BE), [(0, 6, 0, 1)])


def test_generation_bump_requeues_the_pending_head():
    r = run(outdated_head())
    # both heads were set aside (NoFit, no flavor left); the update at 6 requeues the tree and the 7-cpu head fits
    # then, not at the holder's finish (100)
    assert r.cycle_start_ns[:3] == [0, 1, 6] and lists(r.admitted)[:3] == [[0], [], [1]] and r.wl_admit_ns[1] == 6
    assert r.n_reclaims == 1 and r.cq_generation.tolist() == [1]


def at_finish():
    """a step at the finish time is dropped"""
    return steps(cq_case([4], [2], run_ns=50), [(0, 50, 0, 1)])


def test_step_at_finish_is_dropped():
    r = run(at_finish())
    assert r.n_reclaims == 0 and r.ps_remaining.tolist() == [4] and r.cq_generation.tolist() == [0]


def evicting():
    """a step on a row whose preemption is issued is dropped (eviction latency 20, issued at 3): the record's step
    applies only in its next run"""
    s = cq_case([4, 1], [2, 8], strategy=BE)
    s.set("wl_priority", [0, 10]); s.set("cq_within_cq", [abi.POLICY_LOWER_PRIORITY]); s.set("wl_evict_ns", [20, 20])
    s.set("wl_create_ns", [0, 3])
    return steps(s, [(0, 10, 0, 1)])


def test_step_on_evicting_row_is_dropped():
    r = run(evicting())
    k = [i for i, x in enumerate(r.reclaims) if len(x)]
    assert r.n_evicted == 1 and r.n_reclaims == 1 and r.wl_admit_ns[0] >= 23
    assert len(k) == 1 and r.cycle_start_ns[k[0]] >= r.wl_admit_ns[0]


def same_boundary():
    """a step in the boundary of its row's admission (cycle 0, 10 ns a cycle) and one in the boundary of a Ready verdict
    (StrictFIFO: the second record is admitted in cycle 1 at 10, Ready at 13, its step at 15)"""
    s = cq_case([4, 4], [1, 1], nominal=10)
    s.drain_cycle_ns = 10
    s.set("wl_check_ns", [0, 3]); s.set("wl_check_fail", [0, 0])
    return steps(s, [(0, 4, 0, 2), (1, 2, 1, 1)])


def test_steps_in_the_admission_and_verdict_boundary():
    r = run(same_boundary())
    assert lists(r.reclaims)[:2] == [[0], [1]] and r.ps_remaining.tolist() == [2, 1]


def readmission():
    """a preempted row is readmitted: its steps replay from the first, those at or above the count change nothing"""
    s = cq_case([4, 1], [2, 7], strategy=BE, run_ns=[100, 5])
    s.set("wl_priority", [0, 10]); s.set("cq_within_cq", [abi.POLICY_LOWER_PRIORITY]); s.set("wl_create_ns", [0, 20])
    return steps(s, [(0, 3, 0, 2), (0, 30, 0, 1)])


def test_readmission_replays_steps():
    r = run(readmission())
    assert r.wl_evictions.tolist() == [1, 0] and r.n_reclaims == 2 and r.ps_remaining.tolist() == [1, 1]


def afs_decay():
    s = cq_case([4], [2], nominal=20, strategy=BE)
    s.set("wl_lq", [0]); s.set("lq_cq", [0]); s.set("cq_afs", [1]); s.set("lq_weight", [1.0])
    s.set("lq_consumed", [[0]]); s.set("lq_consumed_scale", [[0]]); s.set("afs_res_weight", [1.0]); s.set("afs_milli_mul", [1000])
    s.set("lq_last_update_ns", [0]); s.set("adm_lq", np.zeros(0))
    s.afs_half_life_ns, s.afs_sampling_ns, s.afs_alpha = 10, 10, 0.5
    return steps(s, [(0, 15, 0, 1)])


def test_afs_decay_with_a_shrinking_admitted_usage():
    """one LocalQueue, alpha 0.5 a sample: wl0 (4 pods x 2 cpu) is admitted at 0 (consumed 0 + entry penalty 4000m).
    The sample at 10 sees 8 cpu admitted: 2000 + 4000 = 6000m.  The step at 15 leaves 1 pod: 2 cpu admitted from then
    on, so the samples at 20 .. 100 halve towards 2000m: 4000, 3000, 2500, 2250, 2125, 2062, 2031, 2015, 2007 (each
    term truncated to whole milli-units).  The completion at 100 comes after that boundary's sample."""
    r = run(afs_decay())
    assert r.n_reclaims == 1 and r.end_ns == 100
    assert r.lq_consumed.tolist() == [[2007]] and r.lq_consumed_scale.tolist() == [[-3]]


def step_and_stop():
    """a step and a stop of the same record at one instant: the step goes first"""
    s = steps(cq_case([4], [2]), [(0, 6, 0, 1)])
    s.set("ac_ns", [6]); s.set("ac_wl", [0]); s.set("ac_active", [0])
    return s


def test_step_and_stop_at_one_instant():
    r = run(step_and_stop())
    assert r.n_reclaims == 1 and r.n_stopped == 1 and r.ps_remaining.tolist() == [1] and r.cq_usage.tolist() == [[0]]


def hashes(with_table):
    """the scheduling hash after a step decides where the record goes when it re-enters its queue.  wl0 (4 pods x 1
    cpu, hash 5) and h (5 cpu) are admitted; wl0 reclaims 1 pod 2 after its start (hash 11 with the table, 0 without)
    and is stopped at 3.  w2 (11 cpu, above the nominal quota, hash 11, created at 4) goes NoFit: 11 joins the ClusterQueue's NoFit set.  wl0 is
    resumed at 10 asking 3 cpu: with hash 11 it goes straight to the inadmissible set (PushOrUpdate,
    cluster_queue.go:288-293) and waits for h's finish at 101; with hash 0 it is queued and admitted at once."""
    s = cq_case([4, 1, 1], [1, 5, 11], strategy=BE, create=[0, 0, 4])
    s.set("wl_sched_hash", [5, 0, 11])
    s.set("ac_ns", [3, 10]); s.set("ac_wl", [0, 0]); s.set("ac_active", [0, 1])
    return steps(s, [(0, 2, 0, 3)], hashes=[11] if with_table else None)


@pytest.mark.parametrize("with_table", [False, True])
def test_sched_hash_after_a_step(with_table):
    r = run(hashes(with_table))
    assert r.n_reclaims == 1 and r.n_stopped == 1 and r.n_resumed == 1 and r.ps_remaining.tolist() == [3, 1, 1]
    assert int(r.wl_admit_ns[0]) == (int(r.wl_finish_ns[1]) if with_table else 10)


# ---------------------------------------------------------------- equivalence, invariants, refusals
def _cfg3():
    return synth.add_events(synth.make_snapshot(3, W=1200, Q=40), seed=2)


def _cfg4():
    return synth.add_events(synth.make_snapshot(4, W=1000, Q=24, preemption=True, evictable=True), seed=3)


def _no_steps(s):
    s.finalize()
    if "adm_wl" not in s.arrays:
        s.set("adm_wl", np.zeros(0))
    s.set("wl_rc_start", np.zeros(s.n_wl + 1)); s.set("rc_after_ns", []); s.set("rc_ps", []); s.set("rc_remaining", [])
    return s


@pytest.mark.parametrize("mk", [_cfg4, lambda: synth.perf_scenario(0.02)])
def test_no_steps_is_no_block(mk):
    base, got = mk(), _no_steps(mk())
    if "adm_wl" not in base.arrays:
        base.set("adm_wl", np.zeros(0))
    a, b = run(base, 400), run(got, 400)
    assert lists(a.heads) == lists(b.heads) and lists(a.decisions) == lists(b.decisions)
    assert a.cycle_start_ns == b.cycle_start_ns and np.array_equal(a.cq_usage, b.cq_usage) and b.n_reclaims == 0
    assert np.array_equal(b.ps_remaining, base.arrays["ps_count"])


@pytest.mark.parametrize("seed", [1, 2])
def test_seeded_invariants(seed):
    s = synth.perf_scenario(0.02, reclaim=seed)
    spec = s.arrays["ps_count"].copy()
    r = run(s)
    assert r.n_reclaims > 0 and (r.ps_remaining <= spec).all() and (r.ps_remaining >= 0).all()
    usage = np.zeros_like(r.cq_usage)
    for row in range(len(r.adm["adm_cq"])):
        for k in range(int(r.adm["adm_use_start"][row]), int(r.adm["adm_use_start"][row + 1])):
            usage[r.adm["adm_cq"][row], r.adm["adm_use_fr"][k]] += r.adm["adm_use_qty"][k]
    assert np.array_equal(usage, r.cq_usage)


def _refusal_case():
    return partial_row(second=2)


REFUSALS = {
    "no-adm-wl": (lambda s: s.arrays.pop("adm_wl") and None, "the tables need adm_wl"),
    "csr": (lambda s: s.set("wl_rc_start", [0, 3]), "not a CSR"),
    "ps-outside": (lambda s: s.set("rc_ps", [1, 0]), "rc_ps outside its record"),
    "after": (lambda s: s.set("rc_after_ns", [10, 5]), "rc_after_ns <= 0 or decreasing"),
    "remaining": (lambda s: s.set("rc_remaining", [2, 3]), "rc_remaining negative or increasing"),
    "divisible": (lambda s: s.set("ps_req", [[31]]), "not divisible"),
    "run-start-late": (lambda s: s.set("adm_run_start_ns", [6]), "adm_run_start_ns after now_ns"),
    "run-start-idle": (lambda s: s.set("adm_evicted", [1]), "on a row that is not running"),
    "missing-adm": (lambda s: s.arrays.pop("ps_adm_usage") and None, "ps_adm_* missing"),
    "cells": (lambda s: s.set("ps_adm_usage", [[33]]), "do not add up"),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_host_definition_refuses_bad_tables(name):
    s = _refusal_case()
    if name == "ps-outside":
        s.set("ps_count", [3]); s.set("rc_ps", [1, 0])
    REFUSALS[name][0](s)
    s.finalize()
    with pytest.raises(ValueError, match=REFUSALS[name][1].replace("*", r"\*")):
        check_reclaims(s)


def test_partially_admissible_record_is_unsupported():
    s = _refusal_case()
    s.set("ps_min_count", [1]); s.finalize()
    with pytest.raises(ReclaimUnsupported):
        check_reclaims(s)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _cfg4_reclaim():
    s = synth.make_snapshot(4, W=1000, Q=24, preemption=True, evictable=True)
    s.set("ps_count", np.full(s.n_podset, 2)); s.set("ps_req", s.arrays["ps_req"] * 2)
    s.flags &= ~abi.F_PARTIAL_ADMISSION
    return synth.add_reclaims(synth.add_events(s, seed=3), seed=8)


def _cfg3_reclaim():
    s = synth.make_snapshot(3, W=1200, Q=40)
    s.set("ps_count", np.full(s.n_podset, 3)); s.set("ps_req", s.arrays["ps_req"] * 3)
    s.flags &= ~abi.F_PARTIAL_ADMISSION
    return synth.add_reclaims(synth.add_events(s, seed=2), seed=9)


CPU_CASES = {
    "dynamically-reclaimed": dynamically_reclaimed, "gradually-released": gradually_released,
    "partial-row": lambda: partial_row(), "partial-row-increased": lambda: partial_row(second=2), "shared-cell": shared_cell,
    "cohort-borrower": cohort_borrower, "outdated-head": outdated_head, "at-finish": at_finish, "evicting": evicting,
    "same-boundary": same_boundary, "readmission": readmission, "afs-decay": afs_decay, "step-and-stop": step_and_stop,
    "hash-null": lambda: hashes(False), "hash-set": lambda: hashes(True),
}
DEVICE_CASES = dict(CPU_CASES)
DEVICE_CASES.update({
    "cfg3": _cfg3_reclaim, "cfg4": _cfg4_reclaim, "baseline": lambda: synth.perf_scenario(0.1, reclaim=5),
    "baseline-all-blocks": lambda: synth.perf_scenario(0.1, evict_ns=30_000_000, checks=7, pods_ready=9, max_exec=3, quota=11,
                                                       active=5, reclaim=5),
})


def compare(want, got):
    assert got.n_cycles == want.cycles and got.n_decisions == want.n_decisions
    cyc = got.cycles()
    for k in range(want.cycles):
        assert np.array_equal(cyc[k][0], want.heads[k]), k
        assert np.array_equal(cyc[k][1], want.decisions[k]), k
        assert int(got.cycle_start_ns[k]) == want.cycle_start_ns[k], k
        assert int(got.cycle_admitted[k]) == len(want.admitted[k]), k
        assert int(got.cycle_evicted[k]) == len(want.evicted[k]), k
        assert int(got.cycle_finished[k]) == len(want.finished[k]), k
        assert int(got.cycle_reclaims[k]) == len(want.reclaims[k]), k
    assert got.n_reclaims == want.n_reclaims and got.end_ns == want.end_ns and got.n_finished == want.n_finished
    for f in ("wl_admit_ns", "wl_finish_ns", "wl_evictions", "wl_admit_cycle", "cq_usage", "cq_generation"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    assert np.array_equal(got.ps_remaining_out, want.ps_remaining)
    if want.lq_consumed is not None:
        assert np.array_equal(got.lq_consumed, want.lq_consumed)
    if want.wl_deactivated is not None:
        assert np.array_equal(got.wl_deactivation_reason, want.wl_deactivation_reason)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DEVICE_CASES))
def test_kb_run_drain_reclaims_like_the_host_definition(name):
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = DEVICE_CASES[name]()
        mc = 100_000 if name.startswith("baseline") else 400
        want = run(snap, mc)
        got = ev.run_drain(snap, abi.DrainOut(snap, mc, trace_capacity=want.n_decisions))
        compare(want, got)
        if name.startswith(("cfg", "baseline")):
            assert got.n_reclaims > 0
    finally:
        ev.close()


@pytest.fixture
def evaluator():
    from kueue_b200 import native
    ev = native.Evaluator(0)
    yield ev
    ev.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REFUSALS))
def test_kb_run_drain_refuses_bad_tables(evaluator, name):
    from kueue_b200 import native
    s = _refusal_case()
    if name == "ps-outside":
        s.set("ps_count", [3])
    REFUSALS[name][0](s)
    s.finalize()
    st = s.as_struct()
    out = abi.DrainOut(s, 5)
    rc = native.lib().kb_run_drain(evaluator._h, C.byref(st), C.byref(out.struct))
    assert rc == abi.KB_ERR_INVALID and REFUSALS[name][1] in native.lib().kb_last_error(evaluator._h).decode()


@pytest.mark.gpu
def test_kb_run_drain_refuses_partially_admissible_records(evaluator):
    from kueue_b200 import native
    s = _refusal_case()
    s.set("ps_min_count", [1]); s.finalize()
    st = s.as_struct()
    out = abi.DrainOut(s, 5)
    rc = native.lib().kb_run_drain(evaluator._h, C.byref(st), C.byref(out.struct))
    assert rc == abi.KB_ERR_UNSUPPORTED and "partially admitted" in native.lib().kb_last_error(evaluator._h).decode()
