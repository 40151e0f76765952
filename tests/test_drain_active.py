"""Workload deactivation and reactivation in the drain's event mode (kb_snapshot.ac_ns, ac_wl, ac_active, wl_inactive;
kueue_b200/drain.py).  A stop (spec.active false) takes a workload out of its queue, or takes its row's quota at once;
a resume returns a deactivated workload to its queue.  CPU: the reference's test cases transcribed as hand-derived
schedules on the oracle, hand-derived schedules for the interactions with the other blocks, the equivalence without
edits and the refusals.  GPU: kb_run_drain equals the host definition cycle by cycle, alone and with every other event
block, and refuses bad tables."""
import ctypes as C

import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from kueue_b200.drain import ALL_FAIL, DEACTIVATED, FINISHED, HELD, QUEUED, USER, check_active_changes, drain

N_, PN_, P_, A_ = abi.DEC_NOFIT, abi.DEC_PREEMPT_NO_TARGETS, abi.DEC_PREEMPTING, abi.DEC_ASSUMED
BE, STRICT = abi.QUEUE_BEST_EFFORT_FIFO, abi.QUEUE_STRICT_FIFO


def run(snap, max_cycles=100_000, run_cycle=None):
    snap.finalize()
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000
    return drain(snap, run_cycle or (lambda s: oracle.run_cycle(s, cap)), max_cycles=max_cycles)


def edits(snap, table):
    """table: [(time, record, active)]"""
    snap.set("ac_ns", [t for t, _, _ in table]); snap.set("ac_wl", [w for _, w, _ in table])
    snap.set("ac_active", [on for _, _, on in table])
    return snap


def one_cq(cpu, held=(), prio=None, strategy=BE, nominal=10, within=None, evict_ns=None):
    """one ClusterQueue with `nominal` cpu; record w asks cpu[w] and is created at 0 with timestamp w; the records in
    `held` hold rows admitted at 0.  One cycle takes 1 ns."""
    W = len(cpu)
    prio = [0] * W if prio is None else prio
    s = abi.FlatSnapshot(n_cq=1, n_cohort=0, n_flavor=1, n_resource=1)
    s.set("parent", [-1]); s.set("nominal", [[nominal]])
    s.set("cq_rg_start", [0, 1]); s.set("rg_res_mask", [1]); s.set("rg_flavor_start", [0, 1]); s.set("rg_flavors", [0])
    s.set("cq_strategy", [strategy])
    if within is not None:
        s.set("cq_within_cq", [within])
    s.set("wl_cq", np.zeros(W)); s.set("wl_priority", prio); s.set("wl_uid", np.arange(W)); s.set("wl_ts", np.arange(W))
    s.set("ps_req", np.asarray(cpu)[:, None]); s.set("ps_req_mask", np.ones(W))
    _rows(s, held, [0] * len(held), prio, cpu, 1)
    if evict_ns is not None:
        s.set("wl_evict_ns", np.full(W, evict_ns))
    s.now_ns, s.drain_cycle_ns = 0, 1
    return s


def _rows(s, held, cqs, prio, cpu, Q):
    n = len(held)
    s.set("adm_cq", cqs); s.set("adm_priority", [prio[w] for w in held]); s.set("adm_ts", list(held))
    s.set("adm_qr_ts", np.zeros(n)); s.set("adm_uid", list(held)); s.set("adm_evicted", np.zeros(n))
    s.set("adm_use_start", np.arange(n + 1)); s.set("adm_use_fr", np.zeros(n)); s.set("adm_use_qty", [cpu[w] for w in held])
    usage = np.zeros((Q, 1), np.int64)
    for q, w in zip(cqs, held):
        usage[q, 0] += cpu[w]
    s.set("cq_usage", usage); s.set("adm_wl", list(held))


def lists(x):
    return [v.tolist() for v in x]


# ---------------------------------------------------------------- the reference's cases, transcribed
def test_deactivated_pending_workload():
    """workload_controller_test.go:1450 "should set the Evicted condition with Deactivated reason when the
    .spec.active=False": a pending workload (StrictFIFO head that does not fit) is stopped at 3.  It leaves its queue,
    DEACTIVATED with reason 4; its queue-order timestamp stays the creation time; the drain then has nothing to run."""
    s = edits(one_cq([20], strategy=STRICT), [(3, 0, 0)])
    r = run(s)
    assert r.cycle_start_ns == [0] and lists(r.decisions) == [[N_]]
    assert r.state.tolist() == [DEACTIVATED] and r.wl_deactivation_reason.tolist() == [USER] and r.wl_deactivated.tolist() == [1]
    assert lists(r.stopped) == [[0]] and r.n_stopped == 1 and r.n_active_changes == 1 and r.end_ns == 3


def test_deactivated_admitted_workload():
    """workload_controller_test.go:1468 "...when the .spec.active=False and Admitted": the admitted row of record 0 is
    stopped at 4 while record 1 waits set aside (Preempt without targets); its cells leave the usage at 4 (the `!active`
    branch deletes it from the cache at once), the record is DEACTIVATED with reason 4, and record 1 is admitted at 4.
    (:1500 differs only by an Evicted=False condition, which the drain does not carry: the same schedule.)"""
    r = run(edits(one_cq([10, 10], held=[0]), [(4, 0, 0)]))
    assert r.cycle_start_ns == [0, 4] and lists(r.heads) == [[1], [1]] and lists(r.decisions) == [[PN_], [A_]]
    assert r.state.tolist() == [DEACTIVATED, HELD] and r.cq_usage.tolist() == [[10]]
    assert r.wl_deactivation_reason.tolist() == [USER, 0] and r.adm["adm_wl"].tolist() == [1]


def test_requeued_on_reactivation():
    """workload_controller_test.go:1262 "should set the WorkloadRequeued condition to true on re-activated": a record
    deactivated before the drain (wl_inactive 4) is resumed at 2; it joins its queue and is admitted at 2."""
    s = one_cq([5])
    s.set("wl_inactive", [USER])
    r = run(edits(s, [(2, 0, 1)]))
    assert r.cycle_start_ns == [2] and lists(r.decisions) == [[A_]] and r.n_resumed == 1 and r.n_stopped == 0
    assert r.state.tolist() == [HELD] and r.wl_deactivated.tolist() == [0]


def _pods_ready(s, limit=-1):
    s.set("wl_pods_ready_ns", np.full(s.n_wl, 10)); s.set("wl_pods_ready_fail", np.full(s.n_wl, ALL_FAIL))
    s.pods_ready_timeout_ns, s.pods_ready_backoff_base_s, s.pods_ready_backoff_max_s = 5, 1, 0
    s.pods_ready_backoff_limit = limit
    return s


def test_clear_requeue_state_after_deactivation():
    """integration workload_controller_test.go:169 "should clear workload requeue state after deactivation": a workload
    whose pods never get ready times out at 5 (Count 1, RequeueAt 5 + 1 s) and waits in BACKOFF; the stop at 7 clears
    RequeueState (Count 0, no RequeueAt): it is DEACTIVATED and never requeued."""
    s = _pods_ready(one_cq([5]))
    r = run(edits(s, [(7, 0, 0)]))
    assert r.cycle_start_ns == [0] and lists(r.pods_ready_timeout) == [[0]] and lists(r.stopped) == [[0]]
    assert r.state.tolist() == [DEACTIVATED] and r.wl_pods_ready_count.tolist() == [0] and r.end_ns == 7


def test_podsready_reactivation_restarts_the_count():
    """scheduler/podsready/scheduler_test.go:292 "...After that re-activating a workload": the pods never get ready
    (timeout 5, backoff 1 s, limit 1).  Admitted at 0, timed out at 5 (Count 1, BACKOFF until 5 + 1 s); stopped at 6
    (Count 0); resumed at 8 and admitted at 8; the next timeout at 13 leaves Count 1, not 2 (no deactivation), and
    the record is admitted again after its 1 s backoff."""
    s = _pods_ready(one_cq([5]), limit=1)
    r = run(edits(s, [(6, 0, 0), (8, 0, 1)]), max_cycles=3)
    assert r.cycle_start_ns == [0, 8, 1_000_000_013] and lists(r.decisions) == [[A_], [A_], [A_]]
    assert lists(r.pods_ready_timeout) == [[0], [0], []] and r.n_pods_ready_deactivated == 0
    assert r.wl_pods_ready_count.tolist() == [1] and r.state.tolist() == [HELD] and r.wl_deactivated.tolist() == [0]


# ---------------------------------------------------------------- hand-derived schedules
def _checks(s):
    s.set("wl_check_ns", [5] + [0] * (s.n_wl - 1)); s.set("wl_check_fail", [1] + [0] * (s.n_wl - 1))
    s.check_backoff_base_s, s.check_backoff_max_s, s.check_backoff_limit = 1, 8, 3
    return s


TIES = {  # a stop at the time of the record's own event that puts it in BACKOFF: the event first, then the stop
    "stop-at-pods-ready-timeout": lambda: edits(_pods_ready(one_cq([5, 20], strategy=STRICT)), [(5, 0, 0)]),
    "stop-at-check-retry": lambda: edits(_checks(one_cq([5, 20], strategy=STRICT)), [(5, 0, 0)]),
}


@pytest.mark.parametrize("name", list(TIES))
def test_stop_at_the_time_of_an_own_event(name):
    """record 0 (5 cpu) is admitted at 0 and its PodsReady timeout (or its check's Retry verdict) comes at 5, the time
    of its stop; record 1 (20 cpu, StrictFIFO) never fits.  The own event comes first: a timeout (or Retry) puts the
    record in BACKOFF until 5 + 1 s and counts; the stop then deactivates it and clears its RequeueAt, so nothing is
    left to wake the clock: the drain ends at 5 after the quiet cycle there."""
    r = run(TIES[name]())
    assert r.cycle_start_ns == [0, 1, 5] and lists(r.decisions) == [[A_], [N_], [N_]] and r.end_ns == 5
    assert lists(r.stopped) == [[], [0], []] and r.state.tolist() == [DEACTIVATED, QUEUED]
    if name == "stop-at-pods-ready-timeout":
        assert lists(r.pods_ready_timeout) == [[], [0], []] and r.wl_pods_ready_count.tolist() == [0, 0]
    else:
        assert lists(r.check_retry) == [[], [0], []] and r.wl_check_retries.tolist() == [1, 0]


def test_stopped_head_lets_the_next_in():
    """StrictFIFO: record 0 (20 cpu) never fits and keeps the head; record 1 (5 cpu) waits behind it.  The stop at 5
    takes the head out: record 1 is admitted at 5.  The resume at 7 returns record 0, NoFit again, and the drain ends."""
    s = edits(one_cq([20, 5], strategy=STRICT), [(5, 0, 0), (7, 0, 1)])
    r = run(s)
    assert r.cycle_start_ns == [0, 5, 7] and lists(r.heads) == [[0], [1], [0]] and lists(r.decisions) == [[N_], [A_], [N_]]
    assert lists(r.stopped) == [[0], [], []] and lists(r.resumed) == [[], [0], []]
    assert r.state.tolist() == [QUEUED, HELD] and r.wl_deactivated.tolist() == [0, 0]


def cohort_case():
    """cq0 (0) and cq1 (1), 5 cpu each, in one cohort (2); record 0 of cq0 holds 10 cpu (5 borrowed from cq1).  Record
    1 (5 cpu) of cq1 does not fit (no preemption policy: Preempt without targets) and is set aside.  Record 0 is stopped at 3."""
    s = abi.FlatSnapshot(n_cq=2, n_cohort=1, n_flavor=1, n_resource=1)
    s.set("parent", [2, 2, -1]); s.set("nominal", [[5], [5], [0]])
    s.set("cq_rg_start", [0, 1, 2]); s.set("rg_res_mask", [1, 1]); s.set("rg_flavor_start", [0, 1, 2]); s.set("rg_flavors", [0, 0])
    s.set("cq_strategy", [BE, BE])
    s.set("wl_cq", [0, 1]); s.set("wl_priority", [0, 0]); s.set("wl_uid", [0, 1]); s.set("wl_ts", [0, 1])
    s.set("ps_req", [[10], [5]]); s.set("ps_req_mask", [1, 1])
    _rows(s, [0], [0], [0, 0], [10, 5], 2)
    s.now_ns, s.drain_cycle_ns = 0, 1
    return edits(s, [(3, 0, 0)])


def test_stopped_row_frees_quota_in_the_cohort():
    """t=0: record 1 is set aside; quiet, wait for the stop.  At 3 the row's cells leave the usage and the
    cohort is requeued: record 1 is admitted at 3 on its own nominal quota."""
    r = run(cohort_case())
    assert r.cycle_start_ns == [0, 3] and lists(r.heads) == [[1], [1]] and lists(r.decisions) == [[PN_], [A_]]
    assert r.cq_usage.tolist() == [[0], [5]] and r.state.tolist() == [DEACTIVATED, HELD]


def evicting_target_case(stop_at=4, sticky=False):
    """record 0 (priority 0) holds all 10 cpu; record 1 (priority 1, 10 cpu) preempts it (withinClusterQueue
    LowerPriority); every eviction takes 10 ns."""
    s = one_cq([10, 10], held=[0], prio=[0, 1], within=abi.POLICY_LOWER_PRIORITY, evict_ns=10)
    if sticky:
        s.set("cq_sticky", [-1])
    return s


def test_stop_a_preemption_target_while_it_evicts():
    """t=0: record 1 preempts record 0 (its eviction ends at 10); t=1: the target is already evicting, quiet, wait for
    the stop at 4.  The stop takes the evicting row's cells at 4 (not at 10) and deactivates record 0: record 1 is
    admitted at 4, and no eviction completes."""
    r = run(edits(evicting_target_case(), [(4, 0, 0)]))
    assert r.cycle_start_ns == [0, 1, 4] and lists(r.decisions) == [[P_], [P_], [A_]]
    assert lists(r.evicted) == [[0], [], []] and r.n_evict_done == 0 and lists(r.stopped) == [[], [0], []]
    assert r.state.tolist() == [DEACTIVATED, HELD] and r.cq_usage.tolist() == [[10]]


def test_stop_the_sticky_workload():
    """with the sticky table: record 1 preempts at 0 and becomes the sticky workload; the stop at 2 clears the slot and
    deactivates it.  At 10 the eviction completes and record 0, back in its queue, is admitted again."""
    r = run(edits(evicting_target_case(sticky=True), [(2, 1, 0)]))
    assert r.cycle_start_ns == [0, 1, 10] and lists(r.decisions) == [[P_], [P_], [A_]] and lists(r.heads)[2] == [0]
    assert r.cq_sticky.tolist() == [-1] and r.state.tolist() == [HELD, DEACTIVATED] and r.n_evict_done == 1


def test_stop_and_resume_inside_one_boundary():
    """record 0 holds 10 cpu, record 1 (StrictFIFO, 20 cpu) never fits.  Record 0 is stopped and resumed at 3 and record
    1 likewise at 3: record 0's row goes at 3 and it returns to its queue behind record 1 (timestamps 0 < 1: it is the
    head), readmitted at 3; record 1 is stopped and resumed without leaving the queue's order."""
    s = edits(one_cq([10, 20], held=[0], strategy=STRICT), [(3, 0, 0), (3, 1, 0), (3, 0, 1), (3, 1, 1)])
    r = run(s)
    assert r.cycle_start_ns == [0, 3, 4] and lists(r.heads) == [[1], [0], [1]] and lists(r.decisions) == [[N_], [A_], [N_]]
    assert r.n_stopped == 2 and r.n_resumed == 2 and lists(r.active_changes) == [[0, 1, 2, 3], [], []]
    assert r.state.tolist() == [HELD, QUEUED] and r.wl_deactivated.tolist() == [0, 0] and r.wl_admit_ns.tolist()[0] == 3


def test_noop_edits():
    """record 0 (5 cpu, runs 2 ns) is admitted at 0; at 1 a resume of it (active, holding a row) changes nothing and a
    stop deactivates record 1; at 3 a stop of the FINISHED record 0 and a second stop of record 1 change nothing.  All
    four count as applied, the jumps after cycle 0 count in it."""
    s = one_cq([5, 20], strategy=STRICT)
    s.set("wl_run_ns", [2, -1])
    r = run(edits(s, [(1, 0, 1), (1, 1, 0), (3, 0, 0), (3, 1, 0)]))
    assert r.n_active_changes == 4 and r.n_stopped == 1 and r.n_resumed == 0 and lists(r.stopped) == [[1]]
    assert r.state.tolist() == [FINISHED, DEACTIVATED]


def test_max_exec_accumulates_at_the_stop():
    """MaximumExecutionTimeSeconds: a row admitted at 0 (limit 100 s) with 2 s of termination latency is stopped at
    3 s: acc = 3 + 2 = 5 s (the QuotaReserved unset after the pods are gone), not reset; the quota goes at 3 s and
    record 1 is admitted then.  It later runs out its own 100 s: MaximumExecutionTimeExceeded (reason 3)."""
    S = 1_000_000_000
    s = one_cq([10, 10], evict_ns=2 * S)
    s.set("adm_wl", np.zeros(0)); s.set("wl_max_exec_s", [100, 100]); s.drain_cycle_ns = S
    r = run(edits(s, [(3 * S, 0, 0)]))
    assert r.wl_admit_ns.tolist() == [0, 3 * S]
    assert r.wl_exec_acc_s.tolist()[0] == 5 and r.wl_deactivation_reason.tolist() == [USER, 3]


# ---------------------------------------------------------------- rule 7 and seeded drains
def _cfg3():
    return synth.add_events(synth.make_snapshot(3, W=1200, Q=40), seed=2)


def _cfg4():
    return synth.add_evict_latency(synth.add_events(synth.make_snapshot(4, W=800, Q=40, tight=1.6, evictable=True), seed=3),
                                   (3_000, 40_000), seed=4)


@pytest.mark.parametrize("mk", [_cfg3, _cfg4])
def test_no_edits_no_inactive_is_no_block(mk):
    plain = mk()
    if "adm_wl" not in plain.arrays:
        plain.set("adm_wl", np.zeros(0))
    blk = mk()
    if "adm_wl" not in blk.arrays:
        blk.set("adm_wl", np.zeros(0))
    edits(blk, []); blk.set("wl_inactive", np.zeros(blk.n_wl))
    want, got = run(plain, 400), run(blk, 400)
    assert got.cycles == want.cycles and got.cycle_start_ns == want.cycle_start_ns and got.end_ns == want.end_ns
    for k in range(want.cycles):
        assert np.array_equal(got.heads[k], want.heads[k]) and np.array_equal(got.decisions[k], want.decisions[k]), k
        assert np.array_equal(got.evicted[k], want.evicted[k]) and np.array_equal(got.finished[k], want.finished[k]), k
    for f in ("cq_usage", "state", "wl_admit_ns", "wl_finish_ns", "wl_evictions", "wl_admit_cycle"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    assert not got.wl_deactivated.any() and got.n_active_changes == 0


@pytest.mark.parametrize("mk", [_cfg3, _cfg4])
def test_seeded_invariants(mk):
    """every stopped record ends inactive unless resumed later; usage never negative; a DEACTIVATED record holds no row"""
    s = synth.add_active_changes(mk(), seed=5, inactive_share=0.05)
    r = run(s, 400)
    assert r.n_stopped > 0 and r.n_resumed > 0 and (r.cq_usage >= 0).all()
    dead = np.flatnonzero(r.state == DEACTIVATED)
    assert not np.isin(dead, r.adm["adm_wl"]).any() and (r.wl_deactivated[dead] == 1).all()
    assert (r.wl_deactivated[r.state != DEACTIVATED] == 0).all()


# ---------------------------------------------------------------- refusals of the host definition
REFUSALS = {
    "missing-table": (lambda s: s.arrays.pop("ac_active"), "a NULL table with n_active_change > 0"),
    "at-now": (lambda s: s.set("ac_ns", [0]), "ac_ns at or before now_ns"),
    "decreasing": (lambda s: edits(s, [(5, 0, 0), (4, 0, 1)]), "ac_ns decreasing"),
    "record-range": (lambda s: s.set("ac_wl", [2]), "ac_wl out of range"),
    "active-value": (lambda s: s.set("ac_active", [2]), "ac_active neither 0 nor 1"),
    "before-create": (lambda s: s.set("wl_create_ns", [5, 0]), "an edit at or before its record's wl_create_ns"),
    "inactive-held": (lambda s: s.set("wl_inactive", [0, 4]), "an inactive start record that adm_wl names"),
    "inactive-absent": (lambda s: (s.set("wl_create_ns", [0, 9]), s.set("wl_inactive", [0, 4]), s.set("adm_wl", np.zeros(0)),
                                   _rows(s, [], [], [0, 0], [10, 10], 1)), "an inactive start record created after now_ns"),
    "inactive-reason": (lambda s: s.set("wl_inactive", [5, 0]), "wl_inactive above 4"),
}


def _refusal_case():
    return edits(one_cq([10, 10], held=[1]).finalize(), [(4, 0, 0)])


@pytest.mark.parametrize("name", list(REFUSALS))
def test_host_definition_refuses_bad_tables(name):
    mutate, msg = REFUSALS[name]
    s = _refusal_case()
    mutate(s)
    with pytest.raises(ValueError) as e:
        check_active_changes(s)
    assert msg in str(e.value)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _with_active(mk, seed=5, **kw):
    def f():
        s = mk()
        if "adm_wl" not in s.arrays and s.n_adm == 0:
            s.set("adm_wl", np.zeros(0))
        return synth.add_active_changes(s, seed=seed, **kw)
    return f


def _cfg2():
    return synth.add_events(synth.make_snapshot(2, W=600, Q=12, preemption=True, tight=1.3, evictable=True), seed=1)


def _checks_pr_mx():
    s = _cfg4()
    synth.add_admission_checks(s, seed=3); synth.add_pods_ready(s, seed=4); synth.add_max_exec(s, seed=5)
    return s


def _afs_decay():
    s = synth.add_events(synth.make_snapshot(3, W=1200, Q=40, afs=3), seed=2)
    s.set("adm_wl", np.zeros(0))
    s.set("lq_last_update_ns", np.full(len(s.arrays["lq_cq"]), s.now_ns)); s.set("adm_lq", np.full(s.n_adm, -1))
    s.afs_half_life_ns, s.afs_sampling_ns, s.afs_alpha = 10 * 1_000_000_000, 1_000_000_000, 0.5 ** 0.1
    return s


def _sticky_quota():
    s = synth.add_quota_changes(_cfg4(), seed=6)
    s.set("cq_sticky", np.full(s.n_cq, -1))
    return s


_S60 = 6_000_000_000  # the baseline scenario at scale 0.1 spans 6 s
CPU_CASES = {
    "pending": lambda: edits(one_cq([20], strategy=STRICT), [(3, 0, 0)]),
    "admitted": lambda: edits(one_cq([10, 10], held=[0]), [(4, 0, 0)]),
    "reactivated": lambda: edits((lambda s: (s.set("wl_inactive", [USER]), s)[1])(one_cq([5])), [(2, 0, 1)]),
    "clear-requeue": lambda: edits(_pods_ready(one_cq([5])), [(7, 0, 0)]),
    "podsready-reactivate": lambda: edits(_pods_ready(one_cq([5]), limit=2), [(6, 0, 0), (8, 0, 1)]),
    "stopped-head": lambda: edits(one_cq([20, 5], strategy=STRICT), [(5, 0, 0), (7, 0, 1)]),
    "cohort": cohort_case,
    "evicting-target": lambda: edits(evicting_target_case(), [(4, 0, 0)]),
    "sticky": lambda: edits(evicting_target_case(sticky=True), [(2, 1, 0)]),
    "stop-at-pods-ready-timeout": TIES["stop-at-pods-ready-timeout"], "stop-at-check-retry": TIES["stop-at-check-retry"],
    # a 10 ns step: the timeout (5) and the Retry verdict (5) come before the stop (7) inside one active boundary
    "stop-after-timeout-in-boundary": lambda: (lambda s: (setattr(s, "drain_cycle_ns", 10), s)[1])(
        edits(_pods_ready(one_cq([5, 20], strategy=STRICT)), [(7, 0, 0)])),
    "stop-after-retry-in-boundary": lambda: (lambda s: (setattr(s, "drain_cycle_ns", 10), s)[1])(
        edits(_checks(one_cq([5, 20], strategy=STRICT)), [(7, 0, 0)])),
    "one-boundary": lambda: edits(one_cq([10, 20], held=[0], strategy=STRICT), [(3, 0, 0), (3, 1, 0), (3, 0, 1), (3, 1, 1)]),
}
DEVICE_CASES = dict(CPU_CASES)
DEVICE_CASES.update({
    "cfg2": _with_active(_cfg2), "cfg3": _with_active(_cfg3, inactive_share=0.05), "cfg4-latency": _with_active(_cfg4),
    "cfg4-checks-pr-mx": _with_active(_checks_pr_mx), "cfg4-sticky-quota": _with_active(_sticky_quota),
    "cfg3-afs-decay": _with_active(_afs_decay), "baseline": lambda: synth.perf_scenario(0.1, active=5),
    "baseline-all-blocks": lambda: synth.perf_scenario(0.1, evict_ns=30_000_000, checks=7, pods_ready=9, max_exec=3, quota=11,
                                                       active=5),
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
        assert int(got.cycle_arrived[k]) == len(want.arrived[k]), k
        assert int(got.cycle_evict_done[k]) == len(want.evict_done[k]), k
        assert int(got.cycle_stopped[k]) == len(want.stopped[k]), k
        assert int(got.cycle_resumed[k]) == len(want.resumed[k]), k
        assert int(got.cycle_quota_changes[k]) == len(want.quota_changes[k]), k
        assert int(got.cycle_max_exec_deactivated[k]) == len(want.max_exec_deactivated[k]), k
        assert int(got.cycle_pods_ready_timeout[k]) == len(want.pods_ready_timeout[k]), k
        assert int(got.cycle_check_retry[k]) == len(want.check_retry[k]), k
    assert got.n_evicted == want.n_evicted and got.n_finished == want.n_finished and got.end_ns == want.end_ns
    assert got.n_stopped == want.n_stopped and got.n_resumed == want.n_resumed and got.n_evict_done == want.n_evict_done
    for f in ("wl_admit_ns", "wl_finish_ns", "wl_evictions", "wl_admit_cycle", "cq_usage", "wl_deactivated",
              "wl_deactivation_reason"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    if want.cq_sticky is not None:
        assert np.array_equal(got.cq_sticky, want.cq_sticky)
    if want.wl_exec_acc_s is not None:
        assert np.array_equal(got.wl_exec_acc_s_out, want.wl_exec_acc_s)
    if want.wl_pods_ready_count is not None:
        assert np.array_equal(got.wl_pods_ready_count_out, want.wl_pods_ready_count)
    if want.lq_consumed is not None:
        assert np.array_equal(got.lq_consumed, want.lq_consumed) and np.array_equal(got.lq_last_update_ns, want.lq_last_update_ns)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DEVICE_CASES))
def test_kb_run_drain_active_changes_like_the_host_definition(name):
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = DEVICE_CASES[name]()
        mc = 100_000 if name.startswith("baseline") else 400
        want = run(snap, mc)
        got = ev.run_drain(snap, abi.DrainOut(snap, mc, trace_capacity=want.n_decisions))
        compare(want, got)
        if name.startswith(("cfg", "baseline")):
            assert got.n_stopped > 0 and got.n_resumed > 0
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
    mutate, msg = REFUSALS[name]
    s = _refusal_case()
    if name != "missing-table":
        mutate(s)
    st = s.as_struct()
    if name == "missing-table":
        st.ac_active = None
    out = abi.DrainOut(s, 5)
    out.struct.max_cycles = 5
    rc = native.lib().kb_run_drain(evaluator._h, C.byref(st), C.byref(out.struct))
    assert rc == abi.KB_ERR_INVALID and msg in native.lib().kb_last_error(evaluator._h).decode()
