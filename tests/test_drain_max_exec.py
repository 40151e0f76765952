"""MaximumExecutionTimeSeconds in the drain's event mode (kb_snapshot.wl_max_exec_s, wl_exec_acc_s, adm_exec_since_ns;
kueue_b200/drain.py).  A workload that has spent its limit in the Admitted state, summed over its admissions, is
deactivated (MaximumExecutionTimeExceeded) and evicted; every release of an admitted row adds that attempt's whole
seconds to the accumulated time.  CPU: the reference's test cases transcribed, hand-derived schedules on the oracle, the
equivalence of nil limits with the drain without the block, invariants.  GPU: kb_run_drain equals the host definition
cycle by cycle, refuses bad tables and reports an accumulated time that leaves int32."""
import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from kueue_b200.drain import DEACTIVATED, FINISHED, HELD, MAX_EXEC, REQUEUING_LIMIT, ExecOverflow, drain, exec_seconds

S = 1_000_000_000
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
I32_MAX = np.iinfo(np.int32).max
ALL = I32_MAX


def _run(snap, max_cycles=100_000):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000
    return drain(snap, lambda s: oracle.run_cycle(s, cap), max_cycles=max_cycles)


def _case(cpu, run, limit, acc=None, prio=None, create=None, adm=None, evict=None, pods_ready=None, checks=None):
    """One ClusterQueue of 2 cpu without a cohort, BestEffortFIFO, withinClusterQueue LowerPriority; one cycle takes
    1 s; now is 0.  `limit` / `acc`: the records' limits and accumulated seconds (-1 = nil).  `adm`: (workload, cpu,
    Admitted time) rows admitted before the drain.  `evict`: a termination latency for every workload.  `pods_ready`:
    (delays, fails, timeout, (base, max, limit)).  `checks`: check delays."""
    W = len(cpu)
    prio = prio or [0] * W
    create = create if create is not None else [0] * W
    s = abi.FlatSnapshot(n_cq=1, n_cohort=0, n_flavor=1, n_resource=1)
    s.set("nominal", [[2]])
    s.set("cq_rg_start", [0, 1]); s.set("rg_res_mask", [1]); s.set("rg_flavor_start", [0, 1]); s.set("rg_flavors", [0])
    s.set("cq_strategy", [abi.QUEUE_BEST_EFFORT_FIFO]); s.set("cq_within_cq", [abi.POLICY_LOWER_PRIORITY])
    s.set("wl_cq", np.zeros(W)); s.set("wl_priority", prio); s.set("wl_uid", np.arange(W)); s.set("wl_ts", create)
    s.set("ps_req", np.asarray(cpu)[:, None]); s.set("ps_req_mask", np.ones(W))
    adm = adm or []
    s.set("adm_wl", [w for w, _, _ in adm])
    if adm:
        s.set("adm_cq", np.zeros(len(adm))); s.set("adm_priority", [prio[w] for w, _, _ in adm])
        s.set("adm_ts", [create[w] for w, _, _ in adm]); s.set("adm_qr_ts", [t for _, _, t in adm])
        s.set("adm_uid", 100 + np.arange(len(adm)))
        s.set("adm_use_start", np.arange(len(adm) + 1)); s.set("adm_use_fr", np.zeros(len(adm)))
        s.set("adm_use_qty", [c for _, c, _ in adm]); s.set("cq_usage", [[sum(c for _, c, _ in adm)]])
    s.set("adm_exec_since_ns", [t for _, _, t in adm])
    s.set("wl_create_ns", create); s.set("wl_run_ns", run)
    s.set("wl_max_exec_s", limit)
    if acc is not None:
        s.set("wl_exec_acc_s", acc)
    if evict is not None:
        s.set("wl_evict_ns", np.full(W, evict))
    if pods_ready is not None:
        delay, fail, timeout, backoff = pods_ready
        s.set("wl_pods_ready_ns", delay); s.set("wl_pods_ready_fail", fail)
        s.pods_ready_timeout_ns = timeout
        s.pods_ready_backoff_base_s, s.pods_ready_backoff_max_s, s.pods_ready_backoff_limit = backoff
        if adm:
            s.set("adm_admitted_ns", [t for _, _, t in adm])
    if checks is not None:
        s.set("wl_check_ns", checks); s.set("wl_check_fail", np.zeros(W))
    s.now_ns, s.drain_cycle_ns = 0, S
    return s.finalize()


def _sec(xs):
    return [int(x) / S for x in xs]


# ---------------------------------------------------------------- the reference's cases, transcribed
def reconcile_case():
    """TestReconcile "admitted workload with max execution time": a 120 s limit, Admitted 60 s before now: the deadline is
    now + 60 s (RequeueAfter 1 min).  No queue has a head: the clock jumps there."""
    return _case([2], [-1], [120], adm=[(0, 2, -60 * S)])


def reconcile_expired_case():
    """"admitted workload with max execution time - expired": a 60 s limit, Admitted 120 s before now: past its limit,
    it expires at the first boundary."""
    return _case([2], [-1], [60], adm=[(0, 2, -120 * S)])


def test_reconcile_max_execution_time():
    r = _run(reconcile_case())
    assert r.cycles == 0 and r.end_ns == 60 * S and r.n_max_exec_deactivated == 1
    assert r.state.tolist() == [DEACTIVATED] and r.wl_deactivated.tolist() == [1]
    assert r.wl_deactivation_reason.tolist() == [MAX_EXEC] and r.wl_exec_acc_s.tolist() == [120]
    r = _run(reconcile_expired_case())
    assert r.cycles == 0 and r.end_ns == 0 and r.n_max_exec_deactivated == 1 and r.state.tolist() == [DEACTIVATED]
    assert r.wl_exec_acc_s.tolist() == [120] and r.cq_usage.tolist() == [[0]]


def sync_admitted_case(acc):
    """TestSyncAdmittedCondition "reservation lost with past admitted time": w0 (no limit) was Admitted 1 s before now;
    w1 (priority 1) preempts it at 0 without latency, so the reservation goes 1 s after Admitted."""
    return _case([2, 2], [-1, -1], [0, 0], acc=[acc, -1], prio=[0, 1], adm=[(0, 2, -S)])


@pytest.mark.parametrize("acc,want", [(-1, 1), (1, 2)])
def test_sync_admitted_condition_adds_the_admitted_seconds(acc, want):
    r = _run(sync_admitted_case(acc))
    assert [e.tolist() for e in r.evicted][0] == [0] and r.wl_exec_acc_s.tolist() == [want, -1]
    assert r.n_max_exec_deactivated == 0 and r.wl_deactivation_reason.tolist() == [0, 0]


def multiple_admissions_case():
    """The integration scenario "should deactivate the workload when the time expires with multiple admissions": w0
    (limit 30 s, 28 s accumulated) is admitted at 0; w1 (priority 1, created at 1.5 s, runs 0.5 s) preempts it at 1.5
    after a span of 1.5 s: acc = 29 = max - 1.  w1 runs 2.5-3; w0 is admitted again at 3.5 and deactivated 1 s later."""
    return _case([2, 2], [-1, S // 2], [30, 0], acc=[28, -1], prio=[0, 1], create=[0, 3 * S // 2])


def test_deactivated_after_multiple_admissions():
    r = _run(multiple_admissions_case())
    assert _sec(r.cycle_start_ns) == [0, 1.5, 2.5, 3.5] and r.end_ns == 4.5 * S
    assert [e.tolist() for e in r.evicted][1] == [0] and [a.tolist() for a in r.admitted] == [[0], [], [1], [0]]
    assert [d.tolist() for d in r.max_exec_deactivated] == [[], [], [], [0]]
    assert r.wl_exec_acc_s.tolist() == [1, -1] and r.state.tolist() == [DEACTIVATED, FINISHED]
    assert [(w, d) for w, _, _, d in r.exec_spans] == [(0, 1), (0, 1)]


# ---------------------------------------------------------------- hand-derived schedules
def truncation_case():
    """w0 (limit 5 s) never becomes ready; PodsReady timeout 1.5 s, backoff base 0 (requeued at the release).  Attempts
    at 0, 1.5, 3 and 4.5 each time out after 1.5 s and add 1 s: after three, acc is 3, not 4.  The one at 4.5 has 2 s
    left (times out at 6: acc 4); the one at 6 has 1 s left and expires at 7."""
    return _case([2], [-1], [5], pods_ready=([0], [ALL], 3 * S // 2, (0, 0, -1)))


def test_truncation_is_per_attempt():
    r = _run(truncation_case())
    assert _sec(r.cycle_start_ns) == [0, 1.5, 3, 4.5, 6] and r.end_ns == 7 * S
    assert [d for _, _, _, d in r.exec_spans] == [1, 1, 1, 1, 1] and r.n_pods_ready_timeout == 4
    assert [d.tolist() for d in r.max_exec_deactivated] == [[], [], [], [], [0]]
    assert r.wl_exec_acc_s.tolist() == [1] and r.wl_pods_ready_count.tolist() == [0] and r.state.tolist() == [DEACTIVATED]


def rounding_case(extra_s=0):
    """a snapshot row Admitted 2^30 s + 999,999,999 ns (plus extra_s) before now, limit 1 s: it expires at now and adds
    float64(2^30) + 0.999999999, which rounds to 2^30 + 1"""
    return _case([2], [-1], [1], adm=[(0, 2, -((2**30 + extra_s) * S + 999_999_999))])


def test_float_rounding_of_seconds():
    assert exec_seconds((2**30) * S + 999_999_999) == 2**30 + 1
    assert exec_seconds(2**23 * S + 999_999_999) == 2**23  # exact below 2^24 s
    assert exec_seconds(S + 999_999_999) == 1
    r = _run(rounding_case())
    assert r.wl_exec_acc_s.tolist() == [2**30 + 1] and r.state.tolist() == [DEACTIVATED]


def test_overflow_is_refused():
    with pytest.raises(ExecOverflow):
        exec_seconds((2**31 - 1) * S + 999_999_999)  # rounds to 2^31
    with pytest.raises(ExecOverflow):
        _run(rounding_case(2**30 - 1))


def finish_at_deadline_case():
    """w0 (limit 3 s) runs 3 s from 0: the finish at the deadline finishes; a completion adds nothing"""
    return _case([2], [3 * S], [3])


def test_finish_at_the_deadline_finishes():
    r = _run(finish_at_deadline_case())
    assert r.state.tolist() == [FINISHED] and r.wl_finish_ns.tolist() == [3 * S] and r.n_max_exec_deactivated == 0
    assert r.wl_exec_acc_s.tolist() == [-1] and r.wl_deactivation_reason.tolist() == [0]


def timeout_at_deadline_case():
    """w0 (limit 2 s) never becomes ready, PodsReady timeout 2 s: the timeout at the deadline is a timeout (Count 1), and
    its release at 2 deactivates the workload (Count 0, acc 2)"""
    return _case([2], [-1], [2], pods_ready=([0], [ALL], 2 * S, (1, 8, -1)))


def test_pods_ready_timeout_at_the_deadline():
    r = _run(timeout_at_deadline_case())
    assert r.n_pods_ready_timeout == 1 and r.n_max_exec_deactivated == 1 and r.end_ns == 2 * S
    assert r.wl_pods_ready_count.tolist() == [0] and r.state.tolist() == [DEACTIVATED]
    assert r.wl_deactivation_reason.tolist() == [MAX_EXEC] and r.wl_exec_acc_s.tolist() == [2]


def limit_before_pods_ready_case():
    """w0 (limit 1 s) becomes ready 3 s after Admitted: the deadline at 1 comes first and drops the attempt"""
    return _case([2], [5 * S], [1], pods_ready=([3 * S], [0], 10 * S, (1, 8, -1)))


def test_deadline_before_pods_ready_drops_the_attempt():
    r = _run(limit_before_pods_ready_case())
    assert r.end_ns == S and r.n_pods_ready_timeout == 0 and r.wl_pods_ready_count.tolist() == [0]
    assert r.wl_pods_ready_at.tolist() == [I64_MIN] and r.state.tolist() == [DEACTIVATED] and r.wl_exec_acc_s.tolist() == [1]


def requeuing_limit_case():
    """w0 (limit 2 s) never becomes ready, PodsReady timeout 2 s, backoffLimitCount 0: the timeout at the deadline
    deactivates it for RequeuingLimitExceeded first, which the limit leaves alone; the release adds 2"""
    return _case([2], [-1], [2], acc=[5], pods_ready=([0], [ALL], 2 * S, (1, 8, 0)))


def test_requeuing_limit_keeps_its_reason():
    r = _run(requeuing_limit_case())
    # acc 5 > limit 2: the deadline is before the admission, so the row expires at once (0) instead
    assert r.wl_deactivation_reason.tolist() == [MAX_EXEC] and r.wl_exec_acc_s.tolist() == [0]
    s = requeuing_limit_case(); s.set("wl_exec_acc_s", [-1])
    r = _run(s)
    assert r.n_pods_ready_deactivated == 1 and r.n_max_exec_deactivated == 0
    assert r.wl_deactivation_reason.tolist() == [REQUEUING_LIMIT] and r.wl_exec_acc_s.tolist() == [2]


def latency_deadline_case():
    """w0 (limit 3 s) is admitted at 0; w1 (priority 1, created at 1.5) preempts it with a 5 s termination latency: the
    eviction ends at 6.5, after the deadline at 3, so w0 is DEACTIVATED at its release (acc 6), not requeued"""
    return _case([2, 2], [-1, -1], [3, 0], prio=[0, 1], create=[0, 3 * S // 2], evict=5 * S)


def test_deadline_during_termination_latency():
    r = _run(latency_deadline_case())
    assert _sec(r.cycle_start_ns) == [0, 1.5, 2.5, 6.5] and r.n_evicted == 1 and r.n_evict_done == 1
    assert [d.tolist() for d in r.max_exec_deactivated] == [[], [], [0], []]
    assert r.state.tolist() == [DEACTIVATED, HELD] and r.wl_exec_acc_s.tolist() == [6, -1]


def ongoing_case():
    """w0 (limit 2 s, 5 s termination latency) expires at 2 and evicts until 7; w1 (priority 1, created at 3) targets
    it: "Preemption ongoing", no eviction is issued.  w1 is admitted at 7."""
    return _case([2, 2], [-1, -1], [2, 0], prio=[0, 1], create=[0, 3 * S], evict=5 * S)


def test_preemptor_of_an_expiring_row_is_ongoing():
    r = _run(ongoing_case())
    assert _sec(r.cycle_start_ns) == [0, 3, 7] and r.n_evicted == 0 and r.n_evict_done == 0
    assert [d.tolist() for d in r.decisions] == [[abi.DEC_ASSUMED], [abi.DEC_PREEMPTING], [abi.DEC_ASSUMED]]
    assert r.state.tolist() == [DEACTIVATED, HELD] and r.wl_exec_acc_s.tolist() == [7, -1]


def checks_ready_case():
    """w0 (limit 3 s) has a 2 s admission check: reserved at 0, Admitted at the Ready verdict (2), deadline 5"""
    return _case([2], [-1], [3], checks=[2 * S])


def checks_preempted_case():
    """w0 (limit 1 s) has a 5 s check; w1 (priority 1, created at 1.5, runs 1 s) preempts it while its checks run: the
    release adds nothing.  w0 is admitted again at 3.5 and expires at 3.5 + 5 + 1."""
    return _case([2, 2], [-1, S], [1, 0], prio=[0, 1], create=[0, 3 * S // 2], checks=[5 * S, 0])


def test_clock_starts_at_the_ready_verdict():
    r = _run(checks_ready_case())
    assert r.wl_ready_ns.tolist() == [2 * S] and r.end_ns == 5 * S and r.wl_exec_acc_s.tolist() == [3]
    r = _run(checks_preempted_case())
    assert [e.tolist() for e in r.evicted][1] == [0] and r.exec_spans[0][1] == 9.5 * S - S
    assert r.end_ns == 9.5 * S and r.wl_exec_acc_s.tolist() == [1, -1] and len(r.exec_spans) == 1


def never_finishes_case():
    """w0 runs forever (wl_run_ns < 0); its 4 s limit ends it"""
    return _case([2], [-1], [4])


def test_limit_ends_a_workload_that_never_finishes():
    r = _run(never_finishes_case())
    assert r.end_ns == 4 * S and r.state.tolist() == [DEACTIVATED] and r.wl_exec_acc_s.tolist() == [4]


def negative_left_case():
    """w0 (limit 2 s, 5 s accumulated): max - acc < 0, so the deadline is before the admission at 0; it expires at the
    first boundary, released at 0 (adds 0)"""
    return _case([2], [5 * S], [2], acc=[5])


def test_negative_time_left():
    r = _run(negative_left_case())
    assert r.cycles == 1 and [d.tolist() for d in r.max_exec_deactivated] == [[0]] and r.end_ns == S
    assert r.wl_exec_acc_s.tolist() == [0] and r.state.tolist() == [DEACTIVATED] and r.wl_finish_ns.tolist() == [I64_MAX]


# ---------------------------------------------------------------- equivalence: nil limits, no start state
def _cfg2():
    return synth.add_events(synth.make_snapshot(2, W=600, Q=12, preemption=True, tight=1.3, evictable=True), seed=1)


def _cfg3_decay():
    snap = synth.add_events(synth.make_snapshot(3, W=1200, Q=40, afs=3), seed=2)
    snap.set("adm_wl", np.zeros(0))
    snap.set("lq_last_update_ns", np.full(len(snap.arrays["lq_cq"]), snap.now_ns)); snap.set("adm_lq", np.full(snap.n_adm, -1))
    snap.afs_half_life_ns, snap.afs_sampling_ns, snap.afs_alpha = 10 * S, S, 0.5 ** 0.1
    return snap


def _cfg4_latency():
    return synth.add_evict_latency(synth.add_events(synth.make_snapshot(4, W=800, Q=40, tight=1.6, evictable=True), seed=3),
                                   (3_000, 40_000), seed=4)


def _baseline_checks_pods_ready():
    return synth.perf_scenario(0.1, checks=7, pods_ready=9)


BASE = {"cfg2": _cfg2, "cfg3-afs-decay": _cfg3_decay, "cfg4-latency": _cfg4_latency,
        "baseline-checks-pods-ready": _baseline_checks_pods_ready}
MAX_CYCLES = {"cfg2": 200, "cfg3-afs-decay": 200, "cfg4-latency": 200, "baseline-checks-pods-ready": 100_000}


def _limits(snap, value):
    """every limit `value` (0 = nil), nothing accumulated, an Admitted time for every row of the snapshot"""
    synth.add_max_exec(snap, seed=11, share=0.0)
    snap.set("wl_max_exec_s", np.full(snap.n_wl, value))
    return snap


def _same_schedule(got, want):
    assert got.cycles == want.cycles and got.cycle_start_ns == want.cycle_start_ns and got.end_ns == want.end_ns
    for k in range(want.cycles):
        assert np.array_equal(got.heads[k], want.heads[k]) and np.array_equal(got.decisions[k], want.decisions[k]), k
        assert np.array_equal(got.evicted[k], want.evicted[k]) and np.array_equal(got.finished[k], want.finished[k]), k
    assert np.array_equal(got.cq_usage, want.cq_usage)
    for f in ("wl_admit_cycle", "wl_evictions", "wl_admit_ns", "wl_finish_ns", "state"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    for f in ("wl_deactivated", "wl_ready_ns", "wl_pods_ready_at", "wl_pods_ready_count"):
        if getattr(want, f) is not None:
            assert np.array_equal(getattr(got, f), getattr(want, f)), f
    assert got.n_max_exec_deactivated == 0


@pytest.mark.parametrize("name", list(BASE))
def test_nil_limits_change_nothing(name):
    want = _run(BASE[name](), MAX_CYCLES[name])
    got = _run(_limits(BASE[name](), 0), MAX_CYCLES[name])
    _same_schedule(got, want)


def _spans_from_the_schedule(snap, res):
    """the accumulated seconds of every record from the schedule alone: an admission at t_c opens a span, a preemption
    in cycle k closes it at t_k plus the record's termination latency"""
    a = snap.arrays
    lat = a.get("wl_evict_ns")
    since = {int(w): int(t) for w, t in zip(a["adm_wl"], a["adm_exec_since_ns"])}
    acc = np.full(snap.n_wl, -1, np.int64)
    for k in range(res.cycles):
        t = res.cycle_start_ns[k]
        for w in res.evicted[k].tolist():
            end = t + (int(lat[w]) if lat is not None else 0)
            acc[w] = max(acc[w], 0) + exec_seconds(end - since.pop(w))
        for w in res.admitted[k].tolist():
            since[w] = t
    return acc


def _finite(snap):
    """every run finishes (a workload that runs forever meets even an INT32_MAX limit, 68 years on)"""
    run = snap.arrays["wl_run_ns"]
    snap.set("wl_run_ns", np.where(run < 0, 25_000, run))
    return snap


@pytest.mark.parametrize("name", ["cfg2", "cfg4-latency"])
def test_int32_max_limits_keep_the_schedule_and_sum_the_spans(name):
    want = _run(_finite(BASE[name]()), MAX_CYCLES[name])
    snap = _limits(_finite(BASE[name]()), I32_MAX)
    got = _run(snap, MAX_CYCLES[name])
    _same_schedule(got, want)
    if name == "cfg4-latency":  # every eviction issued in the drain completed before it ended
        assert got.n_evict_done == got.n_evicted
    assert got.n_evicted > 0 and np.array_equal(got.wl_exec_acc_s, _spans_from_the_schedule(snap, got))


# ---------------------------------------------------------------- invariants on seeded drains
def _cfg4_max_exec():
    """cfg4 on a clock in seconds (runs 0.5-4 s, 0.2 s cycles), termination latencies up to 1 s, PodsReady (delays up to
    1 s, timeout 0.8 s, limit 3) and limits of 1-3 s on half of the workloads"""
    snap = synth.add_events(synth.make_snapshot(4, W=800, Q=40, tight=1.6, evictable=True), seed=3, span_ns=20 * S,
                            run_ns=(S // 2, 4 * S), step_ns=S // 5)
    synth.add_evict_latency(snap, (0, S), seed=4)
    synth.add_pods_ready(snap, seed=5, delay_ns=(0, S), timeout_ns=4 * S // 5, base_s=0, max_s=0, limit=3)
    return synth.add_max_exec(snap, seed=6, share=0.5, limit_s=(1, 3), spent_share=0.1)


def _baseline_max_exec():
    return synth.perf_scenario(0.1, evict_ns=30_000_000, pods_ready=9, max_exec=3)


SEEDED = {"cfg4-max-exec": _cfg4_max_exec, "baseline-max-exec": _baseline_max_exec}


class _Watch:
    """run_cycle that records, for every cycle, (t_c, uid and reservation time of each row that is not evicting)"""

    def __init__(self, cap):
        self.cap, self.seen = cap, []

    def __call__(self, cs):
        a = cs.arrays
        live = a["adm_evicted"] == 0
        self.seen.append((int(cs.now_ns), a["adm_uid"][live].copy(), a["adm_qr_ts"][live].copy()))
        return oracle.run_cycle(cs, self.cap)


@pytest.mark.parametrize("name", list(SEEDED))
def test_max_exec_invariants(name):
    snap = SEEDED[name]()
    a = snap.arrays
    watch = _Watch(40 * (snap.n_adm + snap.n_wl) + 10000)
    res = drain(snap, watch, max_cycles=100_000)
    assert res.n_max_exec_deactivated > 0 and len(res.exec_spans) > 0
    # reasons and counts agree
    reason = res.wl_deactivation_reason
    assert np.array_equal(res.wl_deactivated, (reason != 0).astype(np.uint8))
    assert set(np.flatnonzero(res.state == DEACTIVATED).tolist()) == set(np.flatnonzero(reason).tolist())
    assert res.n_max_exec_deactivated == int((reason == MAX_EXEC).sum())
    per_cycle = [w for d in res.max_exec_deactivated for w in d.tolist()]
    assert len(per_cycle) == len(set(per_cycle)) and set(per_cycle) <= set(np.flatnonzero(reason == MAX_EXEC).tolist())
    # acc_out is the sum of the truncated spans of each record's releases; a deactivation leaves the last one
    acc0 = a["wl_exec_acc_s"].astype(np.int64)
    want = acc0.copy()
    last = {}
    for w, A, t, d in res.exec_spans:
        assert t >= A and d == (t - A) // S
        want[w] = max(want[w], 0) + d
        last[w] = d
    for w in np.flatnonzero(reason == MAX_EXEC):
        want[w] = last[int(w)]
    assert np.array_equal(res.wl_exec_acc_s, want)
    # no live row of a record with a limit is past its effective deadline at a cycle (rows admitted in the drain; the
    # record's accumulated time is what its earlier releases left)
    uid_of = {int(u): w for w, u in enumerate(a["wl_uid"])}
    spans = {}
    for w, A, t, d in res.exec_spans:
        spans.setdefault(w, []).append((t, d))
    limit, checked = a["wl_max_exec_s"], 0
    admissions = {(int(w), res.cycle_start_ns[k]) for k, adm in enumerate(res.admitted) for w in adm.tolist()}
    for t_c, uids, qr in watch.seen:
        for u, A in zip(uids.tolist(), qr.tolist()):
            w = uid_of.get(u)
            if w is None or (w, A) not in admissions or limit[w] <= 0:
                continue
            acc = acc0[w]
            for t_rel, d in spans.get(w, []):
                if t_rel <= A:
                    acc = max(acc, 0) + d
            assert max(A + (int(limit[w]) - max(int(acc), 0)) * S, A) > t_c, (w, t_c)
            checked += 1
    assert checked > 0


# ---------------------------------------------------------------------------------------------------------------- GPU
DEVICE_CASES = {
    "reconcile": reconcile_case, "reconcile-expired": reconcile_expired_case,
    "sync-admitted-nil": lambda: sync_admitted_case(-1), "sync-admitted-add": lambda: sync_admitted_case(1),
    "multiple-admissions": multiple_admissions_case, "truncation": truncation_case, "rounding": rounding_case,
    "finish-at-deadline": finish_at_deadline_case, "timeout-at-deadline": timeout_at_deadline_case,
    "before-pods-ready": limit_before_pods_ready_case, "requeuing-limit": requeuing_limit_case,
    "latency-deadline": latency_deadline_case, "ongoing": ongoing_case, "checks-ready": checks_ready_case,
    "checks-preempted": checks_preempted_case, "never-finishes": never_finishes_case, "negative-left": negative_left_case,
    "nil-cfg2": lambda: _limits(_cfg2(), 0), "nil-cfg3-afs-decay": lambda: _limits(_cfg3_decay(), 0),
    "nil-cfg4-latency": lambda: _limits(_cfg4_latency(), 0),
    "nil-baseline-checks-pods-ready": lambda: _limits(_baseline_checks_pods_ready(), 0),
    "int32-max-cfg2": lambda: _limits(_finite(_cfg2()), I32_MAX),
    "int32-max-cfg4-latency": lambda: _limits(_finite(_cfg4_latency()), I32_MAX),
    "cfg4-max-exec": _cfg4_max_exec, "baseline-max-exec": _baseline_max_exec,
    "baseline-full": lambda: synth.perf_scenario(1.0, evict_ns=30_000_000, checks=7, pods_ready=9, max_exec=3),
}


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
        assert int(got.cycle_pods_ready_timeout[k]) == len(want.pods_ready_timeout[k]), k
        assert int(got.cycle_pods_ready_deactivated[k]) == len(want.pods_ready_deactivated[k]), k
        assert int(got.cycle_check_retry[k]) == len(want.check_retry[k]), k
        assert int(got.cycle_max_exec_deactivated[k]) == len(want.max_exec_deactivated[k]), k
    assert got.n_evicted == want.n_evicted and got.n_finished == want.n_finished and got.end_ns == want.end_ns
    assert got.n_evict_done == want.n_evict_done and got.n_resorts == want.n_resorts
    assert (got.n_pods_ready_timeout, got.n_pods_ready_deactivated) == (want.n_pods_ready_timeout, want.n_pods_ready_deactivated)
    assert got.n_max_exec_deactivated == want.n_max_exec_deactivated
    for f in ("wl_admit_ns", "wl_finish_ns", "wl_evictions", "wl_admit_cycle", "cq_usage", "wl_deactivated",
              "wl_deactivation_reason"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    assert np.array_equal(got.wl_exec_acc_s_out, want.wl_exec_acc_s)
    if want.wl_pods_ready_at is not None:
        assert np.array_equal(got.wl_pods_ready_at_ns, want.wl_pods_ready_at)
        assert np.array_equal(got.wl_pods_ready_count_out, want.wl_pods_ready_count)
    if want.wl_ready_ns is not None:
        assert np.array_equal(got.wl_ready_ns, want.wl_ready_ns)
        assert (got.n_check_ready, got.n_check_retry, got.n_check_rejected) == (want.n_check_ready, want.n_check_retry, want.n_check_rejected)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DEVICE_CASES))
def test_kb_run_drain_max_exec_like_the_host_definition(name):
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = DEVICE_CASES[name]()
        mc = 100_000 if "baseline" in name or "max-exec" in name else 400
        want = _run(snap, mc)
        got = ev.run_drain(snap, abi.DrainOut(snap, mc, trace_capacity=want.n_decisions))
        compare(want, got)
        if name == "baseline-full":
            assert got.n_max_exec_deactivated > 0 and got.n_pods_ready_timeout > 0 and got.n_check_retry > 0
    finally:
        ev.close()


@pytest.fixture
def evaluator():
    from kueue_b200 import native
    ev = native.Evaluator(0)
    yield ev
    ev.close()


def _refused(ev, snap, match, code=abi.KB_ERR_INVALID):
    """refused with `code` by the check whose message contains `match`"""
    from kueue_b200 import native
    with pytest.raises(native.KueueB200Error, match=match) as e:
        ev.run_drain(snap, max_cycles=5)
    assert e.value.code == code


@pytest.mark.gpu
def test_refuses_tables_without_adm_wl(evaluator):
    s = never_finishes_case(); del s.arrays["adm_wl"]
    _refused(evaluator, s, "max exec: the tables need adm_wl")


@pytest.mark.gpu
@pytest.mark.parametrize("field", ["wl_exec_acc_s", "adm_exec_since_ns"])
def test_refuses_tables_without_the_limits(evaluator, field):
    s = reconcile_case(); s.set("wl_exec_acc_s", [-1]); del s.arrays["wl_max_exec_s"]
    if field == "wl_exec_acc_s":
        del s.arrays["adm_exec_since_ns"]
    _refused(evaluator, s, "max exec: the tables need wl_max_exec_s")


@pytest.mark.gpu
def test_refuses_a_negative_limit(evaluator):
    s = reconcile_case(); s.set("wl_max_exec_s", [-1])
    _refused(evaluator, s, "max exec: wl_max_exec_s < 0")


@pytest.mark.gpu
def test_refuses_an_accumulated_time_below_nil(evaluator):
    s = reconcile_case(); s.set("wl_exec_acc_s", [-2])
    _refused(evaluator, s, "max exec: wl_exec_acc_s < -1")


@pytest.mark.gpu
def test_refuses_missing_admitted_times(evaluator):
    s = reconcile_case(); del s.arrays["adm_exec_since_ns"]
    _refused(evaluator, s, "max exec: adm_exec_since_ns is NULL while n_adm > 0")
    s = reconcile_case(); s.set("adm_exec_since_ns", [I64_MIN])
    _refused(evaluator, s, "max exec: adm_exec_since_ns missing on a row whose checks do not run")


@pytest.mark.gpu
def test_refuses_an_admitted_time_after_now(evaluator):
    s = reconcile_case(); s.set("adm_exec_since_ns", [S])
    _refused(evaluator, s, "max exec: adm_exec_since_ns after now_ns")


@pytest.mark.gpu
def test_refuses_an_admitted_time_on_a_row_whose_checks_run(evaluator):
    s = reconcile_case(); s.set("wl_check_ns", [0]); s.set("adm_check_end_ns", [5 * S])
    _refused(evaluator, s, "max exec: adm_exec_since_ns set on a row whose checks run")


@pytest.mark.gpu
def test_refuses_an_admitted_time_other_than_adm_admitted_ns(evaluator):
    s = reconcile_case(); s.set("wl_pods_ready_ns", [0]); s.set("adm_admitted_ns", [-30 * S])
    _refused(evaluator, s, "max exec: adm_exec_since_ns differs from adm_admitted_ns")


@pytest.mark.gpu
def test_overflow_status(evaluator):
    _refused(evaluator, rounding_case(2**30 - 1), "max exec: an accumulated execution time leaves int32", abi.KB_ERR_UNSUPPORTED)
