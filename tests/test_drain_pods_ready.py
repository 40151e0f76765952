"""WaitForPodsReady in the drain's event mode (kb_snapshot.wl_pods_ready_ns and the start-state tables;
kueue_b200/drain.py).  An attempt starts at Admitted; a ready one reaches PodsReady after its delay and runs from there,
a failing one is evicted at Admitted + timeout, requeued after its backoff (or deactivated past the limit) and releases
its quota once its pods are gone.  CPU: hand-derived schedules on the oracle, the backoff edges, the equivalence of zero
delays with the drain without the block, invariants.  GPU: kb_run_drain equals the host definition cycle by cycle, and
refuses bad tables."""
import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from kueue_b200.drain import BACKOFF, DEACTIVATED, FINISHED, HELD, QUEUED, SET_ASIDE, drain, pods_ready_wait_ns

S = 1_000_000_000
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
ALL = np.iinfo(np.int32).max


def _run(snap, max_cycles=100_000):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000
    return drain(snap, lambda s: oracle.run_cycle(s, cap), max_cycles=max_cycles)


def _case(cpu, ts, run, delay, fail, timeout=10 * S, backoff=(1, 8, -1), creation=0, prio=None, create=None,
          within=abi.POLICY_NEVER, adm=None, evict=None):
    """One ClusterQueue of 2 cpu without a cohort, BestEffortFIFO, withinClusterQueue `within`; one cycle takes 1 s.
    `backoff` = (base s, max s, limit).  `adm`: (workload, cpu, Admitted time or INT64_MIN) rows admitted before the
    drain; `evict`: a termination latency for every workload."""
    W = len(cpu)
    s = abi.FlatSnapshot(n_cq=1, n_cohort=0, n_flavor=1, n_resource=1)
    s.set("nominal", [[2]])
    s.set("cq_rg_start", [0, 1]); s.set("rg_res_mask", [1]); s.set("rg_flavor_start", [0, 1]); s.set("rg_flavors", [0])
    s.set("cq_strategy", [abi.QUEUE_BEST_EFFORT_FIFO]); s.set("cq_within_cq", [within])
    s.set("wl_cq", np.zeros(W)); s.set("wl_priority", prio or [0] * W); s.set("wl_uid", np.arange(W)); s.set("wl_ts", ts)
    s.set("ps_req", np.asarray(cpu)[:, None]); s.set("ps_req_mask", np.ones(W))
    adm = adm or []
    s.set("adm_wl", [w for w, _, _ in adm])
    if adm:
        s.set("adm_cq", np.zeros(len(adm))); s.set("adm_priority", [(prio or [0] * W)[w] for w, _, _ in adm])
        s.set("adm_ts", [ts[w] for w, _, _ in adm]); s.set("adm_qr_ts", np.zeros(len(adm))); s.set("adm_uid", 100 + np.arange(len(adm)))
        s.set("adm_use_start", np.arange(len(adm) + 1)); s.set("adm_use_fr", np.zeros(len(adm)))
        s.set("adm_use_qty", [c for _, c, _ in adm]); s.set("cq_usage", [[sum(c for _, c, _ in adm)]])
        s.set("adm_admitted_ns", [t for _, _, t in adm])
    s.set("wl_create_ns", create if create is not None else np.minimum(ts, 0)); s.set("wl_run_ns", run)
    s.set("wl_pods_ready_ns", delay); s.set("wl_pods_ready_fail", fail)
    if evict is not None:
        s.set("wl_evict_ns", np.full(W, evict))
    s.pods_ready_timeout_ns = timeout
    s.pods_ready_backoff_base_s, s.pods_ready_backoff_max_s, s.pods_ready_backoff_limit = backoff
    s.pods_ready_requeue_creation = creation
    s.now_ns, s.drain_cycle_ns = 0, S
    return s.finalize()


def _sec(xs):
    return [int(x) // S for x in xs]


# ---------------------------------------------------------------- hand-derived schedules
def ready_case():
    """w0 and w1 need the whole 2 cpu and run 5 s.  0: w0 admitted, PodsReady at 3 (delay 3 s), finishes at 8.  1: w1
    NoFit, set aside; the quiet cycle waits for 8: w0 finishes, w1 is admitted with a delay equal to the timeout (ready:
    the tie-break), PodsReady at 18, finishes at 23."""
    return _case([2, 2], [0, 1], [5 * S] * 2, [3 * S, 10 * S], [0, 0])


def test_ready_within_the_timeout_shifts_the_finish():
    r = _run(ready_case())
    assert _sec(r.cycle_start_ns) == [0, 1, 8] and [h.tolist() for h in r.heads] == [[0], [1], [1]]
    assert _sec(r.wl_pods_ready_at) == [3, 18] and _sec(r.wl_finish_ns) == [8, 23] and r.end_ns == 23 * S
    assert r.n_pods_ready_timeout == r.n_pods_ready_deactivated == 0 and r.n_evicted == 0 and r.n_resorts == 0
    assert r.wl_pods_ready_count.tolist() == [0, 0] and (r.state == FINISHED).all()


def readmit_case():
    """The reference's "Should re-admit a timed out workload" with backoffLimitCount nil: w0's first two attempts never
    become ready (timeout 10 s, base 1 s).  0 admitted, times out at 10 (Count 1, back at 11, timestamp 10: a re-sort);
    11 admitted, times out at 21 (Count 2, back at 23); 23 admitted, ready at once, finishes at 28."""
    return _case([2], [0], [5 * S], [0], [2])


def test_timed_out_workload_is_readmitted():
    r = _run(readmit_case())
    assert _sec(r.cycle_start_ns) == [0, 11, 23] and r.end_ns == 28 * S
    assert [x.tolist() for x in r.pods_ready_timeout] == [[0], [0], []] and r.n_pods_ready_deactivated == 0
    assert r.wl_pods_ready_count.tolist() == [2] and r.wl_deactivated.tolist() == [0] and r.state.tolist() == [FINISHED]
    assert _sec(r.wl_pods_ready_at) == [23] and r.n_resorts == 2 and r.n_evicted == 0 and r.n_finished == 1


def deactivate_case():
    """The reference's "deactivate a workload exceeded the re-queue count limit": limit 2, base 1 s, w0 never ready.
    Admitted at 0, 11 (10 + 1 s) and 23 (21 + 2 s); the third timeout at 33 has Count + 1 = 3 > 2: deactivated."""
    return _case([2], [0], [5 * S], [0], [ALL], backoff=(1, 8, 2))


def test_deactivated_past_the_requeue_limit():
    r = _run(deactivate_case())
    assert _sec(r.cycle_start_ns) == [0, 11, 23] and r.end_ns == 33 * S
    assert [x.tolist() for x in r.pods_ready_timeout] == [[0], [0], []]
    assert [x.tolist() for x in r.pods_ready_deactivated] == [[], [], [0]]
    assert r.n_pods_ready_timeout == 2 and r.n_pods_ready_deactivated == 1
    assert r.wl_deactivated.tolist() == [1] and r.wl_pods_ready_count.tolist() == [0] and r.state.tolist() == [DEACTIVATED]
    assert r.cq_usage.tolist() == [[0]] and r.wl_pods_ready_at.tolist() == [I64_MIN]


def ordering_case(creation):
    """The reference's eviction-ordering scenarios: w0, w1, w2 (created 0, 1, 2 s) each fill the ClusterQueue and
    never become ready; timeout 10 s, base 1 s, no limit."""
    return _case([2, 2, 2], [0, S, 2 * S], [-1] * 3, [0] * 3, [ALL] * 3, creation=creation)


def _admitted(r):
    return [int(w) for adm in r.admitted for w in adm]


def test_eviction_timestamp_moves_the_evicted_workload_to_the_back():
    """Eviction: each timed-out workload sorts by its eviction time, behind the others: w0, w1, w2, w0, w1, w2, ..."""
    r = _run(ordering_case(0), max_cycles=40)
    got = _admitted(r)
    assert got[:7] == [0, 1, 2, 0, 1, 2, 0]
    assert _sec(r.cycle_start_ns)[:4] == [0, 1, 10, 11]  # 10: w0 times out, w1 admitted; 11: w0 back behind w2


def test_creation_timestamp_keeps_the_evicted_workload_at_the_front():
    """Creation: w0 keeps timestamp 0.  It is back at 11 and first in the queue; when w1 times out at 20, w0 is admitted
    again ahead of w2, and so on: w2 never runs."""
    r = _run(ordering_case(1), max_cycles=40)
    got = _admitted(r)
    assert got[:5] == [0, 1, 0, 1, 0] and 2 not in got
    assert r.n_resorts == 0


def latency_case():
    """"low" (priority -1) never becomes ready (timeout 10 s, base 60 s) and its pods take 5 s to terminate; "hi"
    (priority 1, created at 12) needs the quota and may preempt lower priorities.  10: low times out, evicting until 15
    (it holds its quota).  12: hi targets it: ongoing, no eviction issued.  15: low is released to BACKOFF (RequeueAt
    70) and hi is admitted at 15."""
    return _case([2, 2], [0, 12 * S], [-1, -1], [0, 0], [ALL, 0], backoff=(60, 0, -1), prio=[-1, 1], create=[0, 12 * S],
                 within=abi.POLICY_LOWER_PRIORITY, evict=5 * S)


def test_timeout_with_eviction_latency_holds_the_quota():
    r = _run(latency_case(), max_cycles=6)
    assert _sec(r.cycle_start_ns)[:3] == [0, 12, 15]
    assert [d.tolist() for d in r.decisions][1] == [abi.DEC_PREEMPTING]
    assert r.n_evicted == 0 and r.wl_evictions.tolist() == [0, 0] and r.n_evict_done == 0
    assert r.n_pods_ready_timeout == 1 and r.wl_admit_ns[1] == 15 * S
    short = _run(latency_case(), max_cycles=3)  # after the release at 15 the record waits in BACKOFF, not QUEUED
    assert _sec(short.cycle_start_ns) == [0, 12, 15] and short.state.tolist() == [BACKOFF, HELD]
    assert _sec(r.cycle_start_ns)[3] == 70 and [h.tolist() for h in r.heads][3] == [0]  # back at RequeueAt 70


def preempt_waiting_case():
    """"low" (priority -1, 2 cpu) fails one attempt; "hi" (priority 1, created at 5, runs 10 s) preempts it at 5 with
    no latency: low is released at once, hi is admitted at 6 and finishes at 16, low is NoFit at 7.  The dropped attempt
    is not counted and uses no failure: low is readmitted at 16, fails (its failure is still left) at 26 with Count 1,
    returns at 27, becomes ready at once and finishes at 30."""
    return _case([2, 2], [0, 5 * S], [3 * S, 10 * S], [0, 0], [1, 0], prio=[-1, 1], create=[0, 5 * S],
                 within=abi.POLICY_LOWER_PRIORITY)


def test_preempted_while_waiting_drops_the_attempt():
    r = _run(preempt_waiting_case())
    assert _sec(r.cycle_start_ns) == [0, 5, 6, 7, 16, 27]
    assert [e.tolist() for e in r.evicted][1] == [0] and r.n_pods_ready_timeout == 1
    assert r.wl_pods_ready_count.tolist() == [1, 0] and _sec(r.wl_pods_ready_at) == [27, 6]
    assert _sec(r.wl_finish_ns) == [30, 16]


def checks_case():
    """Admission checks: w0's check takes 0.3 s and its first PodsReady attempt never becomes ready (timeout 0.5 s).  The
    cycle at 0 admits it, so the next boundary is 1 s: the Ready verdict at 0.3 and the timeout at 0.8 fall in it.  w0
    returns at 1.8, its check is Ready at 2.1, and it is ready at once: it runs 5 s until 7.1."""
    s = _case([2], [0], [5 * S], [0], [1], timeout=S // 2)
    s.set("wl_check_ns", [3 * S // 10])
    return s


def test_timer_starts_at_the_ready_verdict():
    r = _run(checks_case())
    assert r.cycle_start_ns == [0, 1_800_000_000] and [x.tolist() for x in r.pods_ready_timeout] == [[0], []]
    assert r.wl_ready_ns.tolist() == [2_100_000_000] and r.wl_pods_ready_at.tolist() == [2_100_000_000]
    assert r.wl_finish_ns.tolist() == [7_100_000_000] and r.n_check_ready == 2 and r.wl_pods_ready_count.tolist() == [1]


def base_zero_case():
    """Base 0 and a starting Count of 2^31 - 2: the timeout at 10 requeues w0 in that boundary (RequeueAt = 10) with
    Count 2^31 - 1; it is admitted again at 10 and is ready."""
    s = _case([2], [0], [5 * S], [0], [1], backoff=(0, 0, -1))
    s.set("wl_pods_ready_count", [2**31 - 2])
    return s


def test_backoff_base_zero_requeues_at_the_release_boundary():
    r = _run(base_zero_case())
    assert _sec(r.cycle_start_ns) == [0, 10] and r.wl_pods_ready_count.tolist() == [2**31 - 1]
    assert _sec(r.wl_finish_ns) == [15] and pods_ready_wait_ns(2**31 - 1, 0, 0) == 0


def test_backoff_base_above_max_and_no_cap():
    assert [pods_ready_wait_ns(k, 60, 30) // S for k in (1, 2, 3)] == [60, 30, 30]
    assert [pods_ready_wait_ns(k, 1, 0) // S for k in (1, 2, 3, 4)] == [1, 2, 4, 8]
    assert pods_ready_wait_ns(200, 1, 0) == 2**62  # MaxInt64 / 2 in float64, as time.Duration(math.MaxInt64 / 2)
    r = _run(_case([2], [0], [5 * S], [0], [1], backoff=(60, 30, -1)))
    assert _sec(r.cycle_start_ns) == [0, 70]  # the base, uncapped, first


def saturating_case():
    """max 0 = no cap: with Count 200 the wait is the cap 2^62 and RequeueAt saturates at INT64_MAX, so w0 never
    returns; the clock starts at 5e18 ns."""
    s = _case([2], [0], [5 * S], [0], [1], backoff=(1, 0, -1))
    s.set("wl_pods_ready_count", [200])
    s.now_ns = 5 * 10**18
    s.set("wl_ts", [s.now_ns]); s.set("wl_create_ns", [s.now_ns])
    return s.finalize()


def test_backoff_without_cap_saturates():
    r = _run(saturating_case())
    assert r.cycles == 1 and r.end_ns == 5 * 10**18 + 10 * S and r.state.tolist() == [BACKOFF]
    assert r.wl_pods_ready_count.tolist() == [201]


def start_state_case():
    """Start state (now 0): row r0 (w0, 1 cpu) was Admitted at -15 s and never becomes ready, so its timeout (-5 s) is
    already due; row r1 (w1, 1 cpu) was Admitted at -2 s with a 4 s delay: PodsReady at 2, finishes at 7.  w2 is in
    backoff until 30 (evicted by a timeout at 20, Count 2 = the limit) and never becomes ready.
      0: no head (w2 waits); the first boundary applies r0's timeout: w0 Count 1, back at -5 + 1 = -4 < 0: queued,
         admitted at 0 (T 10)   7: w1 finishes   10: w0 times out, Count 2, back at 12, admitted at 12, times out at 22:
         deactivated   30: w2 returns, admitted, times out at 40: Count 3 > 2, deactivated."""
    s = _case([1, 1, 2], [0, 0, 0], [5 * S] * 3, [0, 4 * S, 0], [ALL, 0, ALL], backoff=(1, 8, 2),
              adm=[(0, 1, -15 * S), (1, 1, -2 * S)])
    s.set("wl_requeue_at_ns", [I64_MIN, I64_MIN, 30 * S]); s.set("wl_pods_ready_evict_ns", [I64_MIN, I64_MIN, 20 * S])
    s.set("wl_pods_ready_count", [0, 0, 2])
    return s


def start_preempted_case():
    """Start state: w0 holds the 2 cpu, Admitted at -2 s with a 4 s delay (PodsReady would come at 2 s); w1 (priority 1)
    preempts it at 0 without latency and runs forever.  w0's attempt is dropped before PodsReady: it has no PodsReady
    time.  w1 is admitted at 1 and is ready at once."""
    return _case([2, 2], [0, 0], [-1, -1], [4 * S, 0], [0, 0], prio=[0, 1], within=abi.POLICY_LOWER_PRIORITY,
                 adm=[(0, 2, -2 * S)])


def test_start_state_row_preempted_before_pods_ready():
    r = _run(start_preempted_case())
    assert _sec(r.cycle_start_ns)[:2] == [0, 1] and [e.tolist() for e in r.evicted][0] == [0]
    assert r.wl_pods_ready_at.tolist() == [I64_MIN, S] and r.state.tolist() == [SET_ASIDE, HELD]
    assert r.wl_pods_ready_count.tolist() == [0, 0] and r.n_pods_ready_timeout == 0


def test_start_state_tables():
    r = _run(start_state_case())
    assert r.n_pods_ready_timeout == 2 and r.n_pods_ready_deactivated == 2
    assert r.wl_deactivated.tolist() == [1, 0, 1] and r.wl_pods_ready_count.tolist() == [0, 0, 0]
    assert _sec(r.wl_pods_ready_at)[1] == 2 and _sec(r.wl_finish_ns)[1] == 7
    assert r.state.tolist() == [DEACTIVATED, FINISHED, DEACTIVATED]
    assert 30 * S in r.cycle_start_ns and r.end_ns == 40 * S


# ---------------------------------------------------------------- equivalence: zero delays, no start state
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


def _baseline():
    return synth.perf_scenario(0.1)


def _baseline_checks():
    return synth.perf_scenario(0.1, checks=7)


BASE = {"cfg2": _cfg2, "cfg3-afs-decay": _cfg3_decay, "cfg4-latency": _cfg4_latency, "baseline": _baseline,
        "baseline-checks": _baseline_checks}
MAX_CYCLES = {"cfg2": 200, "cfg3-afs-decay": 200, "cfg4-latency": 200, "baseline": 100_000, "baseline-checks": 100_000}


def _zero(snap):
    snap.set("wl_pods_ready_ns", np.zeros(snap.n_wl)); snap.set("wl_pods_ready_fail", np.zeros(snap.n_wl))
    return snap


@pytest.mark.parametrize("name", list(BASE))
def test_zero_delays_change_nothing(name):
    want = _run(BASE[name](), MAX_CYCLES[name])
    got = _run(_zero(BASE[name]()), MAX_CYCLES[name])
    assert got.cycles == want.cycles and got.cycle_start_ns == want.cycle_start_ns and got.end_ns == want.end_ns
    for k in range(want.cycles):
        assert np.array_equal(got.heads[k], want.heads[k]) and np.array_equal(got.decisions[k], want.decisions[k]), k
        assert np.array_equal(got.evicted[k], want.evicted[k]) and np.array_equal(got.finished[k], want.finished[k]), k
    assert np.array_equal(got.cq_usage, want.cq_usage)
    for f in ("wl_admit_cycle", "wl_evictions", "wl_admit_ns", "wl_finish_ns", "state"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    assert got.n_pods_ready_timeout == got.n_pods_ready_deactivated == 0
    if "checks" in name:
        assert got.n_resorts == want.n_resorts and np.array_equal(got.wl_ready_ns, want.wl_ready_ns)
    else:
        assert got.n_resorts == 0


# ---------------------------------------------------------------- invariants on seeded drains
def _cfg4_pods_ready():
    return synth.add_pods_ready(synth.add_evict_latency(synth.add_events(
        synth.make_snapshot(4, W=800, Q=40, tight=1.6, evictable=True), seed=3), (3_000, 40_000), seed=4), seed=5,
        delay_ns=(0, 3_000), timeout_ns=2_500, base_s=0, max_s=0, limit=3)


def _baseline_pods_ready():
    return synth.perf_scenario(0.1, pods_ready=9)


SEEDED = {"cfg4-pods-ready": _cfg4_pods_ready, "baseline-pods-ready": _baseline_pods_ready}


def _cells_of(adm, Q, FR):
    use = np.zeros((Q, FR), np.int64)
    st = adm["adm_use_start"]
    for a in range(len(adm["adm_cq"])):
        for k in range(int(st[a]), int(st[a + 1])):
            use[int(adm["adm_cq"][a]), int(adm["adm_use_fr"][k])] += int(adm["adm_use_qty"][k])
    return use


@pytest.mark.parametrize("name", list(SEEDED))
def test_pods_ready_invariants(name):
    snap = SEEDED[name]()
    a = snap.arrays
    res = _run(snap, 100_000)
    assert res.n_pods_ready_timeout > 0
    Q, FR = snap.n_cq, snap.n_fr
    init = {k: a[k] for k in ("adm_cq", "adm_use_start", "adm_use_fr", "adm_use_qty")}
    assert np.array_equal(res.cq_usage - _cells_of(res.adm, Q, FR), a["cq_usage"].reshape(Q, FR) - _cells_of(init, Q, FR))
    assert set(np.flatnonzero(res.state == HELD).tolist()) == set(res.adm["adm_wl"].tolist())
    gone = set(np.flatnonzero(res.wl_deactivated).tolist())
    assert gone == set(np.flatnonzero(res.state == DEACTIVATED).tolist()) and len(gone) == res.n_pods_ready_deactivated
    deact_at, timeouts = {}, np.zeros(snap.n_wl, np.int64)
    for k in range(res.cycles):
        for w in res.pods_ready_deactivated[k].tolist():
            deact_at[w] = k
        for w in res.pods_ready_timeout[k].tolist():
            timeouts[w] += 1
    for k in range(res.cycles):  # a deactivated record is never admitted again
        for w in res.admitted[k].tolist():
            assert w not in deact_at or k <= deact_at[w], (w, k)
    start = a["wl_pods_ready_count"] if "wl_pods_ready_count" in a else np.zeros(snap.n_wl)
    for w in range(snap.n_wl):
        assert res.wl_pods_ready_count[w] == (0 if w in gone else start[w] + timeouts[w]), w
    # no record is queued before its RequeueAt: after a timeout applied in cycle k (its T in (t_k, t_{k+1}]), with
    # RequeueAt = T + WaitTime(Count) from the Count sequence, the record is no cycle's head before RequeueAt (a head is a
    # queued record), and it is next admitted at a cycle start >= RequeueAt
    base, mx = snap.pods_ready_backoff_base_s, snap.pods_ready_backoff_max_s
    count, checked = start.astype(np.int64).copy(), 0
    starts = res.cycle_start_ns
    for k in range(res.cycles):
        for w, (T, at) in zip(res.pods_ready_timeout[k].tolist(), res.pods_ready_timeout_at[k].tolist()):
            count[w] += 1
            assert starts[k] < T and (k + 1 == res.cycles or T <= starts[k + 1]), (w, k)
            assert at == min(T + pods_ready_wait_ns(int(count[w]), base, mx), I64_MAX), (w, k)
            for j in range(k + 1, res.cycles):
                if w in res.heads[j].tolist():
                    assert starts[j] >= at, (w, k, j)
                    checked += 1
                if w in res.admitted[j].tolist():
                    break
    assert checked > 0


# ---------------------------------------------------------------------------------------------------------------- GPU
DEVICE_CASES = {
    "ready": ready_case, "readmit": readmit_case, "deactivate": deactivate_case,
    "ordering-eviction": lambda: ordering_case(0), "ordering-creation": lambda: ordering_case(1),
    "latency": latency_case, "preempt-waiting": preempt_waiting_case, "checks": checks_case, "base-zero": base_zero_case,
    "saturating": saturating_case, "start-state": start_state_case, "start-preempted": start_preempted_case,
    "zero-cfg2": lambda: _zero(_cfg2()), "zero-cfg3-afs-decay": lambda: _zero(_cfg3_decay()),
    "zero-cfg4-latency": lambda: _zero(_cfg4_latency()), "zero-baseline": lambda: _zero(_baseline()),
    "zero-baseline-checks": lambda: _zero(_baseline_checks()),
    "cfg4-pods-ready": _cfg4_pods_ready, "baseline-pods-ready": _baseline_pods_ready,
    "baseline-full": lambda: synth.perf_scenario(1.0, evict_ns=30_000_000, checks=7, pods_ready=9),
}
DEVICE_MAX_CYCLES = {"ordering-eviction": 40, "ordering-creation": 40}


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
        assert int(got.cycle_pods_ready_timeout[k]) == len(want.pods_ready_timeout[k]), k
        assert int(got.cycle_pods_ready_deactivated[k]) == len(want.pods_ready_deactivated[k]), k
    assert got.n_evicted == want.n_evicted and got.n_finished == want.n_finished and got.end_ns == want.end_ns
    assert got.n_evict_done == want.n_evict_done and got.n_resorts == want.n_resorts
    assert (got.n_pods_ready_timeout, got.n_pods_ready_deactivated) == (want.n_pods_ready_timeout, want.n_pods_ready_deactivated)
    for f in ("wl_admit_ns", "wl_finish_ns", "wl_evictions", "wl_admit_cycle", "cq_usage", "wl_deactivated"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    assert np.array_equal(got.wl_pods_ready_at_ns, want.wl_pods_ready_at)
    assert np.array_equal(got.wl_pods_ready_count_out, want.wl_pods_ready_count)
    if want.wl_ready_ns is not None:
        assert np.array_equal(got.wl_ready_ns, want.wl_ready_ns)
        assert (got.n_check_ready, got.n_check_retry, got.n_check_rejected) == (want.n_check_ready, want.n_check_retry, want.n_check_rejected)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DEVICE_CASES))
def test_kb_run_drain_pods_ready_like_the_host_definition(name):
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = DEVICE_CASES[name]()
        mc = DEVICE_MAX_CYCLES.get(name, 100_000 if "baseline" in name else 400)
        want = _run(snap, mc)
        got = ev.run_drain(snap, abi.DrainOut(snap, mc, trace_capacity=want.n_decisions))
        compare(want, got)
        if name == "baseline-full":
            assert got.n_pods_ready_timeout > 0 and got.n_check_retry > 0 and got.n_resorts > 0
    finally:
        ev.close()


@pytest.fixture
def evaluator():
    from kueue_b200 import native
    ev = native.Evaluator(0)
    yield ev
    ev.close()


def _refused(ev, snap, match):
    """refused with KB_ERR_INVALID by the check whose message contains `match`"""
    from kueue_b200 import native
    with pytest.raises(native.KueueB200Error, match=match) as e:
        ev.run_drain(snap, max_cycles=5)
    assert e.value.code == abi.KB_ERR_INVALID


@pytest.mark.gpu
def test_refuses_tables_without_adm_wl(evaluator):
    s = ready_case(); del s.arrays["adm_wl"]
    _refused(evaluator, s, "pods ready: the tables need adm_wl")


@pytest.mark.gpu
def test_refuses_tables_without_the_delays(evaluator):
    s = ready_case(); del s.arrays["wl_pods_ready_ns"]
    _refused(evaluator, s, "pods ready: the tables need wl_pods_ready_ns")


@pytest.mark.gpu
@pytest.mark.parametrize("field", ["wl_pods_ready_ns", "wl_pods_ready_fail", "wl_pods_ready_count"])
def test_refuses_a_negative_delay_fail_or_count(evaluator, field):
    s = ready_case(); s.set(field, [-1, 0])
    _refused(evaluator, s, "pods ready: a negative delay, fail count or requeue count")


@pytest.mark.gpu
@pytest.mark.parametrize("attr,value,match", [
    ("pods_ready_timeout_ns", 0, "pods ready: timeout <= 0"),
    ("pods_ready_backoff_base_s", -1, "pods ready: backoff base < 0, max < 0 or limit < -1"),
    ("pods_ready_backoff_max_s", -1, "pods ready: backoff base < 0, max < 0 or limit < -1"),
    ("pods_ready_backoff_limit", -2, "pods ready: backoff base < 0, max < 0 or limit < -1"),
    ("pods_ready_requeue_creation", 2, "pods ready: pods_ready_requeue_creation is neither")])
def test_refuses_a_bad_setting(evaluator, attr, value, match):
    s = ready_case(); setattr(s, attr, value)
    _refused(evaluator, s, match)


@pytest.mark.gpu
def test_refuses_an_admitted_time_after_now(evaluator):
    s = start_state_case(); s.set("adm_admitted_ns", [S, I64_MIN])
    _refused(evaluator, s, "pods ready: adm_admitted_ns after now_ns")


@pytest.mark.gpu
def test_refuses_an_admitted_time_on_a_row_whose_checks_run(evaluator):
    s = start_state_case(); s.set("wl_check_ns", np.zeros(3)); s.set("adm_check_end_ns", [5 * S, I64_MIN])
    _refused(evaluator, s, "pods ready: adm_admitted_ns on a row whose checks run")


@pytest.mark.gpu
def test_refuses_an_admitted_time_on_an_evicting_row(evaluator):
    s = start_state_case()
    s.set("wl_evict_ns", np.full(3, S)); s.set("adm_evicted", [1, 0]); s.set("adm_evict_end_ns", [5 * S, I64_MIN])
    _refused(evaluator, s, "pods ready: adm_admitted_ns on a row whose eviction is under way")


@pytest.mark.gpu
def test_refuses_an_eviction_time_on_a_held_record(evaluator):
    s = start_state_case(); s.set("wl_pods_ready_evict_ns", [20 * S, I64_MIN, I64_MIN])
    _refused(evaluator, s, "pods ready: wl_pods_ready_evict_ns on a record that holds quota")


@pytest.mark.gpu
def test_refuses_two_eviction_times_on_one_record(evaluator):
    s = start_state_case(); s.set("wl_check_ns", np.zeros(3)); s.set("wl_check_evict_ns", [I64_MIN, I64_MIN, 20 * S])
    _refused(evaluator, s, "pods ready: a record with both wl_pods_ready_evict_ns and wl_check_evict_ns")
