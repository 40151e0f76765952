"""Eviction latency in the drain's event mode (kb_snapshot.wl_evict_ns / adm_evict_end_ns; kueue_b200/drain.py).  An
eviction is issued at once and releases its quota on the clock.  CPU: the host definition on the oracle against
hand-derived schedules, the degenerate latency against the drain without the table, and invariants; GPU: kb_run_drain
equals the host definition cycle by cycle, and refuses bad tables."""
import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from kueue_b200.drain import FINISHED, HELD, NEVER, QUEUED, drain

I64_MAX = np.iinfo(np.int64).max


def _run(snap, max_cycles=100_000, record=None):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000

    def cycle(s):
        out = oracle.run_cycle(s, cap)
        if record is not None:
            record.append((s, out))
        return out
    return drain(snap, cycle, max_cycles=max_cycles)


def _cq_case(prio, cpu, create=None, evict_ns=5, adm_evicted=False, adm_evict_end=None, within=abi.POLICY_LOWER_PRIORITY,
             now=0):
    """One ClusterQueue of 2 cpu without a cohort, withinClusterQueue `within`, BestEffortFIFO.  Pending workload 0 is
    "low" (priority -1, 2 cpu), admitted before the drain (adm_wl names it); the others are pending with `prio` / `cpu`.
    One cycle takes 1 ns; no workload ever finishes."""
    W = 1 + len(prio)
    s = abi.FlatSnapshot(n_cq=1, n_cohort=0, n_flavor=1, n_resource=1)
    s.set("nominal", [[2]])
    s.set("cq_rg_start", [0, 1]); s.set("rg_res_mask", [1]); s.set("rg_flavor_start", [0, 1]); s.set("rg_flavors", [0])
    s.set("cq_strategy", [abi.QUEUE_BEST_EFFORT_FIFO]); s.set("cq_within_cq", [within])
    s.set("wl_cq", np.zeros(W)); s.set("wl_priority", [-1] + list(prio)); s.set("wl_uid", np.arange(W))
    s.set("wl_ts", np.arange(W))
    s.set("ps_req", np.asarray([2] + list(cpu))[:, None]); s.set("ps_req_mask", np.ones(W))
    s.set("adm_cq", [0]); s.set("adm_priority", [-1]); s.set("adm_ts", [0]); s.set("adm_qr_ts", [0]); s.set("adm_uid", [100])
    s.set("adm_evicted", [int(adm_evicted)])
    s.set("adm_use_start", [0, 1]); s.set("adm_use_fr", [0]); s.set("adm_use_qty", [2]); s.set("cq_usage", [[2]])
    s.set("adm_wl", [0])
    if create is not None:
        s.set("wl_create_ns", create)
    s.set("wl_evict_ns", np.full(W, evict_ns))
    if adm_evict_end is not None:
        s.set("adm_evict_end_ns", [adm_evict_end])
    s.now_ns, s.drain_cycle_ns = now, 1
    return s.finalize()


def skips_duplicate_case():
    """TestIssuePreemptionsSkipsDuplicate (preemption_test.go:4401) on the clock: "low" (0) and "in" (1, priority 1)."""
    return _cq_case([1], [2])


def test_issue_then_ongoing_then_release():
    """t=0: "in" preempts "low", the eviction is issued (end 0 + 5).  t=1: "in" targets "low" again, the eviction is under
    way: nothing is issued and the cycle is quiet, so the clock waits for E = 5.  At 5 low's quota is released and low
    is queued again; "in" (priority 1) is the head and is admitted.  t=6: low is evaluated and finds no target (a
    priority-1 workload cannot be preempted by a priority -1 one): the cycle is quiet and nothing is left to wait for."""
    r = _run(skips_duplicate_case())
    assert r.cycle_start_ns == [0, 1, 5, 6]
    assert [h.tolist() for h in r.heads] == [[1], [1], [1], [0]]
    assert [d.tolist() for d in r.decisions[:3]] == [[abi.DEC_PREEMPTING], [abi.DEC_PREEMPTING], [abi.DEC_ASSUMED]]
    assert r.decisions[3].tolist() in ([abi.DEC_PREEMPT_NO_TARGETS], [abi.DEC_NOFIT])
    assert [e.tolist() for e in r.evicted] == [[0], [], [], []] and r.n_evicted == 1
    assert [e.tolist() for e in r.evict_done] == [[], [0], [], []] and r.n_evict_done == 1
    assert r.wl_evictions.tolist() == [1, 0]
    assert r.wl_admit_ns.tolist() == [np.iinfo(np.int64).min, 5] and r.wl_admit_cycle.tolist() == [-1, 2]
    assert r.cq_usage.tolist() == [[2]] and r.end_ns == 6
    assert r.adm["adm_wl"].tolist() == [1] and r.adm["adm_evicting"].tolist() == [False]


def test_second_preemptor_retargets_the_evicting_row():
    """"in1" (priority 1) issues the eviction of "low" at 0.  "in2" (priority 2) is created at 2 and becomes the head: it
    targets "low" too, whose eviction is under way, so it issues nothing and waits.  At 5 the quota is released and
    in2, ordered first, takes it; in1 then finds no target."""
    r = _run(_cq_case([1, 2], [2, 2], create=[0, 0, 2]))
    assert r.cycle_start_ns == [0, 1, 2, 5, 6]
    assert [h.tolist() for h in r.heads] == [[1], [1], [2], [2], [1]]
    assert [int(d[0]) for d in r.decisions[:4]] == [abi.DEC_PREEMPTING] * 3 + [abi.DEC_ASSUMED]
    assert [e.tolist() for e in r.evicted] == [[0], [], [], [], []]
    assert [e.tolist() for e in r.evict_done] == [[], [], [0], [], []]
    assert [a.tolist() for a in r.arrived] == [[], [2], [], [], []]
    assert r.wl_evictions.tolist() == [1, 0, 0]
    assert r.wl_admit_ns[2] == 5 and r.state[2] == HELD and r.state[0] == QUEUED


def test_eviction_under_way_before_the_drain_completes_untargeted():
    """"low" carries adm_evicted with an end time of 3; "in" (priority 0) cannot preempt (policy Never) and is set aside
    at 0.  At 3 the eviction completes without a cycle targeting it: the quota is released and the root tree's
    set-aside workloads are requeued, so "in" is admitted at 3."""
    r = _run(_cq_case([0], [2], adm_evicted=True, adm_evict_end=3, within=abi.POLICY_NEVER))
    assert r.cycle_start_ns == [0, 3, 4]
    assert [h.tolist() for h in r.heads] == [[1], [1], [0]]
    assert int(r.decisions[1][0]) == abi.DEC_ASSUMED
    assert r.n_evicted == 0 and r.n_evict_done == 1 and [e.tolist() for e in r.evict_done] == [[0], [], []]
    assert r.wl_evictions.tolist() == [0, 0]


def test_eviction_under_way_before_the_drain_is_ongoing_when_targeted():
    """the same row targeted by "in" (priority 1): the eviction under way counts as ongoing, nothing is issued, and the
    quiet cycle waits for its end at 3"""
    r = _run(_cq_case([1], [2], adm_evicted=True, adm_evict_end=3))
    assert r.cycle_start_ns == [0, 3, 4]
    assert int(r.decisions[0][0]) == abi.DEC_PREEMPTING and int(r.decisions[1][0]) == abi.DEC_ASSUMED
    assert r.n_evicted == 0 and r.n_evict_done == 1


def test_eviction_before_the_drain_without_end_times_is_issued_when_targeted():
    r = _run(_cq_case([1], [2], adm_evicted=True))
    assert r.cycle_start_ns == [0, 1, 5, 6] and r.n_evicted == 1 and r.n_evict_done == 1


def test_end_time_saturates():
    """now_ns 10 and a latency of INT64_MAX - 5: the end time saturates at INT64_MAX, the eviction never completes and
    the drain ends after the quiet cycle that finds it under way"""
    r = _run(_cq_case([1], [2], evict_ns=I64_MAX - 5, now=10))
    assert r.cycle_start_ns == [10, 11]
    assert [e.tolist() for e in r.evicted] == [[0], []] and r.n_evict_done == 0
    assert r.adm["adm_finish_ns"].tolist() == [NEVER] and r.adm["adm_evicting"].tolist() == [True]
    assert r.adm["adm_evicted"].tolist() == [1] and r.state[0] == HELD and r.cq_usage.tolist() == [[2]]


# ---- degenerate latency: every wl_evict_ns <= max(drain_cycle_ns, 1), no adm_evict_end_ns -> the drain without it
def _cfg2():
    return synth.add_events(synth.make_snapshot(2, W=600, Q=12, preemption=True, tight=1.3, evictable=True), seed=1)


def _cfg3_afs():
    snap = synth.add_events(synth.make_snapshot(3, W=1200, Q=40, afs=3), seed=2)
    snap.set("adm_wl", np.zeros(0))
    return snap


def _cfg4():
    return synth.add_events(synth.make_snapshot(4, W=800, Q=40, tight=1.6, evictable=True), seed=3)


def _baseline():
    return synth.perf_scenario(0.1)


BASE = {"cfg2": _cfg2, "cfg3-afs": _cfg3_afs, "cfg4-evictable": _cfg4, "baseline": _baseline}
MAX_CYCLES = {"cfg2": 200, "cfg3-afs": 200, "cfg4-evictable": 200, "baseline": 100_000}


def _degenerate(snap, seed=0):
    step = max(1, int(snap.drain_cycle_ns))
    return synth.add_evict_latency(snap, (0, step), seed)


def _same(want, got):
    assert got.cycles == want.cycles
    assert got.cycle_start_ns == want.cycle_start_ns
    for k in range(want.cycles):
        assert np.array_equal(got.heads[k], want.heads[k]) and np.array_equal(got.decisions[k], want.decisions[k]), k
        assert np.array_equal(got.evicted[k], want.evicted[k]), k
        assert np.array_equal(got.finished[k], want.finished[k]) and np.array_equal(got.arrived[k], want.arrived[k]), k
    assert np.array_equal(got.cq_usage, want.cq_usage)
    for f in ("wl_admit_cycle", "wl_evictions", "wl_admit_ns", "wl_finish_ns", "state"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    assert got.n_evict_done == want.n_evicted and got.end_ns == want.end_ns


@pytest.mark.parametrize("name", list(BASE))
def test_degenerate_latency_changes_nothing(name):
    want = _run(BASE[name](), MAX_CYCLES[name])
    got = _run(_degenerate(BASE[name]()), MAX_CYCLES[name])
    _same(want, got)
    if name in ("cfg2", "cfg4-evictable", "baseline"):
        assert want.n_evicted > 0
    if name == "cfg4-evictable":
        assert BASE[name]().arrays["adm_evicted"].any(), "rows evicted before the drain are issued like any other"


# ---- invariants with latencies longer than a cycle
def _cfg4_latency():
    return synth.add_evict_latency(_cfg4(), (3_000, 40_000), seed=4)


def _baseline_latency():
    return synth.perf_scenario(0.1, evict_ns=30 * 1_000_000)


LATENCY = {"cfg4-evictable": _cfg4_latency, "baseline": _baseline_latency}


def _cells_of(adm, Q, FR):
    use = np.zeros((Q, FR), np.int64)
    st = adm["adm_use_start"]
    for a in range(len(adm["adm_cq"])):
        for k in range(int(st[a]), int(st[a + 1])):
            use[int(adm["adm_cq"][a]), int(adm["adm_use_fr"][k])] += int(adm["adm_use_qty"][k])
    return use


def check_latency_invariants(snap, res):
    a = snap.arrays
    Q, FR = snap.n_cq, snap.n_fr
    init = {k: a[k] for k in ("adm_cq", "adm_use_start", "adm_use_fr", "adm_use_qty")}
    # usage conservation: evicting rows keep their cells until the release
    assert np.array_equal(res.cq_usage - _cells_of(res.adm, Q, FR), a["cq_usage"].reshape(Q, FR) - _cells_of(init, Q, FR))
    # every issued eviction completed or is still under way
    assert res.n_evicted == res.n_evict_done + int(res.adm["adm_evicting"].sum())
    assert res.n_evicted == int(res.wl_evictions.sum())
    # an evicting record is never finished nor evaluated until its release
    under_way = set()
    for k in range(res.cycles):
        assert not under_way & set(res.heads[k].tolist()), k
        under_way |= set(res.evicted[k].tolist())
        assert not under_way & set(res.finished[k].tolist()), k
        assert set(res.evict_done[k].tolist()) <= under_way, k
        under_way -= set(res.evict_done[k].tolist())
    assert under_way == set(res.adm["adm_wl"][res.adm["adm_evicting"]].tolist())
    assert (res.adm["adm_evicted"][res.adm["adm_evicting"]] == 1).all()
    assert not (res.state[list(under_way)] != HELD).any()


@pytest.mark.parametrize("name", list(LATENCY))
def test_latency_invariants(name):
    snap = LATENCY[name]()
    res = _run(snap, MAX_CYCLES[name])
    assert res.n_evicted > 0 and res.n_evict_done > 0
    check_latency_invariants(snap, res)
    if name == "baseline":
        assert res.n_finished == snap.n_wl and (res.state == FINISHED).all(), "the scenario runs to the end"
        plain = _run(_baseline(), MAX_CYCLES[name])
        print(f"baseline x0.1: {res.cycles} cycles with a 30 ms termination latency, {plain.cycles} without; "
              f"evictions {res.n_evicted} / {plain.n_evicted}; end {res.end_ns / 1e9:.3f} s / {plain.end_ns / 1e9:.3f} s")


# ---------------------------------------------------------------------------------------------------------------- GPU
DEVICE_CASES = {
    "skips-duplicate": skips_duplicate_case,
    "second-preemptor": lambda: _cq_case([1, 2], [2, 2], create=[0, 0, 2]),
    "before-drain-untargeted": lambda: _cq_case([0], [2], adm_evicted=True, adm_evict_end=3, within=abi.POLICY_NEVER),
    "before-drain-ongoing": lambda: _cq_case([1], [2], adm_evicted=True, adm_evict_end=3),
    "before-drain-issued": lambda: _cq_case([1], [2], adm_evicted=True),
    "saturates": lambda: _cq_case([1], [2], evict_ns=I64_MAX - 5, now=10),
    "cfg4-latency": _cfg4_latency,
    "cfg4-latency-end-times": lambda: _with_end_times(_cfg4_latency()),
    "baseline-latency": lambda: synth.perf_scenario(1.0, evict_ns=30 * 1_000_000),
    "degenerate-cfg2": lambda: _degenerate(_cfg2()),
    "degenerate-cfg3-afs": lambda: _degenerate(_cfg3_afs()),
    "degenerate-cfg4": lambda: _degenerate(_cfg4()),
    "degenerate-baseline": lambda: _degenerate(synth.perf_scenario(1.0)),
}


def _with_end_times(snap):
    """end times for the rows evicted before the drain, seeded after now_ns"""
    rng = np.random.default_rng(9)
    snap.set("adm_evict_end_ns", snap.now_ns + rng.integers(1, 20_000, snap.n_adm))
    return snap


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
    assert got.n_evicted == want.n_evicted and got.n_evict_done == want.n_evict_done
    assert got.n_finished == want.n_finished and got.n_arrived == want.n_arrived and got.end_ns == want.end_ns
    for f in ("wl_admit_ns", "wl_finish_ns", "wl_evictions", "wl_admit_cycle", "cq_usage"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DEVICE_CASES))
def test_kb_run_drain_evict_latency_like_the_host_definition(name):
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = DEVICE_CASES[name]()
        mc = 100_000 if "baseline" in name else 400
        want = _run(snap, mc)
        got = ev.run_drain(snap, abi.DrainOut(snap, mc, trace_capacity=want.n_decisions))
        compare(want, got)
        if name == "baseline-latency":
            assert got.n_finished == snap.n_wl and got.n_evict_done == got.n_evicted > 0
    finally:
        ev.close()


@pytest.mark.gpu
def test_kb_run_drain_refuses_bad_latency_tables():
    from kueue_b200 import native
    ev = native.Evaluator(0)

    def refused(snap):
        with pytest.raises(native.KueueB200Error) as e:
            ev.run_drain(snap, max_cycles=5)
        assert e.value.code == abi.KB_ERR_INVALID

    try:
        no_adm_wl = skips_duplicate_case()
        del no_adm_wl.arrays["adm_wl"]
        refused(no_adm_wl)                                       # wl_evict_ns without adm_wl
        ends_only = _cq_case([1], [2], adm_evicted=True, adm_evict_end=3)
        del ends_only.arrays["adm_wl"]
        del ends_only.arrays["wl_evict_ns"]
        refused(ends_only)                                       # adm_evict_end_ns without adm_wl
        no_lat = _cq_case([1], [2], adm_evicted=True, adm_evict_end=3)
        del no_lat.arrays["wl_evict_ns"]
        refused(no_lat)                                          # adm_evict_end_ns without wl_evict_ns
        refused(_cq_case([1], [2], evict_ns=-1))                 # wl_evict_ns < 0
        refused(_cq_case([1], [2], adm_evicted=True, adm_evict_end=0))  # an end at or before now_ns
        ok = _cq_case([1], [2], adm_evicted=False, adm_evict_end=0)     # read only where adm_evicted is set
        assert ev.run_drain(ok, max_cycles=5).n_evicted == 1
    finally:
        ev.close()
