"""Arrivals and completions in the drain (event mode of kb_run_drain; kueue_b200/drain.py).  CPU: the host definition
on the oracle against a hand-derived schedule, the plain drain and invariants; GPU: kb_run_drain equals the host
definition cycle by cycle."""
import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from kueue_b200.drain import ABSENT, FINISHED, HELD, NEVER, NoFitSets, drain

I64_MIN = np.iinfo(np.int64).min


def _run(snap, max_cycles=100_000, record=None):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000

    def cycle(s):
        out = oracle.run_cycle(s, cap)
        if record is not None:
            record.append((s, out))
        return out
    return drain(snap, cycle, max_cycles=max_cycles)


def _one_cq(n_wl, nominal=2, cpu=None, create=None, run=None, ts=None, hashes=None, strategy=abi.QUEUE_BEST_EFFORT_FIFO,
            lender=False):
    """One ClusterQueue without a cohort, one flavor, cpu only, no preemption; workloads of priority 0, UIDs in index
    order, wl_ts = create unless given.  lender: the ClusterQueue has no quota of its own and borrows `nominal` from a
    second ClusterQueue of its cohort (a request that does not fit is NoFit there, not Preempt)."""
    Q = 2 if lender else 1
    s = abi.FlatSnapshot(n_cq=Q, n_cohort=1 if lender else 0, n_flavor=1, n_resource=1)
    if lender:
        s.set("parent", [2, 2, -1]); s.set("nominal", [[0], [nominal], [0]])
    else:
        s.set("nominal", [[nominal]])
    s.set("cq_rg_start", np.arange(Q + 1)); s.set("rg_res_mask", np.ones(Q)); s.set("rg_flavor_start", np.arange(Q + 1))
    s.set("rg_flavors", np.zeros(Q)); s.set("cq_strategy", np.full(Q, strategy))
    s.set("wl_cq", np.zeros(n_wl)); s.set("wl_priority", np.zeros(n_wl)); s.set("wl_uid", np.arange(n_wl))
    s.set("wl_ts", create if ts is None else ts)
    s.set("ps_req", np.asarray(cpu if cpu is not None else [1] * n_wl)[:, None]); s.set("ps_req_mask", np.ones(n_wl))
    s.set("wl_create_ns", create); s.set("wl_run_ns", run)
    if hashes is not None:
        s.set("wl_sched_hash", hashes)
    s.now_ns, s.drain_cycle_ns = 0, 1
    return s.finalize()


def hand_case():
    return _one_cq(4, create=[0, 0, 3, 3], run=[10] * 4)


def test_hand_derived_schedule():
    """nominal 2 cpu, four 1-cpu workloads of run 10 created at 0, 0, 3, 3.  t=0: w0 admitted; t=1: w1 admitted; t=2: no
    head, the clock jumps to 3 where w2 and w3 arrive; t=3: w2 NoFit, set aside (a quiet cycle: wait for E = 10);
    t=10: w0 finishes and w2 is requeued, w2 admitted; t=11: w1 finishes, w3 admitted; jumps to 20 and 21."""
    r = _run(hand_case())
    assert r.cycles == 5
    assert r.cycle_start_ns == [0, 1, 3, 10, 11]
    assert [h.tolist() for h in r.heads] == [[0], [1], [2], [2], [3]]
    # w2 fits the nominal quota, so the assigner offers Preempt mode; without a policy there are no targets, and the
    # entry goes to the inadmissible set like a NoFit one
    assert [d.tolist() for d in r.decisions] == [[abi.DEC_ASSUMED], [abi.DEC_ASSUMED], [abi.DEC_PREEMPT_NO_TARGETS], [abi.DEC_ASSUMED],
                                                 [abi.DEC_ASSUMED]]
    assert r.wl_admit_ns.tolist() == [0, 1, 10, 11]
    assert r.wl_finish_ns.tolist() == [10, 11, 20, 21]
    assert r.end_ns == 21 and int(r.cq_usage.sum()) == 0
    assert [len(a) for a in r.arrived] == [0, 2, 0, 0, 0] and r.n_arrived == 2
    assert [f.tolist() for f in r.finished] == [[], [], [0], [1], [2, 3]] and r.n_finished == 4
    assert (r.state == FINISHED).all() and (r.wl_admit_cycle == -1).all()


# ---- degenerate tables: every run time < 0, every creation <= now_ns, no adm_finish_ns -> the plain drain
def _afs3():
    return synth.make_snapshot(3, W=1200, Q=40, afs=3)


DEGENERATE = {
    "cfg2-strict": lambda: synth.make_snapshot(2, W=1500, Q=30),
    "cfg3": lambda: synth.make_snapshot(3, W=1500, Q=40),
    "cfg3-afs": _afs3,
    "cfg4-evictable": lambda: synth.make_snapshot(4, W=600, Q=40, tight=1.2, evictable=True),
}


def _degenerate(snap):
    W = snap.n_wl
    snap.set("wl_create_ns", snap.now_ns - np.arange(W) % 3)
    snap.set("wl_run_ns", np.full(W, -1))
    snap.drain_cycle_ns = 0
    return snap


def _same_as_plain(want, got):
    assert got.cycles == want.cycles
    for k in range(want.cycles):
        assert np.array_equal(got.heads[k], want.heads[k]) and np.array_equal(got.decisions[k], want.decisions[k]), k
        assert np.array_equal(got.evicted[k], want.evicted[k]), k
    assert np.array_equal(got.cq_usage, want.cq_usage)
    assert np.array_equal(got.wl_admit_cycle, want.wl_admit_cycle)
    assert np.array_equal(got.wl_evictions, want.wl_evictions)


@pytest.mark.parametrize("name", list(DEGENERATE))
def test_degenerate_tables_change_nothing(name):
    want = _run(DEGENERATE[name](), 60)
    got = _run(_degenerate(DEGENERATE[name]()), 60)
    _same_as_plain(want, got)
    assert got.cycle_start_ns == [int(DEGENERATE[name]().now_ns) + c for c in range(got.cycles)]
    assert got.n_finished == 0 and got.n_arrived == 0


# ---- invariants on seeded event drains
def _hashes_with_arrivals():
    snap = synth.make_snapshot(3, W=1200, Q=30)
    snap.set("wl_sched_hash", np.random.default_rng(3).integers(0, 5, snap.n_wl))
    return synth.add_events(snap, seed=11, present=0.3, run_ns=(2_000, 30_000))


EVENT_CASES = {
    "cfg2": lambda: synth.add_events(synth.make_snapshot(2, W=1500, Q=30), seed=1),
    "cfg3-afs": lambda: synth.add_events(_afs3(), seed=2),
    "cfg4-evictable": lambda: synth.add_events(synth.make_snapshot(4, W=800, Q=40, tight=1.2, evictable=True), seed=3),
    "hashes-arrivals": _hashes_with_arrivals,
}


def _cells_of(adm, Q, FR):
    use = np.zeros((Q, FR), np.int64)
    st = adm["adm_use_start"]
    for a in range(len(adm["adm_cq"])):
        for k in range(int(st[a]), int(st[a + 1])):
            use[int(adm["adm_cq"][a]), int(adm["adm_use_fr"][k])] += int(adm["adm_use_qty"][k])
    return use


def check_invariants(snap, res):
    a = snap.arrays
    Q, FR = snap.n_cq, snap.n_fr
    init = {k: a[k] for k in ("adm_cq", "adm_use_start", "adm_use_fr", "adm_use_qty")}
    # usage conservation: the usage outside the admitted tables never changes, the rest is the live rows' cells
    assert np.array_equal(res.cq_usage - _cells_of(res.adm, Q, FR), a["cq_usage"].reshape(Q, FR) - _cells_of(init, Q, FR))
    create = a.get("wl_create_ns", np.full(snap.n_wl, snap.now_ns))
    run = a.get("wl_run_ns", np.full(snap.n_wl, -1))
    adm = res.wl_admit_ns != I64_MIN
    assert (res.wl_admit_ns[adm] >= create[adm]).all(), "a workload admitted before its creation"
    fin = res.wl_finish_ns != NEVER
    drain_fin = fin & adm  # finished after an admission in the drain (the others held a row of the snapshot)
    assert np.array_equal(res.wl_finish_ns[drain_fin], res.wl_admit_ns[drain_fin] + run[drain_fin]), "finish != last admit + run"
    assert np.array_equal(res.state == FINISHED, fin), "FINISHED is exactly the workloads with a finish time"
    assert (create[res.state == ABSENT] > res.end_ns).all(), "a workload created by the end is still absent"
    # a FINISHED workload is never evaluated again
    for k in range(res.cycles):
        t = res.cycle_start_ns[k]
        h = res.heads[k]
        assert not (fin[h] & (res.wl_finish_ns[h] <= t)).any(), k
        assert (create[h] <= t).all(), k
    assert all(b > x for x, b in zip(res.cycle_start_ns, res.cycle_start_ns[1:])), "clock not monotone"
    assert res.end_ns >= (res.cycle_start_ns[-1] if res.cycles else snap.now_ns)
    # completions: the finished workloads, plus the finished rows of the snapshot that name no record
    assert res.n_finished == int(fin.sum()) + int(sum((f < 0).sum() for f in res.finished))
    assert int((res.state == HELD).sum()) <= len(res.adm["adm_cq"])


@pytest.mark.parametrize("name", list(EVENT_CASES))
def test_event_drain_invariants(name):
    snap = EVENT_CASES[name]()
    res = _run(snap, 400)
    assert res.n_finished > 0 and res.n_admitted > 0
    if "wl_create_ns" in snap.arrays and (snap.arrays["wl_create_ns"] > snap.now_ns).any():
        assert res.n_arrived > 0
    check_invariants(snap, res)
    again = _run(EVENT_CASES[name](), 400)
    assert again.cycles == res.cycles and again.cycle_start_ns == res.cycle_start_ns
    for k in range(res.cycles):
        assert np.array_equal(again.heads[k], res.heads[k]) and np.array_equal(again.decisions[k], res.decisions[k])
    assert np.array_equal(again.wl_finish_ns, res.wl_finish_ns) and np.array_equal(again.cq_usage, res.cq_usage)


# ---- the NoFit set and arrivals
def test_nofit_sets():
    n = NoFitSets()
    assert not n.arrival_goes_aside(0, False, 5)
    n.insert(0, 5)
    assert n.arrival_goes_aside(0, False, 5)
    assert not n.arrival_goes_aside(0, True, 5), "StrictFIFO has no NoFit set"
    assert not n.arrival_goes_aside(0, False, 0), "an unknown hash"
    assert not n.arrival_goes_aside(1, False, 5), "the set is per ClusterQueue"
    n.clear(0)
    assert not n.arrival_goes_aside(0, False, 5)


def nofit_case(w0_run):
    """w0 (2 cpu, hash 7) fills the ClusterQueue at t=0; w1 (1 cpu, hash 5) is NoFit at t=1, so hash 5 joins the NoFit
    set; w2 (1 cpu, hash 5) is created at 2."""
    return _one_cq(3, cpu=[2, 1, 1], create=[0, 0, 2], run=[w0_run, 10, 10], hashes=[7, 5, 5], lender=True)


def test_arrival_of_a_nofit_class_is_set_aside():
    r = _run(nofit_case(100))
    assert r.decisions[1].tolist() == [abi.DEC_NOFIT]
    # t=2: w2 arrives straight into the inadmissible set (no head, the clock jumps on to 100 where w0 finishes)
    assert r.cycle_start_ns == [0, 1, 100, 101]
    assert [h.tolist() for h in r.heads] == [[0], [1], [1], [2]]
    assert r.wl_admit_ns.tolist() == [0, 100, 101]


def test_requeue_before_the_arrival_lets_it_in():
    # w0 finishes at 2, the time w2 arrives: the requeue clears the NoFit set, so w2 joins its queue whatever the order
    r = _run(nofit_case(2))
    assert r.cycle_start_ns == [0, 1, 2, 3]
    assert [h.tolist() for h in r.heads] == [[0], [1], [1], [2]]
    assert r.wl_admit_ns.tolist() == [0, 2, 3]


def test_nofit_arrival_waits_for_the_requeue_even_with_room_elsewhere():
    # without the hash, w2 would be queued at 2 and evaluated at once
    s = _one_cq(3, cpu=[2, 1, 1], create=[0, 0, 2], run=[100, 10, 10], hashes=[7, 5, 6], lender=True)
    r = _run(s)
    assert r.cycle_start_ns[:3] == [0, 1, 2] and r.heads[2].tolist() == [2]


# ---- the reference's baseline scenario
def test_baseline_scenario_runs_to_the_end():
    snap = synth.perf_scenario(0.1)
    assert snap.n_wl == 1500 and synth.perf_scenario().n_wl == 15_000
    res = _run(snap)
    assert res.n_finished == snap.n_wl and (res.state == FINISHED).all()
    assert res.n_arrived == snap.n_wl and len(res.adm["adm_cq"]) == 0 and int(res.cq_usage.sum()) == 0
    check_invariants(snap, res)
    print(f"baseline x0.1: {res.cycles} cycles, {res.n_admitted} admissions, {res.n_evicted} preemptions replayed, "
          f"end {res.end_ns / 1e9:.3f} s")
    assert res.n_evicted > 0, "the scenario replays preemptions"


def test_run_time_zero_finishes_at_the_boundary_of_its_admission():
    s = _one_cq(3, create=[0, 0, 0], run=[0, 0, 0], nominal=1)
    r = _run(s)
    assert r.cycle_start_ns == [0, 1, 2] and r.wl_admit_ns.tolist() == [0, 1, 2] and r.wl_finish_ns.tolist() == [0, 1, 2]
    assert len(r.adm["adm_cq"]) == 0


def adm_finish_without_adm_wl():
    snap = synth.make_snapshot(3, W=1200, Q=40, admitted=300)
    snap.set("adm_finish_ns", snap.now_ns + 1 + np.arange(snap.n_adm) * 3)
    snap.drain_cycle_ns = 2
    return snap


def test_adm_finish_without_adm_wl():
    snap = adm_finish_without_adm_wl()
    res = _run(snap, 300)
    assert res.n_finished == snap.n_adm and (res.wl_finish_ns == NEVER).all()
    check_invariants(snap, res)


# ---------------------------------------------------------------------------------------------------------------- GPU
DEVICE_CASES = {
    "hand": hand_case,
    "nofit-aside": lambda: nofit_case(100),
    "nofit-requeue": lambda: nofit_case(2),
    "run-zero": lambda: _one_cq(3, create=[0, 0, 0], run=[0, 0, 0], nominal=1),
    "adm-finish-without-adm-wl": adm_finish_without_adm_wl,
    "cfg2": EVENT_CASES["cfg2"],
    "cfg3-afs": EVENT_CASES["cfg3-afs"],
    "cfg4-evictable": EVENT_CASES["cfg4-evictable"],
    "hashes-arrivals": _hashes_with_arrivals,
    "cfg4-degenerate": DEGENERATE["cfg4-evictable"],
    "baseline": lambda: synth.perf_scenario(1.0),
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
    assert got.n_finished == want.n_finished and got.n_arrived == want.n_arrived and got.end_ns == want.end_ns
    assert np.array_equal(got.wl_admit_ns, want.wl_admit_ns)
    assert np.array_equal(got.wl_finish_ns, want.wl_finish_ns)
    assert np.array_equal(got.wl_evictions, want.wl_evictions)
    assert np.array_equal(got.wl_admit_cycle, want.wl_admit_cycle)
    assert np.array_equal(got.cq_usage, want.cq_usage)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DEVICE_CASES))
def test_kb_run_drain_events_like_the_host_definition(name):
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = DEVICE_CASES[name]()
        if name == "cfg4-degenerate":
            snap = _degenerate(snap)
        mc = 100_000 if name == "baseline" else 400
        want = _run(snap, mc)
        got = ev.run_drain(snap, abi.DrainOut(snap, mc, trace_capacity=want.n_decisions))
        compare(want, got)
    finally:
        ev.close()


@pytest.mark.gpu
def test_kb_run_drain_full_size_config3_events():
    """cfg3 at full size with seeded events, on the device alone: usage conservation, admit >= create, finish = admit +
    run, and every workload is finished, holding quota or still pending."""
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = synth.add_events(synth.make_snapshot(3), seed=7, span_ns=200_000, step_ns=2_000)
        got = ev.run_drain(snap, max_cycles=300)
        a = snap.arrays
        assert got.n_finished > 0 and got.n_arrived > 0
        adm = got.wl_admit_ns != I64_MIN
        assert (got.wl_admit_ns[adm] >= a["wl_create_ns"][adm]).all()
        fin = got.wl_finish_ns != NEVER
        assert (fin <= adm).all()
        assert np.array_equal(got.wl_finish_ns[fin], got.wl_admit_ns[fin] + a["wl_run_ns"][fin])
        held = got.wl_admit_cycle >= 0
        assert not (held & fin).any()
        # rows of the snapshot without a record finish too: completions = finished workloads + finished snapshot rows
        assert got.n_finished == int(fin.sum()) + int((a["adm_finish_ns"] <= got.end_ns).sum())
        pending = ~fin & ~held
        assert int(fin.sum()) + int(held.sum()) + int(pending.sum()) == snap.n_wl
        print(f"cfg3 events: {got.n_cycles} cycles, {got.n_admitted} admitted, {got.n_finished} finished, "
              f"{got.n_arrived} arrived, {got.gpu_ms / max(1, got.n_cycles):.3f} ms/cycle")
    finally:
        ev.close()


@pytest.mark.gpu
def test_kb_run_drain_refuses_bad_event_tables():
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = synth.add_events(synth.make_snapshot(4, W=300, Q=20, evictable=True), seed=1)
        fin = snap.arrays["adm_finish_ns"].copy()
        fin[3] = snap.now_ns
        snap.set("adm_finish_ns", fin)
        with pytest.raises(native.KueueB200Error) as e:
            ev.run_drain(snap, max_cycles=5)
        assert e.value.code == abi.KB_ERR_INVALID
        snap = synth.add_events(synth.make_snapshot(4, W=300, Q=20, evictable=True), seed=1)
        cr = snap.arrays["wl_create_ns"].copy()
        cr[snap.arrays["adm_wl"][0]] = snap.now_ns + 1
        snap.set("wl_create_ns", cr)
        with pytest.raises(native.KueueB200Error) as e:
            ev.run_drain(snap, max_cycles=5)
        assert e.value.code == abi.KB_ERR_INVALID
    finally:
        ev.close()
