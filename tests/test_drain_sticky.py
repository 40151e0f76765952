"""The sticky workload in kb_run_drain (kb_snapshot.cq_sticky; kueue_b200/drain.py).  A BestEffortFIFO ClusterQueue keeps a
preemptor that waits for its evictions at its head until it is admitted.  CPU: the host definition on the oracle against
hand-derived schedules, the degenerate equivalences (a)-(c) of the header against the drain without the table, and
invariants on seeded drains; GPU: kb_run_drain equals the host definition cycle by cycle, final slots included, and
refuses bad tables."""
import numpy as np
import pytest

import oracle
from kueue_b200 import abi, shard, synth
from kueue_b200.drain import FINISHED, HELD, drain
from tests.test_drain_evict_latency import _cq_case, check_latency_invariants

MS = 1_000_000


def _run(snap, max_cycles=100_000):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000
    return drain(snap, lambda s: oracle.run_cycle(s, cap), max_cycles=max_cycles)


def _sticky(snap, slots=None):
    """the snapshot with the table: every slot -1 unless `slots` are given"""
    snap.set("cq_sticky", np.full(snap.n_cq, -1) if slots is None else slots)
    return snap


def second_preemptor(strategy=abi.QUEUE_BEST_EFFORT_FIFO):
    """the "second preemptor" case of the eviction-latency tests: "low" (0, priority -1) holds the ClusterQueue's 2 cpu;
    "in1" (1, priority 1) and "in2" (2, priority 2, created at 2) want 2 cpu each; every eviction takes 5 ns"""
    snap = _cq_case([1, 2], [2, 2], create=[0, 0, 2])
    snap.set("cq_strategy", [strategy])
    return snap


def test_sticky_preemptor_keeps_the_head():
    """t=0: in1 preempts low (end 5) and becomes the sticky workload.  t=1: in1 re-targets the evicting row: quiet, the
    clock waits for in2's creation.  t=2: in2 (priority 2) sorts first, but in1 is sticky and keeps the head; quiet, wait
    for E = 5.  At 5 low is released, in1 takes the quota and the slot is cleared.  t=6: in2 preempts in1 (end 11) and
    becomes sticky; t=7 re-targets, quiet, wait for 11.  At 11 in1 is released and in2 is admitted (slot cleared).
    t=12: in1 finds no target (a priority-2 workload) and nothing is left to wait for.  Without the table in2 takes the
    quota at 5 (test_second_preemptor_retargets_the_evicting_row)."""
    r = _run(_sticky(second_preemptor(), [-1]))
    assert r.cycle_start_ns == [0, 1, 2, 5, 6, 7, 11, 12]
    assert [h.tolist() for h in r.heads] == [[1], [1], [1], [1], [2], [2], [2], [1]]
    P, A = abi.DEC_PREEMPTING, abi.DEC_ASSUMED
    assert [int(d[0]) for d in r.decisions[:7]] == [P, P, P, A, P, P, A]
    assert int(r.decisions[7][0]) in (abi.DEC_PREEMPT_NO_TARGETS, abi.DEC_NOFIT)
    assert [e.tolist() for e in r.evicted] == [[0], [], [], [], [1], [], [], []]
    assert [e.tolist() for e in r.evict_done] == [[], [], [0], [], [], [1], [], []]
    assert r.wl_evictions.tolist() == [1, 1, 0]
    assert r.wl_admit_ns[1:].tolist() == [5, 11]
    assert r.cq_sticky.tolist() == [-1]
    assert [h.tolist() for h in r.sticky_heads] == [[], [], [1], [1], [], [], [], []]


def test_seeded_sticky_workload_is_the_head():
    """in1 is the sticky workload at the start and in2 (priority 2) exists at 0: in1 is still the head at 0"""
    snap = _cq_case([1, 2], [2, 2], create=[0, 0, 0])
    r = _run(_sticky(snap, [1]))
    assert r.heads[0].tolist() == [1] and r.sticky_heads[0].tolist() == [1]
    assert int(r.decisions[0][0]) == abi.DEC_PREEMPTING
    plain = _run(_cq_case([1, 2], [2, 2], create=[0, 0, 0]))
    assert plain.heads[0].tolist() == [2]


def _same(want, got):
    """heads, decisions, evictions, events, usage and per-workload results"""
    assert got.cycles == want.cycles
    assert got.cycle_start_ns == want.cycle_start_ns
    for k in range(want.cycles):
        assert np.array_equal(got.heads[k], want.heads[k]) and np.array_equal(got.decisions[k], want.decisions[k]), k
        assert np.array_equal(got.evicted[k], want.evicted[k]) and np.array_equal(got.evict_done[k], want.evict_done[k]), k
        assert np.array_equal(got.finished[k], want.finished[k]) and np.array_equal(got.arrived[k], want.arrived[k]), k
    assert np.array_equal(got.cq_usage, want.cq_usage)
    for f in ("wl_admit_cycle", "wl_evictions", "wl_admit_ns", "wl_finish_ns", "state"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    assert got.end_ns == want.end_ns
    if got.lq_consumed is not None:
        assert np.array_equal(got.lq_consumed, want.lq_consumed) and np.array_equal(got.lq_last_update_ns, want.lq_last_update_ns)


def test_strict_fifo_second_preemptor_is_the_drain_without_the_table():
    want = _run(second_preemptor(abi.QUEUE_STRICT_FIFO))
    got = _run(_sticky(second_preemptor(abi.QUEUE_STRICT_FIFO)))
    _same(want, got)
    assert not any(len(h) for h in got.sticky_heads) and got.cq_sticky.tolist() == [-1]


# ---- a classical restatement of kueue#6929 ("workload which fits behind ClusterQueue head", fair_sharing_test.go:841)
def fits_behind_head():
    """Nodes: cq1 (0), cq2 (1), cohort "a" (2) with 3 cpu under cohort "root" (3).  cq1 (in a) and cq2 (in root) have
    nominal 0, reclaimWithinCohort Any, withinClusterQueue LowerPriority, BestEffortFIFO; the classical scheduler (no
    fair sharing).  cq2 borrows two 1-cpu workloads (records 0 and 1, admitted before the drain).  In cq1 "big" (2, 4 cpu,
    priority 999) exists at 0 and "fits" (3, 3 cpu, priority 0) is created at 1.  Every eviction takes 5 ns; one cycle
    takes 1 ns; nothing finishes."""
    s = abi.FlatSnapshot(n_cq=2, n_cohort=2, n_flavor=1, n_resource=1)
    s.flags = abi.FLAGS_DEFAULT & ~abi.F_FAIR_SHARING
    s.set("parent", [2, 3, 3, -1])
    s.set("nominal", [[0], [0], [3000], [0]])
    s.set("cq_rg_start", [0, 1, 2]); s.set("rg_res_mask", [1, 1]); s.set("rg_flavor_start", [0, 1, 2]); s.set("rg_flavors", [0, 0])
    s.set("cq_strategy", [abi.QUEUE_BEST_EFFORT_FIFO] * 2)
    s.set("cq_within_cq", [abi.POLICY_LOWER_PRIORITY] * 2); s.set("cq_reclaim_within", [abi.POLICY_ANY] * 2)
    s.set("wl_cq", [1, 1, 0, 0]); s.set("wl_priority", [0, 0, 999, 0])
    s.set("wl_ts", [0, 1, 2, 3]); s.set("wl_uid", [0, 1, 2, 3])
    s.set("ps_req", [[1000], [1000], [4000], [3000]]); s.set("ps_req_mask", np.ones(4))
    s.set("adm_cq", [1, 1]); s.set("adm_priority", [0, 0]); s.set("adm_ts", [0, 1]); s.set("adm_qr_ts", [0, 0])
    s.set("adm_uid", [0, 1]); s.set("adm_evicted", [0, 0])
    s.set("adm_use_start", [0, 1, 2]); s.set("adm_use_fr", [0, 0]); s.set("adm_use_qty", [1000, 1000])
    s.set("cq_usage", [[0], [2000]])
    s.set("adm_wl", [0, 1])
    s.set("wl_create_ns", [0, 0, 0, 1])
    s.set("wl_evict_ns", np.full(4, 5))
    s.now_ns, s.drain_cycle_ns = 0, 1
    return s.finalize()


def test_fits_behind_the_head():
    """t=0: big (4 cpu > the 3 of the tree) is NoFit and set aside; quiet, wait for fits' creation.  t=1: fits reclaims
    cohort a's quota from cq2's borrowing workloads (both evictions end at 6) and becomes cq1's sticky workload; t=2 it
    re-targets them: quiet, wait for 6.  At 6 both evictions complete: records 0 and 1 return to cq2's queue, and the
    root tree's requeue returns big to cq1's.
      with the table: fits is still cq1's head at 6 and is admitted.  The classical iterator orders it before record 0:
      the lowest subtree fits fits in is cohort a (height 1), record 0's is root (height 2; Assignment.Borrows,
      FindHeightOfLowestSubtreeThatFits hierarchical_preemption.go:214).  Record 0 then no longer fits and is skipped.
      The slot is cleared.  t=7: big and record 0 are NoFit and set aside, and the drain ends.
      without it: big (priority 999) takes cq1's head at 6 and is set aside again while record 0 borrows 1 cpu; at 7
      fits reclaims from record 0 (end 12), at 8 it waits, at 12 the release requeues big, and the three cycles repeat
      every 6 ns: fits is never admitted (the livelock kueue#6929 reports).
    Left out: the mid-run quota change of "sticky workload becomes inadmissible" (:866) and the deletion of "sticky
    workload deleted" (:918): a drain has no spec changes and no deletions."""
    N, P, A, S = abi.DEC_NOFIT, abi.DEC_PREEMPTING, abi.DEC_ASSUMED, abi.DEC_SKIPPED_NO_FIT
    r = _run(_sticky(fits_behind_head()))
    assert r.cycle_start_ns == [0, 1, 2, 6, 7]
    assert [h.tolist() for h in r.heads] == [[2], [3], [3], [3, 0], [2, 0]]
    assert [d.tolist() for d in r.decisions] == [[N], [P], [P], [A, S], [N, N]]
    assert [e.tolist() for e in r.evicted] == [[], [0, 1], [], [], []]
    assert [e.tolist() for e in r.evict_done] == [[], [], [0, 1], [], []]
    assert [h.tolist() for h in r.sticky_heads] == [[], [], [], [3], []]
    assert r.wl_admit_ns[3] == 6 and r.state[3] == HELD and r.cq_sticky.tolist() == [-1, -1]
    plain = _run(fits_behind_head(), 30)
    assert plain.cycle_start_ns[:6] == [0, 1, 2, 6, 7, 8]
    assert [h.tolist() for h in plain.heads[:6]] == [[2], [3], [3], [2, 0], [3, 1], [3, 1]]
    assert [d.tolist() for d in plain.decisions[:6]] == [[N], [P], [P], [N, A], [P, S], [P, S]]
    for k in range(6, 30):  # from t=6 the period: big's cycle, the reclaim, the wait
        assert plain.cycle_start_ns[k] == plain.cycle_start_ns[k - 3] + 6
        assert np.array_equal(plain.heads[k], plain.heads[k - 3]) and np.array_equal(plain.decisions[k], plain.decisions[k - 3])
    assert plain.wl_admit_ns[3] == np.iinfo(np.int64).min


# ---- the degenerate equivalences: every slot -1 at the start and (a) no adm_wl and no event table, (b) every ClusterQueue
# StrictFIFO, or (c) no preemption policy -> the drain without the table
def _no_policy(snap):
    for nm in ("cq_within_cq", "cq_reclaim_within", "cq_borrow_within"):
        snap.set(nm, np.full(snap.n_cq, abi.POLICY_NEVER))
    return snap


def _cfg3_afs_events():
    snap = synth.add_events(synth.make_snapshot(3, W=1200, Q=40, afs=3), seed=2)
    snap.set("adm_wl", np.zeros(0))
    return snap


DEGENERATE = {
    "a-cfg2": lambda: synth.make_snapshot(2, W=1500, Q=30, preemption=True, tight=1.2),
    "a-cfg4": lambda: synth.make_snapshot(4, W=2000, Q=100, tight=1.06),
    "b-cfg2-evictable-events": lambda: synth.add_events(synth.make_snapshot(2, W=600, Q=12, preemption=True, tight=1.3,
                                                                            evictable=True), seed=1),
    "c-cfg3-afs-events": _cfg3_afs_events,
    "c-cfg4-evictable-events": lambda: _no_policy(synth.add_events(synth.make_snapshot(4, W=800, Q=40, tight=1.6,
                                                                                       evictable=True), seed=3)),
}
DEGENERATE_CYCLES = 200


@pytest.mark.parametrize("name", list(DEGENERATE))
def test_degenerate_table_changes_nothing(name):
    snap = DEGENERATE[name]()
    a = snap.arrays
    if name.startswith("a-"):
        assert "adm_wl" not in a and not any(k in a for k in abi.EVENT_FIELDS)
    if name.startswith("b-"):
        assert (a["cq_strategy"] == abi.QUEUE_STRICT_FIFO).all()
    want = _run(snap, DEGENERATE_CYCLES)
    got = _run(_sticky(DEGENERATE[name]()), DEGENERATE_CYCLES)
    _same(want, got)
    assert not any(len(h) for h in got.sticky_heads)
    if not name.startswith("c-"):  # Preempting heads happen: without (a) or (b) they could make the rule matter
        assert (np.concatenate(want.decisions) == abi.DEC_PREEMPTING).any()


# ---- invariants with the rule on
def _cfg4_latency():
    snap = synth.add_events(synth.make_snapshot(4, W=800, Q=40, tight=1.6, evictable=True), seed=2)
    return synth.add_evict_latency(snap, (3_000, 40_000), seed=4)


# The baseline scenario creates its workloads on a 100 ms lattice: with a 30 ms termination latency the rule chose no head
# in these drains, with 150 ms it does (a preemptor still waits when the next arrivals come).
INVARIANT = {"cfg4-evictable-latency": (_cfg4_latency, 400),
             "baseline-latency": (lambda: synth.perf_scenario(0.1, evict_ns=30 * MS), 100_000),
             "baseline-latency-150ms": (lambda: synth.perf_scenario(0.1, evict_ns=150 * MS), 100_000)}


def check_sticky_invariants(snap, res):
    """Replays the slots from the heads and decisions: each cycle a head is its ClusterQueue's sticky workload when the
    rule chose it, and otherwise the slot is empty, the head itself, or a workload that left the queue by a NoFit or
    Preempt-without-targets decision; a slot is cleared exactly at its workload's admission; the final slots match and
    name no record that holds quota."""
    a = snap.arrays
    strict = a["cq_strategy"] == abi.QUEUE_STRICT_FIFO
    slot = a["cq_sticky"].astype(np.int64).copy()
    last = {}
    for k in range(res.cycles):
        chosen = set(res.sticky_heads[k].tolist())
        for w in res.heads[k].tolist():
            q = int(a["wl_cq"][w])
            if w in chosen:
                assert slot[q] == w, k
            elif slot[q] >= 0 and slot[q] != w:
                assert last.get(int(slot[q])) in (abi.DEC_NOFIT, abi.DEC_PREEMPT_NO_TARGETS), k
        for w, d in zip(res.heads[k].tolist(), res.decisions[k].tolist()):
            q = int(a["wl_cq"][w])
            last[w] = d
            if d == abi.DEC_ASSUMED:
                if slot[q] == w:
                    slot[q] = -1
                assert w not in slot, k  # an admitted workload is never left in a slot
            elif d == abi.DEC_PREEMPTING and not strict[q]:
                slot[q] = w
    assert np.array_equal(slot, res.cq_sticky)
    held = res.cq_sticky[res.cq_sticky >= 0]
    assert not (res.state[held] == HELD).any()


@pytest.mark.parametrize("name", list(INVARIANT))
def test_sticky_invariants(name):
    make, mc = INVARIANT[name]
    snap = _sticky(make())
    res = _run(snap, mc)
    check_sticky_invariants(snap, res)
    check_latency_invariants(snap, res)
    assert res.n_evicted > 0
    if name != "baseline-latency":
        assert any(len(h) for h in res.sticky_heads), "the rule chose a head"
    if name.startswith("baseline"):
        assert res.n_finished == snap.n_wl and (res.state == FINISHED).all(), "the scenario runs to the end"


def test_shard_carries_the_table():
    snap = synth.make_snapshot(4, W=400, Q=20, evictable=True)
    a = snap.arrays
    sticky = np.full(snap.n_cq, -1)
    held = set(a["adm_wl"].tolist())
    for q in range(snap.n_cq):
        free = [w for w in np.flatnonzero(a["wl_cq"] == q).tolist() if w not in held]
        if free and q % 2 == 0:
            sticky[q] = free[-1]
    _sticky(snap, sticky)
    for rank in range(3):
        part, m = shard.shard(snap, rank, 3)
        want = sticky[m.nodes[:part.n_cq]]
        got = part.arrays["cq_sticky"]
        assert np.array_equal(got >= 0, want >= 0)
        assert np.array_equal(m.wls[got[got >= 0]], want[want >= 0])


# ---------------------------------------------------------------------------------------------------------------- GPU
DEVICE_CASES = {
    "second-preemptor": lambda: _sticky(second_preemptor()),
    "second-preemptor-strict": lambda: _sticky(second_preemptor(abi.QUEUE_STRICT_FIFO)),
    "seeded": lambda: _sticky(_cq_case([1, 2], [2, 2], create=[0, 0, 0]), [1]),
    "fits-behind-head": lambda: _sticky(fits_behind_head()),
    "fits-behind-head-without-table": fits_behind_head,
    "cfg4-evictable-latency": lambda: _sticky(_cfg4_latency()),
    "baseline-latency": lambda: _sticky(synth.perf_scenario(1.0, evict_ns=30 * MS)),
    "baseline-latency-150ms": lambda: _sticky(synth.perf_scenario(1.0, evict_ns=150 * MS)),
    "baseline": lambda: _sticky(synth.perf_scenario(1.0)),
    **{f"degenerate-{k}": (lambda k=k: _sticky(DEGENERATE[k]())) for k in DEGENERATE},
}


def compare(snap, want, got):
    a = snap.arrays
    events = any(k in a for k in abi.EVENT_FIELDS)
    assert got.n_cycles == want.cycles and got.n_decisions == want.n_decisions
    cyc = got.cycles()
    for k in range(want.cycles):
        assert np.array_equal(cyc[k][0], want.heads[k]), k
        assert np.array_equal(cyc[k][1], want.decisions[k]), k
        assert int(got.cycle_admitted[k]) == len(want.admitted[k]), k
        assert int(got.cycle_evicted[k]) == len(want.evicted[k]), k
        if events:
            assert int(got.cycle_start_ns[k]) == want.cycle_start_ns[k], k
            assert int(got.cycle_finished[k]) == len(want.finished[k]), k
            assert int(got.cycle_arrived[k]) == len(want.arrived[k]), k
            assert int(got.cycle_evict_done[k]) == len(want.evict_done[k]), k
    assert got.n_evicted == want.n_evicted
    if events:
        assert got.n_finished == want.n_finished and got.n_arrived == want.n_arrived and got.end_ns == want.end_ns
        assert got.n_evict_done == want.n_evict_done
        assert np.array_equal(got.wl_admit_ns, want.wl_admit_ns) and np.array_equal(got.wl_finish_ns, want.wl_finish_ns)
    if "adm_wl" in a:
        assert np.array_equal(got.wl_evictions, want.wl_evictions)
    assert np.array_equal(got.wl_admit_cycle, want.wl_admit_cycle)
    assert np.array_equal(got.cq_usage, want.cq_usage)
    if "cq_sticky" in a:
        assert np.array_equal(got.cq_sticky, want.cq_sticky)
    else:
        assert (got.cq_sticky == -1).all(), "written only when the table is given"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DEVICE_CASES))
def test_kb_run_drain_sticky_like_the_host_definition(name):
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = DEVICE_CASES[name]()
        mc = 100_000 if name.startswith("baseline") else 400 if name.startswith("cfg4") else DEGENERATE_CYCLES if "degenerate" in name else 30
        want = _run(snap, mc)
        got = ev.run_drain(snap, abi.DrainOut(snap, mc, trace_capacity=want.n_decisions))
        compare(snap, want, got)
        if name.startswith("baseline"):
            assert got.n_finished == snap.n_wl
        if name in ("second-preemptor", "seeded", "fits-behind-head", "cfg4-evictable-latency", "baseline-latency-150ms"):
            assert any(len(h) for h in want.sticky_heads), "the rule chose a head"
    finally:
        ev.close()


@pytest.mark.gpu
def test_kb_run_drain_refuses_bad_sticky_tables():
    from kueue_b200 import native
    ev = native.Evaluator(0)

    def refused(snap, code=abi.KB_ERR_INVALID):
        with pytest.raises(native.KueueB200Error) as e:
            ev.run_drain(snap, max_cycles=5)
        assert e.value.code == code

    try:
        refused(_sticky(second_preemptor(), [3]))                 # outside [-1, n_wl)
        refused(_sticky(second_preemptor(), [-2]))
        refused(_sticky(fits_behind_head(), [-1, 3]))             # not in the ClusterQueue's queue
        refused(_sticky(second_preemptor(), [0]))                 # named by adm_wl: holds quota
        refused(_sticky(second_preemptor(), [2]))                 # created after now_ns
        afs = _cfg3_afs_events()
        q = int(np.flatnonzero(afs.arrays["cq_afs"])[0])
        w = int(np.flatnonzero((afs.arrays["wl_cq"] == q) & (afs.arrays["wl_create_ns"] <= afs.now_ns))[0])
        slots = np.full(afs.n_cq, -1)
        slots[q] = w
        refused(_sticky(afs, slots), abi.KB_ERR_UNSUPPORTED)      # a sticky workload on an AFS ClusterQueue
        ok = _sticky(second_preemptor(), [1])
        out = ev.run_drain(ok, abi.DrainOut(ok, 30))
        assert out.n_cycles > 0 and out.cq_sticky.tolist() == [-1]
        none = _sticky(second_preemptor(), [1])                   # a drain that runs no cycle returns the slots as given
        out = ev.run_drain(none, abi.DrainOut(none, 0))
        assert out.n_cycles == 0 and out.cq_sticky.tolist() == [1]
    finally:
        ev.close()
