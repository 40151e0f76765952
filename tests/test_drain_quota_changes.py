"""ClusterQueue and Cohort quota changes in the drain's event mode (kb_snapshot.qc_ns, qc_node, qc_nominal, qc_borrow_limit,
qc_lend_limit; kueue_b200/drain.py).  An edit replaces a node's three quota rows on the clock: unless it changes
nothing it bumps the generation of every ClusterQueue of the node's root tree and requeues that tree's inadmissible
workloads; nothing is evicted.  CPU: the reference's test cases transcribed as hand-derived schedules on the oracle, a
generation case, the equivalences, invariants on seeded drains and the refusals.  GPU: kb_run_drain equals the host
definition cycle by cycle, leaves no edited quota resident on its handle, refuses bad tables and changes nothing
without the table."""
import ctypes as C

import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from kueue_b200.drain import HELD, SET_ASIDE, check_quota_changes, drain, root_of

S = 1_000_000_000
N_, P_, A_, SK = abi.DEC_NOFIT, abi.DEC_PREEMPTING, abi.DEC_ASSUMED, abi.DEC_SKIPPED_NO_FIT


def run(snap, max_cycles=100_000, run_cycle=None):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000
    return drain(snap, run_cycle or (lambda s: oracle.run_cycle(s, cap)), max_cycles=max_cycles)


def edits(snap, table):
    """table: [(time, node, nominal row, borrowing-limit row or None, lending-limit row or None)]; None keeps the row
    in force at that point (the snapshot's, or the node's previous edit's)"""
    a = snap.arrays
    N, FR = snap.n_nodes, snap.n_fr
    cur = {k: a[k].reshape(N, FR).astype(np.int64).copy() for k in ("nominal", "borrow_limit", "lend_limit")}
    ns, node, rows = [], [], {k: [] for k in cur}
    for t, n, nom, bl, ll in table:
        for k, v in (("nominal", nom), ("borrow_limit", bl), ("lend_limit", ll)):
            if v is not None:
                cur[k][n] = v
            rows[k].append(cur[k][n].copy())
        ns.append(t); node.append(n)
    snap.set("qc_ns", ns); snap.set("qc_node", node)
    for k, nm in (("nominal", "qc_nominal"), ("borrow_limit", "qc_borrow_limit"), ("lend_limit", "qc_lend_limit")):
        snap.set(nm, np.asarray(rows[k], np.int64).reshape(len(ns), FR))
    return snap


# ---------------------------------------------------------------- the reference's cases, transcribed
def borrowed_from_cohort_case():
    """scheduler_test.go:1579 "Should admit workload using resources borrowed from cohort": ClusterQueue cq (0) with
    nominal 0 on-demand cpu in cohort (1); the cohort's nominal goes 0 -> 5 (t=5) -> 10 (t=10); a 10-cpu workload exists
    at 0.  One cycle takes 1 ns."""
    s = abi.FlatSnapshot(n_cq=1, n_cohort=1, n_flavor=1, n_resource=1)
    s.set("parent", [1, -1]); s.set("nominal", [[0], [0]])
    s.set("cq_rg_start", [0, 1]); s.set("rg_res_mask", [1]); s.set("rg_flavor_start", [0, 1]); s.set("rg_flavors", [0])
    s.set("wl_cq", [0]); s.set("ps_req", [[10]]); s.set("ps_req_mask", [1])
    s.now_ns, s.drain_cycle_ns = 0, 1
    return edits(s.finalize(), [(5, 1, [5], None, None), (10, 1, [10], None, None)])


def test_admit_using_resources_borrowed_from_cohort():
    """t=0: the workload is NoFit (the tree has 0 cpu) and set aside; the cycle is quiet and waits for the first edit.
    At 5 the edit bumps cq's generation and requeues the root: NoFit again (5 < 10), set aside, wait for 10.  At 10 the
    second edit requeues it and it is admitted on on-demand with 10 cpu (all borrowed from the cohort)."""
    r = run(borrowed_from_cohort_case())
    assert r.cycle_start_ns == [0, 5, 10] and [d.tolist() for d in r.decisions] == [[N_], [N_], [A_]]
    assert [q.tolist() for q in r.quota_changes] == [[0], [1], []] and r.n_quota_changes == 2
    assert r.cq_generation.tolist() == [2] and r.cq_usage.tolist() == [[10]] and r.state.tolist() == [HELD]


def lending_limit_case():
    """scheduler_test.go:1786 "Should admit workloads after updating lending limit": prod-cq (0) and dev-cq (1), 5 cpu
    nominal each, in one cohort (2); dev-cq lends nothing (lendingLimit 0).  wl-1 (5 cpu) and wl-2 (5 cpu, created later)
    wait in prod-cq.  dev-cq's lending limit becomes 5 at t=5."""
    s = abi.FlatSnapshot(n_cq=2, n_cohort=1, n_flavor=1, n_resource=1)
    s.set("parent", [2, 2, -1]); s.set("nominal", [[5], [5], [0]])
    s.set("lend_limit", [[abi.KB_NO_LIMIT], [0], [abi.KB_NO_LIMIT]])
    s.set("cq_rg_start", [0, 1, 2]); s.set("rg_res_mask", [1, 1]); s.set("rg_flavor_start", [0, 1, 2]); s.set("rg_flavors", [0, 0])
    s.set("wl_cq", [0, 0]); s.set("wl_ts", [0, 1]); s.set("ps_req", [[5], [5]]); s.set("ps_req_mask", [1, 1])
    s.now_ns, s.drain_cycle_ns = 0, 1
    return edits(s.finalize(), [(5, 1, None, None, [5])])


def test_admit_after_updating_lending_limit():
    """t=0: wl-1 is admitted within prod-cq's nominal quota.  t=1: wl-2 needs to borrow 5 cpu that dev-cq does not lend
    (Preempt without targets), set aside; quiet, wait for the edit.  At 5 the edit bumps both generations and requeues the cohort: wl-2 is
    admitted, borrowing dev-cq's 5 cpu."""
    r = run(lending_limit_case())
    assert r.cycle_start_ns == [0, 1, 5] and [h.tolist() for h in r.heads] == [[0], [1], [1]]
    assert [d.tolist() for d in r.decisions] == [[A_], [abi.DEC_PREEMPT_NO_TARGETS], [A_]]
    assert [q.tolist() for q in r.quota_changes] == [[], [0], []] and r.cq_generation.tolist() == [1, 1]
    assert r.cq_usage.tolist() == [[10], [0]]


def sticky_inadmissible_case(sticky=True):
    """fair_sharing_test.go:866 "sticky workload becomes inadmissible. next workload admits", on the shape of
    test_drain_sticky.fits_behind_head: cq1 (0) in cohort a (2, 3 cpu) under root (3, 0 cpu), cq2 (1) under root; both
    reclaimWithinCohort Any, withinClusterQueue LowerPriority, BestEffortFIFO, the classical scheduler.  cq2 borrows two
    1-cpu workloads (records 0 and 1).  In cq1 the 3-cpu preemptor (2) exists at 0 and the 2-cpu workload (3) is created
    at 3.  Every eviction takes 5 ns, one cycle 1 ns.  At t=2 cohort a's nominal goes 3 -> 2 cpu."""
    s = abi.FlatSnapshot(n_cq=2, n_cohort=2, n_flavor=1, n_resource=1)
    s.flags = abi.FLAGS_DEFAULT & ~abi.F_FAIR_SHARING
    s.set("parent", [2, 3, 3, -1]); s.set("nominal", [[0], [0], [3000], [0]])
    s.set("cq_rg_start", [0, 1, 2]); s.set("rg_res_mask", [1, 1]); s.set("rg_flavor_start", [0, 1, 2]); s.set("rg_flavors", [0, 0])
    s.set("cq_strategy", [abi.QUEUE_BEST_EFFORT_FIFO] * 2)
    s.set("cq_within_cq", [abi.POLICY_LOWER_PRIORITY] * 2); s.set("cq_reclaim_within", [abi.POLICY_ANY] * 2)
    s.set("wl_cq", [1, 1, 0, 0]); s.set("wl_priority", [0, 0, 0, 0])
    s.set("wl_ts", [0, 1, 2, 3]); s.set("wl_uid", [0, 1, 2, 3])
    s.set("ps_req", [[1000], [1000], [3000], [2000]]); s.set("ps_req_mask", np.ones(4))
    s.set("adm_cq", [1, 1]); s.set("adm_priority", [0, 0]); s.set("adm_ts", [0, 1]); s.set("adm_qr_ts", [0, 0])
    s.set("adm_uid", [0, 1]); s.set("adm_evicted", [0, 0])
    s.set("adm_use_start", [0, 1, 2]); s.set("adm_use_fr", [0, 0]); s.set("adm_use_qty", [1000, 1000])
    s.set("cq_usage", [[0], [2000]])
    s.set("adm_wl", [0, 1])
    s.set("wl_create_ns", [0, 0, 0, 3])
    s.set("wl_evict_ns", np.full(4, 5))
    if sticky:
        s.set("cq_sticky", [-1, -1])
    s.now_ns, s.drain_cycle_ns = 0, 1
    return edits(s.finalize(), [(2, 2, [2000], None, None)])


CPU_CASES = {"borrowed-from-cohort": borrowed_from_cohort_case, "lending-limit": lending_limit_case,
             "sticky-inadmissible": sticky_inadmissible_case}


def test_sticky_workload_becomes_inadmissible():
    """t=0: the preemptor reclaims cohort a's 2 cpu from cq2's two borrowing rows (their evictions end at 5) and becomes
    cq1's sticky workload; t=1 it re-targets them: quiet, wait for the edit at 2.  The edit leaves the tree 2 cpu: at 2
    the sticky preemptor is NoFit and set aside (the slot keeps it).  t=3: the 2-cpu workload arrives, takes the head
    and re-targets the evicting rows ("Preemption ongoing"), replacing the sticky workload; quiet, wait for 5.  At 5 the
    evictions complete (records 0 and 1 back in cq2's queue) and the root's requeue returns the preemptor: the 2-cpu
    workload is cq1's sticky head and is admitted, record 0 is skipped.  t=6: the preemptor (3 > 2) and record 0 are
    NoFit, and the drain ends with one admitted workload in cq1."""
    r = run(sticky_inadmissible_case())
    assert r.cycle_start_ns == [0, 1, 2, 3, 5, 6] and r.end_ns == 6
    assert [h.tolist() for h in r.heads] == [[2], [2], [2], [3], [3, 0], [2, 0]]
    assert [d.tolist() for d in r.decisions] == [[P_], [P_], [N_], [P_], [A_, SK], [N_, N_]]
    assert [e.tolist() for e in r.evicted] == [[0, 1], [], [], [], [], []]
    assert [e.tolist() for e in r.evict_done] == [[], [], [], [0, 1], [], []]
    assert [q.tolist() for q in r.quota_changes] == [[], [0], [], [], [], []]
    assert [h.tolist() for h in r.sticky_heads] == [[], [], [], [], [3], []]
    assert r.state[3] == HELD and r.state[2] == SET_ASIDE and r.cq_usage.tolist() == [[2000], [0]]
    assert r.cq_generation.tolist() == [1, 1] and len(r.adm["adm_cq"]) == 1


# ---------------------------------------------------------------- generations
def generation_case(noop=False):
    """one ClusterQueue with flavors f0, f1 (one resource group, no cohort), nominal 0 on both; the pending 1-cpu
    workload's LastAssignment tried f0 at generation 0.  At t=5 an edit raises f0 to 1 cpu (noop: repeats the rows)."""
    s = abi.FlatSnapshot(n_cq=1, n_cohort=0, n_flavor=2, n_resource=1)
    s.set("nominal", [[0, 0]])
    s.set("cq_rg_start", [0, 1]); s.set("rg_res_mask", [1]); s.set("rg_flavor_start", [0, 2]); s.set("rg_flavors", [0, 1])
    s.set("wl_cq", [0]); s.set("ps_req", [[1]]); s.set("ps_req_mask", [1])
    s.set("wl_last_gen", [0]); s.set("ps_last_tried", [[0]])
    s.set("wl_create_ns", [0])
    s.now_ns, s.drain_cycle_ns = 0, 1
    return edits(s.finalize(), [(5, 0, [0, 0] if noop else [1, 0], None, None)])


def test_generation_bump_restarts_the_flavor_search():
    """t=0: the LastAssignment is in force (generation 0), the attempt resumes after f0: f1 has no quota, NoFit, set
    aside.  At 5 the edit bumps the generation to 1 and requeues the ClusterQueue: the LastAssignment is outdated, the
    search starts at f0 and the workload is admitted there.  As a no-op the edit bumps nothing and requeues nothing: the
    workload stays set aside and the drain ends at the edit."""
    r = run(generation_case())
    assert r.cycle_start_ns == [0, 5] and [d.tolist() for d in r.decisions] == [[N_], [A_]]
    assert r.cq_generation.tolist() == [1] and r.cq_usage.tolist() == [[1, 0]]
    r = run(generation_case(noop=True))
    assert r.cycle_start_ns == [0] and [d.tolist() for d in r.decisions] == [[N_]] and r.end_ns == 5
    assert r.cq_generation.tolist() == [0] and r.n_quota_changes == 1 and r.state.tolist() == [SET_ASIDE]
    # the same LastAssignment without the edit: the attempt at t=0 is the same
    plain = generation_case(); [plain.arrays.pop(k) for k in abi.QUOTA_CHANGE_FIELDS]
    assert [d.tolist() for d in run(plain).decisions] == [[N_]]


# ---------------------------------------------------------------- equivalences
def _same_schedule(got, want, end=True):
    assert got.cycles == want.cycles and got.cycle_start_ns == want.cycle_start_ns
    if end:
        assert got.end_ns == want.end_ns
    for k in range(want.cycles):
        assert np.array_equal(got.heads[k], want.heads[k]) and np.array_equal(got.decisions[k], want.decisions[k]), k
        assert np.array_equal(got.admitted[k], want.admitted[k]) and np.array_equal(got.evicted[k], want.evicted[k]), k
        assert np.array_equal(got.finished[k], want.finished[k]), k
    assert np.array_equal(got.cq_usage, want.cq_usage)
    for f in ("wl_admit_cycle", "wl_evictions", "wl_admit_ns", "wl_finish_ns", "state"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f


def _cfg2():
    return synth.add_events(synth.make_snapshot(2, W=600, Q=12, preemption=True, tight=1.3, evictable=True), seed=1)


def test_empty_table_is_no_table():
    want = run(_cfg2(), 200)
    s = _cfg2(); FR = s.n_fr
    s.set("qc_ns", np.zeros(0)); s.set("qc_node", np.zeros(0))
    for k in ("qc_nominal", "qc_borrow_limit", "qc_lend_limit"):
        s.set(k, np.zeros((0, FR)))
    got = run(s, 200)
    _same_schedule(got, want)
    assert got.n_quota_changes == 0 and got.cq_generation is None


def _final_rows(snap):
    """the snapshot with the rows its last edits leave, and no table"""
    a = snap.arrays
    N, FR = snap.n_nodes, snap.n_fr
    for k, q in (("nominal", "qc_nominal"), ("borrow_limit", "qc_borrow_limit"), ("lend_limit", "qc_lend_limit")):
        rows = a[k].reshape(N, FR).copy()
        for i, n in enumerate(a["qc_node"]):
            rows[n] = a[q].reshape(-1, FR)[i]
        snap.set(k, rows)
    for k in abi.QUOTA_CHANGE_FIELDS:
        a.pop(k)
    return snap


def _early_edits():
    """the baseline scenario at scale 0.1 (every workload created from 100 ms on) with edits in the first 50 ms: halved
    nominal quotas (never restored: the restore is dropped), lending limits, no-op edits"""
    s = synth.add_quota_changes(synth.perf_scenario(0.1), seed=4, span_ns=50_000_000, lend_share=0.5, noop_share=0.3)
    a = s.arrays
    keep = np.ones(len(a["qc_ns"]), bool)
    seen = set()
    for i in range(len(keep) - 1, -1, -1):  # the later of the two edits of a dipped node is its restore
        n = int(a["qc_node"][i])
        if n < s.n_cq and n not in seen and (a["qc_nominal"].reshape(-1, s.n_fr)[i] == a["nominal"].reshape(-1, s.n_fr)[n]).all():
            keep[i] = False
        seen.add(n)
    for k in abi.QUOTA_CHANGE_FIELDS:
        s.set(k, a[k][keep])
    return s


def test_edits_before_every_creation_are_the_final_rows():
    got = run(_early_edits())
    want = run(_final_rows(_early_edits()))
    _same_schedule(got, want)
    assert got.n_quota_changes == len(_early_edits().arrays["qc_ns"]) and got.cycles > 0
    assert (got.cq_generation > 0).any()


def test_noop_edits_after_the_natural_end():
    """no-op edits just after the drain's natural end: the last cycle of the drain without the table is quiet (its
    StrictFIFO heads stay) and ends it.  With the edits it waits for them instead: t_{c+1} = t_c + step, since they all
    fall in that step and are applied at that boundary (counted in that cycle), they change nothing, and the same heads
    get the same decisions once more before the drain ends.  That one cycle is all that differs."""
    want = run(_cfg2(), 400)
    s = _cfg2()
    n = s.n_nodes
    t_end = want.end_ns + 10
    edits(s, [(t_end + 3 * i, i % n, None, None, None) for i in range(5)])
    got = run(s, 400)
    K = want.cycles
    assert got.cycles == K + 1 and got.cycle_start_ns[:K] == want.cycle_start_ns
    assert got.cycle_start_ns[K] == want.end_ns + s.drain_cycle_ns == got.end_ns
    for k in range(K):
        assert np.array_equal(got.heads[k], want.heads[k]) and np.array_equal(got.decisions[k], want.decisions[k]), k
        assert np.array_equal(got.admitted[k], want.admitted[k]) and np.array_equal(got.evicted[k], want.evicted[k]), k
    assert np.array_equal(got.heads[K], want.heads[-1]) and np.array_equal(got.decisions[K], want.decisions[-1])
    assert len(got.admitted[K]) == 0 and len(got.evicted[K]) == 0 and len(got.finished[K]) == 0
    assert np.array_equal(got.cq_usage, want.cq_usage) and np.array_equal(got.state, want.state)
    assert got.quota_changes[K - 1].tolist() == [0, 1, 2, 3, 4] and got.n_quota_changes == 5
    assert np.array_equal(got.cq_generation, s.cq_generation)


# ---------------------------------------------------------------- invariants on seeded drains
def _cfg3_quota():
    return synth.add_quota_changes(synth.add_events(synth.make_snapshot(3, W=1200, Q=40), seed=2), seed=5)


def _cfg4_quota():
    snap = synth.add_evict_latency(synth.add_events(synth.make_snapshot(4, W=800, Q=40, tight=1.6, evictable=True), seed=3),
                                   (3_000, 40_000), seed=4)
    return synth.add_quota_changes(snap, seed=6)


def _cfg2_quota():
    return synth.add_quota_changes(_cfg2(), seed=7, dip=0.25)


SEEDED = {"cfg2": _cfg2_quota, "cfg3": _cfg3_quota, "cfg4-latency": _cfg4_quota}


class _Watch:
    """run_cycle that keeps what every cycle saw: t_c, the quota rows, the generations and the usage"""

    def __init__(self, cap):
        self.cap, self.seen = cap, []

    def __call__(self, cs):
        a = cs.arrays
        self.seen.append((int(cs.now_ns), a["nominal"].copy(), a["borrow_limit"].copy(), a["lend_limit"].copy(),
                          a["cq_generation"].copy(), a["cq_usage"].copy(), int(cs.static_generation)))
        return oracle.run_cycle(cs, self.cap)


@pytest.mark.parametrize("name", list(SEEDED))
def test_quota_change_invariants(name):
    snap = SEEDED[name]()
    snap.static_generation = 7
    a = snap.arrays
    N, Q, FR = snap.n_nodes, snap.n_cq, snap.n_fr
    watch = _Watch(40 * (snap.n_adm + snap.n_wl) + 10000)
    res = drain(snap, watch, max_cycles=400)
    assert res.n_quota_changes > 0
    ns, node = a["qc_ns"], a["qc_node"]
    rows = [a[k].reshape(-1, FR) for k in ("qc_nominal", "qc_borrow_limit", "qc_lend_limit")]
    root = root_of(a["parent"])
    tree_nodes = {int(r): np.flatnonzero(root == r) for r in np.unique(root)}
    prev_gen, prev_sg, prev_rows = a["cq_generation"].astype(np.int64), snap.static_generation, None
    for k, (t_c, nom, bl, ll, gen, usage, sg) in enumerate(watch.seen):
        # the rows in force at t_c: the snapshot's, then every edit with qc_ns <= t_c in table order
        want = [a[x].reshape(N, FR).astype(np.int64).copy() for x in ("nominal", "borrow_limit", "lend_limit")]
        want_gen = a["cq_generation"].astype(np.int64).copy()
        for i in np.flatnonzero(ns <= t_c):
            n = int(node[i])
            if all(np.array_equal(w[n], r[i]) for w, r in zip(want, rows)):
                continue
            for w, r in zip(want, rows):
                w[n] = r[i]
            want_gen[root[:Q] == root[n]] += 1  # exactly one per edit that changes the rows of the tree
        assert all(np.array_equal(x.reshape(N, FR), w) for x, w in zip((nom, bl, ll), want)), k
        assert np.array_equal(gen, want_gen) and (gen >= prev_gen).all(), k
        rows_now = [x.reshape(N, FR) for x in (nom, bl, ll)]
        if prev_rows is not None:  # the static generation changes with the rows, and only with them
            same = all(np.array_equal(x, y) for x, y in zip(rows_now, prev_rows))
            assert (sg == prev_sg) == same and sg != 0, k
        prev_gen, prev_sg, prev_rows = gen, sg, rows_now
        u = usage.reshape(Q, FR)
        assert (u >= 0).all(), k
        # an admission never takes a root tree past the sum of its nominal rows in a cycle without evictions
        if len(res.evicted[k]) == 0 and len(res.admitted[k]):
            after = u.copy()
            nxt = watch.seen[k + 1][5].reshape(Q, FR) if k + 1 < len(watch.seen) else res.cq_usage
            for r, nodes in tree_nodes.items():
                cqs = nodes[nodes < Q]
                cap = nom.reshape(N, FR)[nodes].sum(0)
                added = np.zeros(FR, np.int64)
                for w in res.admitted[k]:
                    if root[int(a["wl_cq"][w])] == r:
                        added += 1
                if not added.any():
                    continue
                before = after[cqs].sum(0)
                grown = nxt[cqs].sum(0)
                if not len(res.finished[k]):
                    assert ((grown <= np.maximum(before, cap)) | (grown <= before)).all(), (k, r)
    assert (res.cq_usage >= 0).all()
    # the generations after the drain: one per edit that changed its tree's rows (the edits applied)
    applied = np.concatenate(res.quota_changes) if res.quota_changes else np.zeros(0, np.int64)
    want = [a[x].reshape(N, FR).astype(np.int64).copy() for x in ("nominal", "borrow_limit", "lend_limit")]
    want_gen = a["cq_generation"].astype(np.int64).copy()
    for i in range(res.n_quota_changes):
        n = int(node[i])
        if not all(np.array_equal(w[n], r[i]) for w, r in zip(want, rows)):
            for w, r in zip(want, rows):
                w[n] = r[i]
            want_gen[root[:Q] == root[n]] += 1
    assert np.array_equal(res.cq_generation, want_gen) and len(applied) <= res.n_quota_changes


# ---------------------------------------------------------------- refusals of the host definition
def _bad(mutate):
    s = lending_limit_case()
    mutate(s)
    with pytest.raises(ValueError) as e:
        check_quota_changes(s)
    return str(e.value)


REFUSALS = {
    "missing-table": (lambda s: s.arrays.pop("qc_lend_limit"), "a NULL table with n_quota_change > 0"),
    "at-now": (lambda s: s.set("qc_ns", [0]), "qc_ns at or before now_ns"),
    "decreasing": (lambda s: edits(s, [(5, 1, None, None, [5]), (4, 1, None, None, [4])]), "qc_ns decreasing"),
    "node-range": (lambda s: s.set("qc_node", [3]), "qc_node out of range"),
    "negative-nominal": (lambda s: s.set("qc_nominal", [[-1]]), "a negative nominal or KB_NO_LIMIT in a nominal row"),
    "nil-nominal": (lambda s: s.set("qc_nominal", [[abi.KB_NO_LIMIT]]), "a negative nominal or KB_NO_LIMIT in a nominal row"),
    "negative-limit": (lambda s: s.set("qc_borrow_limit", [[-2]]), "a negative limit"),
    "uncovered-cell": (lambda s: s.set("cq_rg_start", [0, 1, 1]), "a ClusterQueue cell its resource groups do not cover"),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_host_definition_refuses_bad_tables(name):
    mutate, msg = REFUSALS[name]
    if name == "uncovered-cell":  # dev-cq (1) without resource groups: its lending-limit cell is not covered
        def mutate(s):
            s.set("cq_rg_start", [0, 1, 1]); s.set("rg_res_mask", [1]); s.set("rg_flavor_start", [0, 1]); s.set("rg_flavors", [0])
    assert msg in _bad(mutate)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _cfg4_sticky_quota():
    s = _cfg4_quota()
    s.set("cq_sticky", np.full(s.n_cq, -1))
    return s


def _baseline_all():
    return synth.perf_scenario(0.1, evict_ns=30_000_000, checks=7, pods_ready=9, max_exec=3, quota=11)


def _afs_decay_quota():
    snap = synth.add_events(synth.make_snapshot(3, W=1200, Q=40, afs=3), seed=2)
    snap.set("adm_wl", np.zeros(0))
    snap.set("lq_last_update_ns", np.full(len(snap.arrays["lq_cq"]), snap.now_ns)); snap.set("adm_lq", np.full(snap.n_adm, -1))
    snap.afs_half_life_ns, snap.afs_sampling_ns, snap.afs_alpha = 10 * S, S, 0.5 ** 0.1
    return synth.add_quota_changes(snap, seed=8)


DEVICE_CASES = dict(CPU_CASES)
DEVICE_CASES.update({
    "generation": generation_case, "generation-noop": lambda: generation_case(noop=True),
    "early-edits": _early_edits, "cfg2": _cfg2_quota, "cfg3-flat": _cfg3_quota, "cfg4-latency-sticky": _cfg4_sticky_quota,
    "baseline-all-blocks": _baseline_all, "cfg3-afs-decay": _afs_decay_quota,
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
        assert int(got.cycle_quota_changes[k]) == len(want.quota_changes[k]), k
        assert int(got.cycle_max_exec_deactivated[k]) == len(want.max_exec_deactivated[k]), k
        assert int(got.cycle_pods_ready_timeout[k]) == len(want.pods_ready_timeout[k]), k
        assert int(got.cycle_check_retry[k]) == len(want.check_retry[k]), k
    assert got.n_evicted == want.n_evicted and got.n_finished == want.n_finished and got.end_ns == want.end_ns
    assert got.n_evict_done == want.n_evict_done and got.n_quota_changes == want.n_quota_changes
    for f in ("wl_admit_ns", "wl_finish_ns", "wl_evictions", "wl_admit_cycle", "cq_usage", "cq_generation"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    if want.cq_sticky is not None:
        assert np.array_equal(got.cq_sticky, want.cq_sticky)
    if want.wl_deactivated is not None:
        assert np.array_equal(got.wl_deactivated, want.wl_deactivated)
    if want.lq_consumed is not None:
        assert np.array_equal(got.lq_consumed, want.lq_consumed) and np.array_equal(got.lq_last_update_ns, want.lq_last_update_ns)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DEVICE_CASES))
def test_kb_run_drain_quota_changes_like_the_host_definition(name):
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = DEVICE_CASES[name]()
        mc = 100_000 if name.startswith(("baseline", "early")) else 400
        want = run(snap, mc)
        got = ev.run_drain(snap, abi.DrainOut(snap, mc, trace_capacity=want.n_decisions))
        compare(want, got)
        if name == "baseline-all-blocks":
            assert got.n_quota_changes > 0 and got.n_max_exec_deactivated > 0 and got.n_check_retry > 0
    finally:
        ev.close()


@pytest.mark.gpu
def test_drain_with_edits_leaves_no_quota_resident():
    """on one handle with static_generation 7: a cycle, a drain whose edits change the rows and generations, then a cycle
    on the original snapshot with the same static_generation: its outputs are those of a fresh handle"""
    from kueue_b200 import native
    snap = _cfg3_quota()
    snap.static_generation = 7
    first = []  # the drain's first cycle as a kb_run_cycle snapshot: one head per ClusterQueue, the snapshot's quotas
    run(snap, 1, lambda cs: first.append(cs) or oracle.run_cycle(cs, 100_000))
    cyc = first[0]
    cyc.static_generation = 7
    ev, fresh = native.Evaluator(0), native.Evaluator(0)
    try:
        before = ev.run_cycle(cyc)
        d = ev.run_drain(snap, max_cycles=400)
        assert d.n_quota_changes > 0 and (d.cq_generation != snap.cq_generation).any()
        after, want = ev.run_cycle(cyc), fresh.run_cycle(cyc)
        for f in ("decision", "mode", "borrow", "ps_flavor", "ps_count", "node_usage"):
            assert np.array_equal(getattr(after, f), getattr(want, f)), f
            assert np.array_equal(getattr(before, f), getattr(want, f)), f
    finally:
        ev.close(); fresh.close()


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
    s = lending_limit_case()
    if name == "uncovered-cell":
        s.set("cq_rg_start", [0, 1, 1]); s.set("rg_res_mask", [1]); s.set("rg_flavor_start", [0, 1]); s.set("rg_flavors", [0])
    elif name != "missing-table":
        mutate(s)
    st = s.as_struct()
    if name == "missing-table":
        st.n_quota_change = 1
        st.qc_lend_limit = None
    out = abi.DrainOut(s, 5)
    out.struct.max_cycles = 5
    rc = native.lib().kb_run_drain(evaluator._h, C.byref(st), C.byref(out.struct))
    assert rc == abi.KB_ERR_INVALID and msg in native.lib().kb_last_error(evaluator._h).decode()


@pytest.mark.gpu
def test_without_the_table_nothing_changes():
    """an event drain with an empty table: the launches and every result are the drain's without the block"""
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        plain = _cfg2()
        empty = _cfg2(); FR = empty.n_fr
        empty.set("qc_ns", np.zeros(0)); empty.set("qc_node", np.zeros(0))
        for k in ("qc_nominal", "qc_borrow_limit", "qc_lend_limit"):
            empty.set(k, np.zeros((0, FR)))
        want = run(plain, 200)
        a = ev.run_drain(plain, abi.DrainOut(plain, 200, trace_capacity=want.n_decisions))
        la = ev.stats().kernel_launches
        b = ev.run_drain(empty, abi.DrainOut(empty, 200, trace_capacity=want.n_decisions))
        lb = ev.stats().kernel_launches
        assert la == lb and b.n_quota_changes == 0
        for f in ("cycle_heads", "cycle_admitted", "cycle_start_ns", "trace_wl", "trace_decision", "wl_admit_ns",
                  "wl_finish_ns", "cq_usage", "wl_evictions"):
            assert np.array_equal(getattr(a, f), getattr(b, f)), f
        assert not b.cq_generation.any()  # untouched without the block
    finally:
        ev.close()
