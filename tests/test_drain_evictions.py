"""Eviction replay in the drain (kb_snapshot.adm_wl; kueue_b200/drain.py).  CPU: the requeue rule against the reference's
tables and the host definition on the oracle; GPU: kb_run_drain equals the host definition cycle by cycle."""
import json
import os

import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from kueue_b200.drain import HELD, drain, requeue_inadmissible

_GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "queue_requeue_cases.json")
_CASES = json.load(open(_GOLDEN))["cases"]


@pytest.mark.parametrize("case", _CASES, ids=[c["name"] for c in _CASES])
def test_requeue_rule_matches_reference_table(case):
    cohorts = [c[0] for c in case["cohorts"]]
    cqs = [q[0] for q in case["cluster_queues"]]
    Q = len(cqs)
    node = {n: i for i, n in enumerate(cqs + cohorts)}
    parent = [node[p] if p else -1 for _, p in case["cluster_queues"]] + [node[p] if p else -1 for _, p in case["cohorts"]]
    aside = {}
    for w, q in case["workloads"]:
        aside.setdefault(node[q], []).append(w)
    moved, roots = requeue_inadmissible(parent, Q, [node[q] for q in case["notified"]], aside)
    assert {cqs[q]: sorted(ws) for q, ws in moved.items()} == case["want_active"]
    assert sum(len(ws) for ws in moved.values()) == case["want_moved"]
    assert len(roots) == case["want_roots"]


def test_requeue_rule_stays_inside_the_root_tree():
    # two trees: root0 <- c0 <- {cq0, cq1}, root1 <- cq2; a lone cq3.  A victim in cq1 requeues cq0 and cq1 only.
    parent = [5, 5, 6, -1, -1, 4, -1]  # nodes 0..3 ClusterQueues, 4 = root0, 5 = c0, 6 = root1
    aside = {0: [10], 1: [11], 2: [12], 3: [13]}
    moved, roots = requeue_inadmissible(parent, 4, [1], aside)
    assert moved == {0: [10], 1: [11]} and roots == [4]
    moved, roots = requeue_inadmissible(parent, 4, [3], aside)
    assert moved == {3: [13]} and roots == [3]


def _with_hashes(snap):
    rng = np.random.default_rng(3)
    snap.set("wl_sched_hash", rng.integers(0, 6, snap.n_wl))  # few classes, 0 = unknown
    return snap


def _evicted_marked(snap, frac=0.3):
    rng = np.random.default_rng(5)
    snap.set("adm_evicted", rng.random(snap.n_adm) < frac)
    return snap


HOST_CASES = {
    "cfg2-within-cq": lambda: synth.make_snapshot(2, W=600, Q=12, preemption=True, tight=1.3, evictable=True),
    "cfg4": lambda: synth.make_snapshot(4, W=600, Q=40, tight=1.2, evictable=True),
    "cfg4-hashes": lambda: _with_hashes(synth.make_snapshot(4, W=600, Q=40, tight=1.2, evictable=True)),
    "cfg4-partial": lambda: synth.make_snapshot(4, W=500, Q=40, partial=True, podsets_max=2, tight=1.2, evictable=True),
}


def _run(snap, max_cycles, record=None):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000

    def cycle(s):
        out = oracle.run_cycle(s, cap)
        if record is not None:
            record.append((s, out))
        return out
    return drain(snap, cycle, max_cycles=max_cycles)


def _cells(adm, rows, Q, FR):
    use = np.zeros((Q, FR), np.int64)
    st = adm["adm_use_start"]
    for a in rows:
        for k in range(int(st[a]), int(st[a + 1])):
            use[int(adm["adm_cq"][a]), int(adm["adm_use_fr"][k])] += int(adm["adm_use_qty"][k])
    return use


def _check_replay(snap, res, seen):
    a = snap.arrays
    Q, FR = snap.n_cq, snap.n_fr
    init = {k: a[k] for k in ("adm_cq", "adm_use_start", "adm_use_fr", "adm_use_qty")}
    # usage is conserved per ClusterQueue: initial usage - cells that left + cells that joined = final usage
    final_rows = _cells(res.adm, range(len(res.adm["adm_cq"])), Q, FR)
    init_rows = _cells(init, range(snap.n_adm), Q, FR)
    assert np.array_equal(res.cq_usage, a["cq_usage"].reshape(Q, FR) - init_rows + final_rows)
    # every row names a distinct record, and exactly the records that hold quota
    wl = res.adm["adm_wl"]
    assert len(np.unique(wl)) == len(wl), "a workload holds two rows"
    assert set(np.flatnonzero(res.state == HELD).tolist()) == set(wl.tolist()), "a workload is both queued and holding quota"
    # every workload evicted in cycle c was a target of a Preempting entry of cycle c and is not held at the start of c+1
    uid_to_wl = {int(u): w for w, u in enumerate(a["wl_uid"])}
    for c, (s, out) in enumerate(seen):
        targets = set()
        for e in np.flatnonzero(np.asarray(out.decision) == abi.DEC_PREEMPTING):
            for k in range(int(out.tgt_start[e]), int(out.tgt_start[e + 1])):
                targets.add(uid_to_wl[int(s.arrays["adm_uid"][int(out.tgt_adm[k])])])
        assert set(res.evicted[c].tolist()) == targets, c
        if c + 1 < res.cycles:
            later = set(np.concatenate(res.admitted[c + 1:]).tolist()) if res.admitted[c + 1:] else set()
            for w in res.evicted[c]:
                assert int(w) not in res.admitted[c].tolist()
                if int(w) in set(wl.tolist()):
                    assert int(w) in later, "an evicted workload holds quota without a later admission"


@pytest.mark.parametrize("name", list(HOST_CASES))
def test_host_definition_replays_evictions(name):
    snap = HOST_CASES[name]()
    seen = []
    res = _run(snap, 25, seen)
    assert res.n_evicted > 0 and res.n_admitted > 0
    _check_replay(snap, res, seen)
    assert res.wl_evictions.sum() == res.n_evicted
    again = _run(snap, 25)
    assert again.cycles == res.cycles
    for k in range(res.cycles):
        assert np.array_equal(again.heads[k], res.heads[k]) and np.array_equal(again.decisions[k], res.decisions[k])
        assert np.array_equal(again.evicted[k], res.evicted[k])
    assert np.array_equal(again.cq_usage, res.cq_usage)


def test_adm_wl_without_preemption_policies_changes_nothing():
    base = synth.make_snapshot(3, W=800, Q=40, admitted=200)  # admitted workloads, no preemption policy
    ev = synth.make_snapshot(3, W=800, Q=40, admitted=200, evictable=True)
    assert ev.n_wl == base.n_wl + base.n_adm
    want = _run(base, 200)
    got = _run(ev, 200)
    assert got.cycles == want.cycles and got.n_evicted == 0
    for k in range(want.cycles):
        assert np.array_equal(got.heads[k], want.heads[k]) and np.array_equal(got.decisions[k], want.decisions[k]), k
    assert np.array_equal(got.cq_usage, want.cq_usage)


def test_evictable_records_match_their_usage():
    snap = synth.make_snapshot(4, W=300, Q=20, evictable=True)
    a = snap.arrays
    R, W0 = snap.n_resource, snap.n_wl - snap.n_adm
    assert np.array_equal(a["adm_wl"], W0 + np.arange(snap.n_adm))
    for k in ("cq", "priority", "ts", "uid"):
        assert np.array_equal(a["wl_" + k][a["adm_wl"]], a["adm_" + k])
    assert not set(a["wl_uid"][:W0].tolist()) & set(a["adm_uid"].tolist())
    req = a["ps_req"].reshape(-1, R)[a["wl_ps_start"][a["adm_wl"]]]
    st = a["adm_use_start"]
    for i in range(snap.n_adm):
        cells = np.zeros(R, np.int64)
        for k in range(st[i], st[i + 1]):
            cells[a["adm_use_fr"][k] % R] += a["adm_use_qty"][k]
        assert np.array_equal(req[i], cells)


# ---------------------------------------------------------------------------------------------------------------- GPU
DEVICE_CASES = {
    "cfg2-within-cq-strict": lambda: synth.make_snapshot(2, W=3000, Q=30, preemption=True, tight=1.2, evictable=True),
    "cfg4-reclaim-borrow-within": lambda: synth.make_snapshot(4, W=2000, Q=100, tight=1.06, evictable=True),
    "cfg3-fair-preemption": lambda: synth.make_snapshot(3, W=1500, Q=40, preemption=True, tight=1.1, evictable=True),
    "cfg4-hashes": lambda: _with_hashes(synth.make_snapshot(4, W=2000, Q=100, tight=1.06, evictable=True)),
    "cfg4-partial": lambda: synth.make_snapshot(4, W=1500, Q=60, partial=True, podsets_max=2, tight=1.1, evictable=True),
    "cfg4-tight-churn": lambda: synth.make_snapshot(4, W=1200, Q=40, tight=1.6, evictable=True),
    "cfg4-adm-evicted": lambda: _evicted_marked(synth.make_snapshot(4, W=1500, Q=60, tight=1.2, evictable=True)),
}


def _compare(snap, want, got):
    assert got.n_cycles == want.cycles
    cyc = got.cycles()
    for k in range(want.cycles):
        assert np.array_equal(cyc[k][0], want.heads[k]), k
        assert np.array_equal(cyc[k][1], want.decisions[k]), k
        assert int(got.cycle_evicted[k]) == len(want.evicted[k]), k
    assert got.n_evicted == want.n_evicted
    assert np.array_equal(got.wl_evictions, want.wl_evictions)
    assert np.array_equal(got.wl_admit_cycle, want.wl_admit_cycle)
    assert np.array_equal(got.cq_usage, want.cq_usage)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DEVICE_CASES))
def test_kb_run_drain_replays_evictions_like_the_host_definition(name):
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = DEVICE_CASES[name]()
        mc = 60
        want = _run(snap, mc)
        assert want.n_evicted > 0
        got = ev.run_drain(snap, max_cycles=mc)
        _compare(snap, want, got)
    finally:
        ev.close()


@pytest.mark.gpu
def test_kb_run_drain_full_size_config4_evictable():
    """cfg4 at full size with every admitted workload evictable: the first cycles equal the host definition; a drain
    on the device alone then conserves usage and leaves one live row per workload."""
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = synth.make_snapshot(4, evictable=True)
        want = _run(snap, 3)
        got = ev.run_drain(snap, max_cycles=3)
        _compare(snap, want, got)
        mc = 400
        got = ev.run_drain(snap, max_cycles=mc)
        a = snap.arrays
        Q, R, FR = snap.n_cq, snap.n_resource, snap.n_fr
        held_init = (got.wl_evictions[a["adm_wl"]] == 0) & (got.wl_admit_cycle[a["adm_wl"]] < 0)
        init_rows = _cells({k: a[k] for k in ("adm_cq", "adm_use_start", "adm_use_fr", "adm_use_qty")}, range(snap.n_adm), Q, FR)
        kept = _cells({k: a[k] for k in ("adm_cq", "adm_use_start", "adm_use_fr", "adm_use_qty")}, np.flatnonzero(held_init), Q, FR)
        joined = np.zeros((Q, FR), np.int64)  # Assignment.Usage of the admissions still held (assignment of the last evaluation)
        ps = a["wl_ps_start"]
        for w in np.flatnonzero(got.wl_admit_cycle >= 0):
            q = int(a["wl_cq"][w])
            cells = {}
            for row in range(int(ps[w]), int(ps[w + 1])):
                full, cnt = int(a["ps_count"][row]), int(got.ps_count[row])
                for r in range(R):
                    f = int(got.ps_flavor[row, r])
                    if f < 0:
                        continue
                    qty = int(a["ps_req"].reshape(-1, R)[row, r])
                    if full != 0 and full != cnt:
                        qty = qty // full * cnt
                    cells[f * R + r] = cells.get(f * R + r, 0) + qty
            for fr, qty in cells.items():
                joined[q, fr] += qty
        assert np.array_equal(got.cq_usage, a["cq_usage"].reshape(Q, FR) - init_rows + kept + joined)
        live_rows = snap.n_adm + got.n_admitted - got.n_evicted
        assert live_rows == int(held_init.sum()) + int((got.wl_admit_cycle >= 0).sum()), "a workload holds two rows"
        assert got.n_evicted > 0
        print(f"cfg4 evictable drain: {got.n_cycles} cycles (max {mc}), ended early: {got.n_cycles < mc}, "
              f"admitted {got.n_admitted}, evicted {got.n_evicted}, {got.gpu_ms / max(1, got.n_cycles):.3f} ms/cycle")
    finally:
        ev.close()


@pytest.mark.gpu
def test_kb_run_drain_refuses_bad_adm_wl():
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        base = synth.make_snapshot(4, W=300, Q=20, evictable=True)
        bad = []
        for fn in (lambda w: w.__setitem__(0, base.n_wl),      # out of range
                   lambda w: w.__setitem__(1, w[0]),           # named twice
                   lambda w: w.__setitem__(0, 0 if base.arrays["wl_cq"][0] != base.arrays["adm_cq"][0] else  # wrong ClusterQueue
                                           int(np.flatnonzero(base.arrays["wl_cq"] != base.arrays["adm_cq"][0])[0]))):
            w = base.arrays["adm_wl"].copy()
            fn(w)
            bad.append(w)
        for w in bad:
            base.set("adm_wl", w)
            with pytest.raises(native.KueueB200Error) as e:
                ev.run_drain(base, max_cycles=5)
            assert e.value.code == abi.KB_ERR_INVALID
        ok = synth.make_snapshot(4, W=300, Q=20, evictable=True)
        ok.flags &= ~abi.F_PRIORITY_SORTING_WITHIN_COHORT
        with pytest.raises(native.KueueB200Error) as e:
            ev.run_drain(ok, max_cycles=5)
        assert e.value.code == abi.KB_ERR_UNSUPPORTED
    finally:
        ev.close()
