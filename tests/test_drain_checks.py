"""Admission checks in the drain's event mode (kb_snapshot.wl_check_ns and the start-state tables; kueue_b200/drain.py).
A reservation starts an attempt whose verdict comes after the check delay: Ready starts the run, Retry releases the quota
and requeues the workload after its backoff with the eviction time as its queue-order timestamp, Rejected deactivates it.
CPU: the backoff goldens on the Python function and on the header's host build, hand-derived schedules on the oracle, the
equivalence of zero delays with the drain without the tables, invariants.  GPU: kb_run_drain equals the host definition
cycle by cycle, and refuses bad tables."""
import json
import os
import subprocess

import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from kueue_b200.drain import (ABSENT, BACKOFF, DEACTIVATED, FINISHED, HELD, QUEUED, SET_ASIDE, check_wait_bound_s,
                              check_wait_s, drain, wait_time)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "check_backoff_cases.json")))
S = 1_000_000_000
I64_MIN = np.iinfo(np.int64).min
ALL = np.iinfo(np.int32).max


def _run(snap, max_cycles=100_000, record=None):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000

    def cycle(s):
        out = oracle.run_cycle(s, cap)
        if record is not None:
            record.append((s, out))
        return out
    return drain(snap, cycle, max_cycles=max_cycles)


# ---------------------------------------------------------------- backoff
def test_backoff_goldens_on_the_python_function():
    for c in GOLDEN["wait_time"]:
        assert wait_time(c["base_ns"], c["cap_ns"], c["factor"], c["iteration"]) == c["want_ns"], c["name"]
    for c in GOLDEN["consecutive"]:
        got = [wait_time(c["base_ns"], c["cap_ns"], c["factor"], it) for it in c["iterations"]]
        assert got == c["want_ns"], c["name"]
    assert [check_wait_s(k, 60, 1800) for k in range(1, 8)] == [60, 120, 240, 480, 960, 1800, 1800]
    # base > max: the first Step returns the base uncapped, every later one the cap
    assert [check_wait_s(k, 60, 30) for k in range(1, 5)] == [60, 30, 30, 30]
    assert check_wait_bound_s(60, 30, 3) == 60 and check_wait_bound_s(20_000, 5_000, 1) == 20_000
    assert check_wait_bound_s(60, 0, 9) == 15_360 and check_wait_bound_s(60, 1800, 0) == 0


def test_backoff_goldens_on_the_host_build_of_the_header(tmp_path):
    """kb_backoff_wait / kb_check_wait_ns compiled from kb_drain.cuh for the host"""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = tmp_path / "backoff.cu"
    src.write_text('#include <cstdio>\n#include "kb_drain.cuh"\n'
                   "int main() { long long b, c, k; double f; while (scanf(\"%lld %lld %lf %lld\", &b, &c, &f, &k) == 4) "
                   "printf(\"%lld %lld %lld\\n\", (long long)kb_backoff_wait(b, c, f, (int)k), (long long)kb_check_wait_ns((int)k, 60, 1800), "
                   "(long long)kb_check_wait_ns((int)k, 60, 30)); "
                   "return 0; }\n")
    exe = tmp_path / "backoff"
    subprocess.check_call([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I", os.path.join(ROOT, "kueue_b200", "csrc"),
                           "-o", str(exe), str(src)])
    cases = [(c["base_ns"], c["cap_ns"], c["factor"], c["iteration"], c["want_ns"]) for c in GOLDEN["wait_time"]]
    cases += [(c["base_ns"], c["cap_ns"], c["factor"], it, w) for c in GOLDEN["consecutive"] for it, w in zip(c["iterations"], c["want_ns"])]
    inp = "\n".join(f"{b} {cap} {f} {it}" for b, cap, f, it, _ in cases)
    out = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout.split("\n")
    for (b, cap, f, it, want), line in zip(cases, out):
        got, drain_wait, inverted = (int(v) for v in line.split())
        assert got == want, (b, cap, f, it)
        assert drain_wait == (check_wait_s(it, 60, 1800) * S if it > 0 else 0)
        assert inverted == (check_wait_s(it, 60, 30) * S if it > 0 else 0)


# ---------------------------------------------------------------- hand-derived schedules
def _case(cpu, ts, create, run, check, fail, prio=None, nominal=2, within=abi.POLICY_NEVER, adm=None):
    """One ClusterQueue of `nominal` cpu without a cohort, BestEffortFIFO, withinClusterQueue `within`; one cycle takes
    1 s; backoff base 60 s, max 1800 s, limit 3 (the defaults).  `adm`: (workload, cpu, check end or INT64_MIN) rows
    admitted before the drain."""
    W = len(cpu)
    s = abi.FlatSnapshot(n_cq=1, n_cohort=0, n_flavor=1, n_resource=1)
    s.set("nominal", [[nominal]])
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
        s.set("adm_check_end_ns", [e for _, _, e in adm])
    s.set("wl_create_ns", create); s.set("wl_run_ns", run)
    s.set("wl_check_ns", check); s.set("wl_check_fail", fail)
    s.now_ns, s.drain_cycle_ns = 0, S
    return s.finalize()


def delay_case():
    """w0 and w1 need the whole 2 cpu.  0: w0 reserves, its check runs until 10.  1: w1 does not fit and is set aside;
    the quiet cycle waits for the verdict at 10: Ready, Admitted at 10, w0 runs until 15 (not 5).  No queue has a head,
    so the clock jumps to 15: w0 finishes, its root tree is requeued, and w1 is admitted at 15 and finishes at 20."""
    return _case([2, 2], [0, 1], [0, 0], [5 * S] * 2, [10 * S, 0], [0, 0])


def test_check_delay_holds_quota_and_shifts_the_finish():
    r = _run(delay_case())
    assert [t // S for t in r.cycle_start_ns] == [0, 1, 15]
    assert [h.tolist() for h in r.heads] == [[0], [1], [1]]
    assert (r.wl_admit_ns // S).tolist() == [0, 15] and (r.wl_ready_ns // S).tolist() == [10, 15]
    assert (r.wl_finish_ns // S).tolist() == [15, 20] and r.end_ns == 20 * S
    assert r.n_check_ready == 1 and r.n_check_retry == 0 and r.n_resorts == 0


def retry_case():
    """w0 (created 0) fails its first attempt; w1 (created 1 s) waits behind it; "early" is created at 5 s and "late" at
    20 s; all need the 2 cpu and run 100 s.
      0 w0 reserves (verdict at 10) | 1 w1 NoFit, aside | 5 early arrives, NoFit, aside
      10 Retry: the quota goes, the root tree is requeued, w0 waits until 10 + 60 = 70 with queue timestamp 10; w1 admitted
      11 early NoFit | 20 late arrives, NoFit | 70 w0 returns (a re-sort: its key was 0), NoFit
      110 w1 finishes, the tree is requeued: early (5) is admitted; 111 w0 (10) is the head, ahead of late (20)
      210 early finishes: w0 reserves again, Ready at 220, runs until 320 | 211 late NoFit | 320 late admitted."""
    return _case([2, 2, 2, 2], [0, S, 5 * S, 20 * S], [0, 0, 5 * S, 20 * S], [100 * S] * 4, [10 * S, 0, 0, 0], [1, 0, 0, 0])


def test_retry_releases_quota_and_requeues_after_the_backoff():
    r = _run(retry_case())
    assert [t // S for t in r.cycle_start_ns] == [0, 1, 5, 10, 11, 20, 70, 110, 111, 210, 211, 320]
    assert [h.tolist() for h in r.heads] == [[0], [1], [2], [1], [2], [3], [0], [2], [0], [0], [3], [3]]
    assert [x.tolist() for x in r.check_retry] == [[], [], [0]] + [[]] * 9  # the verdict at 10 is cycle 2's
    assert r.n_check_retry == 1 and r.n_check_ready == 1 and r.n_resorts == 1
    assert (r.wl_admit_ns // S).tolist() == [210, 10, 110, 320] and (r.wl_ready_ns // S).tolist() == [220, 10, 110, 320]
    assert r.wl_check_retries.tolist() == [1, 0, 0, 0] and r.wl_queue_ts[0] == 0  # readmission: back to its creation


def rejected_case():
    """w0 fails every attempt: Retry at 10 (back at 70), 80 (back at 80 + 120 = 200), 210 (back at 210 + 240 = 450),
    then attempt 4 > BackoffLimitCount 3 is Rejected at 460: deactivated, never queued again."""
    return _case([2], [0], [0], [100 * S], [10 * S], [ALL])


def test_three_retries_then_rejected():
    r = _run(rejected_case())
    assert [t // S for t in r.cycle_start_ns] == [0, 70, 200, 450] and r.end_ns == 460 * S
    assert [x.tolist() for x in r.check_retry] == [[0], [0], [0], []]
    assert r.n_check_retry == 3 and r.n_check_rejected == 1 and r.n_check_ready == 0 and r.n_resorts == 3
    assert r.wl_check_retries.tolist() == [3] and r.wl_deactivated.tolist() == [1] and r.state.tolist() == [DEACTIVATED]
    assert r.cq_usage.tolist() == [[0]] and r.wl_ready_ns.tolist() == [I64_MIN]


def inverted_backoff_case():
    """BackoffBaseSeconds 60 > BackoffMaxSeconds 30 (the reference accepts it): w0 fails twice.  Retry at 10 waits the
    uncapped base, 60 s (back at 70); the attempt at 70 fails at 80 and waits the cap, 30 s (back at 110); the attempt at
    110 is Ready at 120."""
    s = _case([2], [0], [0], [100 * S], [10 * S], [2])
    s.check_backoff_base_s, s.check_backoff_max_s = 60, 30
    return s


def test_base_above_max_waits_the_base_first():
    r = _run(inverted_backoff_case())
    assert [t // S for t in r.cycle_start_ns] == [0, 70, 110]
    assert r.n_check_retry == 2 and r.wl_check_retries.tolist() == [2] and r.wl_ready_ns.tolist() == [120 * S]


def preempt_checking_case():
    """"low" (0, priority -1) holds the 2 cpu with its checks running until 50 and would fail them; "in" (1, priority 1)
    preempts it at 0 with a 5 s termination latency.  low holds no pods: it is released at the next boundary (1), the
    attempt is dropped (no verdict, no failure used), and "in" is admitted at 1."""
    s = _case([2, 2], [0, S], [0, 0], [-1, -1], [10 * S, 0], [1, 0], prio=[-1, 1], within=abi.POLICY_LOWER_PRIORITY,
              adm=[(0, 2, 50 * S)])
    s.set("wl_evict_ns", [5 * S, 5 * S])
    return s


def test_preempting_a_row_whose_checks_run_releases_at_once():
    r = _run(preempt_checking_case())
    assert [t // S for t in r.cycle_start_ns] == [0, 1, 2]
    assert [e.tolist() for e in r.evicted][:2] == [[0], []] and [e.tolist() for e in r.evict_done][:1] == [[0]]
    assert r.n_check_ready == r.n_check_retry == r.n_check_rejected == 0
    assert r.wl_check_retries.tolist() == [0, 0] and r.wl_admit_ns[1] == S and r.state.tolist() == [SET_ASIDE, HELD]


def readmit_preempt_case():
    """w0 fails once (Retry at 10, back at 70 with timestamp 10), is reserved again at 70 and Admitted at 80; "hi"
    (priority 5) is created at 100 and preempts it (no latency).  w0 returns with its creation timestamp 0: a second
    re-sort, and the cycle at 102 sees wl_ts 0."""
    return _case([2, 2], [0, S], [0, 100 * S], [-1, -1], [10 * S, 0], [1, 0], prio=[0, 5], within=abi.POLICY_LOWER_PRIORITY)


def test_readmitted_then_preempted_goes_back_to_its_creation_timestamp():
    rec = []
    r = _run(readmit_preempt_case(), record=rec)
    assert [t // S for t in r.cycle_start_ns] == [0, 70, 100, 101, 102]
    assert [h.tolist() for h in r.heads] == [[0], [0], [1], [1], [0]]
    assert r.wl_ready_ns[0] == 80 * S and r.n_resorts == 2 and [e.tolist() for e in r.evicted][2] == [0]
    assert int(rec[1][0].arrays["wl_ts"][0]) == 10 * S and int(rec[4][0].arrays["wl_ts"][0]) == 0
    assert r.resort_orders[-1]["qts"][0] == 0


def start_state_case():
    """6 cpu.  Row r0 (w0, 2 cpu) has its checks running until 30 s; w1 is in backoff until 50 s (evicted by a check at
    20 s, RetryCount 2) and fails one more attempt; w2 (2 cpu, runs 1000 s) is queued.
      0 w2 admitted | 30 r0 Ready, runs until 130 | 50 w1 returns (its key, 20 s, is unchanged: no re-sort), reserves
      60 Retry: RetryCount 3, back at 60 + 240 = 300 | 130 w0 finishes | 300 w1 returns (a re-sort), reserves, Ready at 310
      410 w1 finishes | 1000 w2 finishes."""
    s = _case([2, 2, 2], [0, 0, 0], [0, 0, 0], [100 * S, 100 * S, 1000 * S], [10 * S] * 2 + [0], [0, 1, 0], nominal=6,
              adm=[(0, 2, 30 * S)])
    s.set("wl_requeue_at_ns", [I64_MIN, 50 * S, I64_MIN]); s.set("wl_check_evict_ns", [I64_MIN, 20 * S, I64_MIN])
    s.set("wl_check_retries", [0, 2, 0])
    return s


def test_start_state_tables():
    r = _run(start_state_case())
    assert [t // S for t in r.cycle_start_ns] == [0, 50, 300]
    assert [h.tolist() for h in r.heads] == [[2], [1], [1]]
    assert (r.wl_ready_ns // S).tolist() == [30, 310, 0] and r.wl_check_retries.tolist() == [0, 3, 0]
    assert (r.wl_finish_ns // S).tolist() == [130, 410, 1000] and r.end_ns == 1000 * S
    assert r.n_check_ready == 2 and r.n_check_retry == 1 and r.n_resorts == 1 and (r.state == FINISHED).all()


# ---------------------------------------------------------------- equivalence: zero delays, no start state
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


def _zero(snap):
    snap.set("wl_check_ns", np.zeros(snap.n_wl)); snap.set("wl_check_fail", np.zeros(snap.n_wl))
    return snap


@pytest.mark.parametrize("name", list(BASE))
def test_zero_delays_change_nothing(name):
    want = _run(BASE[name](), MAX_CYCLES[name])
    got = _run(_zero(BASE[name]()), MAX_CYCLES[name])
    assert got.cycles == want.cycles and got.cycle_start_ns == want.cycle_start_ns
    for k in range(want.cycles):
        assert np.array_equal(got.heads[k], want.heads[k]) and np.array_equal(got.decisions[k], want.decisions[k]), k
        assert np.array_equal(got.evicted[k], want.evicted[k]) and np.array_equal(got.finished[k], want.finished[k]), k
    assert np.array_equal(got.cq_usage, want.cq_usage)
    for f in ("wl_admit_cycle", "wl_evictions", "wl_admit_ns", "wl_finish_ns", "state"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    assert got.n_check_retry == got.n_check_ready == got.n_resorts == 0
    assert np.array_equal(got.wl_ready_ns, want.wl_admit_ns)


# ---------------------------------------------------------------- invariants on seeded drains
def _cfg4_checks():
    return synth.add_admission_checks(_cfg4(), seed=5)


def _baseline_checks():
    return synth.perf_scenario(0.1, checks=7)


SEEDED = {"cfg4-checks": _cfg4_checks, "baseline-checks": _baseline_checks}


def _cells_of(adm, Q, FR):
    use = np.zeros((Q, FR), np.int64)
    st = adm["adm_use_start"]
    for a in range(len(adm["adm_cq"])):
        for k in range(int(st[a]), int(st[a + 1])):
            use[int(adm["adm_cq"][a]), int(adm["adm_use_fr"][k])] += int(adm["adm_use_qty"][k])
    return use


@pytest.mark.parametrize("name", list(SEEDED))
def test_check_invariants(name):
    snap = SEEDED[name]()
    a = snap.arrays
    res = _run(snap, 100_000)
    assert res.n_check_retry > 0 and res.n_check_ready > 0
    Q, FR = snap.n_cq, snap.n_fr
    init = {k: a[k] for k in ("adm_cq", "adm_use_start", "adm_use_fr", "adm_use_qty")}
    assert np.array_equal(res.cq_usage - _cells_of(res.adm, Q, FR), a["cq_usage"].reshape(Q, FR) - _cells_of(init, Q, FR))
    assert set(np.unique(res.state).tolist()) <= {QUEUED, SET_ASIDE, HELD, ABSENT, FINISHED, BACKOFF, DEACTIVATED}
    held = set(res.adm["adm_wl"].tolist())
    assert held == set(np.flatnonzero(res.state == HELD).tolist())  # one state per record: HELD iff it has a row
    assert (res.wl_check_retries <= snap.check_backoff_limit).all()
    gone = set(np.flatnonzero(res.wl_deactivated).tolist())
    assert gone == set(np.flatnonzero(res.state == DEACTIVATED).tolist()) and len(gone) == res.n_check_rejected
    rejected_at = {}
    for k in range(res.cycles):
        for w in res.check_rejected[k].tolist():
            rejected_at[w] = k
    for k in range(res.cycles):  # a deactivated record is never a head again
        for w in res.heads[k].tolist():
            assert w not in rejected_at or k <= rejected_at[w], (w, k)
    key = lambda w: (-int(a["wl_priority"][w]), int(qts[w]), int(a["wl_uid"][w]))  # noqa: E731
    for rs in res.resort_orders:  # the state every re-sort rebuilt, checked element by element
        order, qstart, qts, st = rs["order"], rs["qstart"], rs["qts"], rs["state"]
        assert sorted(order.tolist()) == list(range(snap.n_wl))
        for s in range(len(qstart) - 1):
            seg = order[qstart[s]:qstart[s + 1]]
            assert (rs["seg_of"][seg] == s).all() and (rs["pos_of"][seg] == np.arange(len(seg))).all()
            assert all(key(x) < key(y) for x, y in zip(seg[:-1], seg[1:])), s  # queueOrderingFunc, strictly
            q = np.flatnonzero(st[seg] == QUEUED)
            aside = np.flatnonzero(st[seg] == SET_ASIDE)
            assert rs["cursor"][s] == (q[0] if len(q) else len(seg)), s
            assert rs["first_aside"][s] == (aside[0] if len(aside) else len(seg)), s
    assert res.n_resorts > 0
    if name == "baseline-checks":
        plain = _run(_baseline(), 100_000)
        print(f"baseline x0.1 with checks: {res.cycles} cycles, end {res.end_ns / 1e9:.3f} s, verdicts ready/retry/rejected "
              f"{res.n_check_ready}/{res.n_check_retry}/{res.n_check_rejected}, {res.n_resorts} re-sorts; without: "
              f"{plain.cycles} cycles, end {plain.end_ns / 1e9:.3f} s")


# ---------------------------------------------------------------------------------------------------------------- GPU
DEVICE_CASES = {
    "delay": delay_case, "retry": retry_case, "rejected": rejected_case, "preempt-checking": preempt_checking_case,
    "readmit-preempt": readmit_preempt_case, "start-state": start_state_case, "base-above-max": inverted_backoff_case,
    "zero-cfg2": lambda: _zero(_cfg2()), "zero-cfg3-afs": lambda: _zero(_cfg3_afs()), "zero-cfg4": lambda: _zero(_cfg4()),
    "zero-baseline": lambda: _zero(_baseline()),
    "cfg4-checks": _cfg4_checks, "cfg4-checks-latency": lambda: synth.add_evict_latency(_cfg4_checks(), (3_000, 40_000), seed=4),
    "baseline-checks": lambda: synth.perf_scenario(1.0, checks=7),
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
        assert int(got.cycle_check_retry[k]) == len(want.check_retry[k]), k
        assert int(got.cycle_check_rejected[k]) == len(want.check_rejected[k]), k
    assert got.n_evicted == want.n_evicted and got.n_finished == want.n_finished and got.end_ns == want.end_ns
    assert (got.n_check_ready, got.n_check_retry, got.n_check_rejected) == (want.n_check_ready, want.n_check_retry, want.n_check_rejected)
    assert got.n_resorts == want.n_resorts
    for f in ("wl_admit_ns", "wl_finish_ns", "wl_evictions", "wl_admit_cycle", "cq_usage", "wl_ready_ns"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    assert np.array_equal(got.wl_check_retries_out, want.wl_check_retries)
    assert np.array_equal(got.wl_deactivated, want.wl_deactivated)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DEVICE_CASES))
def test_kb_run_drain_checks_like_the_host_definition(name):
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = DEVICE_CASES[name]()
        mc = 100_000 if "baseline" in name else 400
        want = _run(snap, mc)
        got = ev.run_drain(snap, abi.DrainOut(snap, mc, trace_capacity=want.n_decisions))
        compare(want, got)
        if name == "baseline-checks":
            assert got.n_check_retry > 0 and got.n_resorts > 0
    finally:
        ev.close()


def _refused(ev, snap, code):
    from kueue_b200 import native
    with pytest.raises(native.KueueB200Error) as e:
        ev.run_drain(snap, max_cycles=5)
    assert e.value.code == code


@pytest.fixture
def evaluator():
    from kueue_b200 import native
    ev = native.Evaluator(0)
    yield ev
    ev.close()


@pytest.mark.gpu
def test_refuses_a_negative_delay(evaluator):
    s = delay_case(); s.set("wl_check_ns", [-1, 0])
    _refused(evaluator, s, abi.KB_ERR_INVALID)


@pytest.mark.gpu
def test_refuses_a_negative_fail_count(evaluator):
    s = delay_case(); s.set("wl_check_fail", [-1, 0])
    _refused(evaluator, s, abi.KB_ERR_INVALID)


@pytest.mark.gpu
def test_refuses_a_check_end_at_or_before_now(evaluator):
    s = start_state_case(); s.set("adm_check_end_ns", [0])
    _refused(evaluator, s, abi.KB_ERR_INVALID)


@pytest.mark.gpu
def test_refuses_tables_without_adm_wl(evaluator):
    s = delay_case(); del s.arrays["adm_wl"]
    _refused(evaluator, s, abi.KB_ERR_INVALID)


@pytest.mark.gpu
def test_refuses_a_requeue_time_on_a_held_record(evaluator):
    s = start_state_case(); s.set("wl_requeue_at_ns", [50 * S, I64_MIN, I64_MIN])
    _refused(evaluator, s, abi.KB_ERR_INVALID)


@pytest.mark.gpu
@pytest.mark.parametrize("base,mx,limit", [(0, 1800, 3), (60, -1, 3), (60, 1800, -1)])
def test_refuses_a_bad_retry_strategy(evaluator, base, mx, limit):
    s = delay_case()
    s.check_backoff_base_s, s.check_backoff_max_s, s.check_backoff_limit = base, mx, limit
    _refused(evaluator, s, abi.KB_ERR_INVALID)


@pytest.mark.gpu
def test_refuses_a_random_backoff(evaluator):
    s = delay_case()
    s.check_backoff_base_s, s.check_backoff_max_s, s.check_backoff_limit = 60, 0, 9  # 60 * 2^8 = 15,360 s
    _refused(evaluator, s, abi.KB_ERR_UNSUPPORTED)
    s.check_backoff_max_s = 9_999  # capped below the bound: accepted
    assert evaluator.run_drain(s, max_cycles=5).n_cycles > 0
    s.check_backoff_base_s, s.check_backoff_max_s, s.check_backoff_limit = 20_000, 5_000, 1  # attempt 1 waits the base
    _refused(evaluator, s, abi.KB_ERR_UNSUPPORTED)


@pytest.mark.gpu
def test_refuses_a_row_with_an_eviction_and_a_check_under_way(evaluator):
    s = start_state_case()
    s.set("wl_evict_ns", np.full(s.n_wl, S)); s.set("adm_evicted", [1]); s.set("adm_evict_end_ns", [40 * S])
    _refused(evaluator, s, abi.KB_ERR_INVALID)
    s.set("adm_evicted", [0])  # the end time is read only where adm_evicted is set: accepted
    assert evaluator.run_drain(s, max_cycles=5).n_cycles > 0


@pytest.mark.gpu
def test_refuses_checks_with_afs_decay(evaluator):
    snap = synth.add_events(synth.make_snapshot(3, W=200, Q=8, afs=2), seed=2)
    snap.set("adm_wl", np.zeros(0))
    snap.set("lq_last_update_ns", np.full(len(snap.arrays["lq_cq"]), snap.now_ns)); snap.set("adm_lq", np.full(snap.n_adm, -1))
    snap.afs_half_life_ns, snap.afs_sampling_ns = 10 * S, S
    _refused(evaluator, _zero(snap), abi.KB_ERR_UNSUPPORTED)
