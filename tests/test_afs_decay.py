"""Decay of AdmissionFairSharing consumed usage on the event clock of the drain (kueue_b200/drain.py, kb_run_drain with
kb_snapshot.lq_last_update_ns): samples every UsageSamplingInterval, decay at admission, completions leaving the
admitted usage.

CPU: the reference's reconcile cases (tests/golden/afs_decay_cases.json) on the host definition, the power function
against math.pow and against its host build from kb_drain.cuh, hand-derived admission-time decay, a queue order that
decay flips, the fixed point of a long jump, half-life 0.  GPU: kb_run_drain equals the host definition cycle by cycle
and in its final consumed usage, and refuses bad tables on the host."""
import json
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import oracle
from kueue_b200 import abi, api, synth
from kueue_b200.drain import decay_quantities, drain, half_pow, milli_value

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "afs_decay_cases.json")))["cases"]
S = 1_000_000_000
NOW = 1_000 * S


# ---------------------------------------------------------------- power function
def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


SWEEP = [i / 4096.0 for i in range(64 * 4096 + 1)] + [k + d for k in range(64) for d in (0.5, 0.5 + 2**-40, 1 - 2**-40, 2**-30)]


def test_half_pow_is_within_one_ulp_of_pow_and_exact_at_integers():
    assert half_pow(0.0) == 1.0
    for n in range(65):
        assert half_pow(float(n)) == 2.0**-n
    worst = max(abs(half_pow(x) - math.pow(0.5, x)) / math.ulp(math.pow(0.5, x)) for x in SWEEP)
    assert worst <= 1.0, worst


def test_half_pow_host_build_of_the_header_has_the_same_bits(tmp_path):
    """afs_half_pow compiled from kb_drain.cuh for the host (nvcc, -ffp-contract=off) against the Python restatement."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    src = tmp_path / "half_pow.cu"
    src.write_text('#include <cstdio>\n#include <cstring>\n#include "kb_drain.cuh"\n'
                   "int main() { double x; while (scanf(\"%lf\", &x) == 1) { double y = afs_half_pow(x); unsigned long long b; "
                   "memcpy(&b, &y, 8); printf(\"%llu\\n\", b); } return 0; }\n")
    exe = tmp_path / "half_pow"
    subprocess.check_call([nvcc, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-ffp-contract=off",
                           "-I", os.path.join(ROOT, "kueue_b200", "csrc"), "-o", str(exe), str(src)])
    xs = SWEEP[::7] + [0.3466, 12.5, 0.49999999999]
    out = subprocess.run([str(exe)], input="\n".join(repr(x) for x in xs), capture_output=True, text=True, check=True).stdout.split()
    assert [int(v) for v in out] == [_bits(half_pow(x)) for x in xs]


def test_milli_value_rounds_a_finer_scale_away_from_zero():
    assert milli_value(8, 0) == 8000 and milli_value(6827, -3) == 6827 and milli_value(3, 3) == 3_000_000
    assert milli_value(1501, -6) == 2 and milli_value(-1501, -6) == -2 and milli_value(1000, -6) == 1 and milli_value(1, -22) == 1


# ---------------------------------------------------------------- goldens on the host definition
def _golden_snapshot(case):
    """One LocalQueue, its running workloads admitted, one pending workload that never fits (no quota): the drain
    evaluates it once, waits for an event that never comes and ends, so it only takes its start-of-drain samples."""
    cq = api.MakeClusterQueue("cq").AdmissionMode("UsageBasedAdmissionFairSharing")
    lq = api.MakeLocalQueue("lq").FairSharing("1").ClusterQueue("cq")
    running = []
    for i, (res, flavor, q) in enumerate(case["running"]):
        running.append(api.MakeWorkload(f"run-{i}").Queue("lq").Request(res, q).ReserveQuota(api.MakeAdmission("cq").Assignment(res, flavor, q)))
    pending = [api.MakeWorkload("pending").Queue("lq").Request("cpu", "1")]
    cfg = api.AdmissionFairSharing(usage_half_life_s=case["half_life_s"], usage_sampling_s=case["sampling_s"])
    snap, idx = api.flatten([cq], pending=pending, admitted=running, local_queues=[lq], afs_config=cfg,
                            consumed={"lq": case["consumed"]}, extra_resources=["cpu"], now_ns=NOW)
    snap.set("wl_run_ns", [-1])
    snap.drain_cycle_ns = S
    last = None if case["elapsed_s"] is None else NOW - case["elapsed_s"] * S
    api.add_afs_decay(snap, cfg, [last], [0] * snap.n_adm)
    return snap, idx


def _milli_of(res, snap, l):
    R = snap.n_resource
    return [milli_value(int(v), int(s)) for v, s in zip(res.lq_consumed.reshape(-1, R)[l], res.lq_consumed_scale.reshape(-1, R)[l])]


def _want_milli(case, idx):
    want = [0] * len(idx.resources)
    for r, q in case["want"].items():
        want[idx.resources.index(r)] = milli_value(*api.parse_quantity(q))
    return want


@pytest.mark.parametrize("name", [c["name"] for c in GOLDEN])
def test_reconcile_goldens_on_the_host_definition(name):
    case = next(c for c in GOLDEN if c["name"] == name)
    snap, idx = _golden_snapshot(case)
    res = drain(snap, oracle.run_cycle)
    assert res.cycles == 1 and res.n_admitted == 0
    assert _milli_of(res, snap, 0) == _want_milli(case, idx)
    elapsed = case["elapsed_s"]
    want_last = NOW - elapsed * S if case["want_last"] == "unchanged" else NOW
    assert int(res.lq_last_update_ns[0]) == want_last
    assert res.n_afs_samples == (0 if elapsed is None or elapsed < case["sampling_s"] else 1)


# ---------------------------------------------------------------- hand-derived drains
def _one_queue(quota, workloads, consumed, half_life_s=300, sampling_s=300, last=NOW, lq_names=("lq",)):
    """ClusterQueue 'cq' with `quota` cpu in flavor 'default', LocalQueues `lq_names`; `workloads`: (name, lq, cpu,
    create_ns, run_ns, priority) pending at NOW or later."""
    cq = (api.MakeClusterQueue("cq").ResourceGroup(api.MakeFlavorQuotas("default").Resource("cpu", str(quota)))
          .AdmissionMode("UsageBasedAdmissionFairSharing"))
    lqs = [api.MakeLocalQueue(n).FairSharing("1").ClusterQueue("cq") for n in lq_names]
    wls = [api.MakeWorkload(n).Queue(lq).Request("cpu", cpu).Creation(c).Priority(p) for n, lq, cpu, c, _, p in workloads]
    cfg = api.AdmissionFairSharing(usage_half_life_s=half_life_s, usage_sampling_s=sampling_s)
    snap, idx = api.flatten([cq], pending=wls, local_queues=lqs, afs_config=cfg, consumed=consumed, flavors=["default"], now_ns=NOW)
    snap.set("wl_create_ns", [c for _, _, _, c, _, _ in workloads])
    snap.set("wl_run_ns", [r for _, _, _, _, r, _ in workloads])
    snap.drain_cycle_ns = S
    lasts = last if isinstance(last, list) else [last] * len(lq_names)
    api.add_afs_decay(snap, cfg, lasts, [])
    return snap, idx


def _admission_case(run_ns):
    # 8 cpu consumed, LastUpdate 150 s before the drain; a 4-cpu workload admitted at NOW; a workload that never fits
    # arrives 300 s later (the clock jumps there; the running one finishes first when run_ns < 300 s)
    return _one_queue(4, [("w", "lq", "4", NOW - S, run_ns, 0), ("big", "lq", "8", NOW + 300 * S, -1, 0)], {"lq": {"cpu": "8"}},
                      last=NOW - 150 * S)


def _admit_only(snap):
    """the same snapshot cut before the arrival: the drain ends after the admission"""
    snap.set("wl_create_ns", np.where(snap.arrays["wl_create_ns"] > NOW, abi.KB_NO_LIMIT, snap.arrays["wl_create_ns"]))
    return snap


def test_admission_decays_then_takes_the_penalty():
    """alpha(150 s, 5 min) = 1 - 0.5^0.5: 8000m * 0.5^0.5 -> 5656m, 4000m * (1 - 0.5^0.5) -> 1171m, penalty 4000m * 0.5
    = 2000m: 8827m, LastUpdate = the admission time."""
    snap, _ = _admission_case(-1)
    res = drain(_admit_only(snap), oracle.run_cycle)
    assert res.n_admitted == 1 and res.cycle_start_ns[0] == NOW
    assert _milli_of(res, snap, 0) == [8827] and int(res.lq_last_update_ns[0]) == NOW and res.n_afs_samples == 0
    assert res.lq_consumed_scale.tolist() == [[-3]]


def test_sample_while_it_runs_and_after_it_finished():
    """300 s after the admission: 8827m * 0.5 -> 4413m plus 4000m * 0.5 while the workload runs (6413m); 4413m when it
    finished before the sample."""
    snap, _ = _admission_case(-1)
    res = drain(snap, oracle.run_cycle)
    assert _milli_of(res, snap, 0) == [6413] and int(res.lq_last_update_ns[0]) == NOW + 300 * S and res.n_afs_samples == 1
    snap, _ = _admission_case(100 * S)
    res = drain(snap, oracle.run_cycle)
    assert res.n_finished == 1 and _milli_of(res, snap, 0) == [4413] and res.n_afs_samples == 1


def _order_flip(decay: bool):
    """Shaped after fair_sharing_test.go:1355-1377 ('should promote a workload from LQ with lower recent usage'): lq-a
    runs a 32-cpu workload for 100 s, then wl-a (lq-a, created first) and wl-b (lq-b) wait for the quota.  lq-b's
    40 cpu of consumed usage is old: with decay it fades every 10 s while lq-a's consumed usage rises towards what it
    runs, so wl-b comes first; without the decay tables the 40 cpu stay and wl-a comes first."""
    snap, idx = _one_queue(32, [("wl", "lq-a", "32", NOW, 100 * S, 0), ("wl-a", "lq-a", "32", NOW + 50 * S, -1, 0),
                                ("wl-b", "lq-b", "32", NOW + 50 * S + 1, -1, 0)],
                           {"lq-b": {"cpu": "40"}}, half_life_s=10, sampling_s=10, lq_names=("lq-a", "lq-b"))
    if not decay:
        for k in abi.AFS_DECAY_FIELDS:
            snap.arrays.pop(k)
    return snap, idx


def test_decay_flips_the_order_of_two_localqueues():
    first = {}
    for decay in (True, False):
        snap, idx = _order_flip(decay)
        res = drain(snap, oracle.run_cycle)
        later = [idx.pending[int(w)] for a in res.admitted[1:] for w in a]
        first[decay] = later[0]
    assert first == {True: "wl-b", False: "wl-a"}


def _long_jump(half_life_s=1, finish_ns=None):
    # 8 cpu consumed, 4 cpu running (a row of the snapshot), nothing pending until 500 s later: the clock jumps over 500
    # sampling intervals
    cq = (api.MakeClusterQueue("cq").ResourceGroup(api.MakeFlavorQuotas("default").Resource("cpu", "4"))
          .AdmissionMode("UsageBasedAdmissionFairSharing"))
    lq = api.MakeLocalQueue("lq").FairSharing("1").ClusterQueue("cq")
    run = api.MakeWorkload("run").Queue("lq").Request("cpu", "4").ReserveQuota(api.MakeAdmission("cq").Assignment("cpu", "default", "4"))
    big = api.MakeWorkload("big").Queue("lq").Request("cpu", "8")
    cfg = api.AdmissionFairSharing(usage_half_life_s=half_life_s, usage_sampling_s=1)
    snap, _ = api.flatten([cq], pending=[big], admitted=[run], local_queues=[lq], afs_config=cfg, consumed={"lq": {"cpu": "8"}},
                          flavors=["default"], now_ns=NOW)
    snap.set("wl_create_ns", [NOW + 500 * S]); snap.set("wl_run_ns", [-1])
    snap.drain_cycle_ns = S
    api.add_afs_decay(snap, cfg, [NOW], [0])
    if finish_ns is not None:
        snap.set("adm_finish_ns", [finish_ns])
    return snap, cfg


def test_long_jump_stops_at_the_fixed_point():
    snap, cfg = _long_jump()
    res = drain(snap, oracle.run_cycle)
    cons, sc = [8], [0]
    for _ in range(500):  # every sample, no early stop
        cons, _ = decay_quantities(cons, sc, [4000], [1], cfg.alpha)
        sc = [-3]
    assert cons == [4000]
    assert _milli_of(res, snap, 0) == cons and int(res.lq_last_update_ns[0]) == NOW + 500 * S and res.n_afs_samples == 500


def test_a_row_of_the_snapshot_leaves_the_admitted_usage_when_it_finishes():
    """the running row finishes 100 s in: the samples before it move consumed towards 4 cpu, the ones after towards 0"""
    snap, cfg = _long_jump(finish_ns=NOW + 100 * S)
    res = drain(snap, oracle.run_cycle)
    assert res.n_finished == 1 and res.n_afs_samples == 500
    cons, sc = [8], [0]
    for k in range(500):
        cons, _ = decay_quantities(cons, sc, [4000 if k < 100 else 0], [1], cfg.alpha)
        sc = [-3]
    assert _milli_of(res, snap, 0) == cons == [0]


def test_half_life_zero_resets_consumed_to_empty():
    snap, _ = _long_jump(half_life_s=0)
    assert snap.afs_alpha == 0.0
    res = drain(snap, oracle.run_cycle)
    assert res.lq_consumed.tolist() == [[0]] and res.lq_consumed_scale.tolist() == [[0]] and res.n_afs_samples == 500


def test_without_the_decay_tables_the_drain_is_unchanged():
    snap = synth.add_events(synth.make_snapshot(2, W=2000, Q=20, afs=3), seed=4)
    plain = drain(snap, oracle.run_cycle)
    assert plain.lq_consumed is None and plain.n_afs_samples == 0


# ---------------------------------------------------------------- device
def _decay_cfg(config, W=None, Q=None, seed=0, half_life_cycles=100, sampling_cycles=20):
    snap = synth.make_snapshot(config, W=W, Q=Q, afs=8)
    synth.add_events(snap, seed=seed)
    step = snap.drain_cycle_ns
    return synth.add_afs_decay(snap, seed=seed + 1, half_life_ns=half_life_cycles * step, sampling_ns=sampling_cycles * step)


def _device_equals_host(ev, snap, max_cycles=10_000):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000
    want = drain(snap, lambda s: oracle.run_cycle(s, cap), max_cycles=max_cycles)
    got = ev.run_drain(snap, max_cycles=max_cycles)
    assert got.n_cycles == want.cycles
    cyc = got.cycles()
    for k in range(want.cycles):
        assert np.array_equal(cyc[k][0], want.heads[k]), k
        assert np.array_equal(cyc[k][1], want.decisions[k]), k
        assert int(got.cycle_admitted[k]) == len(want.admitted[k]) and int(got.cycle_start_ns[k]) == want.cycle_start_ns[k], k
    assert np.array_equal(got.cq_usage, want.cq_usage)
    assert got.end_ns == want.end_ns and got.n_finished == want.n_finished
    assert np.array_equal(got.lq_consumed, want.lq_consumed.reshape(got.lq_consumed.shape))
    assert np.array_equal(got.lq_consumed_scale, want.lq_consumed_scale.reshape(got.lq_consumed_scale.shape))
    assert np.array_equal(got.lq_last_update_ns, want.lq_last_update_ns)
    assert got.n_afs_samples == want.n_afs_samples
    return want, got


@pytest.fixture(scope="module")
def ev():
    from kueue_b200 import native
    e = native.Evaluator(0)
    yield e
    e.close()


HAND_CASES = {
    "admission": lambda: _admit_only(_admission_case(-1)[0]),
    "sample-while-running": lambda: _admission_case(-1)[0],
    "sample-after-finish": lambda: _admission_case(100 * S)[0],
    "order-flip": lambda: _order_flip(True)[0],
    "order-flip-off": lambda: _order_flip(False)[0],
    "long-jump": lambda: _long_jump()[0],
    "snapshot-row-finishes": lambda: _long_jump(finish_ns=NOW + 100 * S)[0],
    "half-life-0": lambda: _long_jump(half_life_s=0)[0],
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(HAND_CASES))
def test_kb_run_drain_decay_hand_cases(ev, name):
    snap = HAND_CASES[name]()
    if "lq_last_update_ns" in snap.arrays:
        _device_equals_host(ev, snap)
    else:
        got, want = ev.run_drain(snap), drain(snap, oracle.run_cycle)
        assert [list(h) for h, _ in got.cycles()] == [list(h) for h in want.heads] and got.n_afs_samples == 0


@pytest.mark.gpu
def test_kb_run_drain_decay_goldens(ev):
    for case in GOLDEN:
        snap, idx = _golden_snapshot(case)
        _, got = _device_equals_host(ev, snap)
        lq = [milli_value(int(v), int(s)) for v, s in zip(got.lq_consumed[0], got.lq_consumed_scale[0])]
        assert lq == _want_milli(case, idx), case["name"]


@pytest.mark.gpu
def test_kb_run_drain_decay_config2(ev):
    snap = _decay_cfg(2, W=6000, Q=60, seed=5)
    want, got = _device_equals_host(ev, snap)
    assert want.cycles >= 60 and want.n_afs_samples > 0 and want.n_finished > 0
    full = _decay_cfg(2, seed=7)
    want, _ = _device_equals_host(ev, full, max_cycles=80)
    assert want.cycles >= 60


@pytest.mark.gpu
def test_kb_run_drain_decay_full_size_config3(ev):
    """cfg3 at full size with 8 LocalQueues per ClusterQueue (80k LocalQueues), events, a sample every 20 cycles and a
    half-life of 100 cycles."""
    want, got = _device_equals_host(ev, _decay_cfg(3, seed=11), max_cycles=64)
    assert want.cycles == 64 and want.n_afs_samples > 0


@pytest.mark.gpu
def test_bad_decay_tables_are_refused_on_the_host(ev):
    from kueue_b200 import native

    def code(edit):
        snap = _two_cqs()
        edit(snap)
        with pytest.raises(native.KueueB200Error) as e:
            ev.run_drain(snap, max_cycles=3)
        return e.value.code

    def no_events(s):
        for k in abi.EVENT_FIELDS:
            s.arrays.pop(k, None)

    def no_lq(s):
        for k in abi.AFS_FIELDS:
            s.arrays.pop(k, None)

    def set_(name, fn):
        return lambda s: s.set(name, fn(s.arrays[name]))
    edits = {
        "no event mode": no_events,
        "no wl_lq": no_lq,
        "adm_lq missing": lambda s: s.arrays.pop("adm_lq"),
        "adm_lq out of range": set_("adm_lq", lambda v: [2]),
        "adm_lq below -1": set_("adm_lq", lambda v: [-2]),
        "adm_lq of another ClusterQueue": set_("adm_lq", lambda v: [1]),
        "last update after now": set_("lq_last_update_ns", lambda v: v + 10**9),
        "alpha of 1": lambda s: setattr(s, "afs_alpha", 1.0),
        "negative alpha": lambda s: setattr(s, "afs_alpha", -0.1),
        "alpha with half-life 0": lambda s: setattr(s, "afs_half_life_ns", 0),
        "negative half-life": lambda s: setattr(s, "afs_half_life_ns", -1),
        "sampling 0": lambda s: setattr(s, "afs_sampling_ns", 0),
    }
    for name, edit in edits.items():
        assert code(edit) == abi.KB_ERR_INVALID, name
    for ok in (lambda s: None, lambda s: s.set("adm_lq", [-1]), lambda s: (setattr(s, "afs_half_life_ns", 0), setattr(s, "afs_alpha", 0.0))):
        snap = _two_cqs()
        ok(snap)
        assert ev.run_drain(snap, max_cycles=3).n_cycles > 0


def _two_cqs():
    """two ClusterQueues with one LocalQueue each, a running row of lq-1 in cq-1, one pending workload per queue"""
    cqs = [(api.MakeClusterQueue(f"cq-{i}").ResourceGroup(api.MakeFlavorQuotas("default").Resource("cpu", "4"))
            .AdmissionMode("UsageBasedAdmissionFairSharing")) for i in (1, 2)]
    lqs = [api.MakeLocalQueue(f"lq-{i}").FairSharing("1").ClusterQueue(f"cq-{i}") for i in (1, 2)]
    run = api.MakeWorkload("run").Queue("lq-1").Request("cpu", "2").ReserveQuota(api.MakeAdmission("cq-1").Assignment("cpu", "default", "2"))
    wls = [api.MakeWorkload(f"w-{i}").Queue(f"lq-{i}").Request("cpu", "1") for i in (1, 2)]
    cfg = api.AdmissionFairSharing(usage_half_life_s=10, usage_sampling_s=1)
    snap, _ = api.flatten(cqs, pending=wls, admitted=[run], local_queues=lqs, afs_config=cfg, consumed={"lq-1": {"cpu": "3"}},
                          flavors=["default"], now_ns=NOW)
    snap.set("wl_run_ns", [5 * S, 5 * S]); snap.drain_cycle_ns = S
    return api.add_afs_decay(snap, cfg, [NOW - 3 * S, None], [0])
