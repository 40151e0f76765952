"""AdmissionFairSharing in the drain (kueue_b200/drain.py, kb_run_drain): ClusterQueues in UsageBasedAdmissionFairSharing
mode order their queue by LocalQueue usage first, and every admission adds an entry penalty to its LocalQueue.

CPU: the quantity rules, the reference's cases (tests/golden/afs_cases.json, transcribed by hand from
cluster_queue_test.go:1054-1225, scheduler_afs_test.go:47-657 and preemption_test.go:4525-4641) on the host definition
over the oracle, and invariants.  GPU: kb_run_drain equals the host definition cycle by cycle."""
import json
import math
import os

import numpy as np
import pytest

import oracle
from kueue_b200 import abi, api, synth
from kueue_b200.drain import (AfsOverflow, compare_usage, drain, entry_penalty, lq_usage, quantity_add, quantity_float)

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "afs_cases.json")))
S = 1_000_000_000


# ---------------------------------------------------------------- quantity rules
def test_quantity_add_zero_shortcuts_keep_the_other_scale():
    # int64Amount.Add (amount.go:162-169): b == 0 keeps a as it is, a == 0 takes b with its scale
    assert quantity_add((5, 0), (0, -3)) == (5, 0)
    assert quantity_add((0, 0), (7, -3)) == (7, -3)
    assert quantity_add((0, 3), (0, -3)) == (0, 3)
    assert quantity_add((7, -9), (0, -3)) == (7, -9)


@pytest.mark.parametrize("consumed,want", [
    ((2, 0), (2267, -3)),          # "2" + 267m: aligned to the smaller scale
    ((15, -1), (1767, -3)),        # "1.5"
    ((3500, -3), (3767, -3)),      # "3500m": same scale, values add
    ((5, -9), (5 + 267 * 10**6, -9)),  # "5n": the penalty is scaled up instead
    ((1, 3), (1000267, -3)),       # "1k"
])
def test_quantity_add_aligns_to_the_smaller_scale(consumed, want):
    assert quantity_add(consumed, (267, -3)) == want


def test_quantity_add_overflow_is_reported():
    with pytest.raises(AfsOverflow):
        quantity_add((2**62, 0), (1, -3))       # 2^62 * 1000 leaves int64
    with pytest.raises(AfsOverflow):
        quantity_add((2**63 - 1, -3), (1, -3))  # int64Add


def test_milli_float_is_a_product_with_the_reciprocal():
    # AsApproximateFloat64: value * math.Pow10(-3), and Pow10(-3) = 1/1000 — not value / 1000
    differ = [v for v in range(1, 5000) if v * (1.0 / 1000) != v / 1000.0]
    assert differ, "no value where the two roundings differ"
    v = differ[0]
    assert quantity_float(v, -3) == v * (1.0 / 1000) != v / 1000.0
    assert quantity_float(7, 0) == 7.0 and quantity_float(3, 3) == 3000.0


def test_usage_sums_in_resource_order_and_divides_by_the_weight():
    cons, sc, pen = [2, 1, 0], [0, 0, 0], [267, 0, 500]
    want = (2.0 * quantity_float(2267, -3) + 0.5 * 1.0 + 1.0 * quantity_float(500, -3)) / 2.0
    assert lq_usage(cons, sc, pen, [2.0, 0.5, 1.0], 2.0) == want


def test_weight_zero_orders_like_cmp_compare():
    inf = lq_usage([3], [0], [0], [1.0], 0.0)
    nan = lq_usage([0], [0], [0], [1.0], 0.0)
    assert inf == math.inf and math.isnan(nan)
    keys = [inf, 1.5, nan, 0.0, -0.0]
    import functools
    ordered = sorted(keys, key=functools.cmp_to_key(compare_usage))
    assert math.isnan(ordered[0]) and ordered[1:3] == [0.0, 0.0] and ordered[3:] == [1.5, inf]
    assert compare_usage(nan, nan) == 0 and compare_usage(-0.0, 0.0) == 0


def test_entry_penalty_uses_the_keys_of_requests_and_truncates():
    alpha = api.AdmissionFairSharing(10, 1).alpha
    req = np.array([[4000, 2**30, 0], [500, 0, 7]])     # cpu milli, memory bytes, a resource that is not a key
    mask = np.array([0b011, 0b001])
    got = entry_penalty(req, mask, [1, 1000, 1000], alpha)
    assert got == [int(4500.0 * alpha), int(float(2**30 * 1000) * alpha), 0]


# ---------------------------------------------------------------- reference cases
def _fs_admission_snapshot(case):
    cq = api.MakeClusterQueue("cq").AdmissionMode(case["cq_mode"])
    lqs = [api.MakeLocalQueue(q["name"]).FairSharing(q["weight"]).ClusterQueue("cq") for q in case["lqs"]]
    wls = [api.MakeWorkload(w["name"]).Queue(w["queue"]).PodSets(api.MakePodSet("main", 1).Request("cpu", "1")).Priority(w["priority"])
           for w in case["workloads"]]
    cfg = None if case["afs_config"] is None else api.AdmissionFairSharing(resource_weights=case["afs_config"]["resource_weights"])
    return api.flatten([cq], pending=wls, local_queues=lqs, afs_config=cfg, consumed=case["consumed"])


@pytest.mark.parametrize("name", [c["name"] for c in GOLDEN["fs_admission"]])
def test_fs_admission_first_pop(name):
    """TestFsAdmission: the first head of the queue (one cycle of the drain evaluates exactly the first Pop)."""
    case = next(c for c in GOLDEN["fs_admission"] if c["name"] == name)
    snap, idx = _fs_admission_snapshot(case)
    res = drain(snap, oracle.run_cycle, max_cycles=1)
    assert [idx.pending[int(w)] for w in res.heads[0]] == [case["want"]]


def _schedule_snapshot(case):
    cq = (api.MakeClusterQueue("cq1").ResourceGroup(api.MakeFlavorQuotas("default").Resource("cpu", "8").Resource("memory", "8Gi"))
          .AdmissionMode("UsageBasedAdmissionFairSharing"))
    lqs = [api.MakeLocalQueue(n).FairSharing("1").ClusterQueue("cq1") for n in ("lq-a", "lq-b", "lq-c")]
    wls = []
    for w in case["workloads"]:
        mw = api.MakeWorkload(w["name"]).Queue(w["queue"]).PodSets(api.MakePodSet("one", 1).Request("cpu", w["cpu"]))
        wls.append(mw.Creation((w["creation_s"] or 0) * S))
    cfg = api.AdmissionFairSharing(usage_half_life_s=10, usage_sampling_s=1) if case["gate"] else None
    return api.flatten([cq], pending=wls, local_queues=lqs, afs_config=cfg, consumed=case["consumed"], flavors=["default"])


def _check_schedule(case, snap, idx, admitted_wl, ps_flavor, ps_count):
    """The admitted set, flavor and quantity of every admitted workload; the reference's Pending ones stay pending.
    The drain stops at its first cycle without an admission, which can come before the reference's last NoFit
    evaluation (it runs one schedule() per workload): that evaluation admits nothing and changes no outcome."""
    got = {idx.pending[int(w)] for w in admitted_wl}
    assert got == set(case["admitted"])
    assert not got & set(case["pending"])
    cpu = idx.resources.index("cpu")
    for name, want in case["admitted"].items():
        w = idx.pending.index(name)
        row = int(snap.arrays["wl_ps_start"][w])
        assert idx.flavors[int(ps_flavor[row, cpu])] == want["flavor"]
        assert int(ps_count[row]) == want["count"]
        assert int(snap.arrays["ps_req"].reshape(-1, snap.n_resource)[row, cpu]) // want["count"] * int(ps_count[row]) == \
            api.resource_value("cpu", want["cpu"])


@pytest.mark.parametrize("name", [c["name"] for c in GOLDEN["schedule"]])
def test_schedule_for_afs(name):
    case = next(c for c in GOLDEN["schedule"] if c["name"] == name)
    snap, idx = _schedule_snapshot(case)
    outs = []
    res = drain(snap, lambda s: outs.append(oracle.run_cycle(s)) or outs[-1])
    R = snap.n_resource
    flavor = np.full((snap.n_podset, R), -1, np.int8); count = np.zeros(snap.n_podset, np.int32)
    for heads, out in zip(res.heads, outs):  # per-cycle tables hold the heads' podsets in head order
        row = 0
        for w in heads:
            r0, r1 = int(snap.arrays["wl_ps_start"][w]), int(snap.arrays["wl_ps_start"][w + 1])
            flavor[r0:r1] = out.ps_flavor[row:row + r1 - r0]; count[r0:r1] = out.ps_count[row:row + r1 - r0]
            row += r1 - r0
    _check_schedule(case, snap, idx, np.concatenate(res.admitted), flavor, count)


def _candidates_less(a, b, preemptor_cq, afs):
    """CandidatesOrdering (preemption/common/ordering.go:41-100) restated for unevicted candidates with the same
    quota-reservation time: other ClusterQueues first; with AFS, inside one ClusterQueue and across LocalQueues,
    higher LocalQueue usage first; then lower priority first."""
    if (a["cq"] == preemptor_cq) != (b["cq"] == preemptor_cq):
        return -1 if b["cq"] == preemptor_cq else 1
    if afs and a["cq"] == b["cq"] and a["queue"] != b["queue"]:
        c = compare_usage(b["lq_usage"], a["lq_usage"])
        if c:
            return c
    return (a["priority"] > b["priority"]) - (a["priority"] < b["priority"])


@pytest.mark.parametrize("name", [c["name"] for c in GOLDEN["candidates_ordering"]])
def test_candidates_ordering_afs_cases(name):
    import functools
    case = next(c for c in GOLDEN["candidates_ordering"] if c["name"] == name)
    got = sorted(case["candidates"], key=functools.cmp_to_key(lambda a, b: _candidates_less(a, b, "preemptor", True)))
    assert [c["name"] for c in got] == case["want"]


def test_candidates_ordering_with_afs_is_not_transitive():
    """Why kb_run_cycle / kb_run_drain refuse AFS with a possible target search: across ClusterQueues the comparator
    above has cycles (c < a by usage, a < b by priority, b < c by priority), so the order slices.SortFunc gives depends
    on the algorithm, and no preemptor-independent rank reproduces it."""
    a = {"cq": "cq1", "queue": "lq1", "priority": 1, "lq_usage": 0.1}
    c = {"cq": "cq1", "queue": "lq2", "priority": 3, "lq_usage": 0.9}
    b = {"cq": "cq2", "queue": "lq3", "priority": 2, "lq_usage": 0.5}
    less = lambda x, y: _candidates_less(x, y, "preemptor", True) < 0  # noqa: E731
    assert less(c, a) and less(a, b) and less(b, c)
    assert not (less(a, c) or less(b, a) or less(c, b))


def test_afs_tables_need_their_ClusterQueue_mode():
    snap, _ = _schedule_snapshot(GOLDEN["schedule"][0])
    assert snap.arrays["cq_afs"].tolist() == [1] and snap.afs_alpha == 1.0 - 0.5 ** 0.1
    snap2, _ = _schedule_snapshot(GOLDEN["schedule"][1])
    assert snap2.arrays["cq_afs"].tolist() == [0]


# ---------------------------------------------------------------- invariants
def _same(x, y):
    return x.cycles == y.cycles and all(np.array_equal(p, q) for p, q in zip(x.heads, y.heads)) and \
        all(np.array_equal(p, q) for p, q in zip(x.decisions, y.decisions)) and np.array_equal(x.cq_usage, y.cq_usage)


def _with_hashes(snap):
    rng = np.random.default_rng(3)
    snap.set("wl_sched_hash", rng.integers(0, 6, snap.n_wl))
    return snap


INVARIANT_CASES = [
    lambda: synth.make_snapshot(2, W=3000, Q=30, podsets_max=2),        # StrictFIFO
    lambda: synth.make_snapshot(3, W=2000, Q=40),                       # flat cohorts, fair sharing
    lambda: _with_hashes(synth.make_snapshot(3, W=4000, Q=40)),         # scheduling-hash bulk move
]


@pytest.mark.parametrize("make", INVARIANT_CASES)
def test_afs_off_or_one_localqueue_is_the_plain_drain(make):
    plain = drain(make(), oracle.run_cycle)
    off = synth.add_afs(make(), 4); off.set("cq_afs", np.zeros(off.n_cq))
    assert _same(drain(off, oracle.run_cycle), plain)
    one = synth.add_afs(make(), 1)
    assert _same(drain(one, oracle.run_cycle), plain)


def _afs_key(a, w, usage):
    return (0 if usage != usage else 1, 0.0 if usage != usage else usage, -int(a["wl_priority"][w]), int(a["wl_ts"][w]), int(a["wl_uid"][w]))


@pytest.mark.parametrize("make", INVARIANT_CASES)
def test_afs_heads_follow_usage_then_priority(make):
    """Along every AFS ClusterQueue, the head of a cycle precedes (usage with the penalties of that cycle, -priority,
    timestamp, UID) every workload of the queue evaluated in a later cycle.  Penalties are recomputed here from the
    admitted sequence."""
    snap = synth.add_afs(make(), 4)
    a, R = snap.arrays, snap.n_resource
    L = len(a["lq_cq"])
    res = drain(snap, oracle.run_cycle)
    assert res.n_admitted > 0
    pen = a["lq_penalty"].reshape(L, R).astype(object).copy()
    cons, sc = a["lq_consumed"].reshape(L, R), a["lq_consumed_scale"].reshape(L, R)
    ps, req = a["wl_ps_start"], a["ps_req"].reshape(-1, R)
    later = [set() for _ in range(res.cycles)]
    for k in range(res.cycles - 2, -1, -1):
        later[k] = later[k + 1] | {int(w) for w in res.heads[k + 1]}
    lqs_changed = 0
    for k in range(res.cycles):
        usage = [lq_usage(cons[l], sc[l], pen[l], a["afs_res_weight"], a["lq_weight"][l]) for l in range(L)]
        for w in res.heads[k]:
            q = int(a["wl_cq"][w])
            hk = _afs_key(a, w, usage[int(a["wl_lq"][w])])
            for w2 in later[k]:
                if int(a["wl_cq"][w2]) == q and w2 != w:
                    assert hk <= _afs_key(a, w2, usage[int(a["wl_lq"][w2])]), (k, w, w2)
        for w in res.admitted[k]:
            l = int(a["wl_lq"][w])
            for r, d in enumerate(entry_penalty(req[ps[w]:ps[w + 1]], a["ps_req_mask"][ps[w]:ps[w + 1]], a["afs_milli_mul"], snap.afs_alpha)):
                pen[l, r] += d
            lqs_changed += 1
    assert lqs_changed == res.n_admitted


# ---------------------------------------------------------------- device
def _with_mixed_modes(snap):
    snap.set("cq_afs", np.arange(snap.n_cq) % 2)  # every other ClusterQueue keeps the plain order
    return snap


DEVICE_CASES = {
    "flat-cohorts-fair-sharing": lambda: synth.make_snapshot(3, W=2000, Q=40, afs=4),
    "strict-fifo": lambda: synth.make_snapshot(2, W=3000, Q=30, podsets_max=2, afs=3),
    "partial-admission": lambda: synth.make_snapshot(3, W=1500, Q=60, partial=True, podsets_max=2, afs=4),
    "scheduling-hash": lambda: _with_hashes(synth.make_snapshot(3, W=4000, Q=40, afs=4)),
    "64-localqueues": lambda: synth.make_snapshot(3, W=12000, Q=20, afs=64),
    "mixed-modes": lambda: _with_mixed_modes(synth.make_snapshot(3, W=2000, Q=40, afs=5)),
    "no-cohort": lambda: synth.make_snapshot(1, afs=3),
}


def _device_equals_host(ev, snap, max_cycles=10_000):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000
    want = drain(snap, lambda s: oracle.run_cycle(s, cap), max_cycles=max_cycles)
    got = ev.run_drain(snap, max_cycles=max_cycles)
    assert got.n_cycles == want.cycles
    cyc = got.cycles()
    for k in range(want.cycles):
        assert np.array_equal(cyc[k][0], want.heads[k]), k
        assert np.array_equal(cyc[k][1], want.decisions[k]), k
    assert np.array_equal(got.cq_usage, want.cq_usage)
    adm = np.concatenate(want.admitted) if want.admitted else np.zeros(0, np.int64)
    assert got.n_admitted == len(adm) and np.array_equal(np.flatnonzero(got.wl_admit_cycle >= 0), np.sort(adm))
    return want, got


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DEVICE_CASES))
def test_kb_run_drain_afs_equals_host_definition(name):
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        want, _ = _device_equals_host(ev, DEVICE_CASES[name]())
        assert want.n_admitted > 0
    finally:
        ev.close()


@pytest.mark.gpu
def test_kb_run_drain_afs_full_size_config3():
    """cfg3 at full size, 8 LocalQueues per ClusterQueue: 80k LocalQueues, one warp per ClusterQueue picks the heads."""
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        _device_equals_host(ev, synth.make_snapshot(3, afs=8), max_cycles=6)
    finally:
        ev.close()


@pytest.mark.gpu
def test_kb_run_drain_afs_goldens():
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        for case in GOLDEN["fs_admission"]:
            snap, idx = _fs_admission_snapshot(case)
            got = ev.run_drain(snap, max_cycles=1)
            assert [idx.pending[int(w)] for w in got.cycles()[0][0]] == [case["want"]], case["name"]
        for case in GOLDEN["schedule"]:
            snap, idx = _schedule_snapshot(case)
            got = ev.run_drain(snap)
            _check_schedule(case, snap, idx, np.flatnonzero(got.wl_admit_cycle >= 0), got.ps_flavor, got.ps_count)
    finally:
        ev.close()


@pytest.mark.gpu
def test_afs_with_preemption_policies_is_refused():
    """A possible target search with an AFS ClusterQueue: KB_ERR_UNSUPPORTED from the host-side checks (the caller
    then runs the Go cycle).  Without AFS ClusterQueues, or without a possible target search, the tables are accepted."""
    from kueue_b200 import native
    ev = native.Evaluator(0)
    try:
        snap = synth.make_snapshot(2, W=3000, Q=30, preemption=True, tight=1.2, afs=2)
        for call in (lambda: ev.run_drain(snap), lambda: ev.run_cycle(snap)):
            with pytest.raises(native.KueueB200Error) as e:
                call()
            assert e.value.code == abi.KB_ERR_UNSUPPORTED
        snap.set("cq_afs", np.zeros(snap.n_cq))
        plain = synth.make_snapshot(2, W=3000, Q=30, preemption=True, tight=1.2)
        assert ev.run_drain(snap, max_cycles=3).n_admitted == ev.run_drain(plain, max_cycles=3).n_admitted
        one = synth.make_snapshot(3, W=3000, Q=300, heads="one_per_cq", afs=4)  # kb_run_cycle ignores the tables
        got, want = ev.run_cycle(one), oracle.run_cycle(one)
        assert np.array_equal(got.decision, want.decision) and np.array_equal(got.ps_flavor, want.ps_flavor)
    finally:
        ev.close()


@pytest.mark.gpu
def test_invalid_afs_tables_are_rejected_on_the_host():
    """The host-side O(n) checks: indices, the ClusterQueue of a workload's LocalQueue, ClusterQueue-major numbering
    (KB_ERR_INVALID), and quantities outside the int64Amount arithmetic (KB_ERR_UNSUPPORTED)."""
    from kueue_b200 import native
    ev = native.Evaluator(0)

    def code(edit):
        snap = synth.make_snapshot(1, afs=2)
        edit(snap)
        with pytest.raises(native.KueueB200Error) as e:
            ev.run_drain(snap)
        return e.value.code
    try:
        assert code(lambda s: s.set("wl_lq", np.where(np.arange(s.n_wl) == 0, 99, s.arrays["wl_lq"]))) == abi.KB_ERR_INVALID
        assert code(lambda s: s.set("wl_lq", (s.arrays["wl_lq"] + 2) % len(s.arrays["lq_cq"]))) == abi.KB_ERR_INVALID
        assert code(lambda s: s.set("lq_cq", s.arrays["lq_cq"][::-1])) == abi.KB_ERR_INVALID
        assert code(lambda s: s.set("lq_consumed_scale", np.full_like(s.arrays["lq_consumed_scale"], 30))) == abi.KB_ERR_UNSUPPORTED
        assert code(lambda s: (s.set("lq_consumed", np.full_like(s.arrays["lq_consumed"], 2**62)),
                               s.set("lq_penalty", np.ones_like(s.arrays["lq_penalty"])))) == abi.KB_ERR_UNSUPPORTED
    finally:
        ev.close()


def test_shard_carries_the_localqueue_tables():
    from kueue_b200 import shard
    snap = synth.make_snapshot(3, W=2000, Q=40, afs=3)
    a = snap.arrays
    total = 0
    for rank in range(2):
        sub, m = shard.shard(snap, rank, 2)
        b = sub.arrays
        assert (b["lq_cq"][b["wl_lq"]] == b["wl_cq"]).all() and (np.diff(b["lq_cq"]) >= 0).all()
        assert sub.afs_alpha == snap.afs_alpha
        # every pending workload keeps its LocalQueue's consumed usage and weight
        gl = a["wl_lq"][m.wls]
        assert np.array_equal(b["lq_consumed"].reshape(-1, 4)[b["wl_lq"]], a["lq_consumed"].reshape(-1, 4)[gl])
        assert np.array_equal(b["lq_weight"][b["wl_lq"]], a["lq_weight"][gl])
        total += len(b["lq_cq"])
    assert total == len(a["lq_cq"])
