"""The flavor walk (findFlavorForPodSets, flavorassigner.go:762-897) on every cycle route and in kb_run_drain, against the
CPU oracle, on snapshots whose walk inputs are not synth's defaults.

synth.make_snapshot gives every ClusterQueue one resource group over all resources and all flavors in index order, with
default fungibility, no preference and no last-scheduling context.  The builders below replace those inputs while
keeping the snapshot API-valid:
  - `ragged`: 1-3 resource groups per ClusterQueue with disjoint resources, ordered flavor lists of varying length,
    sometimes a resource that no group covers;
  - `policies`: whenCanBorrow, whenCanPreempt and the preference drawn per ClusterQueue;
  - `last_tried`: ClusterQueue generations, current / stale / nil LastAssignments and a start index per (podset, group);
  - `pods`: the last resource is corev1.ResourcePods, covered by some ClusterQueues only.

Every device case proves the route it names from the per-kernel timings (kb_set_profile) and the group-walk counters,
and every fixture shows, on the oracle, that each of the three inputs changes the cycle's answer."""
import copy

import numpy as np
import pytest

import oracle
from kueue_b200 import abi, shard, synth
from kueue_b200.drain import drain
from tests.helpers import assert_cycle_equal

# ------------------------------------------------------------------------------------------------------------- builders


def _groups(snap):
    """[(ClusterQueue, resource mask, flavor list)] of every resource group"""
    a = snap.arrays
    out = []
    for q in range(snap.n_cq):
        for g in range(int(a["cq_rg_start"][q]), int(a["cq_rg_start"][q + 1])):
            fl = a["rg_flavors"][int(a["rg_flavor_start"][g]):int(a["rg_flavor_start"][g + 1])]
            out.append((q, int(a["rg_res_mask"][g]), fl.astype(np.int64)))
    return out


def _covered_resources(snap):
    """[n_cq] mask of the resources some resource group of the ClusterQueue covers"""
    cov = np.zeros(snap.n_cq, np.int64)
    for q, m, _ in _groups(snap):
        cov[q] |= m
    return cov


def ragged(snap, seed):
    """1-3 resource groups per ClusterQueue with disjoint resource masks (in about 15 % of the ClusterQueues one
    resource belongs to no group), each an ordered list of distinct flavors, no flavor in two groups of a ClusterQueue.
    Uncovered cells get no quota (nominal 0, no limits, no usage); admitted workloads lose their usage cells outside the
    cover (a row left without cells is dropped: an admitted workload holds quota) and cq_usage is their sum again.  About
    90 % of the podsets drop their requests for uncovered resources; the rest keep them (NoFit, flavorassigner.go:770)."""
    rng = np.random.default_rng(seed)
    a = snap.arrays
    Q, F, R, N, FR = snap.n_cq, snap.n_flavor, snap.n_resource, snap.n_nodes, snap.n_fr
    assert "adm_wl" not in a, "build evictable records after ragged: they copy the admitted usage"
    rg_start, masks, fl_start, flavors = [0], [], [0], []
    for _ in range(Q):
        ng = int(rng.integers(1, min(3, R, F) + 1))
        res = rng.permutation(R)
        owner = np.empty(R, np.int64)
        owner[res[:ng]] = np.arange(ng)                        # every group covers a resource
        owner[res[ng:]] = rng.integers(0, ng, R - ng)
        if R > ng and rng.random() < 0.15:
            owner[res[ng]] = -1                                 # a resource without a group
        used = int(rng.integers(ng, F + 1))
        perm = rng.permutation(F)[:used]
        cuts = np.sort(rng.choice(np.arange(1, used), ng - 1, replace=False)) if ng > 1 else []
        for g, fl in enumerate(np.split(perm, cuts)):
            masks.append(int(sum(1 << r for r in range(R) if owner[r] == g)))
            flavors += fl.tolist()
            fl_start.append(len(flavors))
        rg_start.append(len(masks))
    snap.set("cq_rg_start", rg_start); snap.set("rg_res_mask", masks)
    snap.set("rg_flavor_start", fl_start); snap.set("rg_flavors", flavors)
    cov = synth._covered_cells(snap)
    nominal, bl, ll = (a[k].reshape(N, FR).copy() for k in ("nominal", "borrow_limit", "lend_limit"))
    nominal[:Q][~cov] = 0
    bl[:Q][~cov] = abi.KB_NO_LIMIT
    ll[:Q][~cov] = abi.KB_NO_LIMIT
    snap.set("nominal", nominal); snap.set("borrow_limit", bl); snap.set("lend_limit", ll)
    usage = a["cq_usage"].reshape(Q, FR).copy()
    if snap.n_adm:
        A = snap.n_adm
        st = a["adm_use_start"].astype(np.int64)
        row = np.repeat(np.arange(A), np.diff(st))
        fr = a["adm_use_fr"].astype(np.int64)
        cq, qty = a["adm_cq"].astype(np.int64), a["adm_use_qty"].astype(np.int64)
        keep = cov[cq[row], fr]
        left = np.bincount(row[keep], minlength=A)
        rows = left > 0
        for k in [k for k in a if k.startswith("adm_") and not k.startswith("adm_use_")]:
            snap.set(k, a[k][rows])
        snap.set("adm_use_start", np.concatenate([[0], np.cumsum(left[rows])]))
        snap.set("adm_use_fr", fr[keep]); snap.set("adm_use_qty", qty[keep])
        usage = np.zeros((Q, FR), np.int64)
        np.add.at(usage, (cq[row[keep]], fr[keep]), qty[keep])
    else:
        usage[~cov] = 0
    snap.set("cq_usage", usage)
    covres = _covered_resources(snap)
    ps_cq = np.repeat(a["wl_cq"].astype(np.int64), np.diff(a["wl_ps_start"].astype(np.int64)))
    mask = a["ps_req_mask"].astype(np.int64)
    strip = ((mask & ~covres[ps_cq]) != 0) & (rng.random(len(mask)) < 0.9)
    new_mask = np.where(strip, mask & covres[ps_cq], mask)
    req = a["ps_req"].reshape(-1, R).copy()
    req[(new_mask[:, None] >> np.arange(R)[None, :] & 1) == 0] = 0
    snap.set("ps_req_mask", new_mask); snap.set("ps_req", req)
    return snap.finalize()


def policies(snap, seed):
    """whenCanBorrow, whenCanPreempt and the preference drawn uniformly per ClusterQueue (synth's preemption policies
    stay: reclaimWithinCohort Never still excludes borrowWithinCohort)"""
    rng = np.random.default_rng(seed)
    Q = snap.n_cq
    snap.set("cq_when_can_borrow", rng.integers(0, 2, Q))
    snap.set("cq_when_can_preempt", rng.integers(0, 2, Q))
    snap.set("cq_preference", rng.integers(0, 3, Q))
    return snap.finalize()


def last_tried(snap, seed):
    """cq_generation in 0..4; the LastAssignment of about half of the workloads is current, of a quarter stale, of the
    rest nil; ps_last_tried holds one start per (podset, resource group) in [-1, len(flavor list) - 2], on every
    resource of the group (the walk reads it at the group's first requested resource, workload.go:178-191)"""
    rng = np.random.default_rng(seed)
    a = snap.arrays
    Q, R, W = snap.n_cq, snap.n_resource, snap.n_wl
    gen = rng.integers(0, 5, Q)
    snap.set("cq_generation", gen)
    wg = gen[a["wl_cq"].astype(np.int64)]
    u = rng.random(W)
    stale = wg - 1 - (rng.random(W) * np.maximum(wg, 1)).astype(np.int64)  # in [0, gen) where gen > 0
    snap.set("wl_last_gen", np.where(u < 0.5, wg, np.where((u < 0.75) & (wg > 0), stale, -1)))
    ps_cq = np.repeat(a["wl_cq"].astype(np.int64), np.diff(a["wl_ps_start"].astype(np.int64)))
    lt = np.full((len(ps_cq), R), -1, np.int64)
    order = np.argsort(ps_cq, kind="stable")
    bounds = np.searchsorted(ps_cq[order], np.arange(Q + 1))
    for q, m, fl in _groups(snap):
        rows = order[bounds[q]:bounds[q + 1]]
        v = rng.integers(-1, len(fl) - 1, len(rows)) if len(fl) > 1 else np.full(len(rows), -1)
        for r in range(R):
            if m >> r & 1:
                lt[rows, r] = v
    snap.set("ps_last_tried", lt)
    return snap.finalize()


def pods(snap):
    """the last resource is corev1.ResourcePods: ClusterQueues whose groups cover it request the pod count there"""
    snap.pods_resource = snap.n_resource - 1
    return snap.finalize()


def fixture(snap, seed, with_pods=False):
    snap = last_tried(policies(ragged(snap, seed), seed + 1), seed + 2)
    return pods(snap) if with_pods else snap


def _fair(snap):
    snap.flags |= abi.F_FAIR_SHARING
    return snap


def _classical(snap):
    snap.flags &= ~abi.F_FAIR_SHARING
    return snap


def _grouped(snap, seed=3):
    """PodSetGroups: in 70 % of the workloads with >= 2 podsets the first two (sometimes three) rows share a group"""
    rng = np.random.default_rng(seed)
    st = np.asarray(snap.arrays["wl_ps_start"])
    grp = np.full(snap.n_podset, -1, np.int32)
    for w in np.flatnonzero(np.diff(st) >= 2):
        if rng.random() < 0.7:
            n = min(int(st[w + 1] - st[w]), 2 + int(rng.random() < 0.3))
            grp[st[w]:st[w] + n] = 0
    snap.set("ps_group", grp)
    return snap.finalize()


def _copy(snap):
    s2 = copy.copy(snap)
    s2.arrays = dict(snap.arrays)
    s2.__dict__["_struct"] = None
    return s2


# ---------------------------------------------------------------------------------------------------------- snapshots
PER_THREAD_W = 132 * 2048 // 8 + 2000  # more nominate lanes than a 132-SM H100 runs at once: one thread per entry

SNAPS = {
    "lone-cfg1": lambda: fixture(synth.make_snapshot(1), 101),
    "lone-cfg2-pods": lambda: fixture(synth.make_snapshot(2, W=5000, Q=50, podsets_max=3), 102, with_pods=True),
    "lone-per-thread": lambda: fixture(synth.make_snapshot(2, W=PER_THREAD_W, Q=400), 103),
    "lone-per-thread-preempt": lambda: fixture(synth.make_snapshot(2, W=PER_THREAD_W, Q=400, preemption=True, tight=1.5), 116),
    "long-lists": lambda: fixture(synth.make_snapshot(2, W=4000, Q=40, F=16, R=4, podsets_max=2), 104),
    "partial-groups": lambda: fixture(_grouped(synth.make_snapshot(2, W=5000, Q=50, partial=True, podsets_max=3)), 105),
    "within-cq": lambda: fixture(synth.make_snapshot(2, W=5000, Q=50, preemption=True, tight=1.5, podsets_max=2), 106),
    "tree-F6R2-pods": lambda: fixture(synth.make_snapshot(4, W=2000, Q=100, F=6, R=2, heads="one_per_cq", preemption=False), 107,
                                      with_pods=True),
    "tree-F12R1": lambda: fixture(synth.make_snapshot(4, W=2000, Q=100, F=12, R=1, heads="one_per_cq", preemption=False), 108),
    "flat-cfg3": lambda: fixture(synth.make_snapshot(3, W=3000, Q=300, heads="one_per_cq"), 109),
    "batched-trees": lambda: fixture(synth.make_snapshot(4, W=4000, Q=200, preemption=False), 110),
    "hier-preempt": lambda: fixture(synth.make_snapshot(4, W=4000, Q=200, heads="one_per_cq", tight=1.3), 111),
    "flat-reclaim": lambda: fixture(_classical(synth.make_snapshot(3, W=3000, Q=300, preemption=True, heads="one_per_cq", tight=1.3)), 112),
    "large-trees": lambda: fixture(synth.make_snapshot(4, W=40000, Q=2000, heads="one_per_cq", tight=1.5), 113),
    "fair-flat": lambda: fixture(synth.make_snapshot(3, W=3000, Q=300, preemption=True, heads="one_per_cq", tight=1.1), 114),
    "fair-hier": lambda: fixture(_fair(synth.make_snapshot(4, W=4000, Q=200, heads="one_per_cq", tight=1.5)), 115),
}


def _cap(snap):
    return 40 * snap.n_adm + 10000


def _targets(snap, want):
    assert want.n_targets > 0, "the fixture must preempt"


def _long_lists(snap, want):
    assert max(len(fl) for _, _, fl in _groups(snap)) > 8, "some flavor list must take several rounds of 8 lanes"
    assert (want.ps_tried_idx >= 8).any(), "some walk must stop in a later round"


def _reduced(snap, want):
    assert (want.ps_count != snap.ps_count[:len(want.ps_count)]).any(), "the PodSetReducer must reduce some count"


# what the oracle's cycle must show for the fixture to reach its branch
ORACLE_CHECKS = {"long-lists": _long_lists, "partial-groups": _reduced, "within-cq": _targets, "hier-preempt": _targets,
                 "flat-reclaim": _targets, "large-trees": _targets, "fair-flat": _targets, "fair-hier": _targets,
                 "lone-per-thread-preempt": _targets}

# ---------------------------------------------------------------------------------------------------------- CPU tests


def check_valid(snap):
    a = snap.arrays
    Q, R, FR, N = snap.n_cq, snap.n_resource, snap.n_fr, snap.n_nodes
    groups = _groups(snap)
    for q in range(Q):
        mine = [(m, fl) for c, m, fl in groups if c == q]
        masks = [m for m, _ in mine]
        assert all(m for m in masks), f"cq {q}: a group without resources"
        assert sum(bin(m).count("1") for m in masks) == bin(int(np.bitwise_or.reduce(masks))).count("1"), f"cq {q}: masks overlap"
        fls = np.concatenate([fl for _, fl in mine])
        assert len(np.unique(fls)) == len(fls), f"cq {q}: a flavor in two places"
        assert ((fls >= 0) & (fls < snap.n_flavor)).all()
    cov = synth._covered_cells(snap)
    assert (a["nominal"].reshape(N, FR)[:Q][~cov] == 0).all(), "quota on an uncovered cell"
    assert (a["cq_usage"].reshape(Q, FR)[~cov] == 0).all(), "usage on an uncovered cell"
    if snap.n_adm:
        st = a["adm_use_start"].astype(np.int64)
        row = np.repeat(np.arange(snap.n_adm), np.diff(st))
        use = np.zeros((Q, FR), np.int64)
        np.add.at(use, (a["adm_cq"].astype(np.int64)[row], a["adm_use_fr"].astype(np.int64)), a["adm_use_qty"])
        assert np.array_equal(use, a["cq_usage"].reshape(Q, FR)), "cq_usage is not the sum of the admitted usage"
    lt = a["ps_last_tried"].reshape(-1, R).astype(np.int64)
    ps_cq = np.repeat(a["wl_cq"].astype(np.int64), np.diff(a["wl_ps_start"].astype(np.int64)))
    hi = np.full((Q, R), -1, np.int64)  # the largest start of every (ClusterQueue, resource): len(list) - 2
    for q, m, fl in groups:
        for r in range(R):
            if m >> r & 1:
                hi[q, r] = len(fl) - 2
    assert (lt >= -1).all() and (lt <= np.maximum(hi[ps_cq], -1)).all(), "ps_last_tried out of its flavor list"
    gen = a["cq_generation"].astype(np.int64)
    assert ((a["wl_last_gen"] >= -1) & (a["wl_last_gen"] <= gen[a["wl_cq"].astype(np.int64)])).all()


def _answer(out):
    return out.decision, out.ps_flavor, out.ps_tried_idx


def _same(x, y):
    return all(np.array_equal(p, q) for p, q in zip(_answer(x), _answer(y)))


def single_group(snap):
    """(a): synth's one resource group over all resources and all flavors replaces the ragged groups"""
    s = _copy(snap)
    Q, F, R = s.n_cq, s.n_flavor, s.n_resource
    s.set("cq_rg_start", np.arange(Q + 1)); s.set("rg_res_mask", np.full(Q, (1 << R) - 1))
    s.set("rg_flavor_start", np.arange(Q + 1) * F); s.set("rg_flavors", np.tile(np.arange(F), Q))
    return s


def default_policies(snap):
    """(b): MayStopSearch, TryNextFlavor, no preference (FlatSnapshot.finalize's defaults)"""
    s = _copy(snap)
    Q = s.n_cq
    s.set("cq_when_can_borrow", np.full(Q, abi.FUNG_MAY_STOP_SEARCH))
    s.set("cq_when_can_preempt", np.full(Q, abi.FUNG_TRY_NEXT_FLAVOR))
    s.set("cq_preference", np.full(Q, abi.PREF_UNSET))
    return s


def no_contexts(snap):
    """(c): no last-scheduling context"""
    s = _copy(snap)
    s.set("wl_last_gen", np.full(s.n_wl, -1)); s.set("ps_last_tried", np.full((s.n_podset, s.n_resource), -1))
    return s


@pytest.fixture(scope="module")
def base_cycles():
    """the oracle's cycle of every fixture, computed once for the CPU tests"""
    cache = {}

    def get(name):
        if name not in cache:
            snap = SNAPS[name]()
            cache[name] = (snap, oracle.run_cycle(snap, _cap(snap)))
        return cache[name]
    return get


@pytest.mark.parametrize("name", list(SNAPS))
def test_fixture_is_valid(name):
    check_valid(SNAPS[name]())


@pytest.mark.parametrize("name", list(SNAPS))
def test_fixture_inputs_change_the_answer(base_cycles, name):
    """each of the three inputs changes (decision, ps_flavor, ps_tried_idx) on the oracle, and the fixture reaches the
    branch its device case is about: a kernel that ignored an input could not pass the device case"""
    snap, want = base_cycles(name)
    ORACLE_CHECKS.get(name, lambda s, w: None)(snap, want)
    cap = _cap(snap)
    for what, change in (("groups", single_group), ("policies", default_policies), ("contexts", no_contexts)):
        other = oracle.run_cycle(change(snap), cap)
        if what == "policies" and snap.n_cohort == 0 and snap.n_adm == 0:
            # without a cohort nothing borrows and without admitted workloads nothing preempts: the fungibility policies
            # and the preference (flavorassigner.go:410-441, :946-963) have nothing to act on
            assert _same(other, want), "the policies changed an answer where they cannot apply"
            continue
        assert not _same(other, want), f"the {what} of the fixture do not change the answer"


@pytest.mark.parametrize("name", ["lone-cfg2-pods", "flat-cfg3", "large-trees", "within-cq"])
@pytest.mark.parametrize("world", [2, 3])
def test_fixture_shard_merge_equals_full(base_cycles, name, world):
    snap, want = base_cycles(name)
    cap = _cap(snap)
    node_rank = shard.partition_roots(snap, world)
    parts = []
    for r in range(world):
        sub, m = shard.shard(snap, r, world, node_rank)
        parts.append((oracle.run_cycle(sub, cap), m))
    assert_cycle_equal(shard.merge(snap, parts), want)


# ----------------------------------------------------------------------------------------------------------- drains
def _events(snap, seed):
    return synth.add_quota_changes(synth.add_events(snap, seed=seed), seed=seed + 1)


def _evictable_events(seed):
    """the records of the admitted workloads are built from the ragged usage, so an evicted workload asks for what it held"""
    snap = synth.add_evictable(fixture(synth.make_snapshot(4, W=2000, Q=100, tight=1.3), seed)).finalize()
    return _events(snap, seed + 10)


DRAINS = {
    "cfg2": lambda: fixture(synth.make_snapshot(2, W=3000, Q=30, podsets_max=2), 201),
    "cfg3": lambda: fixture(synth.make_snapshot(3, W=2000, Q=40), 202),
    "cfg4": lambda: fixture(synth.make_snapshot(4, W=2000, Q=100, tight=1.3), 203),
    "cfg3-events": lambda: _events(fixture(synth.make_snapshot(3, W=2000, Q=40), 204), 214),
    "cfg4-events-evictable": lambda: _evictable_events(205),
}
EVENT_DRAINS = ("cfg3-events", "cfg4-events-evictable")
DRAIN_CYCLES = 10_000


def _drain_on_oracle(snap, run_cycle=None):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000
    return drain(snap, run_cycle or (lambda s: oracle.run_cycle(s, cap)), max_cycles=DRAIN_CYCLES)


@pytest.mark.parametrize("name", list(DRAINS))
def test_drain_fixture_is_valid(name):
    check_valid(DRAINS[name]())


@pytest.mark.parametrize("name", list(DRAINS))
def test_drain_carries_contexts(name):
    """from snapshots without any last-scheduling context, the drain hands later cycles heads with a current
    LastAssignment and a flavor to resume from: the write-back of ps_tried_idx / the generation reaches the walk"""
    snap = no_contexts(DRAINS[name]())
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000
    counts = []

    def cycle(cs):
        a, R = cs.arrays, cs.n_resource
        st, lt, gen = a["wl_ps_start"], a["ps_last_tried"].reshape(-1, R), a["wl_last_gen"]
        counts.append(sum(int(gen[w] >= 0 and (lt[st[w]:st[w + 1]] >= 0).any()) for w in a["heads"]))
        return oracle.run_cycle(cs, cap)
    res = _drain_on_oracle(snap, cycle)
    assert res.cycles > 1 and counts[0] == 0
    assert sum(counts[1:]) > 0, "no head resumed a flavor walk"


# ------------------------------------------------------------------------------------------------------------ device
@pytest.fixture(scope="module")
def ev():
    from kueue_b200 import native
    e = native.Evaluator(0)
    e.set_profile(True)
    yield e
    e.close()


FUSED = "k_cycle_flat"  # this slot times whichever fused per-root kernel ran: k_cycle_flat or k_cycle_root


def _ms(st, name):
    return st.kernel_ms[abi.KERNEL_NAMES.index(name)]


def _coop(snap, st):
    """k_nominate_coop (KB_NG = 8 lanes per entry) runs while the lanes fit the device, k_nominate otherwise; both are
    timed in the k_nominate slot"""
    return snap.n_heads * 8 <= st.sm_count * 2048


def _lone(snap, st):
    assert _ms(st, "k_lone") > 0 and _ms(st, "k_nominate") > 0 and _ms(st, "k_admit") > 0
    assert _ms(st, "k_tree") == 0 and _ms(st, FUSED) == 0


def lone_coop(snap, st):
    _lone(snap, st)
    assert _coop(snap, st)


def lone_per_thread(snap, st):
    _lone(snap, st)
    assert not _coop(snap, st)


def classical_search(snap, st):
    assert _ms(st, "k_nominate") > 0 and _ms(st, "k_search_cells") > 0 and _ms(st, "k_nominate_walk") > 0
    assert _ms(st, "k_admit") > 0 and _ms(st, FUSED) == 0 and _ms(st, "k_nominate_search_fair") == 0


def lone_per_thread_search(snap, st):
    classical_search(snap, st)
    assert not _coop(snap, st)


def fair_search(snap, st):
    assert _ms(st, "k_nominate") > 0 and _ms(st, "k_nominate_search_fair") > 0 and _ms(st, "k_admit") > 0
    assert _ms(st, FUSED) == 0 and _ms(st, "k_nominate_walk") == 0


def cycle_root_tree(snap, st):
    assert _ms(st, FUSED) > 0 and _ms(st, "k_nominate") == 0 and _ms(st, "k_tree") == 0
    assert list(st.flat_group_walk) == [0, 0], "k_cycle_flat ran instead of k_cycle_root"


def general_chain_tree(snap, st):
    assert _ms(st, "k_tree") > 0 and _ms(st, "k_nominate") > 0 and _ms(st, "k_admit") > 0 and _ms(st, FUSED) == 0


def cycle_root_flat(snap, st):
    assert _ms(st, FUSED) > 0 and _ms(st, "k_nominate") == 0
    assert st.flat_group_walk[1] == 0, "k_cycle_flat ran instead of k_cycle_root"


def cycle_flat(snap, st):
    assert _ms(st, FUSED) > 0 and _ms(st, "k_nominate") == 0
    assert st.flat_group_walk[1] > 0, "k_cycle_root ran instead of k_cycle_flat"


def batched_trees(snap, st):
    assert _ms(st, "k_tree") > 0 and _ms(st, "k_nominate") > 0 and _ms(st, "k_admit") > 0 and _ms(st, FUSED) == 0
    assert _coop(snap, st)


ROUTES = {  # case: (fixture, environment, route check)
    "lone-coop-cfg1": ("lone-cfg1", {}, lone_coop),
    "lone-coop-cfg2-pods": ("lone-cfg2-pods", {}, lone_coop),
    "lone-per-thread": ("lone-per-thread", {}, lone_per_thread),
    "lone-per-thread-preempt": ("lone-per-thread-preempt", {}, lone_per_thread_search),
    "long-lists": ("long-lists", {}, lone_coop),
    "partial-groups": ("partial-groups", {}, lone_coop),
    "within-cq": ("within-cq", {}, classical_search),
    "cycle-root-tree-F6R2-pods": ("tree-F6R2-pods", {}, cycle_root_tree),
    "cycle-root-tree-F12R1": ("tree-F12R1", {}, cycle_root_tree),
    "no-fused-tree-F6R2-pods": ("tree-F6R2-pods", {"KB_NO_FUSED": "1"}, general_chain_tree),
    "no-fused-tree-F12R1": ("tree-F12R1", {"KB_NO_FUSED": "1"}, general_chain_tree),
    "cycle-root-flat": ("flat-cfg3", {"KB_FUSED_V1": "1"}, cycle_root_flat),
    "cycle-flat": ("flat-cfg3", {}, cycle_flat),
    "batched-trees": ("batched-trees", {}, batched_trees),
    "hier-preempt": ("hier-preempt", {}, classical_search),
    "flat-reclaim": ("flat-reclaim", {}, classical_search),
    "large-trees": ("large-trees", {}, classical_search),
    "fair-flat": ("fair-flat", {}, fair_search),
    "fair-hier": ("fair-hier", {}, fair_search),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(ROUTES))
def test_route_matches_oracle(ev, monkeypatch, case):
    name, env, route = ROUTES[case]
    for k in ("KB_NO_FUSED", "KB_FUSED_V1"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    snap = SNAPS[name]()
    cap = _cap(snap)
    got = ev.run_cycle(snap, abi.CycleOut(snap, cap))
    st = ev.stats()
    want = oracle.run_cycle(snap, cap)
    ORACLE_CHECKS.get(name, lambda s, w: None)(snap, want)
    assert_cycle_equal(got, want)
    route(snap, st)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DRAINS))
def test_kb_run_drain_matches_host_definition(name):
    from kueue_b200 import native
    from tests.test_drain_quota_changes import compare
    snap = DRAINS[name]()
    want = _drain_on_oracle(snap)
    assert want.n_admitted > 0 and want.cycles > 1
    ev = native.Evaluator(0)
    try:
        got = ev.run_drain(snap, abi.DrainOut(snap, DRAIN_CYCLES, trace_capacity=want.n_decisions))
    finally:
        ev.close()
    if name in EVENT_DRAINS:
        assert want.n_quota_changes > 0
        compare(want, got)
        return
    assert got.n_cycles == want.cycles
    cyc = got.cycles()
    for k in range(want.cycles):
        assert np.array_equal(cyc[k][0], want.heads[k]), k
        assert np.array_equal(cyc[k][1], want.decisions[k]), k
    assert np.array_equal(got.cq_usage, want.cq_usage)
    adm = np.concatenate(want.admitted) if want.admitted else np.zeros(0, np.int64)
    assert got.n_admitted == len(adm) and np.array_equal(np.flatnonzero(got.wl_admit_cycle >= 0), np.sort(adm))


@pytest.mark.gpu
def test_target_lists_longer_than_four_per_admitted_workload(ev):
    """Regression: heads of one large tree that all reclaim from the same admitted workloads list 120 330 targets over
    16 000 admitted rows.  The device pool held 4 per admitted row + 1024 (65 024), so kb_run_cycle failed with
    KB_ERR_CAPACITY although the caller's buffer, exactly the oracle's count here, holds every target."""
    snap = synth.make_snapshot(4, W=10000, Q=1000, heads="one_per_cq", tight=1.3)
    want = oracle.run_cycle(snap, _cap(snap))
    assert want.n_targets > 4 * snap.n_adm + 1024
    got = ev.run_cycle(snap, abi.CycleOut(snap, want.n_targets))
    assert_cycle_equal(got, want)
