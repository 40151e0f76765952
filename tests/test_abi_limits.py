"""The scheduling cycle, kb_tree_eval and kb_run_drain against the CPU oracle at the size limits the C-ABI accepts:
64 flavors, 16 resources (1,024 flavor-resource cells), 8 podsets per workload and cohort paths of 17 nodes (a
ClusterQueue 16 parent hops below its root), and the refusals just past them.

synth.make_snapshot builds the wide snapshots.  The builders below add what it cannot: cohort forests of any shape
over a cohort-less snapshot (`forest`, `chains`), podsets eligible on one flavor each (`one_flavor_per_podset`) and
one resource group per resource (`group_per_resource`).  Every fixture has a CPU test that proves the shape it claims
(and, where the case is about a branch, that the oracle's cycle reaches it), and every device case proves the route it
names from the per-kernel timings (kb_set_profile)."""
import ctypes as C

import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from kueue_b200.drain import drain
from tests.helpers import assert_cycle_equal
from tests.test_drain_evictions import _compare as compare_drain
from tests.test_flavor_walk_routes import (_lone, _ms, _targets, classical_search, cycle_flat, cycle_root_tree, fair_search,
                                           general_chain_tree)

KIB = 1024
ADMIT_SMEM = 200 * KIB  # the dynamic shared memory k_admit may use (launch_admit)
KB_PF = 6               # path nodes the global-table admit stages per ClusterQueue (kb_kernels.cuh)

# ------------------------------------------------------------------------------------------------------------- builders


def forest(snap, coh_parent, cq_parent, coh_quota=0.3, seed=0):
    """`snap` (cohort-less) with cohorts: coh_parent[c] is the parent cohort of cohort c (-1 = root), cq_parent[q] the
    cohort of ClusterQueue q (-1 = none).  A share `coh_quota` of the cohorts gets a nominal quota of a quarter of the
    mean ClusterQueue row; every ClusterQueue with a cohort reclaims (Any / LowerPriority / Never), a third of those
    also borrow within the cohort (never together with reclaim Never)."""
    rng = np.random.default_rng(seed)
    a = snap.arrays
    Q, F, R, FR = snap.n_cq, snap.n_flavor, snap.n_resource, snap.n_fr
    assert snap.n_cohort == 0
    coh_parent, cq_parent = np.asarray(coh_parent, np.int64), np.asarray(cq_parent, np.int64)
    Cn = len(coh_parent)
    out = abi.FlatSnapshot(n_cq=Q, n_cohort=Cn, n_flavor=F, n_resource=R, pods_resource=snap.pods_resource, flags=snap.flags,
                           now_ns=snap.now_ns)
    for k, v in a.items():
        if k not in ("parent", "fair_weight", "nominal", "borrow_limit", "lend_limit"):
            out.arrays[k] = v
    out.set("parent", np.concatenate([np.where(cq_parent >= 0, cq_parent + Q, -1), np.where(coh_parent >= 0, coh_parent + Q, -1)]))
    fw = np.ones(Q + Cn)
    fw[:Q] = a["fair_weight"][:Q]
    out.set("fair_weight", fw)
    rows = {}
    for k, fill in (("nominal", 0), ("borrow_limit", abi.KB_NO_LIMIT), ("lend_limit", abi.KB_NO_LIMIT)):
        t = np.full((Q + Cn, FR), fill, np.int64)
        t[:Q] = a[k].reshape(-1, FR)[:Q]
        rows[k] = t
    has = rng.random(Cn) < coh_quota
    rows["nominal"][Q:][has] = rows["nominal"][:Q].mean(axis=0).astype(np.int64) // 4
    for k, t in rows.items():
        out.set(k, t)
    inco = cq_parent >= 0
    reclaim = np.where(inco, rng.choice([abi.POLICY_NEVER, abi.POLICY_LOWER_PRIORITY, abi.POLICY_ANY], Q), abi.POLICY_NEVER)
    bw = inco & (reclaim != abi.POLICY_NEVER) & (rng.random(Q) < 0.33)
    out.set("cq_reclaim_within", reclaim)
    out.set("cq_borrow_within", np.where(bw, abi.POLICY_LOWER_PRIORITY, abi.POLICY_NEVER))
    return out.finalize()


def chains(snap, n_chains, depth, deep_share=0.5, seed=0):
    """`snap` under `n_chains` cohort chains of `depth` cohorts each (root first): a share `deep_share` of the
    ClusterQueues hangs off the last cohort of its chain (depth `depth`), the others off a cohort drawn uniformly along
    the chain; chain k holds the ClusterQueues q with q % n_chains == k"""
    rng = np.random.default_rng(seed)
    coh_parent = np.array([-1 if i % depth == 0 else i - 1 for i in range(n_chains * depth)])
    Q = snap.n_cq
    level = np.where(rng.random(Q) < deep_share, depth - 1, rng.integers(0, depth, Q))
    level[np.arange(Q) < n_chains] = depth - 1  # every chain reaches its full depth
    cq_parent = (np.arange(Q) % n_chains) * depth + level
    return forest(snap, coh_parent, cq_parent, seed=seed + 1)


def cohorts_of(snap, size, seed=0):
    """flat cohorts of `size` ClusterQueues (consecutive indexes) under one parentless cohort each"""
    Q = snap.n_cq
    nco = (Q + size - 1) // size
    return forest(snap, np.full(nco, -1), np.arange(Q) // size, seed=seed)


def one_flavor_per_podset(snap):
    """podset i of every workload is eligible on flavor i only (F >= the most podsets of a workload)"""
    st = snap.arrays["wl_ps_start"].astype(np.int64)
    idx = np.arange(snap.n_podset) - np.repeat(st[:-1], np.diff(st))
    assert idx.max() < snap.n_flavor
    snap.set("ps_flavor_ok", np.left_shift(np.uint64(1), idx.astype(np.uint64)))
    return snap.finalize()


def only_last_flavor(snap, share=0.3, seed=0):
    """a share of the podsets is eligible on the last flavor only (flavor F - 1: bit 63 at F = 64)"""
    rng = np.random.default_rng(seed)
    ok = snap.arrays["ps_flavor_ok"].copy()
    ok[rng.random(len(ok)) < share] = np.uint64(1) << np.uint64(snap.n_flavor - 1)
    snap.set("ps_flavor_ok", ok)
    return snap.finalize()


def group_per_resource(snap, seed=0):
    """R resource groups of one resource each in every ClusterQueue (the API's MaxItems=16), each over its own
    flavors: F // R distinct flavors per group in a random order (a flavor belongs to one group of a ClusterQueue).
    Every flavor is eligible for every podset: a podset needs one eligible flavor in each of the R groups."""
    rng = np.random.default_rng(seed)
    Q, F, R = snap.n_cq, snap.n_flavor, snap.n_resource
    k = F // R
    assert k >= 1
    flavors, fstart = [], [0]
    for _ in range(Q):
        perm = rng.permutation(F)
        for r in range(R):
            flavors += perm[r * k:(r + 1) * k].tolist()
            fstart.append(len(flavors))
    snap.set("cq_rg_start", np.arange(Q + 1) * R); snap.set("rg_res_mask", np.tile(1 << np.arange(R), Q))
    snap.set("rg_flavor_start", fstart); snap.set("rg_flavors", flavors)
    cov = synth._covered_cells(snap)
    N, FR = snap.n_nodes, snap.n_fr
    nominal = snap.arrays["nominal"].reshape(N, FR).copy()
    nominal[:Q][~cov] = 0
    snap.set("nominal", nominal)
    snap.set("cq_usage", np.where(cov, snap.arrays["cq_usage"].reshape(Q, FR), 0))
    snap.set("ps_flavor_ok", np.full(snap.n_podset, np.iinfo(np.uint64).max, np.uint64))
    return snap.finalize()


def _fair(snap):
    snap.flags |= abi.F_FAIR_SHARING
    return snap.finalize()


def _lone_cfg(**kw):
    return synth.make_snapshot(2, **kw)


# ------------------------------------------------------------------------------------------------------------ snapshots
SNAPS = {
    "wide-lone": lambda: _lone_cfg(W=2000, Q=40, F=64, R=16, podsets_max=3),
    "cliff-190": lambda: _lone_cfg(W=1000, Q=20, F=19, R=10, podsets_max=2),
    "cliff-192": lambda: _lone_cfg(W=1000, Q=20, F=12, R=16, podsets_max=2),
    "wide-trees-search": lambda: synth.make_snapshot(4, W=2000, Q=100, F=16, R=16, heads="one_per_cq", tight=1.3),
    "fused-3": lambda: _fair(cohorts_of(_lone_cfg(W=600, Q=60, F=64, R=16, heads="one_per_cq", podsets_max=2), 3)),
    "fused-4": lambda: _fair(cohorts_of(_lone_cfg(W=600, Q=60, F=64, R=16, heads="one_per_cq", podsets_max=2), 4)),
    "flat-F64R1": lambda: only_last_flavor(_fair(cohorts_of(_lone_cfg(W=3000, Q=300, F=64, R=1, heads="one_per_cq"), 20))),
    "groups-F16R16": lambda: group_per_resource(cohorts_of(_lone_cfg(W=600, Q=60, F=16, R=16, heads="one_per_cq"), 3)),
    "wide-fair-search": lambda: synth.make_snapshot(3, W=600, Q=60, F=16, R=16, heads="one_per_cq", preemption=True, tight=1.1),
    "cells-128": lambda: one_flavor_per_podset(_lone_cfg(W=2000, Q=20, F=8, R=16, podsets_max=8, preemption=True, tight=1.5)),
    "cells-128-fair": lambda: one_flavor_per_podset(synth.make_snapshot(3, W=600, Q=60, F=8, R=16, podsets_max=8, heads="one_per_cq",
                                                                        preemption=True, tight=1.2)),
    "cells-64": lambda: one_flavor_per_podset(_lone_cfg(W=2000, Q=20, F=8, R=16, podsets_max=4, preemption=True, tight=1.5)),
    "reducer-8": lambda: _lone_cfg(W=2000, Q=20, F=4, R=16, podsets_max=8, partial=True),
    "depth16-preempt": lambda: chains(_lone_cfg(W=2000, Q=100, F=4, R=4, heads="one_per_cq", preemption=True, tight=1.6), 4, 16),
    "depth16-fair": lambda: _fair(chains(_lone_cfg(W=2000, Q=100, F=4, R=4, heads="one_per_cq", preemption=True, tight=1.6), 4, 16,
                                         seed=1)),
    "depth16-fused": lambda: chains(_lone_cfg(W=2000, Q=100, F=4, R=4, heads="one_per_cq"), 4, 16, seed=2),
    "deep-large-5": lambda: chains(_lone_cfg(W=2000, Q=60, F=16, R=16, heads="one_per_cq", preemption=True, tight=1.6), 2, 5),
    "deep-large-6": lambda: chains(_lone_cfg(W=2000, Q=60, F=16, R=16, heads="one_per_cq", preemption=True, tight=1.6), 2, 6),
    "deep-large-16": lambda: chains(_lone_cfg(W=2000, Q=60, F=16, R=16, heads="one_per_cq", preemption=True, tight=1.6), 2, 16),
    "memo-overflow": lambda: _lone_cfg(W=24000, Q=400, F=64, R=16, preemption=True, tight=1.5),
}


def _cap(snap):
    return 40 * snap.n_adm + 10000


def _depth(snap):
    """[n_nodes] parent hops from every node to its root"""
    p = snap.arrays["parent"].astype(np.int64)
    d = np.zeros(len(p), np.int64)
    cur = np.arange(len(p))
    while (p[cur] >= 0).any():
        m = p[cur] >= 0
        d[m] += 1
        cur = np.where(m, p[cur], cur)
    return d


def _root(snap):
    p = snap.arrays["parent"].astype(np.int64)
    cur = np.arange(len(p))
    while (p[cur] >= 0).any():
        cur = np.where(p[cur] >= 0, p[cur], cur)
    return cur


def _max_tree_nodes(snap):
    r = _root(snap)
    inco = np.bincount(r, minlength=snap.n_nodes)
    trees = [n for n in range(snap.n_cq, snap.n_nodes) if snap.arrays["parent"][n] < 0]
    return max(int(inco[t]) for t in trees) if trees else 0


def _max_podsets(snap):
    return int(np.diff(snap.arrays["wl_ps_start"]).max())


def _memo_items(snap):
    """plan_search: results of min(H, 2^26 / (FR * 16 B)) speculative searches fit the memo"""
    return min(snap.n_heads, (64 << 20) // (snap.n_fr * 16))


def _rows(snap, e):
    """the podset rows of head e (CycleOut's podset tables are indexed like the snapshot's)"""
    st, w = snap.arrays["wl_ps_start"], int(snap.arrays["heads"][e])
    return slice(int(st[w]), int(st[w + 1]))


def _preempt_heads(snap, want):
    """heads whose assignment has a cell in Preempt mode"""
    return [e for e in range(snap.n_heads) if (want.ps_res_mode[_rows(snap, e)] == abi.MODE_PREEMPT).any()]


def _cells_of(snap, want, e):
    R = snap.n_resource
    return {int(f) * R + r for row in want.ps_flavor[_rows(snap, e)] for r, f in enumerate(row) if f >= 0}


# ------------------------------------------------------------------------------------------------- shape proofs (CPU)
def _shape_wide_lone(snap, want):
    assert (snap.n_flavor, snap.n_resource, snap.n_cohort) == (64, 16, 0) and _max_podsets(snap) == 3
    assert 1056 * snap.n_fr > ADMIT_SMEM, "the request tile of k_admit<true> must not fit at a fixed 128 entries"


def _shape_cliff(fr):
    def check(snap, want):
        assert snap.n_fr == fr and snap.n_cohort == 0 and snap.n_fr > 64, "k_admit<true> (no warp-per-root admit) at this FR"
        assert (want.decision == abi.DEC_ASSUMED).any()
    return check


def _shape_wide_trees(snap, want):
    assert snap.n_fr == 256 and _max_tree_nodes(snap) * snap.n_fr * 32 > ADMIT_SMEM, "the tree tables must not fit"
    _targets(snap, want)


def _shape_fused(nodes):
    def check(snap, want):
        assert snap.n_fr == 1024 and _max_tree_nodes(snap) == nodes and snap.n_adm == 0
        assert (_depth(snap)[:snap.n_cq] == 1).all()
        # choose_route: k_cycle_root's tables are 6 x nodes x FR x 8 B (+ small terms) <= 220 KiB
        fits = 6 * nodes * snap.n_fr * 8 + 6 * KIB <= 220 * KIB
        assert fits == (nodes == 4)
        assert (want.decision == abi.DEC_ASSUMED).any()
    return check


def _shape_flat_f64(snap, want):
    assert (snap.n_flavor, snap.n_resource) == (64, 1)
    last = snap.arrays["ps_flavor_ok"] == np.uint64(1 << 63)
    assert last.any()
    assert (want.ps_flavor[:, 0] == 63).any(), "some podset must be assigned flavor 63: the last of 8 rounds of 8 lanes"


def _shape_groups(snap, want):
    a = snap.arrays
    assert snap.n_resource == 16 and (np.diff(a["cq_rg_start"]) == 16).all()
    assert (np.diff(a["rg_flavor_start"]) == 1).all() and (a["rg_res_mask"] == np.tile(1 << np.arange(16), snap.n_cq)).all()
    for q in range(snap.n_cq):
        fl = a["rg_flavors"][16 * q:16 * (q + 1)]
        assert len(np.unique(fl)) == 16, "a flavor in two resource groups of a ClusterQueue"
    assert (want.decision == abi.DEC_ASSUMED).any()


def _shape_wide_fair(snap, want):
    assert snap.flags & abi.F_FAIR_SHARING and snap.n_fr == 256
    # plan_search: the private tree goes to global memory when nodes x FR x 32 B (+ small terms) exceed 190 KiB
    assert _max_tree_nodes(snap) * snap.n_fr * 32 > 190 * KIB
    _targets(snap, want)


def _shape_cells(n_cells):
    def check(snap, want):
        assert snap.n_resource == 16
        pre = [e for e in _preempt_heads(snap, want) if want.tgt_start[e + 1] > want.tgt_start[e]]
        assert pre, "some entry must preempt"
        most = max(len(_cells_of(snap, want, e)) for e in pre)
        assert most == n_cells, f"the largest preempting assignment has {most} distinct cells"
    return check


def _shape_cells_64(snap, want):
    pre = [e for e in _preempt_heads(snap, want) if want.tgt_start[e + 1] > want.tgt_start[e]]
    sizes = {len(_cells_of(snap, want, e)) for e in pre}
    assert any(32 < k <= 64 for k in sizes), f"no preempting assignment with 33..64 cells: {sorted(sizes)}"


def _shape_reducer(snap, want):
    assert _max_podsets(snap) == 8 and snap.n_resource == 16
    eight = [e for e in range(snap.n_heads) if _rows(snap, e).stop - _rows(snap, e).start == 8]
    changed = [e for e in eight if want.decision[e] == abi.DEC_ASSUMED and
               (want.ps_count[_rows(snap, e)] != snap.ps_count[_rows(snap, e)]).any()]
    assert changed, "the PodSetReducer must reduce an admitted 8-podset workload"


def _shape_depth16(preempt):
    def check(snap, want):
        d = _depth(snap)
        assert d[:snap.n_cq].max() == 16 and d.max() == 16, "a ClusterQueue 16 hops below its root (a 17-node path)"
        if preempt:
            _targets(snap, want)
        else:
            assert (want.decision == abi.DEC_ASSUMED).any()
    return check


def _shape_deep_large(depth):
    def check(snap, want):
        d = _depth(snap)
        assert d[:snap.n_cq].max() == depth and snap.n_fr == 256
        assert _max_tree_nodes(snap) * snap.n_fr * 32 > ADMIT_SMEM, "the four tables alone must exceed the admit budget"
        # the global-table admit stages the paths of the ClusterQueues when they have at most KB_PF nodes
        assert (depth + 1 <= KB_PF) == (depth == 5)
        _targets(snap, want)
    return check


def _shape_memo(snap, want):
    assert snap.n_fr == 1024 and snap.n_cohort == 0
    assert len(_preempt_heads(snap, want)) > _memo_items(snap), "more deferred entries than the memo holds"


SHAPES = {
    "wide-lone": _shape_wide_lone, "cliff-190": _shape_cliff(190), "cliff-192": _shape_cliff(192),
    "wide-trees-search": _shape_wide_trees, "fused-3": _shape_fused(4), "fused-4": _shape_fused(5),
    "flat-F64R1": _shape_flat_f64, "groups-F16R16": _shape_groups, "wide-fair-search": _shape_wide_fair,
    "cells-128": _shape_cells(128), "cells-128-fair": _shape_cells(128), "cells-64": _shape_cells_64,
    "reducer-8": _shape_reducer, "depth16-preempt": _shape_depth16(True), "depth16-fair": _shape_depth16(True),
    "depth16-fused": _shape_depth16(False), "deep-large-5": _shape_deep_large(5), "deep-large-6": _shape_deep_large(6),
    "deep-large-16": _shape_deep_large(16), "memo-overflow": _shape_memo,
}


@pytest.mark.parametrize("name", list(SNAPS))
def test_fixture_has_its_shape(name):
    snap = SNAPS[name]()
    SHAPES[name](snap, oracle.run_cycle(snap, _cap(snap)))


# ------------------------------------------------------------------------------------------------------ device cycles
@pytest.fixture(scope="module")
def ev():
    from kueue_b200 import native
    e = native.Evaluator(0)
    e.set_profile(True)
    yield e
    e.close()


def lone(snap, st):
    _lone(snap, st)


def lone_search(snap, st):
    assert _ms(st, "k_lone") > 0 and _ms(st, "k_tree") == 0
    classical_search(snap, st)


ROUTES = {
    "wide-lone": lone, "cliff-190": lone, "cliff-192": lone,
    "wide-trees-search": classical_search,
    "fused-3": cycle_root_tree, "fused-4": general_chain_tree,
    "flat-F64R1": cycle_flat, "groups-F16R16": cycle_root_tree,
    "wide-fair-search": fair_search,
    "cells-128": lone_search, "cells-128-fair": fair_search, "cells-64": lone_search,
    "reducer-8": lone,
    "depth16-preempt": classical_search, "depth16-fair": fair_search, "depth16-fused": cycle_root_tree,
    "deep-large-5": classical_search, "deep-large-6": classical_search, "deep-large-16": classical_search,
    "memo-overflow": lone_search,
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SNAPS))
def test_cycle_at_the_limits_matches_oracle(ev, monkeypatch, name):
    for k in ("KB_NO_FUSED", "KB_FUSED_V1"):
        monkeypatch.delenv(k, raising=False)
    snap = SNAPS[name]()
    cap = _cap(snap)
    got = ev.run_cycle(snap, abi.CycleOut(snap, cap))
    st = ev.stats()
    want = oracle.run_cycle(snap, cap)
    assert_cycle_equal(got, want)
    ROUTES[name](snap, st)


TREE_EVAL = ("wide-lone", "wide-trees-search", "fused-4", "wide-fair-search", "depth16-preempt", "depth16-fair", "deep-large-16")


@pytest.mark.gpu
@pytest.mark.parametrize("name", TREE_EVAL)
def test_tree_eval_at_the_limits_matches_oracle(ev, name):
    snap = SNAPS[name]()
    got, want = ev.tree_eval(snap), oracle.tree_eval(snap)
    for f in ("subtree_quota", "usage", "available", "potential_available", "drs_rounded", "drs_resource", "drs_borrowing"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f


# ----------------------------------------------------------------------------------------------------------- drains
DRAINS = {
    "lone-FR256": lambda: _lone_cfg(W=2000, Q=20, F=16, R=16, podsets_max=2),
    "trees-FR256": lambda: synth.make_snapshot(4, W=1500, Q=60, F=16, R=16, tight=1.2, evictable=True),
    "depth16-evictable": lambda: synth.add_evictable(
        chains(_lone_cfg(W=1500, Q=60, F=4, R=4, preemption=True, tight=1.3), 3, 16, seed=3)).finalize(),
}
DRAIN_CYCLES = 60


def _drain_on_oracle(snap):
    cap = 40 * (snap.n_adm + snap.n_wl) + 10000
    return drain(snap, lambda s: oracle.run_cycle(s, cap), max_cycles=DRAIN_CYCLES)


@pytest.mark.parametrize("name", list(DRAINS))
def test_drain_fixture_has_its_shape(name):
    snap = DRAINS[name]()
    want = _drain_on_oracle(snap)
    assert want.n_admitted > 0 and want.cycles > 1
    if name == "lone-FR256":
        assert snap.n_fr == 256 and snap.n_cohort == 0
    elif name == "trees-FR256":
        assert snap.n_fr == 256 and _max_tree_nodes(snap) * snap.n_fr * 32 > ADMIT_SMEM and want.n_evicted > 0
    else:
        assert _depth(snap)[:snap.n_cq].max() == 16 and "adm_wl" in snap.arrays and want.n_evicted > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DRAINS))
def test_kb_run_drain_at_the_limits_matches_host_definition(name):
    from kueue_b200 import native
    snap = DRAINS[name]()
    want = _drain_on_oracle(snap)
    e = native.Evaluator(0)
    try:
        got = e.run_drain(snap, max_cycles=DRAIN_CYCLES)
    finally:
        e.close()
    compare_drain(snap, want, got)
    adm = np.concatenate(want.admitted) if want.admitted else np.zeros(0, np.int64)
    assert got.n_admitted == len(adm)


# --------------------------------------------------------------------------------------------------------- refusals
def _podsets(snap, n):
    """workload 0 with `n` podsets: its single podset row repeated (eligible everywhere)"""
    a = snap.arrays
    R = snap.n_resource
    st = a["wl_ps_start"].astype(np.int64)
    assert st[1] - st[0] == 1
    rep = np.concatenate([np.zeros(n - 1, np.int64), np.arange(snap.n_podset)])
    for k in ("ps_req_mask", "ps_count", "ps_min_count", "ps_flavor_ok"):
        snap.set(k, a[k][rep])
    for k in ("ps_req", "ps_last_tried"):
        snap.set(k, a[k].reshape(-1, R)[rep])
    snap.set("wl_ps_start", np.concatenate([[0], st[1:] + n - 1]))
    return snap.finalize()


def _small():
    return _lone_cfg(W=200, Q=10, F=4, R=4)


REFUSALS = {  # case: (snapshot, struct edit after finalize)
    "depth-17": (lambda: chains(_small(), 2, 17), None),
    "flavors-65": (lambda: _lone_cfg(W=200, Q=10, F=64, R=1), lambda s: setattr(s, "n_flavor", 65)),
    "resources-17": (lambda: _lone_cfg(W=200, Q=10, F=1, R=16), lambda s: setattr(s, "n_resource", 17)),
    "podsets-9": (lambda: _podsets(_small(), 9), None),
}


def test_refusal_fixtures_are_one_past_the_limits():
    assert _depth(REFUSALS["depth-17"][0]())[:10].max() == 17
    assert _max_podsets(REFUSALS["podsets-9"][0]()) == 9
    assert _max_podsets(_podsets(_small(), 8)) == 8


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REFUSALS))
def test_library_refuses_past_the_limits(name):
    """KB_ERR_INVALID from kb_run_cycle and kb_run_drain (not a launch failure, not a silent answer), and the handle
    still runs a valid cycle afterwards"""
    from kueue_b200 import native
    make, edit = REFUSALS[name]
    snap = make()
    e = native.Evaluator(0)
    try:
        for call in ("kb_run_cycle", "kb_run_drain"):
            s = snap.as_struct()
            if edit:
                edit(s)
            out = abi.CycleOut(snap) if call == "kb_run_cycle" else abi.DrainOut(snap, 5)
            rc = getattr(native.lib(), call)(e._h, C.byref(s), C.byref(out.struct))
            assert rc == -1, (call, rc, native.lib().kb_last_error(e._h).decode())
            ok = _small()
            assert_cycle_equal(e.run_cycle(ok), oracle.run_cycle(ok))
        ok8 = _podsets(_small(), 8)
        assert_cycle_equal(e.run_cycle(ok8), oracle.run_cycle(ok8))
    finally:
        e.close()


# ------------------------------------------------------------------------------------------------------------- synth
SYNTH_DIGESTS = {  # sha256 over every array (name, dtype, shape, bytes) in name order, taken before R could exceed 8
    "cfg1": ("bcdaf224fa3d924f8673f2336211ef61905a59cac5cb44017552412e77584d0e", lambda: synth.make_snapshot(1)),
    "cfg2": ("cd12530629c8813409ca4d23c83ba8875563ec683d802bc5f812a5be29c6f99a",
             lambda: synth.make_snapshot(2, W=2000, Q=20, podsets_max=3, partial=True)),
    "cfg2-afs": ("7b8382b1e70fdfc8c073ac133c0f13b797c8768b81a1410cab5b82bfaed330ee", lambda: synth.make_snapshot(2, W=1000, Q=10, afs=3)),
    "cfg3": ("0c9835ac069d66ba841a6c7c73071495f1d255e0548d95b15fdb4f8da97403c7",
             lambda: synth.make_snapshot(3, W=2000, Q=200, heads="one_per_cq", preemption=True)),
    "cfg4": ("8fbbe30c2dd3a0b0b7b7d79bc9d354fbddaba86e97734f5c8017fff04d787791", lambda: synth.make_snapshot(4, W=3000, Q=100, evictable=True)),
    "cfg4-F4R8": ("4852d9844044c634e964e52da063c22e919658b3db4f4851434bb13d4ce74da4", lambda: synth.make_snapshot(4, W=1000, Q=50, F=4, R=8)),
}


@pytest.mark.parametrize("name", list(SYNTH_DIGESTS))
def test_synth_snapshots_up_to_eight_resources_are_unchanged(name):
    import hashlib
    digest, make = SYNTH_DIGESTS[name]
    snap = make()
    h = hashlib.sha256()
    for k in sorted(snap.arrays):
        v = np.ascontiguousarray(snap.arrays[k])
        h.update(f"{k}:{v.dtype.str}:{v.shape};".encode())
        h.update(v.tobytes())
    assert h.hexdigest() == digest


def test_synth_builds_sixteen_resources():
    snap = synth.make_snapshot(2, W=100, Q=5, F=4, R=16, admitted=50, afs=2)
    assert snap.n_resource == 16 and snap.arrays["lq_consumed"].shape[1] == 16
    scale = synth._scale(16)
    assert np.array_equal(scale[8:], scale[:8])
