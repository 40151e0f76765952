"""k_cycle_flat (kb_flat.cuh) against the CPU oracle on quota shapes the other flat-kernel tests do not set.

The kernel stages SubtreeQuota and localQuota from static tree-local tables (k_tl_static / k_tl_root) and the group
walk computes available / potentialAvailable of each cell it evaluates itself. These cases steer the branches of
those computations: borrowing limits, a root cohort with its own nominal quota, lending limits at 0 and at the
nominal quota, and partial admission, whose reducible heads take the general walk and its availability sweep."""
import numpy as np
import pytest

import oracle
from kueue_b200 import abi, synth
from tests.helpers import assert_cycle_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ev():
    from kueue_b200 import native
    e = native.Evaluator(0)
    e.set_profile(True)
    yield e
    e.close()


def _base(**kw):
    kw.setdefault("W", 3000)
    kw.setdefault("Q", 300)
    return synth.make_snapshot(3, heads="one_per_cq", **kw)


def _nominal(snap):
    return np.array(snap.arrays["nominal"]).reshape(snap.n_cq + snap.n_cohort, -1)


def _borrow_limits(snap, seed=11):
    """A third of the ClusterQueues get a borrowing limit: 0, a quarter of the nominal quota or the nominal quota."""
    rng = np.random.default_rng(seed)
    Q = snap.n_cq
    nom = _nominal(snap)
    bl = np.array(snap.arrays["borrow_limit"]).reshape(nom.shape).copy()
    pick = rng.random(Q) < 1 / 3
    frac = rng.choice([0.0, 0.25, 1.0], Q)
    bl[:Q][pick] = (nom[:Q][pick] * frac[pick][:, None]).astype(np.int64)
    snap.set("borrow_limit", bl)
    return snap


def _cohort_quota(snap, seed=12):
    """Every root cohort has nominal quota of its own, about two ClusterQueues' worth."""
    rng = np.random.default_rng(seed)
    Q, C = snap.n_cq, snap.n_cohort
    nom = _nominal(snap).copy()
    nom[Q:] = (nom[:Q].mean(0)[None, :] * rng.uniform(1.0, 3.0, (C, 1))).astype(np.int64)
    snap.set("nominal", nom)
    return snap


def _lend_limits(snap, seed=13):
    """Lending limits at 0 (nothing lent) and at the nominal quota (everything lent) on a fifth of the ClusterQueues
    each, the cohort's unchanged."""
    rng = np.random.default_rng(seed)
    Q = snap.n_cq
    nom = _nominal(snap)
    ll = np.array(snap.arrays["lend_limit"]).reshape(nom.shape).copy()
    u = rng.random(Q)
    ll[:Q][u < 0.2] = 0
    ll[:Q][(u >= 0.2) & (u < 0.4)] = nom[:Q][(u >= 0.2) & (u < 0.4)]
    snap.set("lend_limit", ll)
    return snap


def _reducible(snap, seed=14):
    """Partial admission on, single-podset heads only; a third of the podsets can be reduced."""
    rng = np.random.default_rng(seed)
    snap.flags |= abi.F_PARTIAL_ADMISSION
    count = np.array(snap.arrays["ps_count"])
    snap.set("ps_min_count", np.where((rng.random(len(count)) < 1 / 3) & (count > 1), np.maximum(1, count // 2), -1))
    return snap


def _classical(snap):
    snap.flags &= ~abi.F_FAIR_SHARING
    return snap


def _run(ev, snap):
    got = ev.run_cycle(snap)
    st = ev.stats()
    assert st.kernel_ms[abi.KERNEL_NAMES.index("k_cycle_flat")] > 0, "the cycle must run k_cycle_flat"
    return got, st


@pytest.mark.parametrize("make", [
    lambda: _borrow_limits(_base()),
    lambda: _cohort_quota(_base()),
    lambda: _lend_limits(_base()),
    lambda: _lend_limits(_cohort_quota(_borrow_limits(_base(tight=0.9)))),
    lambda: _lend_limits(_cohort_quota(_borrow_limits(_base(W=900, Q=90, F=3, R=3)))),  # FR = 9: per-thread staging
    lambda: _classical(_lend_limits(_cohort_quota(_borrow_limits(_base())))),
], ids=["borrow_limits", "cohort_quota", "lend_limits", "all_limits", "all_limits_fr9", "all_limits_classical"])
def test_flat_quota_shapes_match_oracle(ev, make):
    snap = make().finalize()
    got, st = _run(ev, snap)
    assert st.flat_group_walk[1] > 0 and st.flat_group_walk[0] == st.flat_group_walk[1], "every entry must take the group walk"
    assert_cycle_equal(got, oracle.run_cycle(snap))


@pytest.mark.parametrize("make", [
    lambda: _reducible(_base()),
    lambda: _reducible(_lend_limits(_cohort_quota(_borrow_limits(_base())))),
], ids=["reducible", "reducible_all_limits"])
def test_flat_partial_admission_single_podsets_match_oracle(ev, make):
    """Reducible heads take the general walk, the others the group walk in the same root, after the sweep."""
    snap = make().finalize()
    got, st = _run(ev, snap)
    assert 0 < st.flat_group_walk[0] < st.flat_group_walk[1], "the root must mix both walks"
    assert_cycle_equal(got, oracle.run_cycle(snap))
