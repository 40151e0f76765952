"""Seeded synthetic snapshots for the BASELINE.json configs (SURVEY.md §8d).

Generated directly in the flat SoA form with numpy (PCG64, seed = config index)
so 1M-workload snapshots build in about a second.  Value ranges keep every sum far
below 2^62.
"""
from __future__ import annotations

import numpy as np

from . import abi

# mean request per resource; resources past the eighth repeat the row (np.resize), so R <= 8 keeps its old snapshots
_SCALE = np.array([2_000, 2**31, 4, 100_000, 50, 10, 1000, 64], np.int64)


def _scale(R: int) -> np.ndarray:
    return np.resize(_SCALE, R)


def _cohort_forest(n_root: int, fanouts, cqs_per_leaf: int):
    """Cohort forest: n_root roots, then `fanouts` children per level; CQs hang off
    the deepest cohorts.  Returns (parent_of_cohort, leaf cohort ids)."""
    parents = [-1] * n_root
    level = list(range(n_root))
    for f in fanouts:
        nxt = []
        for p in level:
            for _ in range(f):
                parents.append(p)
                nxt.append(len(parents) - 1)
        level = nxt
    return np.array(parents, np.int64), np.array(level, np.int64)


def make_snapshot(config: int = 2, W: int | None = None, Q: int | None = None, F: int | None = None,
                  R: int | None = None, seed: int | None = None, heads: str = "all",
                  podsets_max: int = 1, admitted: int | None = None, preemption: bool | None = None,
                  partial: bool = False, tight: float = 1.0, afs: int = 0, evictable: bool = False) -> abi.FlatSnapshot:
    """config 1: 100 wl x 10 CQ x 2 flavors x 3 resources, no cohort
       config 2: 100k x 1k x 8 x 4, StrictFIFO, no cohort, usage 60-90% of nominal
       config 3: 1M x 10k, 100 flat cohorts x 100 CQ, BestEffortFIFO, fair sharing
       config 4: 1M x 10k, depth-4 cohort forest (10 -> 5 -> 5 -> 4), classical
    heads: "all" (batched evaluator over every pending workload) | "one_per_cq"
    (reference cycle: the best-ordered workload of each CQ).
    afs: k > 0 gives every ClusterQueue k LocalQueues with UsageBasedAdmissionFairSharing (see `add_afs`).
    evictable: every admitted workload also gets a pending record and `adm_wl` names it (see `add_evictable`): a drain
    replays the evictions of its preemptions."""
    dflt = {1: (100, 10, 2, 3), 2: (100_000, 1_000, 8, 4), 3: (1_000_000, 10_000, 8, 4), 4: (1_000_000, 10_000, 8, 4)}[config]
    W = W or dflt[0]; Q = Q or dflt[1]; F = F or dflt[2]; R = R or dflt[3]
    rng = np.random.Generator(np.random.PCG64(config if seed is None else seed))
    FR = F * R
    # ---- cohort structure ----
    if config in (1, 2):
        coh_parent = np.zeros(0, np.int64); cq_parent = np.full(Q, -1, np.int64)
    elif config == 3:
        ncoh = max(1, Q // 100)
        coh_parent = np.full(ncoh, -1, np.int64)
        cq_parent = Q + (np.arange(Q) % ncoh)
    else:
        nroot = max(1, Q // 1000)
        coh_parent, leaves = _cohort_forest(nroot, (5, 5, 4), 10)
        cq_parent = Q + leaves[np.arange(Q) % len(leaves)]
        coh_parent = np.where(coh_parent >= 0, coh_parent + Q, -1)
    C = len(coh_parent); N = Q + C
    snap = abi.FlatSnapshot(n_cq=Q, n_cohort=C, n_flavor=F, n_resource=R)
    flags = abi.FLAGS_DEFAULT
    if config == 3:
        flags |= abi.F_FAIR_SHARING
    snap.flags = flags
    snap.set("parent", np.concatenate([cq_parent, coh_parent]))
    fw = np.ones(N)
    if config == 3:
        fw[:Q] = rng.choice([0.5, 1.0, 2.0], Q)
    snap.set("fair_weight", fw)
    # ---- quotas ----
    scale = _scale(R)
    per_cq = max(1, W // Q)
    k = rng.uniform(4, 16, (Q, F, 1))
    nominal = np.zeros((N, FR), np.int64)
    nominal[:Q] = (k * scale[None, None, :]).astype(np.int64).reshape(Q, FR)
    bl = np.full((N, FR), abi.KB_NO_LIMIT, np.int64)
    ll = np.full((N, FR), abi.KB_NO_LIMIT, np.int64)
    if config == 3:
        lend = rng.random(Q) < 0.2
        ll[:Q][lend] = nominal[:Q][lend] // 2
    if config == 4:
        has_q = rng.random(C) < 0.3
        nominal[Q:][has_q] = (rng.uniform(2, 8, (int(has_q.sum()), F, 1)) * scale[None, None, :]).astype(np.int64).reshape(-1, FR)
        blm = rng.random(Q) < 0.3
        bl[:Q][blm] = nominal[:Q][blm]
    snap.set("nominal", nominal); snap.set("borrow_limit", bl); snap.set("lend_limit", ll)
    lo, hi = {1: (0.6, 0.9), 2: (0.6, 0.9), 3: (0.7, 1.25), 4: (0.85, 1.2)}[config]
    lo, hi = lo * tight, hi * tight
    if preemption is None:
        preemption = config == 4
    if admitted is None:
        admitted = max(W // 5, 2 * Q * F) if preemption else 0
    if admitted:
        # admitted workloads (preemption candidates); ClusterQueue usage is exactly their sum
        A = admitted
        pair = rng.permutation(A) % (Q * F)        # round-robin over (ClusterQueue, flavor) pairs
        a_cq, a_f = pair // F, pair % F
        per = np.bincount(pair, minlength=Q * F)[pair].astype(np.float64)
        frac = rng.uniform(lo, hi, Q * F)[pair]      # target usage of the pair as a fraction of nominal
        qty = (nominal[:Q].reshape(Q, F, R)[a_cq, a_f] * (frac / per)[:, None] * rng.uniform(0.7, 1.3, (A, R))).astype(np.int64)
        usage = np.zeros((Q, F, R), np.int64)
        np.add.at(usage, (a_cq, a_f), qty)
        usage = usage.reshape(Q, FR)
        snap.set("adm_cq", a_cq); snap.set("adm_priority", rng.integers(0, 4, A) * 100)
        snap.set("adm_ts", 1_600_000_000_000_000_000 + rng.permutation(A).astype(np.int64) * 1_000_000)
        qr = 1_650_000_000_000_000_000 + rng.permutation(A).astype(np.int64) * 1_000_000
        qr[rng.random(A) < 0.02] = abi.KB_TS_UNSET
        snap.set("adm_qr_ts", qr); snap.set("adm_uid", rng.permutation(A) + 10_000_000)
        snap.set("adm_evicted", rng.random(A) < 0.01)
        snap.set("adm_use_start", np.arange(A + 1) * R)
        snap.set("adm_use_fr", (a_f[:, None] * R + np.arange(R)[None, :]).reshape(-1))
        snap.set("adm_use_qty", qty.reshape(-1))
        snap.now_ns = 1_700_000_000_000_000_000
    else:
        usage = (nominal[:Q] * rng.uniform(lo, hi, (Q, FR))).astype(np.int64)
        if config in (1, 2):
            usage = np.minimum(usage, nominal[:Q])
    snap.set("cq_usage", usage)
    if preemption:
        snap.set("cq_within_cq", rng.choice([abi.POLICY_NEVER, abi.POLICY_LOWER_PRIORITY, abi.POLICY_LOWER_OR_NEWER_EQUAL_PRIORITY], Q))
        if C:
            snap.set("cq_reclaim_within", rng.choice([abi.POLICY_NEVER, abi.POLICY_LOWER_PRIORITY, abi.POLICY_ANY], Q))
            bw = rng.random(Q) < 0.4
            bw &= snap.arrays["cq_reclaim_within"] != abi.POLICY_NEVER  # API validation: reclaim=Never excludes borrowWithinCohort
            snap.set("cq_borrow_within", np.where(bw, abi.POLICY_LOWER_PRIORITY, abi.POLICY_NEVER))
            thr = bw & (rng.random(Q) < 0.5)
            snap.set("cq_has_bwc_threshold", thr); snap.set("cq_bwc_threshold", np.where(thr, 100, 0))
    # ---- CQ attributes: one resource group covering all resources, all flavors ----
    snap.set("cq_strategy", np.full(Q, abi.QUEUE_STRICT_FIFO if config == 2 else abi.QUEUE_BEST_EFFORT_FIFO))
    snap.set("cq_rg_start", np.arange(Q + 1))
    snap.set("rg_res_mask", np.full(Q, (1 << R) - 1))
    snap.set("rg_flavor_start", np.arange(Q + 1) * F)
    snap.set("rg_flavors", np.tile(np.arange(F), Q))
    # ---- pending workloads, grouped by CQ ----
    wl_cq = np.sort(rng.integers(0, Q, W)) if config != 1 else np.repeat(np.arange(Q), per_cq)[:W]
    snap.set("wl_cq", wl_cq)
    snap.set("wl_priority", rng.integers(0, 4, W) * 100)
    snap.set("wl_ts", 1_700_000_000_000_000_000 + rng.permutation(W).astype(np.int64) * 1_000_000)
    snap.set("wl_uid", rng.permutation(W))
    nps = rng.integers(1, podsets_max + 1, W) if podsets_max > 1 else np.ones(W, np.int64)
    st = np.concatenate([[0], np.cumsum(nps)])
    P = int(st[-1])
    snap.set("wl_ps_start", st)
    count = rng.integers(1, 9, P)
    per_pod = (rng.uniform(0.05, 1.0, (P, R)) * scale[None, :] / 4).astype(np.int64)
    big = rng.random(P) < 0.03  # a few podsets larger than any ClusterQueue can ever hold
    per_pod[big] *= 40
    snap.set("ps_req", per_pod * count[:, None])
    snap.set("ps_req_mask", np.full(P, (1 << R) - 1))
    snap.set("ps_count", count)
    if partial:
        mc = np.where(rng.random(P) < 0.5, np.maximum(1, count // 2), -1)
        snap.set("ps_min_count", mc)
    ok = rng.integers(0, 2**63, P, dtype=np.uint64) | rng.integers(0, 2**63, P, dtype=np.uint64) | np.uint64(1 << (F - 1))
    snap.set("ps_flavor_ok", ok)  # ~75% of flavors eligible, last flavor always
    if evictable:
        add_evictable(snap)
    if afs:
        add_afs(snap, afs, seed=(config if seed is None else seed) + 1000)
    if heads == "all":
        snap.set("heads", np.arange(snap.n_wl))
    else:
        # reference Heads(): per CQ the first in (priority desc, ts asc, uid) order (cluster_queue.go:636-685)
        order = np.lexsort((snap.wl_uid, snap.wl_ts, -snap.wl_priority, snap.wl_cq))
        first = np.concatenate([[True], snap.wl_cq[order][1:] != snap.wl_cq[order][:-1]])
        snap.set("heads", order[first])
    return snap.finalize()


def compact_to_heads(snap: abi.FlatSnapshot) -> abi.FlatSnapshot:
    """The pending tables reduced to the entries of the cycle — what `queues.Heads()` hands the
    reference scheduler (manager.go:721-794): the cycle never sees the workloads deeper in the queues."""
    from .shard import _csr_take
    a = snap.arrays
    R = snap.n_resource
    h = a["heads"].astype(np.int64)
    out = abi.FlatSnapshot(n_cq=snap.n_cq, n_cohort=snap.n_cohort, n_flavor=snap.n_flavor, n_resource=R,
                           pods_resource=snap.pods_resource, flags=snap.flags, now_ns=snap.now_ns)
    for k, v in a.items():
        if not (k.startswith("wl_") or k.startswith("ps_") or k == "heads"):
            out.arrays[k] = v
    for nm in ("wl_cq", "wl_priority", "wl_ts", "wl_uid", "wl_last_gen"):
        out.set(nm, a[nm][h])
    st, rows = _csr_take(a["wl_ps_start"].astype(np.int64), h)
    out.set("wl_ps_start", st)
    out.set("ps_req", a["ps_req"].reshape(-1, R)[rows]); out.set("ps_last_tried", a["ps_last_tried"].reshape(-1, R)[rows])
    for nm in ("ps_req_mask", "ps_count", "ps_min_count", "ps_flavor_ok"):
        out.set(nm, a[nm][rows])
    if "ps_group" in a:  # optional tables (kb_snapshot: NULL when absent)
        out.set("ps_group", a["ps_group"][rows])
    for nm in ("wl_has_quota_reservation", "wl_sched_hash"):
        if nm in a:
            out.set(nm, a[nm][h])
    out.set("heads", np.arange(len(h)))
    return out.finalize()


def add_afs(snap: abi.FlatSnapshot, k: int, seed: int = 0, half_life_s: float = 10.0, sampling_s: float = 1.0) -> abi.FlatSnapshot:
    """AdmissionFairSharing tables (include/kueue_b200.h): k LocalQueues per ClusterQueue (numbered ClusterQueue-major),
    every ClusterQueue in UsageBasedAdmissionFairSharing mode, every pending workload in a random LocalQueue of its
    ClusterQueue.  Seeded LocalQueue weights, consumed usage (cpu as whole or milli quantities, the other resources
    whole), initial entry penalties and ResourceWeights.  Resource 0 is cpu (milli units)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    Q, R, W = snap.n_cq, snap.n_resource, snap.n_wl
    L = Q * k
    snap.set("lq_cq", np.repeat(np.arange(Q), k))
    snap.set("wl_lq", snap.arrays["wl_cq"].astype(np.int64) * k + rng.integers(0, k, W))
    snap.set("cq_afs", np.ones(Q))
    snap.set("lq_weight", rng.choice([0.5, 1.0, 1.5, 2.0], L))
    scale = _scale(R)
    val = (rng.uniform(0, 8, (L, R)) * scale[None, :]).astype(np.int64)
    sc = np.zeros((L, R), np.int64)
    whole = rng.random(L) < 0.5  # cpu as "3" (scale 0) or "3500m" (scale -3)
    val[whole, 0] //= 1000
    sc[~whole, 0] = -3
    val[rng.random((L, R)) < 0.1] = 0  # absent keys
    snap.set("lq_consumed", val); snap.set("lq_consumed_scale", sc)
    snap.set("lq_penalty", np.where(rng.random((L, R)) < 0.3, rng.integers(0, 5000, (L, R)), 0))
    snap.set("afs_res_weight", rng.choice([0.5, 1.0, 2.0], R))
    snap.set("afs_milli_mul", np.where(np.arange(R) == 0, 1, 1000))
    snap.afs_alpha = 1.0 - 0.5 ** (sampling_s / half_life_s) if half_life_s else 0.0
    return snap


def add_afs_decay(snap: abi.FlatSnapshot, seed: int = 0, half_life_ns: int = 100_000, sampling_ns: int = 20_000) -> abi.FlatSnapshot:
    """Decay tables of an event drain (include/kueue_b200.h) on a snapshot with `add_afs` tables: every LocalQueue's
    LastUpdate spread over the last sampling interval, every admitted row in a random LocalQueue of its ClusterQueue
    (-1 where it has none), the two durations, and afs_alpha = calculateAlphaRate(sampling, half-life)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    a = snap.arrays
    L = len(a["lq_cq"])
    now = int(snap.now_ns)
    snap.set("lq_last_update_ns", now - rng.integers(0, sampling_ns, L))
    n_of = np.bincount(a["lq_cq"].astype(np.int64), minlength=snap.n_cq)
    first = np.concatenate([[0], np.cumsum(n_of)])
    cq = a["adm_cq"].astype(np.int64)
    pick = first[cq] + (rng.random(len(cq)) * np.maximum(n_of[cq], 1)).astype(np.int64)
    snap.set("adm_lq", np.where(n_of[cq] > 0, pick, -1))
    snap.afs_half_life_ns, snap.afs_sampling_ns = int(half_life_ns), int(sampling_ns)
    snap.afs_alpha = 1.0 - 0.5 ** (sampling_ns / half_life_ns) if half_life_ns else 0.0
    return snap


def add_evictable(snap: abi.FlatSnapshot) -> abi.FlatSnapshot:
    """Give every admitted workload a pending record consistent with its usage and name it in `adm_wl`
    (include/kueue_b200.h): same ClusterQueue, priority, queue-order timestamp and UID, one podset of count 1 whose
    requests are the workload's usage cells (every flavor eligible).  The records are appended after the existing
    pending workloads; admitted UIDs and pending UIDs stay distinct."""
    a = snap.arrays
    R, A, W = snap.n_resource, snap.n_adm, snap.n_wl
    use_start = a["adm_use_start"].astype(np.int64)
    req = np.zeros((A, R), np.int64)
    rows = np.repeat(np.arange(A), np.diff(use_start))
    np.add.at(req, (rows, a["adm_use_fr"].astype(np.int64) % R), a["adm_use_qty"])
    mask = np.zeros(A, np.int64)
    np.bitwise_or.at(mask, rows, 1 << (a["adm_use_fr"].astype(np.int64) % R))
    P = int(a["wl_ps_start"][-1]) if W else 0
    cat = lambda name, extra: snap.set(name, np.concatenate([a[name], np.asarray(extra).astype(a[name].dtype)]))  # noqa: E731
    cat("wl_cq", a["adm_cq"]); cat("wl_priority", a["adm_priority"]); cat("wl_ts", a["adm_ts"]); cat("wl_uid", a["adm_uid"])
    cat("wl_ps_start", P + 1 + np.arange(A))
    snap.set("ps_req", np.concatenate([a["ps_req"].reshape(-1, R), req]))
    cat("ps_req_mask", mask); cat("ps_count", np.ones(A))
    cat("ps_flavor_ok", np.full(A, np.iinfo(np.uint64).max, np.uint64))
    if "ps_last_tried" in a:
        snap.set("ps_last_tried", np.concatenate([a["ps_last_tried"].reshape(-1, R), np.full((A, R), -1)]))
    for name, fill in (("wl_last_gen", -1), ("ps_min_count", -1), ("wl_sched_hash", 0), ("wl_has_quota_reservation", 0)):
        if name in a:
            cat(name, np.full(A, fill))
    if "ps_group" in a:
        cat("ps_group", np.full(A, -1))
    snap.set("adm_wl", W + np.arange(A))
    return snap


def add_events(snap: abi.FlatSnapshot, seed: int = 0, present: float = 0.5, span_ns: int = 50_000, run_ns=(1_000, 20_000),
               never: float = 0.05, step_ns: int = 1_000) -> abi.FlatSnapshot:
    """Arrival and completion tables of kb_run_drain's event mode (include/kueue_b200.h), seeded, for any config: a
    share `present` of the workloads exists at now_ns, the others are created uniformly in (now_ns, now_ns + span_ns];
    run times are uniform in `run_ns`, a share `never` never finishes; every row admitted before the drain finishes in
    (now_ns, now_ns + span_ns].  Records named by adm_wl exist at now_ns.  One cycle takes step_ns."""
    rng = np.random.Generator(np.random.PCG64(seed))
    W, A, now = snap.n_wl, snap.n_adm, int(snap.now_ns)
    create = np.where(rng.random(W) < present, now - rng.integers(0, 1000, W), now + rng.integers(1, span_ns + 1, W))
    if "adm_wl" in snap.arrays:
        create[snap.arrays["adm_wl"]] = now
    run = np.where(rng.random(W) < never, -1, rng.integers(run_ns[0], run_ns[1] + 1, W))
    snap.set("wl_create_ns", create)
    snap.set("wl_run_ns", run)
    snap.set("adm_finish_ns", now + rng.integers(1, span_ns + 1, A))
    snap.drain_cycle_ns = step_ns
    return snap


def add_evict_latency(snap: abi.FlatSnapshot, ns_range=(0, 0), seed: int = 0) -> abi.FlatSnapshot:
    """Eviction latency of an event drain (include/kueue_b200.h) on a snapshot with `adm_wl`: every workload's time from
    its eviction until its quota is released, seeded uniform in `ns_range` (inclusive; the pods' termination grace period
    defaults to 30 s).  Adds no `adm_evict_end_ns`: rows evicted before the drain are issued when targeted."""
    rng = np.random.Generator(np.random.PCG64(seed))
    lo, hi = int(ns_range[0]), int(ns_range[1])
    snap.set("wl_evict_ns", rng.integers(lo, hi + 1, snap.n_wl))
    return snap


def add_admission_checks(snap: abi.FlatSnapshot, seed: int = 0, delay_ns=(1_000, 5_000), fail_share: float = 0.3,
                         max_fail: int = 2, all_fail_share: float = 0.05, cqs=None, backoff=(1, 8, 3)) -> abi.FlatSnapshot:
    """Admission checks of an event drain (include/kueue_b200.h) on a snapshot with `adm_wl`, seeded: the workloads of
    the ClusterQueues `cqs` (None = all) get a check delay uniform in `delay_ns` (inclusive; 0 elsewhere); a share
    `fail_share` of them fails its next 1..max_fail attempts and a share `all_fail_share` every attempt.  `backoff` is
    the RetryStrategy (base s, max s, limit)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    W = snap.n_wl
    on = np.ones(W, bool) if cqs is None else np.isin(snap.arrays["wl_cq"], np.asarray(cqs))
    delay = np.where(on, rng.integers(int(delay_ns[0]), int(delay_ns[1]) + 1, W), 0)
    u = rng.random(W)
    fail = np.where(u < fail_share, rng.integers(1, max_fail + 1, W), 0)
    fail = np.where(u > 1 - all_fail_share, np.iinfo(np.int32).max, fail)
    snap.set("wl_check_ns", delay)
    snap.set("wl_check_fail", np.where(on, fail, 0))
    snap.check_backoff_base_s, snap.check_backoff_max_s, snap.check_backoff_limit = (int(v) for v in backoff)
    return snap


def add_pods_ready(snap: abi.FlatSnapshot, seed: int = 0, delay_ns=(0, 2_000), fail_share: float = 0.1,
                   timeout_ns: int = 5_000, base_s: int = 1, max_s: int = 8, limit: int = 2, creation: int = 0) -> abi.FlatSnapshot:
    """WaitForPodsReady of an event drain (include/kueue_b200.h) on a snapshot with `adm_wl`, seeded: every workload
    gets an Admitted -> PodsReady delay uniform in `delay_ns` (inclusive), and a share `fail_share` of them never
    becomes ready (wl_pods_ready_fail = INT32_MAX).  timeout_ns, base_s, max_s, limit (-1 = nil) and creation are the
    waitForPodsReady settings."""
    rng = np.random.Generator(np.random.PCG64(seed))
    W = snap.n_wl
    snap.set("wl_pods_ready_ns", rng.integers(int(delay_ns[0]), int(delay_ns[1]) + 1, W))
    snap.set("wl_pods_ready_fail", np.where(rng.random(W) < fail_share, np.iinfo(np.int32).max, 0))
    snap.pods_ready_timeout_ns, snap.pods_ready_backoff_base_s, snap.pods_ready_backoff_max_s = int(timeout_ns), int(base_s), int(max_s)
    snap.pods_ready_backoff_limit, snap.pods_ready_requeue_creation = int(limit), int(creation)
    return snap


def add_max_exec(snap: abi.FlatSnapshot, seed: int = 0, share: float = 0.5, limit_s=(1, 3), spent_share: float = 0.1,
                 since_ns: int = 2_000_000_000) -> abi.FlatSnapshot:
    """MaximumExecutionTimeSeconds of an event drain (include/kueue_b200.h) on a snapshot with `adm_wl`, seeded: a share
    `share` of the workloads gets a limit uniform in `limit_s` seconds (inclusive; 0 = nil elsewhere).  A share
    `spent_share` of those starts with an accumulated time of limit - 1, limit or limit + 1 seconds, so its remaining time
    is 1 s, 0 or negative: below the run time of most workloads; the others start nil.  Every admitted row of the
    snapshot gets an Admitted time up to `since_ns` before now_ns (INT64_MIN where its checks run, adm_admitted_ns where
    that is set)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    W, A, now = snap.n_wl, snap.n_adm if "adm_cq" in snap.arrays else 0, int(snap.now_ns)
    limit = np.where(rng.random(W) < share, rng.integers(int(limit_s[0]), int(limit_s[1]) + 1, W), 0)
    spent = (limit > 0) & (rng.random(W) < spent_share)
    acc = np.where(spent, np.maximum(limit + rng.integers(-1, 2, W), 0), -1)
    since = now - rng.integers(0, int(since_ns) + 1, A)
    a = snap.arrays
    if "adm_admitted_ns" in a:
        since = np.where(a["adm_admitted_ns"] != np.iinfo(np.int64).min, a["adm_admitted_ns"], since)
    if "adm_check_end_ns" in a:
        since = np.where(a["adm_check_end_ns"] != np.iinfo(np.int64).min, np.iinfo(np.int64).min, since)
    snap.set("wl_max_exec_s", limit)
    snap.set("wl_exec_acc_s", acc)
    snap.set("adm_exec_since_ns", since)
    return snap


def _covered_cells(snap: abi.FlatSnapshot) -> np.ndarray:
    """[n_cq][F*R] the cells a ClusterQueue's resource groups cover"""
    a, R = snap.arrays, snap.n_resource
    cov = np.zeros((snap.n_cq, snap.n_fr), bool)
    for q in range(snap.n_cq):
        for g in range(int(a["cq_rg_start"][q]), int(a["cq_rg_start"][q + 1])):
            for f in a["rg_flavors"][int(a["rg_flavor_start"][g]):int(a["rg_flavor_start"][g + 1])]:
                for r in range(R):
                    if int(a["rg_res_mask"][g]) >> r & 1:
                        cov[q, int(f) * R + r] = True
    return cov


def add_quota_changes(snap: abi.FlatSnapshot, seed: int = 0, span_ns: int = 50_000, dip: float = 0.5, lend_share: float = 0.2,
                      noop_share: float = 0.1, start_ns: int | None = None) -> abi.FlatSnapshot:
    """Planned ClusterQueue / Cohort quota edits of an event drain (kb_snapshot.qc_*, include/kueue_b200.h), seeded, in
    (start_ns, start_ns + span_ns] (start_ns defaults to now_ns):
      - a capacity dip per root tree: at a time t1 the nominal row of every node of the tree with some quota is scaled by
        `dip` (a ClusterQueue's covered cells only), and at a later t2 restored;
      - a share `lend_share` of the ClusterQueues with quota get a lending limit of half their nominal quota on their
        covered cells at one time (KB_NO_LIMIT elsewhere stays);
      - a share `noop_share` of the nodes get an edit at one time that repeats the rows in force then (no change).
    The edits are sorted by time (ties keep the order above)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    a = snap.arrays
    N, Q, FR = snap.n_nodes, snap.n_cq, snap.n_fr
    t0 = int(snap.now_ns if start_ns is None else start_ns)
    snap.finalize()  # the default rows of absent tables
    rows = [a[k].reshape(N, FR).astype(np.int64).copy() for k in ("nominal", "borrow_limit", "lend_limit")]
    cov = np.ones((N, FR), bool)
    cov[:Q] = _covered_cells(snap)
    parent = a["parent"].astype(np.int64)
    root = np.arange(N)
    for _ in range(N):
        root = np.where(parent[root] >= 0, parent[root], root)
    plan = []  # (time, kind order, node, kind)
    for r in np.unique(root):
        t1, t2 = np.sort(rng.integers(1, span_ns + 1, 2))
        for n in np.flatnonzero(root == r):
            if (rows[0][n][cov[n]] > 0).any():
                plan += [(t0 + int(t1), 0, int(n), "dip"), (t0 + int(t2) + (t2 == t1), 0, int(n), "restore")]
    for q in range(Q):
        if (rows[0][q][cov[q]] > 0).any() and rng.random() < lend_share:
            plan.append((t0 + int(rng.integers(1, span_ns + 1)), 1, q, "lend"))
    for n in range(N):
        if rng.random() < noop_share:
            plan.append((t0 + int(rng.integers(1, span_ns + 1)), 2, n, "noop"))
    plan.sort(key=lambda e: (e[0], e[1]))
    base = rows[0].copy()
    ns, node, out = [], [], [[], [], []]
    for t, _, n, kind in plan:
        if kind == "dip":
            rows[0][n] = np.where(cov[n], (base[n] * dip).astype(np.int64), rows[0][n])
        elif kind == "restore":
            rows[0][n] = np.where(cov[n], base[n], rows[0][n])
        elif kind == "lend":
            rows[2][n] = np.where(cov[n], rows[0][n] // 2, rows[2][n])
        ns.append(t); node.append(n)
        for k in range(3):
            out[k].append(rows[k][n].copy())
    snap.set("qc_ns", np.asarray(ns, np.int64)); snap.set("qc_node", np.asarray(node, np.int64))
    for k, nm in enumerate(("qc_nominal", "qc_borrow_limit", "qc_lend_limit")):
        snap.set(nm, np.asarray(out[k], np.int64).reshape(len(ns), FR))
    return snap


def add_active_changes(snap: abi.FlatSnapshot, seed: int = 0, span_ns: int = 50_000, stop_share: float = 0.1,
                       resume_share: float = 0.5, inactive_share: float = 0.0, start_ns: int | None = None) -> abi.FlatSnapshot:
    """Stop / resume edits of spec.active for an event drain (kb_snapshot.ac_*, wl_inactive, include/kueue_b200.h),
    seeded: a share `stop_share` of the records get a stop at a time in (t, t + span_ns] with t the later of start_ns
    (default now_ns) and its creation, and a share `resume_share` of those a resume at or after it, within span_ns;
    a share `inactive_share` of the records present at the start that adm_wl does not name start inactive (reason 4).
    The edits are sorted by time (a stop before a resume at the same time).  An empty adm_wl is added when the
    snapshot has no admitted rows and no adm_wl."""
    rng = np.random.Generator(np.random.PCG64(seed))
    a = snap.arrays
    snap.finalize()
    W = snap.n_wl
    if "adm_wl" not in a and snap.n_adm == 0:
        snap.set("adm_wl", np.zeros(0))
    t0 = int(snap.now_ns if start_ns is None else start_ns)
    create = a["wl_create_ns"].astype(np.int64) if "wl_create_ns" in a else np.full(W, np.iinfo(np.int64).min)
    plan = []  # (time, kind, record)
    for w in np.flatnonzero(rng.random(W) < stop_share):
        t = max(t0, int(create[w])) + int(rng.integers(1, span_ns + 1))
        plan.append((t, 0, int(w)))
        if rng.random() < resume_share:
            plan.append((t + int(rng.integers(0, span_ns + 1)), 1, int(w)))
    plan.sort(key=lambda e: (e[0], e[1]))
    snap.set("ac_ns", np.asarray([p[0] for p in plan], np.int64))
    snap.set("ac_wl", np.asarray([p[2] for p in plan], np.int64))
    snap.set("ac_active", np.asarray([p[1] for p in plan], np.int64))
    if inactive_share > 0:
        held = np.zeros(W, bool)
        held[a["adm_wl"].astype(np.int64)] = True
        ok = ~held & (create <= snap.now_ns)
        snap.set("wl_inactive", np.where(ok & (rng.random(W) < inactive_share), 4, 0))
    return snap


# The reference's scheduler performance scenario (test/performance/scheduler/configs/baseline/generator.yaml, generated
# by runner/generator/generator.go): 5 cohorts of 6 ClusterQueues, one flavor, cpu only; per ClusterQueue, workload k of
# a class is created at (k + 1) * interval and runs `run` once admitted (runner/controller/controller.go).
PERF_CLASSES = (  # (name, count per ClusterQueue, interval ms, run time ms, priority, cpu)
    ("small", 350, 100, 200, 50, 1),
    ("medium", 100, 500, 500, 100, 5),
    ("large", 50, 1200, 1000, 200, 20),
)
PERF_COHORTS, PERF_CQS_PER_COHORT = 5, 6
PERF_NOMINAL_CPU, PERF_BORROW_CPU = 20, 100
_MS = 1_000_000


def perf_scenario(scale: float = 1.0, cycle_ns: int = _MS, evict_ns: int | None = None, checks: int | None = None,
                  pods_ready: int | None = None, max_exec: int | None = None, quota: int | None = None,
                  active: int | None = None) -> abi.FlatSnapshot:
    """The baseline scenario as numbers (15,000 workloads at scale 1; `scale` multiplies the count of every class):
    nominal 20 cpu and borrowingLimit 100 cpu per ClusterQueue, preemption reclaimWithinCohort Any and
    withinClusterQueue LowerPriority, BestEffortFIFO.  cpu is in milli-units.  wl_ts is the creation time, an empty
    adm_wl turns eviction replay on, and `snap.perf_class` holds each workload's index into PERF_CLASSES.  One drain cycle takes cycle_ns of simulated time.
    evict_ns: the termination latency of every workload (wl_evict_ns: an eviction releases its quota that long after it
    is issued); None = every eviction completes before the next cycle.
    checks: a seed: every other ClusterQueue of each cohort gets an admission check (add_admission_checks: a
    ProvisioningRequest-like delay of 20-200 ms, a share of failing attempts, backoff base 1 s, max 8 s, limit 3).
    pods_ready: a seed: WaitForPodsReady on every workload (add_pods_ready: a PodsReady delay of 0-50 ms, 10% of the
    workloads never ready, timeout 100 ms, backoff base 1 s, max 8 s, limit 2).
    max_exec: a seed: MaximumExecutionTimeSeconds (add_max_exec: half of the workloads get a limit of 1 s, and 20% of
    those start with 0, 1 or 2 s accumulated, so they expire at admission or race their run time of up to 1 s).
    quota: a seed: a capacity dip (add_quota_changes over the scenario's 60 s: each cohort's ClusterQueues drop to half
    their nominal quota at one time and get it back later, some lending limits, some no-op edits).
    active: a seed: stop / resume edits (add_active_changes over the scenario's 60 s: 5% of the workloads are stopped
    once, half of those resumed later)."""
    Q = PERF_COHORTS * PERF_CQS_PER_COHORT
    snap = abi.FlatSnapshot(n_cq=Q, n_cohort=PERF_COHORTS, n_flavor=1, n_resource=1)
    snap.set("parent", np.concatenate([Q + np.arange(Q) // PERF_CQS_PER_COHORT, np.full(PERF_COHORTS, -1)]))
    nominal = np.zeros((Q + PERF_COHORTS, 1), np.int64)
    nominal[:Q] = PERF_NOMINAL_CPU * 1000
    bl = np.full((Q + PERF_COHORTS, 1), abi.KB_NO_LIMIT, np.int64)
    bl[:Q] = PERF_BORROW_CPU * 1000
    snap.set("nominal", nominal); snap.set("borrow_limit", bl)
    snap.set("cq_within_cq", np.full(Q, abi.POLICY_LOWER_PRIORITY)); snap.set("cq_reclaim_within", np.full(Q, abi.POLICY_ANY))
    snap.set("cq_strategy", np.full(Q, abi.QUEUE_BEST_EFFORT_FIFO))
    snap.set("cq_rg_start", np.arange(Q + 1)); snap.set("rg_res_mask", np.ones(Q)); snap.set("rg_flavor_start", np.arange(Q + 1))
    snap.set("rg_flavors", np.zeros(Q))
    cq, cls, create, run, prio, cpu = [], [], [], [], [], []
    for q in range(Q):
        for c, (_, count, interval, run_ms, p, req) in enumerate(PERF_CLASSES):
            n = max(1, int(round(count * scale)))
            cq += [q] * n; cls += [c] * n
            create += list((np.arange(n) + 1) * interval * _MS)
            run += [run_ms * _MS] * n; prio += [p] * n; cpu += [req * 1000] * n
    W = len(cq)
    snap.set("wl_cq", cq); snap.set("wl_priority", prio)
    snap.set("wl_ts", create); snap.set("wl_uid", np.arange(W))
    snap.set("ps_req", np.asarray(cpu, np.int64)[:, None]); snap.set("ps_req_mask", np.ones(W)); snap.set("ps_count", np.ones(W))
    snap.set("wl_create_ns", create); snap.set("wl_run_ns", run)
    snap.set("adm_wl", np.zeros(0))
    if evict_ns is not None:
        snap.set("wl_evict_ns", np.full(W, evict_ns))
    snap.now_ns = 0
    snap.drain_cycle_ns = cycle_ns
    if checks is not None:
        add_admission_checks(snap, checks, delay_ns=(20 * _MS, 200 * _MS), cqs=np.arange(0, Q, 2))
    if pods_ready is not None:
        add_pods_ready(snap, pods_ready, delay_ns=(0, 50 * _MS), timeout_ns=100 * _MS)
    if max_exec is not None:
        add_max_exec(snap, max_exec, share=0.5, limit_s=(1, 1), spent_share=0.2)
    if quota is not None:
        add_quota_changes(snap, quota, span_ns=int(60_000 * scale) * _MS)
    if active is not None:
        add_active_changes(snap, active, span_ns=int(60_000 * scale) * _MS, stop_share=0.05)
    snap.finalize()
    snap.__dict__["perf_class"] = np.asarray(cls, np.int64)
    return snap
