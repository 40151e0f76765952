"""Multi-GPU sharding of one snapshot by ROOT COHORT (SURVEY.md §8e).

All quota coupling of the cycle is confined to a cohort tree (`available` stops at the
root, resource_node.go:106-108; preemption candidates come from the root's subtree,
preemption.go:523), and a ClusterQueue without a cohort is its own root.  Ranks therefore
take disjoint sets of roots, run the unchanged single-GPU cycle on their sub-snapshot and
the host concatenates the decisions: no collective on the data path.

`partition_roots` bin-packs roots by (entries + admitted workloads + nodes);
`shard` builds rank r's sub-snapshot with re-indexed nodes / workloads / admitted tables;
`merge` scatters the per-rank outputs back into full-size output arrays.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import abi


def root_of_nodes(parent: np.ndarray) -> np.ndarray:
    root = np.arange(len(parent))
    p = parent.copy()
    for _ in range(abi.KB_MAX_RESOURCES + 4):  # depth <= KB_MAX_DEPTH
        has = p[root] >= 0
        if not has.any():
            break
        root = np.where(has, p[root], root)
    return root


def partition_roots(snap: abi.FlatSnapshot, world: int) -> np.ndarray:
    """rank of every node (nodes of one root always share a rank); greedy LPT bin packing."""
    a = snap.arrays
    N = snap.n_nodes
    root = root_of_nodes(a["parent"].astype(np.int64))
    w = np.bincount(root, minlength=N).astype(np.int64)  # nodes
    if snap.n_heads:
        w += np.bincount(root[a["wl_cq"][a["heads"]]], minlength=N) * 4
    if snap.n_adm:
        w += np.bincount(root[a["adm_cq"]], minlength=N)
    roots = np.flatnonzero(a["parent"] < 0)
    order = roots[np.argsort(-w[roots], kind="stable")]
    load = np.zeros(world, np.int64)
    rank_of_root = np.zeros(N, np.int64)
    for r in order:
        k = int(np.argmin(load))
        rank_of_root[r] = k
        load[k] += w[r]
    return rank_of_root[root]


@dataclass
class ShardMap:
    nodes: np.ndarray    # global node id of each local node (CQs first, then cohorts)
    wls: np.ndarray      # global pending index of each local pending workload
    podsets: np.ndarray  # global podset row of each local podset row
    adms: np.ndarray     # global admitted index of each local admitted workload
    heads: np.ndarray    # global ENTRY position of each local entry


def _csr_take(start: np.ndarray, rows: np.ndarray):
    """Rows `rows` of a CSR structure: (new_start, flat index of the kept cells)."""
    lens = start[rows + 1] - start[rows]
    new_start = np.concatenate([[0], np.cumsum(lens)])
    if len(rows) == 0 or new_start[-1] == 0:
        return new_start, np.zeros(0, np.int64)
    idx = np.repeat(start[rows] - new_start[:-1], lens) + np.arange(new_start[-1])
    return new_start, idx


def shard(snap: abi.FlatSnapshot, rank: int, world: int, node_rank: np.ndarray | None = None):
    a = snap.arrays
    Q, N, FR, R = snap.n_cq, snap.n_nodes, snap.n_fr, snap.n_resource
    if node_rank is None:
        node_rank = partition_roots(snap, world)
    keep = np.flatnonzero(node_rank == rank)
    cqs, cohorts = keep[keep < Q], keep[keep >= Q]
    nodes = np.concatenate([cqs, cohorts])
    remap = np.full(N, -1, np.int64)
    remap[nodes] = np.arange(len(nodes))
    out = abi.FlatSnapshot(n_cq=len(cqs), n_cohort=len(cohorts), n_flavor=snap.n_flavor, n_resource=R,
                           pods_resource=snap.pods_resource, flags=snap.flags, now_ns=snap.now_ns)
    par = a["parent"][nodes].astype(np.int64)
    out.set("parent", np.where(par >= 0, remap[np.maximum(par, 0)], -1))
    out.set("fair_weight", a["fair_weight"][nodes])
    for nm in ("nominal", "borrow_limit", "lend_limit"):
        out.set(nm, a[nm].reshape(N, FR)[nodes])
    out.set("cq_usage", a["cq_usage"].reshape(Q, FR)[cqs])
    for nm in ("cq_within_cq", "cq_reclaim_within", "cq_borrow_within", "cq_has_bwc_threshold", "cq_bwc_threshold",
               "cq_when_can_borrow", "cq_when_can_preempt", "cq_preference", "cq_strategy", "cq_generation"):
        out.set(nm, a[nm][cqs])
    rg_start, rg_rows = _csr_take(a["cq_rg_start"].astype(np.int64), cqs)
    out.set("cq_rg_start", rg_start)
    out.set("rg_res_mask", a["rg_res_mask"][rg_rows])
    fl_start, fl_idx = _csr_take(a["rg_flavor_start"].astype(np.int64), rg_rows)
    out.set("rg_flavor_start", fl_start)
    out.set("rg_flavors", a["rg_flavors"][fl_idx])
    # pending workloads
    wls = np.flatnonzero(node_rank[a["wl_cq"]] == rank) if snap.n_wl else np.zeros(0, np.int64)
    wl_remap = np.full(max(1, snap.n_wl), -1, np.int64)
    wl_remap[wls] = np.arange(len(wls))
    out.set("wl_cq", remap[a["wl_cq"][wls]])
    for nm in ("wl_priority", "wl_ts", "wl_uid", "wl_last_gen"):
        out.set(nm, a[nm][wls])
    ps_start, ps_rows = _csr_take(a["wl_ps_start"].astype(np.int64), wls)
    out.set("wl_ps_start", ps_start)
    out.set("ps_req", a["ps_req"].reshape(-1, R)[ps_rows])
    out.set("ps_last_tried", a["ps_last_tried"].reshape(-1, R)[ps_rows])
    for nm in ("ps_req_mask", "ps_count", "ps_min_count", "ps_flavor_ok"):
        out.set(nm, a[nm][ps_rows])
    if "ps_group" in a:  # optional tables (kb_snapshot: NULL when absent)
        out.set("ps_group", a["ps_group"][ps_rows])
    for nm in ("wl_has_quota_reservation", "wl_sched_hash"):
        if nm in a:
            out.set(nm, a[nm][wls])
    hpos = np.flatnonzero(wl_remap[a["heads"]] >= 0) if snap.n_heads else np.zeros(0, np.int64)
    out.set("heads", wl_remap[a["heads"][hpos]])
    # admitted workloads
    adms = np.flatnonzero(node_rank[a["adm_cq"]] == rank) if snap.n_adm else np.zeros(0, np.int64)
    out.set("adm_cq", remap[a["adm_cq"][adms]])
    for nm in ("adm_priority", "adm_ts", "adm_qr_ts", "adm_uid", "adm_evicted"):
        out.set(nm, a[nm][adms])
    us, ui = _csr_take(a["adm_use_start"].astype(np.int64), adms)
    out.set("adm_use_start", us)
    out.set("adm_use_fr", a["adm_use_fr"][ui]); out.set("adm_use_qty", a["adm_use_qty"][ui])
    if "adm_wl" in a:  # eviction replay: a record lives with its ClusterQueue, as does its admitted row
        out.set("adm_wl", wl_remap[a["adm_wl"][adms]])
    if "cq_sticky" in a:  # the sticky workload of a ClusterQueue is one of its records
        sw = a["cq_sticky"][cqs].astype(np.int64)
        out.set("cq_sticky", np.where(sw >= 0, wl_remap[np.maximum(sw, 0)], -1))
    if "wl_lq" in a:  # AdmissionFairSharing: the LocalQueues travel with their ClusterQueues (still ClusterQueue-major)
        L = len(a["lq_cq"])
        lqs = np.flatnonzero(node_rank[a["lq_cq"]] == rank) if L else np.zeros(0, np.int64)
        lq_remap = np.full(max(1, L), -1, np.int64)
        lq_remap[lqs] = np.arange(len(lqs))
        out.set("lq_cq", remap[a["lq_cq"][lqs]])
        out.set("wl_lq", lq_remap[a["wl_lq"][wls]])
        out.set("cq_afs", a["cq_afs"][cqs])
        out.set("lq_weight", a["lq_weight"][lqs])
        for nm in ("lq_consumed", "lq_consumed_scale", "lq_penalty"):
            if nm in a:
                out.set(nm, a[nm].reshape(L, R)[lqs])
        out.set("afs_res_weight", a["afs_res_weight"]); out.set("afs_milli_mul", a["afs_milli_mul"])
        out.afs_alpha = snap.afs_alpha
    out.finalize()
    return out, ShardMap(nodes=nodes, wls=wls, podsets=ps_rows, adms=adms, heads=hpos)


def merge(snap: abi.FlatSnapshot, parts) -> abi.CycleOut:
    """parts: iterable of (CycleOut of the shard, ShardMap).  Returns a full-size CycleOut."""
    parts = list(parts)
    total_t = sum(int(o.tgt_start[-1]) for o, _ in parts)
    full = abi.CycleOut(snap, tgt_capacity=max(16, total_t))
    H = snap.n_heads
    tgt_lists = [[] for _ in range(H)]
    for o, m in parts:
        for f in ("decision", "mode", "borrow", "commit_rank"):
            getattr(full, f)[m.heads] = getattr(o, f)
        for f in ("ps_flavor", "ps_res_mode", "ps_tried_idx", "ps_count"):
            getattr(full, f)[m.podsets] = getattr(o, f)
        if full.node_usage is not None and o.node_usage is not None:
            full.node_usage[m.nodes] = o.node_usage
        for le, ge in enumerate(m.heads):
            a0, a1 = int(o.tgt_start[le]), int(o.tgt_start[le + 1])
            tgt_lists[ge] = [(int(m.adms[o.tgt_adm[k]]), int(o.tgt_reason[k])) for k in range(a0, a1)]
    nt = 0
    for e in range(H):
        full.tgt_start[e] = nt
        for adm, reason in tgt_lists[e]:
            full.tgt_adm[nt] = adm; full.tgt_reason[nt] = reason; nt += 1
    full.tgt_start[H] = nt
    full.n_targets = nt
    return full
