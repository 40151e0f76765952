"""ctypes mirror of include/kueue_b200.h.

`FlatSnapshot` owns the structure-of-arrays buffers (numpy) that a Go host
would fill from pkg/cache/scheduler.Snapshot + queues.Heads(); `as_struct()`
yields the `kb_snapshot` the C-ABI takes.  Field names and order match the
header exactly — tests/test_abi.py checks sizeof/offsets against a C probe.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

KB_NO_LIMIT = np.iinfo(np.int64).max
KB_TS_UNSET = np.iinfo(np.int64).min
KB_MAX_RESOURCES = 16
KB_MAX_FLAVORS = 64

# enums (see header for the reference citations)
MODE_NOFIT, MODE_PREEMPT, MODE_FIT = 0, 1, 2
POLICY_NEVER, POLICY_LOWER_PRIORITY, POLICY_LOWER_OR_NEWER_EQUAL_PRIORITY, POLICY_ANY = 0, 1, 2, 3
FUNG_MAY_STOP_SEARCH, FUNG_TRY_NEXT_FLAVOR = 0, 1
PREF_UNSET, PREF_BORROWING_OVER_PREEMPTION, PREF_PREEMPTION_OVER_BORROWING = 0, 1, 2
QUEUE_BEST_EFFORT_FIFO, QUEUE_STRICT_FIFO = 0, 1
REASON_IN_CLUSTER_QUEUE, REASON_IN_COHORT_RECLAMATION = 1, 2
REASON_IN_COHORT_FAIR_SHARING, REASON_IN_COHORT_RECLAIM_WHILE_BORROWING = 3, 4
DEC_NOFIT, DEC_PREEMPT_NO_TARGETS, DEC_SKIPPED_OVERLAP, DEC_SKIPPED_NO_FIT, DEC_PREEMPTING, DEC_ASSUMED = range(6)
DEC_NAMES = ["NoFit", "PreemptNoTargets", "SkippedOverlap", "SkippedNoFit", "Preempting", "Assumed"]

F_FAIR_SHARING = 1 << 0
F_PARTIAL_ADMISSION = 1 << 1
F_FLAVOR_FUNGIBILITY = 1 << 2
F_PRIORITY_SORTING_WITHIN_COHORT = 1 << 3
F_TS_PREEMPTION_BUFFER = 1 << 9
F_FS_PRIORITIZE_NON_BORROWING = 1 << 4
F_FS_PREEMPT_WITHIN_NOMINAL = 1 << 5
F_FS_STRATEGY_S2A = 1 << 6
F_FS_STRATEGY_S2B = 1 << 7
F_FS_STRATEGY_S2B_FIRST = 1 << 8
F_USAGE_RESIDENT = 1 << 16  # upload hint: keep cq_usage on the device, usage_delta_* may follow (include/kueue_b200.h)
FLAGS_DEFAULT = (F_PARTIAL_ADMISSION | F_FLAVOR_FUNGIBILITY | F_PRIORITY_SORTING_WITHIN_COHORT |
                 F_FS_PRIORITIZE_NON_BORROWING | F_FS_PREEMPT_WITHIN_NOMINAL | F_FS_STRATEGY_S2A | F_FS_STRATEGY_S2B)

KB_OK, KB_ERR_INVALID, KB_ERR_CUDA, KB_ERR_CAPACITY, KB_ERR_UNSUPPORTED, KB_ERR_NO_DEVICE = 0, -1, -2, -3, -4, -5

_P = C.POINTER


class kb_snapshot(C.Structure):
    _fields_ = [
        ("n_cq", C.c_int32), ("n_cohort", C.c_int32), ("n_flavor", C.c_int32), ("n_resource", C.c_int32),
        ("n_rg", C.c_int32), ("n_wl", C.c_int32), ("n_podset", C.c_int32), ("n_adm", C.c_int32),
        ("n_adm_use", C.c_int32), ("n_heads", C.c_int32), ("pods_resource", C.c_int32), ("flags", C.c_uint32),
        ("now_ns", C.c_int64),
        ("parent", _P(C.c_int32)), ("fair_weight", _P(C.c_double)),
        ("nominal", _P(C.c_int64)), ("borrow_limit", _P(C.c_int64)), ("lend_limit", _P(C.c_int64)),
        ("cq_usage", _P(C.c_int64)),
        ("cq_within_cq", _P(C.c_uint8)), ("cq_reclaim_within", _P(C.c_uint8)), ("cq_borrow_within", _P(C.c_uint8)),
        ("cq_has_bwc_threshold", _P(C.c_uint8)), ("cq_bwc_threshold", _P(C.c_int32)),
        ("cq_when_can_borrow", _P(C.c_uint8)), ("cq_when_can_preempt", _P(C.c_uint8)), ("cq_preference", _P(C.c_uint8)),
        ("cq_strategy", _P(C.c_uint8)), ("cq_generation", _P(C.c_int64)),
        ("cq_rg_start", _P(C.c_int32)), ("rg_res_mask", _P(C.c_uint32)), ("rg_flavor_start", _P(C.c_int32)),
        ("rg_flavors", _P(C.c_int32)),
        ("wl_cq", _P(C.c_int32)), ("wl_priority", _P(C.c_int32)), ("wl_ts", _P(C.c_int64)), ("wl_uid", _P(C.c_int64)),
        ("wl_last_gen", _P(C.c_int64)), ("wl_ps_start", _P(C.c_int32)),
        ("ps_req", _P(C.c_int64)), ("ps_req_mask", _P(C.c_uint32)), ("ps_count", _P(C.c_int32)),
        ("ps_min_count", _P(C.c_int32)), ("ps_flavor_ok", _P(C.c_uint64)), ("ps_last_tried", _P(C.c_int8)),
        ("adm_cq", _P(C.c_int32)), ("adm_priority", _P(C.c_int32)), ("adm_ts", _P(C.c_int64)),
        ("adm_qr_ts", _P(C.c_int64)), ("adm_uid", _P(C.c_int64)), ("adm_evicted", _P(C.c_uint8)),
        ("adm_use_start", _P(C.c_int32)), ("adm_use_fr", _P(C.c_int32)), ("adm_use_qty", _P(C.c_int64)),
        ("heads", _P(C.c_int32)),
        ("wl_has_quota_reservation", _P(C.c_uint8)), ("wl_sched_hash", _P(C.c_int64)), ("ps_group", _P(C.c_int32)),
        ("static_generation", C.c_int64),
        ("n_usage_delta", C.c_int32), ("usage_delta_cq", _P(C.c_int32)), ("usage_delta_rows", _P(C.c_int64)),
    ]


class kb_cycle_out(C.Structure):
    _fields_ = [
        ("decision", _P(C.c_uint8)), ("mode", _P(C.c_uint8)), ("borrow", _P(C.c_int32)), ("commit_rank", _P(C.c_int32)),
        ("ps_flavor", _P(C.c_int8)), ("ps_res_mode", _P(C.c_int8)), ("ps_tried_idx", _P(C.c_int8)),
        ("ps_count", _P(C.c_int32)),
        ("tgt_start", _P(C.c_int32)), ("tgt_adm", _P(C.c_int32)), ("tgt_reason", _P(C.c_uint8)),
        ("tgt_capacity", C.c_int32), ("n_targets", C.c_int32),
        ("node_usage", _P(C.c_int64)),
    ]


class kb_tree_out(C.Structure):
    _fields_ = [
        ("subtree_quota", _P(C.c_int64)), ("usage", _P(C.c_int64)), ("available", _P(C.c_int64)),
        ("potential_available", _P(C.c_int64)), ("drs_rounded", _P(C.c_int64)), ("drs_resource", _P(C.c_int32)),
        ("drs_borrowing", _P(C.c_uint8)),
    ]


class kb_stats(C.Structure):
    _fields_ = [
        ("last_cycle_gpu_ms", C.c_double), ("last_h2d_ms", C.c_double), ("last_d2h_ms", C.c_double),
        ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("kernel_launches", C.c_int32), ("sm_count", C.c_int32),
        ("kernel_ms", C.c_float * 20), ("search_stat", C.c_int64 * 8),
        ("flat_group_walk", C.c_int64 * 2),
    ]


KERNEL_NAMES = ["k_tree", "k_lone", "k_nominate", "k_scan_roots", "k_scatter", "k_admit", "k_rank", "k_nominate_search_fair",
                "k_rank_admitted", "k_search_tables", "k_search_cells", "k_nominate_walk", "k_fair_prep", "k_drain", "k_tas", "k_cycle_flat", "k_tas_leaf", "k_tas_reduce", "k_tas_select", "-"]


class kb_drain_out(C.Structure):
    _fields_ = [
        ("max_cycles", C.c_int32), ("n_cycles", C.c_int32), ("n_decisions", C.c_int64), ("n_admitted", C.c_int64),
        ("cycle_heads", _P(C.c_int32)), ("cycle_admitted", _P(C.c_int32)),
        ("wl_admit_cycle", _P(C.c_int32)), ("wl_last_decision", _P(C.c_uint8)), ("wl_evals", _P(C.c_int32)),
        ("ps_flavor", _P(C.c_int8)), ("ps_count", _P(C.c_int32)), ("cq_usage", _P(C.c_int64)),
        ("trace_wl", _P(C.c_int32)), ("trace_decision", _P(C.c_uint8)), ("trace_capacity", C.c_int64),
        ("gpu_ms", C.c_double),
    ]


class kb_tas_topology(C.Structure):
    _fields_ = [
        ("n_levels", C.c_int32), ("n_domains", C.c_int32), ("n_resource", C.c_int32), ("pods_resource", C.c_int32),
        ("level_start", _P(C.c_int32)), ("parent", _P(C.c_int32)),
        ("free_capacity", _P(C.c_int64)), ("cap_mask", _P(C.c_uint32)), ("tas_usage", _P(C.c_int64)), ("usage_mask", _P(C.c_uint32)),
    ]


class kb_tas_requests(C.Structure):
    _fields_ = [
        ("n_req", C.c_int32), ("chain", _P(C.c_int32)), ("pod_request", _P(C.c_int64)), ("request_mask", _P(C.c_uint32)),
        ("count", _P(C.c_int32)), ("slice_size", _P(C.c_int32)), ("level", _P(C.c_int32)), ("slice_level", _P(C.c_int32)),
        ("flags", _P(C.c_uint32)), ("leaf_ok", _P(C.c_uint32)),
    ]


class kb_tas_out(C.Structure):
    _fields_ = [
        ("status", _P(C.c_int32)), ("asg_start", _P(C.c_int32)), ("asg_leaf", _P(C.c_int32)), ("asg_count", _P(C.c_int32)),
        ("capacity", C.c_int32), ("n_assigned", C.c_int32),
    ]


TAS_REQUIRED, TAS_UNCONSTRAINED, TAS_SIMULATE_EMPTY, TAS_PROFILE_MIXED = 1, 2, 4, 8
TAS_OK, TAS_NO_FIT, TAS_BAD_REQUEST = 0, 1, 2


class kb_config(C.Structure):
    _fields_ = [("device", C.c_int32), ("reserved", C.c_int32)]


_DT = {
    "parent": np.int32, "fair_weight": np.float64, "nominal": np.int64, "borrow_limit": np.int64,
    "lend_limit": np.int64, "cq_usage": np.int64,
    "cq_within_cq": np.uint8, "cq_reclaim_within": np.uint8, "cq_borrow_within": np.uint8,
    "cq_has_bwc_threshold": np.uint8, "cq_bwc_threshold": np.int32, "cq_when_can_borrow": np.uint8,
    "cq_when_can_preempt": np.uint8, "cq_preference": np.uint8, "cq_strategy": np.uint8, "cq_generation": np.int64,
    "cq_rg_start": np.int32, "rg_res_mask": np.uint32, "rg_flavor_start": np.int32, "rg_flavors": np.int32,
    "wl_cq": np.int32, "wl_priority": np.int32, "wl_ts": np.int64, "wl_uid": np.int64, "wl_last_gen": np.int64,
    "wl_ps_start": np.int32, "ps_req": np.int64, "ps_req_mask": np.uint32, "ps_count": np.int32,
    "ps_min_count": np.int32, "ps_flavor_ok": np.uint64, "ps_last_tried": np.int8,
    "adm_cq": np.int32, "adm_priority": np.int32, "adm_ts": np.int64, "adm_qr_ts": np.int64, "adm_uid": np.int64,
    "adm_evicted": np.uint8, "adm_use_start": np.int32, "adm_use_fr": np.int32, "adm_use_qty": np.int64,
    "heads": np.int32,
    "wl_has_quota_reservation": np.uint8, "wl_sched_hash": np.int64, "ps_group": np.int32,
    "usage_delta_cq": np.int32, "usage_delta_rows": np.int64,
}
OPTIONAL_FIELDS = ("wl_has_quota_reservation", "wl_sched_hash", "ps_group", "usage_delta_cq", "usage_delta_rows")  # NULL in kb_snapshot when absent
ARRAY_FIELDS = list(_DT.keys())
# tables the library keeps resident while kb_snapshot.static_generation is unchanged (include/kueue_b200.h)
STATIC_FIELDS = ("parent", "fair_weight", "nominal", "borrow_limit", "lend_limit", "cq_within_cq", "cq_reclaim_within",
                 "cq_borrow_within", "cq_has_bwc_threshold", "cq_bwc_threshold", "cq_when_can_borrow", "cq_when_can_preempt",
                 "cq_preference", "cq_strategy", "cq_generation", "cq_rg_start", "rg_res_mask", "rg_flavor_start", "rg_flavors")


def _ptr(arr: np.ndarray, ctype):
    return arr.ctypes.data_as(_P(ctype))


_CT = {np.int32: C.c_int32, np.int64: C.c_int64, np.uint8: C.c_uint8, np.uint32: C.c_uint32,
       np.uint64: C.c_uint64, np.int8: C.c_int8, np.float64: C.c_double}


@dataclass
class FlatSnapshot:
    """SoA buffers of one snapshot.  Arrays are C-contiguous numpy arrays."""
    n_cq: int = 0
    n_cohort: int = 0
    n_flavor: int = 1
    n_resource: int = 1
    pods_resource: int = -1
    flags: int = FLAGS_DEFAULT
    now_ns: int = 0
    static_generation: int = 0
    arrays: dict = field(default_factory=dict)

    def __getattr__(self, name):
        arrays = self.__dict__.get("arrays", {})
        if name in arrays:
            return arrays[name]
        raise AttributeError(name)

    def set(self, name: str, value) -> None:
        self.arrays[name] = np.ascontiguousarray(value, dtype=_DT[name])
        self.__dict__["_struct"] = None

    @property
    def n_nodes(self) -> int:
        return self.n_cq + self.n_cohort

    @property
    def n_fr(self) -> int:
        return self.n_flavor * self.n_resource

    def finalize(self) -> "FlatSnapshot":
        """Fill absent optional tables with empty/default arrays and validate shapes."""
        N, Q, FR, R = self.n_nodes, self.n_cq, self.n_fr, self.n_resource
        a = self.arrays
        def default(name, val):
            if name not in a:
                self.set(name, val)
        default("parent", np.full(N, -1))
        default("fair_weight", np.ones(N))
        default("nominal", np.zeros((N, FR)))
        default("borrow_limit", np.full((N, FR), KB_NO_LIMIT))
        default("lend_limit", np.full((N, FR), KB_NO_LIMIT))
        default("cq_usage", np.zeros((Q, FR)))
        for nm in ("cq_within_cq", "cq_reclaim_within", "cq_borrow_within", "cq_has_bwc_threshold", "cq_bwc_threshold",
                   "cq_when_can_borrow", "cq_preference", "cq_strategy", "cq_generation"):
            default(nm, np.zeros(Q))
        default("cq_when_can_preempt", np.full(Q, FUNG_TRY_NEXT_FLAVOR))
        default("cq_rg_start", np.zeros(Q + 1))
        default("rg_res_mask", np.zeros(0))
        default("rg_flavor_start", np.zeros(len(a["rg_res_mask"]) + 1))
        default("rg_flavors", np.zeros(0))
        W = len(a["wl_cq"]) if "wl_cq" in a else 0
        default("wl_cq", np.zeros(0))
        default("wl_priority", np.zeros(W))
        default("wl_ts", np.arange(W))
        default("wl_uid", np.arange(W))
        default("wl_last_gen", np.full(W, -1))
        default("wl_ps_start", np.arange(W + 1))
        P = int(a["wl_ps_start"][-1]) if W else 0
        default("ps_req", np.zeros((P, R)))
        default("ps_req_mask", np.zeros(P))
        default("ps_count", np.ones(P))
        default("ps_min_count", np.full(P, -1))
        default("ps_flavor_ok", np.full(P, np.iinfo(np.uint64).max, dtype=np.uint64))
        default("ps_last_tried", np.full((P, R), -1))
        A = len(a["adm_cq"]) if "adm_cq" in a else 0
        default("adm_cq", np.zeros(0))
        default("adm_priority", np.zeros(A))
        default("adm_ts", np.zeros(A))
        default("adm_qr_ts", np.full(A, KB_TS_UNSET))
        default("adm_uid", np.arange(A))
        default("adm_evicted", np.zeros(A))
        default("adm_use_start", np.zeros(A + 1))
        default("adm_use_fr", np.zeros(0))
        default("adm_use_qty", np.zeros(0))
        default("heads", np.arange(W))
        assert a["nominal"].size == N * FR and a["cq_usage"].size == Q * FR
        assert a["ps_req"].size == P * R and len(a["ps_count"]) == P
        assert R <= KB_MAX_RESOURCES and self.n_flavor <= KB_MAX_FLAVORS
        return self

    # sizes
    @property
    def n_wl(self): return len(self.arrays["wl_cq"])
    @property
    def n_podset(self): return len(self.arrays["ps_count"])
    @property
    def n_adm(self): return len(self.arrays["adm_cq"])
    @property
    def n_heads(self): return len(self.arrays["heads"])
    @property
    def n_rg(self): return len(self.arrays["rg_res_mask"])

    def head_podsets(self) -> int:
        st = self.arrays["wl_ps_start"]; h = self.arrays["heads"]
        return int((st[h + 1] - st[h]).sum()) if len(h) else 0

    def as_struct(self, cached: bool = False) -> kb_snapshot:
        """ctypes view of the snapshot.  cached=True reuses the struct built by the previous call (only the scalar
        header is refreshed) — valid while no array was replaced through set()."""
        if cached and getattr(self, "_struct", None) is not None:
            s = self._struct
            s.flags, s.now_ns, s.static_generation = self.flags, self.now_ns, self.static_generation
            return s
        s = kb_snapshot()
        s.n_cq, s.n_cohort, s.n_flavor, s.n_resource = self.n_cq, self.n_cohort, self.n_flavor, self.n_resource
        s.n_rg, s.n_wl, s.n_podset, s.n_adm = self.n_rg, self.n_wl, self.n_podset, self.n_adm
        s.n_adm_use = len(self.arrays["adm_use_fr"])
        s.n_usage_delta = len(self.arrays["usage_delta_cq"]) if "usage_delta_cq" in self.arrays else 0
        s.n_heads = self.n_heads
        s.pods_resource, s.flags, s.now_ns = self.pods_resource, self.flags, self.now_ns
        s.static_generation = self.static_generation
        for name in ARRAY_FIELDS:
            if name in OPTIONAL_FIELDS and name not in self.arrays:
                continue  # stays NULL
            arr = self.arrays[name]
            setattr(s, name, _ptr(arr, _CT[_DT[name]]))
        s._keepalive = self  # noqa: keep numpy buffers alive with the struct
        self._struct = s
        return s


class CycleOut:
    """Caller-allocated output buffers of kb_run_cycle."""

    def __init__(self, snap: FlatSnapshot, tgt_capacity: int | None = None, with_usage: bool = True):
        H, R = snap.n_heads, snap.n_resource
        HP = snap.n_podset
        cap = tgt_capacity if tgt_capacity is not None else max(16, 4 * snap.n_adm + 16)
        self.decision = np.zeros(H, np.uint8)
        self.mode = np.zeros(H, np.uint8)
        self.borrow = np.zeros(H, np.int32)
        self.commit_rank = np.full(H, -1, np.int32)
        self.ps_flavor = np.full((HP, R), -1, np.int8)
        self.ps_res_mode = np.full((HP, R), -1, np.int8)
        self.ps_tried_idx = np.full((HP, R), -1, np.int8)
        self.ps_count = np.zeros(HP, np.int32)
        self.tgt_start = np.zeros(H + 1, np.int32)
        self.tgt_adm = np.zeros(cap, np.int32)
        self.tgt_reason = np.zeros(cap, np.uint8)
        self.node_usage = np.zeros((snap.n_nodes, snap.n_fr), np.int64) if with_usage else None
        s = kb_cycle_out()
        s.decision = _ptr(self.decision, C.c_uint8); s.mode = _ptr(self.mode, C.c_uint8)
        s.borrow = _ptr(self.borrow, C.c_int32); s.commit_rank = _ptr(self.commit_rank, C.c_int32)
        s.ps_flavor = _ptr(self.ps_flavor, C.c_int8); s.ps_res_mode = _ptr(self.ps_res_mode, C.c_int8)
        s.ps_tried_idx = _ptr(self.ps_tried_idx, C.c_int8); s.ps_count = _ptr(self.ps_count, C.c_int32)
        s.tgt_start = _ptr(self.tgt_start, C.c_int32); s.tgt_adm = _ptr(self.tgt_adm, C.c_int32)
        s.tgt_reason = _ptr(self.tgt_reason, C.c_uint8)
        s.tgt_capacity = cap; s.n_targets = 0
        s.node_usage = _ptr(self.node_usage, C.c_int64) if with_usage else None
        self.struct = s

    def targets(self, entry: int):
        a, b = self.tgt_start[entry], self.tgt_start[entry + 1]
        return [(int(self.tgt_adm[k]), int(self.tgt_reason[k])) for k in range(a, b)]


class TreeOut:
    def __init__(self, snap: FlatSnapshot):
        N, Q, FR = snap.n_nodes, snap.n_cq, snap.n_fr
        self.subtree_quota = np.zeros((N, FR), np.int64)
        self.usage = np.zeros((N, FR), np.int64)
        self.available = np.zeros((Q, FR), np.int64)
        self.potential_available = np.zeros((Q, FR), np.int64)
        self.drs_rounded = np.zeros(N, np.int64)
        self.drs_resource = np.zeros(N, np.int32)
        self.drs_borrowing = np.zeros(N, np.uint8)
        s = kb_tree_out()
        s.subtree_quota = _ptr(self.subtree_quota, C.c_int64); s.usage = _ptr(self.usage, C.c_int64)
        s.available = _ptr(self.available, C.c_int64); s.potential_available = _ptr(self.potential_available, C.c_int64)
        s.drs_rounded = _ptr(self.drs_rounded, C.c_int64); s.drs_resource = _ptr(self.drs_resource, C.c_int32)
        s.drs_borrowing = _ptr(self.drs_borrowing, C.c_uint8)
        self.struct = s


class DrainOut:
    """Caller-allocated output buffers of kb_run_drain."""

    def __init__(self, snap: FlatSnapshot, max_cycles: int = 10_000, trace: bool = True):
        W, Q, R = snap.n_wl, snap.n_cq, snap.n_resource
        self.max_cycles = max_cycles
        self.cycle_heads = np.zeros(max_cycles, np.int32)
        self.cycle_admitted = np.zeros(max_cycles, np.int32)
        self.wl_admit_cycle = np.full(W, -1, np.int32)
        self.wl_last_decision = np.full(W, 0xff, np.uint8)
        self.wl_evals = np.zeros(W, np.int32)
        self.ps_flavor = np.full((snap.n_podset, R), -1, np.int8)
        self.ps_count = np.zeros(snap.n_podset, np.int32)
        self.cq_usage = np.zeros((Q, snap.n_fr), np.int64)
        cap = min(W * 4 + Q, min(Q, W) * max_cycles) if trace else 0
        self.trace_wl = np.zeros(max(1, cap), np.int32)
        self.trace_decision = np.zeros(max(1, cap), np.uint8)
        s = kb_drain_out()
        s.max_cycles = max_cycles
        s.cycle_heads = _ptr(self.cycle_heads, C.c_int32); s.cycle_admitted = _ptr(self.cycle_admitted, C.c_int32)
        s.wl_admit_cycle = _ptr(self.wl_admit_cycle, C.c_int32); s.wl_last_decision = _ptr(self.wl_last_decision, C.c_uint8)
        s.wl_evals = _ptr(self.wl_evals, C.c_int32)
        s.ps_flavor = _ptr(self.ps_flavor, C.c_int8); s.ps_count = _ptr(self.ps_count, C.c_int32)
        s.cq_usage = _ptr(self.cq_usage, C.c_int64)
        if trace:
            s.trace_wl = _ptr(self.trace_wl, C.c_int32); s.trace_decision = _ptr(self.trace_decision, C.c_uint8)
        s.trace_capacity = cap
        self.struct = s

    @property
    def n_cycles(self): return int(self.struct.n_cycles)
    @property
    def n_decisions(self): return int(self.struct.n_decisions)
    @property
    def n_admitted(self): return int(self.struct.n_admitted)
    @property
    def gpu_ms(self): return float(self.struct.gpu_ms)

    def cycles(self):
        """[(heads, decisions)] per cycle from the trace."""
        out, off = [], 0
        for c in range(self.n_cycles):
            n = int(self.cycle_heads[c])
            out.append((self.trace_wl[off:off + n].copy(), self.trace_decision[off:off + n].copy()))
            off += n
        return out
