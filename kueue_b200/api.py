"""Host-side mirror of the reference's API objects for this path.

The classes follow the fluent builders the reference's own tests use
(pkg/util/testing/v1beta2/wrappers.go: MakeClusterQueue :862, MakeFlavorQuotas
:1072, MakeCohort :810, MakeWorkload :65, MakeAdmission :667) so that parity
fixtures transcribed from pkg/scheduler/*_test.go read like the originals.
`flatten()` performs what the Go shim does after `cache.Snapshot()`:
ClusterQueueSnapshot / CohortSnapshot / workload.Info -> SoA int64 tables
(include/kueue_b200.h).
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import abi

# ---------------------------------------------------------------------------
# resource.Quantity -> int64, pkg/resources/requests.go:104-109
# ---------------------------------------------------------------------------
_SUF = {"": 1, "k": 10**3, "M": 10**6, "G": 10**9, "T": 10**12, "P": 10**15,
        "Ki": 2**10, "Mi": 2**20, "Gi": 2**30, "Ti": 2**40, "Pi": 2**50}
_QRE = re.compile(r"^([+-]?[0-9]*\.?[0-9]+)(m|k|M|G|T|P|Ki|Mi|Gi|Ti|Pi)?$")


def resource_value(name: str, q) -> int:
    """ResourceValue: milli-units for cpu, absolute units otherwise."""
    if getattr(q, "_raw_units", False):
        return int(q)
    if isinstance(q, (int, np.integer)):
        return int(q) * (1000 if name == "cpu" else 1)
    m = _QRE.match(str(q))
    if not m:
        raise ValueError(f"bad quantity {q!r}")
    from fractions import Fraction
    num = Fraction(m.group(1))
    suf = m.group(2) or ""
    val = num / 1000 if suf == "m" else num * _SUF[suf]
    if name == "cpu":
        val *= 1000
    # Quantity.Value()/MilliValue() round up
    return int(-((-val.numerator) // val.denominator))


# ---------------------------------------------------------------------------
# builders
# ---------------------------------------------------------------------------
@dataclass
class ResourceQuota:
    nominal: str
    borrowing_limit: Optional[str] = None
    lending_limit: Optional[str] = None


class MakeFlavorQuotas:
    def __init__(self, name: str):
        self.name = name
        self.resources: Dict[str, ResourceQuota] = {}

    def Resource(self, name: str, nominal="0", borrowing_limit="", lending_limit="") -> "MakeFlavorQuotas":
        self.resources[name] = ResourceQuota(nominal, borrowing_limit or None, lending_limit or None)
        return self

    def Obj(self):
        return self


class _QuotaHolder:
    def __init__(self):
        self.resource_groups: List[List[MakeFlavorQuotas]] = []

    def ResourceGroup(self, *flavors: MakeFlavorQuotas):
        self.resource_groups.append(list(flavors))
        return self


class MakeClusterQueue(_QuotaHolder):
    def __init__(self, name: str):
        super().__init__()
        self.name = name
        self.cohort: Optional[str] = None
        self.within_cluster_queue = abi.POLICY_NEVER
        self.reclaim_within_cohort = abi.POLICY_NEVER
        self.borrow_within_cohort = abi.POLICY_NEVER
        self.bwc_threshold: Optional[int] = None
        self.when_can_borrow = abi.FUNG_MAY_STOP_SEARCH
        self.when_can_preempt = abi.FUNG_TRY_NEXT_FLAVOR
        self.preference = abi.PREF_UNSET
        self.strategy = abi.QUEUE_BEST_EFFORT_FIFO
        self.fair_weight = 1.0
        self.generation = 0
        self.admission_mode: Optional[str] = None  # Spec.AdmissionScope.AdmissionMode; None = no AdmissionScope

    def Cohort(self, c: str): self.cohort = c; return self

    def AdmissionMode(self, mode: str):
        assert mode in ("UsageBasedAdmissionFairSharing", "NoAdmissionFairSharing"), mode
        self.admission_mode = mode
        return self

    def Preemption(self, withinClusterQueue="Never", reclaimWithinCohort="Never", borrowWithinCohort=None,
                   maxPriorityThreshold=None):
        pol = {"Never": abi.POLICY_NEVER, "LowerPriority": abi.POLICY_LOWER_PRIORITY,
               "LowerOrNewerEqualPriority": abi.POLICY_LOWER_OR_NEWER_EQUAL_PRIORITY, "Any": abi.POLICY_ANY}
        self.within_cluster_queue = pol[withinClusterQueue]
        self.reclaim_within_cohort = pol[reclaimWithinCohort]
        self.borrow_within_cohort = pol[borrowWithinCohort or "Never"]
        self.bwc_threshold = maxPriorityThreshold
        return self

    def FlavorFungibility(self, whenCanBorrow="MayStopSearch", whenCanPreempt="TryNextFlavor", preference=None):
        f = {"MayStopSearch": abi.FUNG_MAY_STOP_SEARCH, "TryNextFlavor": abi.FUNG_TRY_NEXT_FLAVOR,
             "Borrow": abi.FUNG_MAY_STOP_SEARCH, "Preempt": abi.FUNG_MAY_STOP_SEARCH}
        self.when_can_borrow = f[whenCanBorrow]
        self.when_can_preempt = f[whenCanPreempt]
        self.preference = {None: abi.PREF_UNSET, "BorrowingOverPreemption": abi.PREF_BORROWING_OVER_PREEMPTION,
                           "PreemptionOverBorrowing": abi.PREF_PREEMPTION_OVER_BORROWING}[preference]
        return self

    def QueueingStrategy(self, s: str):
        self.strategy = {"StrictFIFO": abi.QUEUE_STRICT_FIFO, "BestEffortFIFO": abi.QUEUE_BEST_EFFORT_FIFO}[s]
        return self

    def FairWeight(self, w): self.fair_weight = float(w); return self
    def Generation(self, g: int): self.generation = g; return self
    def Obj(self): return self


class MakeLocalQueue:
    """LocalQueue (wrappers.go MakeLocalQueue): the ClusterQueue it feeds and its Spec.FairSharing.Weight."""

    def __init__(self, name: str, ns: str = "default"):
        self.name, self.namespace = name, ns
        self.cq: Optional[str] = None
        self.weight = None  # Spec.FairSharing.Weight quantity; None = nil

    def FairSharing(self, weight=None): self.weight = weight; return self
    def ClusterQueue(self, cq: str): self.cq = cq; return self
    def Obj(self): return self


@dataclass
class AdmissionFairSharing:
    """config.AdmissionFairSharing (apis/config/v1beta2): the Configuration block that, with the feature gate on,
    makes afs.Enabled true.  Durations in seconds; resource_weights = ResourceWeights (1 for a resource not listed)."""
    usage_half_life_s: float = 0.0
    usage_sampling_s: float = 0.0
    resource_weights: Dict[str, float] = field(default_factory=dict)

    @property
    def alpha(self) -> float:
        """calculateAlphaRate(sampling, halfLife) (admission_fair_sharing.go): 1 - 0.5^(sampling/halfLife), 0 without a
        half-life."""
        if self.usage_half_life_s == 0:
            return 0.0
        return 1.0 - 0.5 ** (self.usage_sampling_s / self.usage_half_life_s)


_DEC_EXP = {"": 0, "n": -9, "u": -6, "m": -3, "k": 3, "M": 6, "G": 9, "T": 12, "P": 15, "E": 18}
_BIN_EXP = {"Ki": 10, "Mi": 20, "Gi": 30, "Ti": 40, "Pi": 50, "Ei": 60}
_PQRE = re.compile(r"^([+-]?)([0-9]*)(?:\.([0-9]*))?(Ki|Mi|Gi|Ti|Pi|Ei|[numkMGTPE]?)$")


def parse_quantity(q) -> tuple:
    """resource.MustParse(q) in the int64Amount form it keeps: (value, scale) with quantity = value * 10^scale
    (apimachinery quantity.go ParseQuantity: a decimal suffix sets the scale, the fraction digits lower it; a binary
    suffix multiplies the integer value, scale 0).  Forms that MustParse keeps as inf.Dec raise ValueError."""
    m = _PQRE.match(str(q))
    if not m or not (m.group(2) or m.group(3)):
        raise ValueError(f"bad quantity {q!r}")
    sign = -1 if m.group(1) == "-" else 1
    num, frac, suf = m.group(2) or "0", m.group(3) or "", m.group(4)
    if suf in _BIN_EXP:
        if frac:
            raise ValueError(f"{q!r}: a fractional binary quantity is not in the int64Amount form")
        v, sc = sign * (int(num) << _BIN_EXP[suf]), 0
    else:
        v, sc = sign * int(num + frac), _DEC_EXP[suf] - len(frac)
    if not -2**63 <= v < 2**63:
        raise ValueError(f"{q!r} does not fit the int64Amount form")
    return v, sc


def _flatten_afs(snap, idx, cqs, pending, local_queues, afs_config, consumed, penalties):
    """AdmissionFairSharing tables of `flatten` (include/kueue_b200.h), what the shim fills from
    qManager.AfsConsumedResources / AfsEntryPenalties and the Configuration."""
    from .drain import quantity_float
    R = snap.n_resource
    order = sorted(range(len(local_queues)), key=lambda i: idx.cqs.index(local_queues[i].cq))  # ClusterQueue-major
    lqs = [local_queues[i] for i in order]
    idx.lqs = [lq.name for lq in lqs]
    snap.set("lq_cq", [idx.cqs.index(lq.cq) for lq in lqs])
    snap.set("wl_lq", [idx.lqs.index(w.queue) for w in pending])
    on = afs_config is not None
    snap.set("cq_afs", [on and c.admission_mode == "UsageBasedAdmissionFairSharing" for c in cqs])
    snap.set("lq_weight", [1.0 if lq.weight is None else quantity_float(*parse_quantity(lq.weight)) for lq in lqs])
    val = np.zeros((len(lqs), R), np.int64); sc = np.zeros((len(lqs), R), np.int32); pen = np.zeros((len(lqs), R), np.int64)
    for i, lq in enumerate(lqs):
        for rname, q in (consumed or {}).get(lq.name, {}).items():
            val[i, idx.resources.index(rname)], sc[i, idx.resources.index(rname)] = parse_quantity(q)
        for rname, milli in (penalties or {}).get(lq.name, {}).items():
            pen[i, idx.resources.index(rname)] = milli
    snap.set("lq_consumed", val); snap.set("lq_consumed_scale", sc)
    if penalties:
        snap.set("lq_penalty", pen)
    rw = (afs_config.resource_weights if on else {})
    snap.set("afs_res_weight", [float(rw.get(r, 1.0)) for r in idx.resources])
    snap.set("afs_milli_mul", [1 if r == "cpu" else 1000 for r in idx.resources])  # MilliValue in the library's units
    snap.afs_alpha = afs_config.alpha if on else 0.0


def add_afs_decay(snap, afs_config: AdmissionFairSharing, last_update_ns, adm_lq):
    """Decay tables of an event drain (kb_snapshot.afs_half_life_ns, afs_sampling_ns, lq_last_update_ns, adm_lq;
    include/kueue_b200.h) on a snapshot that carries the AdmissionFairSharing tables.  `last_update_ns[l]`: LastUpdate of
    LocalQueue l's AfsConsumedResources entry, None where the cache has no entry yet: such a LocalQueue is initialised
    as initializeAfsIfNeeded does (localqueue_controller.go:327-353), consumed = its admitted usage (GetAdmittedUsage,
    flattened over flavors, as milli-units) and LastUpdate = now_ns.  `adm_lq[a]`: LocalQueue of admitted row a, -1
    for none.  Durations in seconds as in the Configuration."""
    a, R = snap.arrays, snap.n_resource
    L = len(a["lq_cq"])
    adm_lq = np.asarray(adm_lq, np.int64)
    assert len(last_update_ns) == L and len(adm_lq) == snap.n_adm
    adm = np.zeros((L, R), np.int64)  # admitted usage per LocalQueue in library units
    us = a["adm_use_start"]
    for row in np.flatnonzero(adm_lq >= 0):
        for k in range(int(us[row]), int(us[row + 1])):
            adm[adm_lq[row], int(a["adm_use_fr"][k]) % R] += int(a["adm_use_qty"][k])
    cons = a["lq_consumed"].reshape(L, R).copy()
    sc = a["lq_consumed_scale"].reshape(L, R).copy()
    last = np.zeros(L, np.int64)
    for l, t in enumerate(last_update_ns):
        if t is None:
            cons[l], sc[l] = adm[l] * a["afs_milli_mul"], -3
            last[l] = snap.now_ns
        else:
            last[l] = int(t)
    snap.set("lq_consumed", cons); snap.set("lq_consumed_scale", sc)
    snap.set("lq_last_update_ns", last); snap.set("adm_lq", adm_lq)
    snap.afs_half_life_ns = int(round(afs_config.usage_half_life_s * 1e9))
    snap.afs_sampling_ns = int(round(afs_config.usage_sampling_s * 1e9))
    snap.afs_alpha = afs_config.alpha
    return snap


class MakeCohort(_QuotaHolder):
    def __init__(self, name: str):
        super().__init__()
        self.name = name
        self.parent: Optional[str] = None
        self.fair_weight = 1.0

    def Parent(self, p: str): self.parent = p; return self
    def FairWeight(self, w): self.fair_weight = float(w); return self
    def Obj(self): return self


class MakeResourceFlavor:
    """kueue.ResourceFlavor: node labels, taints and tolerations (wrappers.go MakeResourceFlavor)."""

    def __init__(self, name: str):
        self.name = name
        self.node_labels: Dict[str, str] = {}
        self.taints: List[dict] = []
        self.tolerations: List[dict] = []

    def NodeLabel(self, k: str, v: str): self.node_labels[k] = v; return self
    def Taint(self, **t): self.taints.append(t); return self
    def Toleration(self, **t): self.tolerations.append(t); return self
    def Obj(self): return self

    def spec(self) -> dict:
        return {"nodeLabels": self.node_labels, "taints": self.taints, "tolerations": self.tolerations}


class MakePodSet:
    def __init__(self, name: str = "main", count: int = 1):
        self.name = name
        self.count = count
        self.min_count: Optional[int] = None
        self.requests: Dict[str, str] = {}   # PER-POD requests, like PodSpec containers
        self.flavor_ok: Optional[Sequence[str]] = None  # flavors passing taints/affinity; None = derive / all
        self.tolerations: List[dict] = []
        self.node_selector: Optional[Dict[str, str]] = None
        self.affinity_terms: Optional[List[dict]] = None
        self.group: Optional[str] = None  # TopologyRequest.PodSetGroupName

    def Request(self, res: str, q): self.requests[res] = q; return self
    def PodSetGroup(self, g: Optional[str]): self.group = g; return self
    def Toleration(self, **t): self.tolerations.append(t); return self
    def NodeSelector(self, kv: Dict[str, str]): self.node_selector = dict(kv); return self

    def RequiredDuringSchedulingIgnoredDuringExecution(self, terms: List[dict]):
        self.affinity_terms = (self.affinity_terms or []) + list(terms)
        return self

    def spec(self) -> dict:
        return {"tolerations": self.tolerations, "nodeSelector": self.node_selector, "affinityTerms": self.affinity_terms}
    def SetMinimumCount(self, m: int): self.min_count = m; return self
    def EligibleFlavors(self, *flavors: str): self.flavor_ok = list(flavors); return self
    def Obj(self): return self


class MakeAdmission:
    """kueue.Admission: per podset -> {resource: (flavor, total quantity)}."""

    def __init__(self, cq: str):
        self.cq = cq
        self.podsets: List[Dict[str, tuple]] = [{}]

    def Assignment(self, res: str, flavor: str, q):
        self.podsets[-1][res] = (flavor, q)
        return self

    def PodSet(self):
        self.podsets.append({})
        return self

    def Obj(self): return self


class MakeWorkload:
    _uid = 0

    def __init__(self, name: str, ns: str = "default"):
        self.name, self.ns = name, ns
        self.queue = ""
        self.cq: Optional[str] = None       # resolved ClusterQueue (LocalQueue -> CQ is host-side)
        self.priority = 0
        self.creation_ns = 0
        self.podsets: List[MakePodSet] = [MakePodSet("main", 1)]
        self.admission: Optional[MakeAdmission] = None
        self.quota_reserved_ns: Optional[int] = None
        self.evicted = False
        self.reclaimable: Dict[str, int] = {}
        self.conditions: Dict[str, tuple] = {}  # type -> (status, reason, lastTransitionTime ns); SetStatusCondition keeps one per type
        self.last_tried: Optional[List[Dict[str, int]]] = None
        self.last_gen = 0
        MakeWorkload._uid += 1
        self.uid = MakeWorkload._uid

    def Queue(self, q: str): self.queue = q; return self
    def ClusterQueue(self, cq: str): self.cq = cq; return self
    def Priority(self, p: int): self.priority = p; return self
    def Creation(self, t): self.creation_ns = int(t); return self
    def UID(self, u: int): self.uid = u; return self
    def Request(self, res: str, q): self.podsets[0].Request(res, q); return self
    def PodSets(self, *ps: MakePodSet): self.podsets = list(ps); return self
    def Evicted(self): self.evicted = True; return self
    def ReclaimablePods(self, counts: Dict[str, int]): self.reclaimable = dict(counts); return self  # Status.ReclaimablePods

    def Condition(self, type: str, status: bool, reason: str = "", last_transition_ns: int = 0):
        self.conditions[type] = (bool(status), reason, int(last_transition_ns))
        if type == "Evicted":
            self.evicted = bool(status)
        return self

    def ReserveQuota(self, a: MakeAdmission, at_ns: Optional[int] = None):
        self.admission = a
        self.cq = a.cq
        self.quota_reserved_ns = at_ns
        return self

    def ReserveQuotaAt(self, a: MakeAdmission, at_ns: int): return self.ReserveQuota(a, at_ns)

    def LastAssignment(self, tried: List[Dict[str, int]], generation: int = 0):
        self.last_tried, self.last_gen = tried, generation
        return self

    def Obj(self): return self


@dataclass
class Index:
    """Name <-> index maps of a flattened snapshot."""
    cqs: List[str]
    cohorts: List[str]
    flavors: List[str]
    resources: List[str]
    pending: List[str] = field(default_factory=list)
    admitted: List[str] = field(default_factory=list)
    lqs: List[str] = field(default_factory=list)  # LocalQueues in kb_snapshot order (AdmissionFairSharing)

    def node(self, name: str) -> int:
        return self.cqs.index(name) if name in self.cqs else len(self.cqs) + self.cohorts.index(name)

    def fr(self, flavor: str, res: str) -> int:
        return self.flavors.index(flavor) * len(self.resources) + self.resources.index(res)


def queue_order_timestamp(w: "MakeWorkload", pods_ready_requeuing: str = "Eviction", priority_sorting: bool = True) -> int:
    """Ordering.GetQueueOrderTimestamp (pkg/workload/workload.go:1174-1193), in ns.

    The timestamp the iterators (scheduler.go:808, fair_sharing_iterator.go:196) and the
    LowerOrNewerEqualPriority policy (preemption_policy.go:39) compare: the PodsReady-timeout eviction time when
    requeuing by eviction timestamp, the admission-check eviction time, the reclaim-while-borrowing preemption
    time + 1 ms when priority sorting within the cohort is off, else the creation time."""
    ev = w.conditions.get("Evicted")
    if ev and ev[0]:
        if pods_ready_requeuing == "Eviction" and ev[1] == "PodsReadyTimeout":
            return ev[2]
        if ev[1] == "AdmissionCheck":
            return ev[2]
    if not priority_sorting:
        pre = w.conditions.get("Preempted")
        if pre and pre[0] and pre[1] == "InCohortReclaimWhileBorrowing":
            return pre[2] + 1_000_000
    return w.creation_ns


def queue_order_key(w: "MakeWorkload", pods_ready_requeuing: str = "Eviction", priority_sorting: bool = True):
    """Sort key of queueOrderingFunc (pkg/cache/queue/cluster_queue.go:636-685): higher priority first, then the
    queue-order timestamp, then UID.  (AdmissionFairSharing usage and the sticky workload are not modelled.)"""
    return (-w.priority, queue_order_timestamp(w, pods_ready_requeuing, priority_sorting), w.uid)


def select_heads(pending: Sequence["MakeWorkload"], pods_ready_requeuing: str = "Eviction", priority_sorting: bool = True):
    """queues.Heads (manager.go:770-794): the first workload of every ClusterQueue's heap in queueOrderingFunc order.
    Returns one workload per ClusterQueue, in first-appearance order of the ClusterQueues."""
    best: Dict[str, "MakeWorkload"] = {}
    for w in pending:
        assert w.cq is not None, f"pending workload {w.name} has no ClusterQueue"
        cur = best.get(w.cq)
        if cur is None or queue_order_key(w, pods_ready_requeuing, priority_sorting) < queue_order_key(cur, pods_ready_requeuing, priority_sorting):
            best[w.cq] = w
    return list(best.values())


def flatten(cqs: Sequence[MakeClusterQueue], cohorts: Sequence[MakeCohort] = (),
            pending: Sequence[MakeWorkload] = (), admitted: Sequence[MakeWorkload] = (),
            usage: Optional[Dict[str, Dict[tuple, int]]] = None, flags: int = abi.FLAGS_DEFAULT,
            heads: Optional[Sequence[str]] = None, now_ns: int = 0,
            flavors: Optional[Sequence[str]] = None, extra_resources: Sequence[str] = (),
            resource_flavors: Optional[Sequence["MakeResourceFlavor"]] = None,
            pods_ready_requeuing: str = "Eviction", reclaimable_pods: bool = True,
            local_queues: Sequence[MakeLocalQueue] = (), afs_config: Optional[AdmissionFairSharing] = None,
            consumed: Optional[Dict[str, Dict[str, str]]] = None, penalties: Optional[Dict[str, Dict[str, int]]] = None):
    """Build (FlatSnapshot, Index).

    `usage` optionally overrides ClusterQueue usage as {cq: {(flavor, resource): int64}}
    (already in int64 units, like resources.FlavorResourceQuantities literals in the
    reference tests); otherwise usage is the sum of `admitted` workloads' admissions
    (clusterqueue.go:535-563).

    `local_queues` adds the AdmissionFairSharing tables: a pending workload's LocalQueue is its Queue() (its
    ClusterQueue defaults to the LocalQueue's); `afs_config` None = afs.Enabled false; `consumed` =
    AfsConsumedResources as {lq: {resource: quantity string}}; `penalties` = AfsEntryPenalties as {lq: {resource: milli}}.
    """
    cohorts = list(cohorts)
    lq_of = {lq.name: lq for lq in local_queues}
    for w in pending:  # the queue manager routes a workload to the ClusterQueue of its LocalQueue
        if w.cq is None and w.queue in lq_of:
            w.cq = lq_of[w.queue].cq
    known = {c.name for c in cohorts}
    # implicit cohorts (hierarchy.Manager creates them on reference, manager.go:80-100)
    for holder in list(cqs) + list(cohorts):
        par = holder.cohort if isinstance(holder, MakeClusterQueue) else holder.parent
        if par and par not in known:
            cohorts.append(MakeCohort(par)); known.add(par)
    fl: List[str] = list(flavors) if flavors else []
    res: set = set(extra_resources)
    for m in (consumed or {}).values():
        res.update(m.keys())
    for holder in list(cqs) + cohorts:
        for rg in holder.resource_groups:
            for fq in rg:
                if fq.name not in fl:
                    fl.append(fq.name)
                res.update(fq.resources.keys())
    for w in list(pending) + list(admitted):
        for ps in w.podsets:
            res.update(ps.requests.keys())
        if w.admission:
            for psa in w.admission.podsets:
                for r, (f, _) in psa.items():
                    res.add(r)
                    if f not in fl:
                        fl.append(f)
    resources = sorted(res) or ["cpu"]
    if not fl:
        fl = ["default"]
    idx = Index([c.name for c in cqs], [c.name for c in cohorts], fl, resources)
    Q, Cn, F, R = len(cqs), len(cohorts), len(fl), len(resources)
    N, FR = Q + Cn, F * R
    snap = abi.FlatSnapshot(n_cq=Q, n_cohort=Cn, n_flavor=F, n_resource=R, flags=flags, now_ns=now_ns)
    snap.pods_resource = resources.index("pods") if "pods" in resources else -1
    parent = np.full(N, -1, np.int32)
    nominal = np.zeros((N, FR), np.int64)
    bl = np.full((N, FR), abi.KB_NO_LIMIT, np.int64)
    ll = np.full((N, FR), abi.KB_NO_LIMIT, np.int64)
    fw = np.ones(N)
    cq_rg_start = [0]; rg_mask = []; rg_fl_start = [0]; rg_fl = []
    for n, holder in enumerate(list(cqs) + cohorts):
        par = holder.cohort if isinstance(holder, MakeClusterQueue) else holder.parent
        if par:
            parent[n] = len(idx.cqs) + idx.cohorts.index(par)  # a parent is always a Cohort (a ClusterQueue may share its name)
        fw[n] = holder.fair_weight
        for rg in holder.resource_groups:
            mask = 0
            for fq in rg:
                for rname, q in fq.resources.items():
                    fr = idx.fr(fq.name, rname)
                    nominal[n, fr] = resource_value(rname, q.nominal)
                    if q.borrowing_limit is not None:
                        bl[n, fr] = resource_value(rname, q.borrowing_limit)
                    if q.lending_limit is not None:
                        ll[n, fr] = resource_value(rname, q.lending_limit)
                    mask |= 1 << resources.index(rname)
            if n < Q:
                rg_mask.append(mask)
                rg_fl.extend(fl.index(fq.name) for fq in rg)
                rg_fl_start.append(len(rg_fl))
        if n < Q:
            cq_rg_start.append(len(rg_mask))
    snap.set("parent", parent); snap.set("fair_weight", fw)
    snap.set("nominal", nominal); snap.set("borrow_limit", bl); snap.set("lend_limit", ll)
    snap.set("cq_rg_start", cq_rg_start); snap.set("rg_res_mask", rg_mask)
    snap.set("rg_flavor_start", rg_fl_start); snap.set("rg_flavors", rg_fl)
    snap.set("cq_within_cq", [c.within_cluster_queue for c in cqs])
    snap.set("cq_reclaim_within", [c.reclaim_within_cohort for c in cqs])
    snap.set("cq_borrow_within", [c.borrow_within_cohort for c in cqs])
    snap.set("cq_has_bwc_threshold", [c.bwc_threshold is not None for c in cqs])
    snap.set("cq_bwc_threshold", [c.bwc_threshold or 0 for c in cqs])
    snap.set("cq_when_can_borrow", [c.when_can_borrow for c in cqs])
    snap.set("cq_when_can_preempt", [c.when_can_preempt for c in cqs])
    snap.set("cq_preference", [c.preference for c in cqs])
    snap.set("cq_strategy", [c.strategy for c in cqs])
    snap.set("cq_generation", [c.generation for c in cqs])

    # admitted workloads
    cq_usage = np.zeros((Q, FR), np.int64)
    a_cq, a_pr, a_ts, a_qr, a_uid, a_ev, a_st, a_fr, a_q = [], [], [], [], [], [], [0], [], []
    for w in admitted:
        assert w.admission is not None, f"admitted workload {w.name} lacks an Admission"
        cqi = idx.cqs.index(w.admission.cq)
        a_cq.append(cqi); a_pr.append(w.priority); a_ts.append(w.creation_ns)
        a_qr.append(abi.KB_TS_UNSET if w.quota_reserved_ns is None else w.quota_reserved_ns)
        a_uid.append(w.uid); a_ev.append(w.evicted)
        acc: Dict[int, int] = {}
        for psa in w.admission.podsets:
            for r, (f, q) in psa.items():
                fr = idx.fr(f, r)
                acc[fr] = acc.get(fr, 0) + resource_value(r, q)
        for fr, q in acc.items():
            a_fr.append(fr); a_q.append(q); cq_usage[cqi, fr] += q
        a_st.append(len(a_fr))
        idx.admitted.append(w.name)
    if usage is not None:
        cq_usage[:] = 0
        for cqname, m in usage.items():
            for (f, r), v in m.items():
                cq_usage[idx.cqs.index(cqname), idx.fr(f, r)] = v
    snap.set("cq_usage", cq_usage)
    snap.set("adm_cq", a_cq); snap.set("adm_priority", a_pr); snap.set("adm_ts", a_ts); snap.set("adm_qr_ts", a_qr)
    snap.set("adm_uid", a_uid); snap.set("adm_evicted", a_ev); snap.set("adm_use_start", a_st)
    snap.set("adm_use_fr", a_fr); snap.set("adm_use_qty", a_q)

    # pending workloads
    w_cq, w_pr, w_ts, w_uid, w_lg, w_st = [], [], [], [], [], [0]
    p_req, p_mask, p_cnt, p_min, p_ok, p_lt, p_grp = [], [], [], [], [], [], []
    for w in pending:
        assert w.cq is not None, f"pending workload {w.name} has no ClusterQueue"
        w_cq.append(idx.cqs.index(w.cq)); w_pr.append(w.priority); w_uid.append(w.uid)
        w_ts.append(queue_order_timestamp(w, pods_ready_requeuing, bool(flags & abi.F_PRIORITY_SORTING_WITHIN_COHORT)))
        w_lg.append(w.last_gen if w.last_tried is not None else -1)
        for pi, ps in enumerate(w.podsets):
            row = np.zeros(R, np.int64); mask = 0
            count = ps.count
            if reclaimable_pods:  # podSetsCountsAfterReclaim workload.go:547-559 (feature gate ReclaimablePods, on by default)
                count -= getattr(w, "reclaimable", {}).get(ps.name, 0)
            for rname, q in ps.requests.items():
                r = resources.index(rname)
                row[r] = resource_value(rname, q) * count  # totalRequestsFromPodSets workload.go:567-598
                mask |= 1 << r
            p_req.append(row); p_mask.append(mask); p_cnt.append(count)
            groups = [g.group for g in w.podsets if g.group is not None]
            p_grp.append(-1 if ps.group is None else sorted(set(groups)).index(ps.group))  # groupKey flavorassigner.go:613-616
            p_min.append(-1 if ps.min_count is None else ps.min_count)
            ok = (1 << 64) - 1
            if ps.flavor_ok is not None:
                ok = 0
                for f in ps.flavor_ok:
                    ok |= 1 << fl.index(f)
            elif resource_flavors is not None:
                # checkFlavorForPodSets (flavorassigner.go:899-944) evaluated on the host per (podset, flavor)
                from .eligibility import flavor_eligible
                rf = {f.name: f for f in resource_flavors}
                ok = 0
                cq_obj = cqs[idx.cqs.index(w.cq)]
                for rg in cq_obj.resource_groups:
                    keys = set()
                    for fq in rg:
                        if fq.name in rf:
                            keys.update(rf[fq.name].node_labels.keys())  # ResourceGroup.LabelKeys resource.go:31-38
                    for fq in rg:
                        if fq.name in rf and flavor_eligible(ps.spec(), rf[fq.name].spec(), keys):
                            ok |= 1 << fl.index(fq.name)
            p_ok.append(ok)
            lt = np.full(R, -1, np.int8)
            if w.last_tried is not None and pi < len(w.last_tried):
                for rname, v in w.last_tried[pi].items():
                    lt[resources.index(rname)] = v
            p_lt.append(lt)
        w_st.append(len(p_cnt))
        idx.pending.append(w.name)
    snap.set("wl_cq", w_cq); snap.set("wl_priority", w_pr); snap.set("wl_ts", w_ts); snap.set("wl_uid", w_uid)
    snap.set("wl_last_gen", w_lg); snap.set("wl_ps_start", w_st)
    snap.set("ps_req", np.array(p_req, np.int64).reshape(len(p_cnt), R)); snap.set("ps_req_mask", p_mask)
    snap.set("ps_count", p_cnt); snap.set("ps_min_count", p_min)
    snap.set("ps_flavor_ok", np.array(p_ok, dtype=np.uint64)); snap.set("ps_last_tried", np.array(p_lt, np.int8).reshape(len(p_cnt), R))
    if any(g >= 0 for g in p_grp):
        snap.set("ps_group", np.array(p_grp, np.int32))
    if heads is None:
        snap.set("heads", np.arange(len(w_cq)))
    else:
        snap.set("heads", [idx.pending.index(h) for h in heads])
    if local_queues:
        _flatten_afs(snap, idx, cqs, pending, list(local_queues), afs_config, consumed, penalties)
    snap.finalize()
    return snap, idx


class UsageTracker:
    """Host side of the incremental snapshot (SURVEY f2, `kb_snapshot.usage_delta_*`): what a scheduler cache that
    maintains the flat usage table does between two cycles.  The reference cache changes a ClusterQueue's usage only in
    `AddOrUpdateWorkload` / `DeleteWorkload` / `AssumeWorkload` / `ForgetWorkload` (pkg/cache/scheduler/cache.go:619-711
    -> clusterqueue.go addOrUpdateWorkload / deleteWorkload -> updateWorkloadUsage); each of them calls `touch(cq)` here.
    `prepare(snap)` then turns the next snapshot into its cheapest valid form: the full table (first call, or after the
    static tables changed) tagged KB_F_USAGE_RESIDENT, or only the touched rows."""

    def __init__(self):
        self._gen = None       # static_generation the device-resident table belongs to
        self._dims = None
        self._dirty: set[int] = set()
        self._last = None      # host copy of what the device holds (to make `touch` optional: rows are also diffed)

    def touch(self, cq_index: int) -> None:
        self._dirty.add(int(cq_index))

    def reset(self) -> None:
        """After any library error (the shim falls back to the stock cycle and the resident table is unknown)."""
        self._gen = None; self._dirty.clear(); self._last = None

    def prepare(self, snap: "abi.FlatSnapshot", diff: bool = True) -> "abi.FlatSnapshot":
        import numpy as np
        Q, FR = snap.n_cq, snap.n_fr
        usage = np.asarray(snap.arrays["cq_usage"], dtype=np.int64).reshape(Q, FR)
        dims = (Q, snap.n_cohort, snap.n_flavor, snap.n_resource)
        fresh = snap.static_generation == 0 or self._gen != snap.static_generation or self._dims != dims or self._last is None
        if fresh:
            snap.arrays.pop("usage_delta_cq", None); snap.arrays.pop("usage_delta_rows", None)
            snap.__dict__["_struct"] = None
            if snap.static_generation != 0:  # the library keeps a usage table only next to resident static tables
                snap.flags |= abi.F_USAGE_RESIDENT
                self._gen, self._dims, self._last = snap.static_generation, dims, usage.copy()
            else:
                snap.flags &= ~abi.F_USAGE_RESIDENT
                self._gen = None
            self._dirty.clear()
            return snap
        rows = set(self._dirty)
        if diff:  # rows the caller forgot to touch would silently go stale on the device: diff against the mirror
            rows |= set(np.flatnonzero((usage != self._last).any(axis=1)).tolist())
        idx = np.array(sorted(rows), dtype=np.int32)
        snap.set("usage_delta_cq", idx)
        snap.set("usage_delta_rows", usage[idx] if len(idx) else np.zeros((0, FR), np.int64))
        snap.flags &= ~abi.F_USAGE_RESIDENT
        self._last[idx] = usage[idx]
        self._dirty.clear()
        return snap
