"""Host side of topology-aware scheduling (kb_tas_find, include/kueue_b200.h): flattens one TAS ResourceFlavor the way
TASFlavorCache.snapshot does (pkg/cache/scheduler/tas_flavor.go:118-160, tas_flavor_snapshot.go:153-241) and resolves a
podset's TopologyRequest to the numeric request the device takes (tas_flavor_snapshot.go:789-830,1059-1147).

Nodes: dicts {name, labels, allocatable{res: int64 units}, taints[], ready, unschedulable}.  Only Ready, schedulable
nodes that carry the flavor's nodeLabels and every topology level label become leaves (tas_nodes_cache / SyncNode).
Domains are numbered level-major, inside a level in lexicographic order of their levelValues."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import numpy as np

from . import abi, eligibility

HOSTNAME = "kubernetes.io/hostname"


class TasTopology:
    def __init__(self, levels: List[str], nodes: List[dict], node_labels: Optional[Dict[str, str]] = None,
                 resources: Optional[List[str]] = None, non_tas_usage: Optional[Dict[str, Dict[str, int]]] = None,
                 tas_usage: Optional[Dict[str, Dict[str, int]]] = None):
        self.levels = list(levels)
        L = len(levels)
        node_labels = node_labels or {}
        leaves = {}  # levelValues tuple -> accumulated leaf (several nodes can share a leaf when the lowest level is not the hostname)
        for n in nodes:
            lab = n.get("labels", {})
            if not n.get("ready", True) or n.get("unschedulable", False):
                continue
            if any(lab.get(k) != v for k, v in node_labels.items()) or any(k not in lab for k in levels):
                continue
            vals = tuple(lab[k] for k in levels)
            leaf = leaves.setdefault(vals, {"values": vals, "free": {}, "nodes": []})
            for r, q in n.get("allocatable", {}).items():
                leaf["free"][r] = leaf["free"].get(r, 0) + int(q)  # addCapacity :243-248
            leaf["nodes"].append(n)
        res = set(resources or [])
        for lf in leaves.values():
            res.update(lf["free"])
        for u in list((non_tas_usage or {}).values()) + list((tas_usage or {}).values()):
            res.update(u)
        res.add("pods")
        self.resources = sorted(res)
        R = len(self.resources)
        self.pods_resource = self.resources.index("pods")
        # domains per level, lexicographic
        per_level = [sorted({lf["values"][:l + 1] for lf in leaves.values()}) for l in range(L)]
        self.level_start = np.zeros(L + 1, np.int32)
        for l in range(L):
            self.level_start[l + 1] = self.level_start[l] + len(per_level[l])
        index = {}
        for l in range(L):
            for i, v in enumerate(per_level[l]):
                index[v] = int(self.level_start[l]) + i
        nd = int(self.level_start[L])
        self.parent = np.full(max(1, nd), -1, np.int32)
        for l in range(1, L):
            for v in per_level[l]:
                self.parent[index[v]] = index[v[:-1]]
        self.leaf_values = per_level[L - 1] if L else []
        nleaf = len(self.leaf_values)
        self.n_leaves = nleaf
        self.free = np.zeros((max(1, nleaf), R), np.int64)
        self.cap_mask = np.zeros(max(1, nleaf), np.uint32)
        self.usage = np.zeros((max(1, nleaf), R), np.int64)
        self.usage_mask = np.zeros(max(1, nleaf), np.uint32)
        self.leaf_nodes = []
        by_name = {}
        for i, v in enumerate(self.leaf_values):
            lf = leaves[v]
            self.leaf_nodes.append(lf["nodes"])
            for n in lf["nodes"]:
                by_name[n["name"]] = i
            for r, q in lf["free"].items():
                self.free[i, self.resources.index(r)] = q
                self.cap_mask[i] |= np.uint32(1 << self.resources.index(r))
        for name, u in (non_tas_usage or {}).items():  # addNonTASUsage :250-255: freeCapacity.Sub(usage)
            if name in by_name:
                i = by_name[name]
                for r, q in u.items():
                    self.free[i, self.resources.index(r)] -= int(q)
                    self.cap_mask[i] |= np.uint32(1 << self.resources.index(r))
        for name, u in (tas_usage or {}).items():       # addTASUsage :267-279 (usage already includes pods)
            if name in by_name:
                i = by_name[name]
                for r, q in u.items():
                    self.usage[i, self.resources.index(r)] += int(q)
                    self.usage_mask[i] |= np.uint32(1 << self.resources.index(r))
        self.lowest_is_node = bool(levels) and levels[-1] == HOSTNAME
        s = abi.kb_tas_topology()
        s.n_levels, s.n_domains, s.n_resource, s.pods_resource = L, nd, R, self.pods_resource
        P = C.POINTER
        s.level_start = self.level_start.ctypes.data_as(P(C.c_int32)); s.parent = self.parent.ctypes.data_as(P(C.c_int32))
        s.free_capacity = self.free.ctypes.data_as(P(C.c_int64)); s.cap_mask = self.cap_mask.ctypes.data_as(P(C.c_uint32))
        s.tas_usage = self.usage.ctypes.data_as(P(C.c_int64)); s.usage_mask = self.usage_mask.ctypes.data_as(P(C.c_uint32))
        self.struct = s

    def level_index(self, key: str) -> int:
        return self.levels.index(key) if key in self.levels else -1


class TasRequests:
    """SoA batch of podset requests.  add() resolves a kueue.PodSetTopologyRequest like findTopologyAssignment does."""

    def __init__(self, topo: TasTopology):
        self.topo = topo
        self.rows = []

    def add(self, chain: int, requests: Dict[str, int], count: int, topology_request: Optional[dict] = None, implied: Optional[bool] = None,
            tolerations: Optional[List[dict]] = None, node_selector: Optional[Dict[str, str]] = None, flavor_tolerations: Optional[List[dict]] = None,
            simulate_empty: bool = False, profile_mixed: bool = True):
        t = self.topo
        tr = topology_request
        implied = (tr is None) if implied is None else implied
        slice_only = tr is not None and tr.get("required") is None and tr.get("preferred") is None and tr.get("sliceRequiredTopology") is not None
        # levelKeyWithImpliedFallback :1079-1105
        key = None
        if tr is not None:
            if tr.get("required") is not None: key = tr["required"]
            elif tr.get("preferred") is not None: key = tr["preferred"]
            elif slice_only: key = t.levels[0]
            elif tr.get("unconstrained"): key = t.levels[-1]
        if key is None and implied:
            key = t.levels[-1]
        slice_key = tr["sliceRequiredTopology"] if tr is not None and tr.get("sliceRequiredTopology") is not None else t.levels[-1]
        slice_size = 1
        if tr is not None and tr.get("sliceRequiredTopology") is not None:
            slice_size = tr.get("sliceSize") or 0  # "slice topology requested, but slice size not provided"
        flags = 0
        if tr is not None and tr.get("required") is not None: flags |= abi.TAS_REQUIRED
        if (tr is not None and tr.get("unconstrained")) or implied or slice_only: flags |= abi.TAS_UNCONSTRAINED
        if simulate_empty: flags |= abi.TAS_SIMULATE_EMPTY
        if profile_mixed: flags |= abi.TAS_PROFILE_MIXED
        ok = None
        if t.lowest_is_node and (tolerations is not None or node_selector or flavor_tolerations or any(n.get("taints") for ns in t.leaf_nodes for n in ns)):
            tol = list(tolerations or []) + list(flavor_tolerations or [])
            ok = np.zeros((t.n_leaves + 31) // 32, np.uint32)
            for i, ns in enumerate(t.leaf_nodes):
                n = ns[0]
                if eligibility.untolerated_taint(n.get("taints", []), tol) is not None:  # fillInCounts :1541-1551
                    continue
                if node_selector and any(n.get("labels", {}).get(k) != v for k, v in node_selector.items()):  # :1553-1563
                    continue
                ok[i // 32] |= np.uint32(1 << (i % 32))
        self.rows.append(dict(chain=chain, requests={r: int(q) for r, q in requests.items() if r != "pods"}, count=count, slice_size=slice_size,
                              level=-1 if key is None else t.level_index(key), slice_level=t.level_index(slice_key), flags=flags, ok=ok))
        return self

    def finalize(self):
        t = self.topo
        n, R = len(self.rows), len(t.resources)
        W = (t.n_leaves + 31) // 32
        self.chain = np.array([r["chain"] for r in self.rows], np.int32)
        self.pod_request = np.zeros((max(1, n), R), np.int64)
        self.request_mask = np.zeros(max(1, n), np.uint32)
        for i, r in enumerate(self.rows):
            for res, q in r["requests"].items():
                if res not in t.resources:
                    raise KeyError(f"resource {res} unknown to the topology (pass resources=[...] to TasTopology)")
                self.pod_request[i, t.resources.index(res)] = q
                self.request_mask[i] |= np.uint32(1 << t.resources.index(res))
        self.count = np.array([r["count"] for r in self.rows], np.int32)
        self.slice_size = np.array([r["slice_size"] for r in self.rows], np.int32)
        self.level = np.array([r["level"] for r in self.rows], np.int32)
        self.slice_level = np.array([r["slice_level"] for r in self.rows], np.int32)
        self.flags = np.array([r["flags"] for r in self.rows], np.uint32)
        any_ok = any(r["ok"] is not None for r in self.rows)
        self.leaf_ok = None
        if any_ok:
            self.leaf_ok = np.full((n, max(1, W)), 0xffffffff, np.uint32)
            for i, r in enumerate(self.rows):
                if r["ok"] is not None:
                    self.leaf_ok[i, :W] = r["ok"]
        s = abi.kb_tas_requests()
        P = C.POINTER
        s.n_req = n
        s.chain = self.chain.ctypes.data_as(P(C.c_int32)); s.pod_request = self.pod_request.ctypes.data_as(P(C.c_int64))
        s.request_mask = self.request_mask.ctypes.data_as(P(C.c_uint32)); s.count = self.count.ctypes.data_as(P(C.c_int32))
        s.slice_size = self.slice_size.ctypes.data_as(P(C.c_int32)); s.level = self.level.ctypes.data_as(P(C.c_int32))
        s.slice_level = self.slice_level.ctypes.data_as(P(C.c_int32)); s.flags = self.flags.ctypes.data_as(P(C.c_uint32))
        if self.leaf_ok is not None:
            s.leaf_ok = self.leaf_ok.ctypes.data_as(P(C.c_uint32))
        self.struct = s
        return self


class TasOut:
    def __init__(self, reqs: TasRequests, capacity: int):
        n = len(reqs.rows)
        self.status = np.full(max(1, n), -2, np.int32)
        self.asg_start = np.zeros(n + 1, np.int32)
        self.asg_leaf = np.zeros(max(1, capacity), np.int32)
        self.asg_count = np.zeros(max(1, capacity), np.int32)
        s = abi.kb_tas_out()
        P = C.POINTER
        s.status = self.status.ctypes.data_as(P(C.c_int32)); s.asg_start = self.asg_start.ctypes.data_as(P(C.c_int32))
        s.asg_leaf = self.asg_leaf.ctypes.data_as(P(C.c_int32)); s.asg_count = self.asg_count.ctypes.data_as(P(C.c_int32))
        s.capacity = capacity; s.n_assigned = 0
        self.struct = s

    def assignment(self, q: int):
        a, b = int(self.asg_start[q]), int(self.asg_start[q + 1])
        return [(int(self.asg_leaf[k]), int(self.asg_count[k])) for k in range(a, b)]


def synth_topology(blocks: int = 10, racks: int = 100, hosts: int = 100, seed: int = 5, used: float = 0.5):
    """cfg5-style synthetic topology (BASELINE.json configs[4]): blocks x racks x hosts, node capacity like
    test/performance/scheduler/configs/tas/generator.yaml:12-24 (96 cpu, 256 Gi, 8 gpu, 110 pods); a fraction of every
    node already used by TAS workloads.  Built directly in flat form (no per-node dicts)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    t = object.__new__(TasTopology)
    t.levels = ["cloud.com/topology-block", "cloud.com/topology-rack", HOSTNAME]
    t.resources = ["cpu", "gpu", "memory", "pods"]
    t.pods_resource = 3
    nb, nr, nh = blocks, blocks * racks, blocks * racks * hosts
    t.level_start = np.array([0, nb, nb + nr, nb + nr + nh], np.int32)
    t.parent = np.concatenate([np.full(nb, -1), np.repeat(np.arange(nb), racks), nb + np.repeat(np.arange(nr), hosts)]).astype(np.int32)
    t.n_leaves = nh
    t.leaf_values = None
    cap = np.array([96_000, 8, 256 << 30, 110], np.int64)
    t.free = np.tile(cap, (nh, 1))
    t.cap_mask = np.full(nh, 0xf, np.uint32)
    frac = rng.uniform(0, 2 * used, (nh, 1)).clip(0, 1)
    t.usage = (t.free * frac * rng.uniform(0.7, 1.0, (nh, 4))).astype(np.int64)
    t.usage_mask = np.full(nh, 0xf, np.uint32)
    t.leaf_nodes = []
    t.lowest_is_node = True
    s = abi.kb_tas_topology()
    s.n_levels, s.n_domains, s.n_resource, s.pods_resource = 3, int(t.level_start[3]), 4, 3
    P = C.POINTER
    s.level_start = t.level_start.ctypes.data_as(P(C.c_int32)); s.parent = t.parent.ctypes.data_as(P(C.c_int32))
    s.free_capacity = t.free.ctypes.data_as(P(C.c_int64)); s.cap_mask = t.cap_mask.ctypes.data_as(P(C.c_uint32))
    s.tas_usage = t.usage.ctypes.data_as(P(C.c_int64)); s.usage_mask = t.usage_mask.ctypes.data_as(P(C.c_uint32))
    t.struct = s
    return t


def synth_requests(topo: TasTopology, n: int, seed: int = 7, shapes: int = 16, chains: bool = False, max_pods: int = 64,
                   profile_mixed: Optional[bool] = True) -> TasRequests:
    """n podset requests: `shapes` distinct pod templates, 1..max_pods pods, required / preferred at rack or block level or
    unconstrained; with chains=True some workloads carry two or three podsets.  profile_mixed=None draws the TASProfileMixed
    flag per request, so unconstrained requests run in both LeastFreeCapacity and BestFit order."""
    rng = np.random.Generator(np.random.PCG64(seed))
    tmpl = [{"cpu": int(rng.integers(1, 33)) * 1000, "memory": int(rng.integers(1, 65)) << 30, **({"gpu": int(rng.integers(1, 5))} if rng.random() < 0.5 else {})}
            for _ in range(shapes)]
    reqs = TasRequests(topo)
    chain, left = 0, 0
    for i in range(n):
        if left == 0:
            chain += 1
            left = int(rng.integers(1, 4)) if chains and rng.random() < 0.3 else 1
        left -= 1
        mode = rng.integers(0, 5)
        lvl = topo.levels[int(rng.integers(0, len(topo.levels)))]
        tr = ({"required": lvl}, {"preferred": lvl}, {"unconstrained": True}, None, {"required": topo.levels[1], "sliceRequiredTopology": topo.levels[-1], "sliceSize": 2})[mode]
        count = int(rng.integers(1, max_pods + 1))
        if mode == 4:
            count += count % 2
        mixed = bool(rng.integers(0, 2)) if profile_mixed is None else profile_mixed
        reqs.add(chain, tmpl[int(rng.integers(0, shapes))], count, None if tr is None else {"required": None, "preferred": None, "unconstrained": False, "sliceRequiredTopology": None, "sliceSize": None, **tr},
                 profile_mixed=mixed)
    return reqs.finalize()
