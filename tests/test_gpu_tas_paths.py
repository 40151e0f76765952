"""kb_tas_find on the placement branches the reference cases and the uniform synthetic topologies do not reach: the
sorted-candidate cache of large level sets, BestFit next to LeastFreeCapacity, slices above the leaves, node eligibility
and simulate-empty, 1- / 2- / 5-level and ragged topologies, over-used leaves, status paths and the full cfg5 topology.

Every fixture is built from seeds in this file.  The device must equal the oracle exactly (status, asg_start, leaves,
counts); every output also passes invariants that do not depend on the oracle; and every fixture states which branches
it reaches, computed from the oracle's output (tests/test_tas_paths_fixtures.py, which needs no GPU).

On an NVIDIA H100 80GB HBM3 at a 400 W power limit this file and the fixture check run in about 15 s together, the
oracle included.  They catch a wrong cache or a wrong order: with every cache fill treated as complete
(s_cmeta[5] = 1 in TasSel::next_cached) the five fixtures that walk a cached set past one fill fail (both cache walks,
ragged, the over-used cache walk, cfg5); with LeastFreeCapacity forced in tas_select_one all 15 fixtures with BestFit
placements over several domains fail."""
import ctypes as C
import functools

import numpy as np
import pytest

import oracle
from kueue_b200 import abi, tas

pytestmark = pytest.mark.gpu

CACHE_KEYS = 128 * 4   # KB_TAS_THREADS * KB_TAS_LOCAL: keys one fill of the sorted-candidate cache holds
CACHE_MIN = 2048       # KB_TAS_CACHE_MIN: larger contiguous level sets are walked through the cache
CTA = 128              # KB_TAS_THREADS
NODE_CAP = np.array([96_000, 8, 256 << 30, 110], np.int64)  # cpu, gpu, memory, pods (as tas.synth_topology)


# ---------------------------------------------------------------------------------------------------------------------
# builders
# ---------------------------------------------------------------------------------------------------------------------
def _flat(levels, fanout, seed, used=0.5, over=0.0):
    """Topology in flat form: fanout[0] roots, then per level an int (uniform), a (lo, hi) range drawn per parent or an
    explicit list of child counts.  Usage like tas.synth_topology; a seeded fraction `over` of the leaves is used at
    130 % of its cpu and pods, so CountIn gives those leaves negative counts."""
    rng = np.random.Generator(np.random.PCG64(seed))
    sizes, parents, start = [fanout[0]], [np.full(fanout[0], -1)], 0
    for f in fanout[1:]:
        n_par = sizes[-1]
        k = np.full(n_par, f) if isinstance(f, int) else rng.integers(f[0], f[1] + 1, n_par) if isinstance(f, tuple) else np.asarray(f)
        assert len(k) == n_par and (k >= 1).all()
        parents.append(start + np.repeat(np.arange(n_par), k))
        start += n_par
        sizes.append(int(k.sum()))
    t = object.__new__(tas.TasTopology)
    L = len(levels)
    t.levels = list(levels)
    t.resources = ["cpu", "gpu", "memory", "pods"]
    t.pods_resource = 3
    t.level_start = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    t.parent = np.concatenate(parents).astype(np.int32)
    nh = sizes[-1]
    t.n_leaves, t.leaf_values, t.leaf_nodes = nh, None, []
    t.free = np.tile(NODE_CAP, (nh, 1))
    t.cap_mask = np.full(nh, 0xf, np.uint32)
    frac = rng.uniform(0, 2 * used, (nh, 1)).clip(0, 1)
    t.usage = (t.free * frac * rng.uniform(0.7, 1.0, (nh, 4))).astype(np.int64)
    hot = rng.random(nh) < over
    t.usage[hot, 0] = NODE_CAP[0] * 13 // 10
    t.usage[hot, 3] = NODE_CAP[3] * 13 // 10
    t.usage_mask = np.full(nh, 0xf, np.uint32)
    t.lowest_is_node = levels[-1] == tas.HOSTNAME
    s = abi.kb_tas_topology()
    s.n_levels, s.n_domains, s.n_resource, s.pods_resource = L, int(t.level_start[L]), 4, 3
    P = C.POINTER
    s.level_start = t.level_start.ctypes.data_as(P(C.c_int32)); s.parent = t.parent.ctypes.data_as(P(C.c_int32))
    s.free_capacity = t.free.ctypes.data_as(P(C.c_int64)); s.cap_mask = t.cap_mask.ctypes.data_as(P(C.c_uint32))
    s.tas_usage = t.usage.ctypes.data_as(P(C.c_int64)); s.usage_mask = t.usage_mask.ctypes.data_as(P(C.c_uint32))
    t.struct = s
    return t


def _levels(n):
    return [f"example.com/level-{i}" for i in range(n - 1)] + [tas.HOSTNAME]


def _tr(**kw):
    return {"required": None, "preferred": None, "unconstrained": False, "sliceRequiredTopology": None, "sliceSize": None, **kw}


def _mixed(topo, n, seed, max_pods=64, chains=False, slices=True, sim_empty=False, reqs=None, chain0=0):
    """n requests of every kind (required / preferred / unconstrained / implied / sliced / slice-only) at random levels,
    TASProfileMixed on or off per request."""
    rng = np.random.Generator(np.random.PCG64(seed))
    L = len(topo.levels)
    tmpl = [{"cpu": int(rng.integers(1, 33)) * 1000, "memory": int(rng.integers(1, 65)) << 30,
             **({"gpu": int(rng.integers(1, 5))} if rng.random() < 0.5 else {})} for _ in range(8)]
    reqs = reqs or tas.TasRequests(topo)
    chain, left = chain0, 0
    for _ in range(n):
        if left == 0:
            chain += 1
            left = int(rng.integers(1, 4)) if chains and rng.random() < 0.3 else 1
        left -= 1
        kind = int(rng.integers(0, 6 if slices else 4))
        lv = int(rng.integers(0, L))
        sl = int(rng.integers(lv, L))
        ss = int(rng.integers(1, 5))
        key = topo.levels[lv]
        tr = [_tr(required=key), _tr(preferred=key), _tr(unconstrained=True), None,
              _tr(**{["required", "preferred"][int(rng.integers(0, 2))]: key}, sliceRequiredTopology=topo.levels[sl], sliceSize=ss),
              _tr(sliceRequiredTopology=topo.levels[sl], sliceSize=ss)][kind]
        reqs.add(chain, tmpl[int(rng.integers(0, len(tmpl)))], int(rng.integers(1, max_pods + 1)), tr,
                 simulate_empty=sim_empty and rng.random() < 0.3, profile_mixed=bool(rng.integers(0, 2)))
    return reqs


def _unconstrained(reqs, chain, res, counts, both=True):
    for c in counts:
        for mixed in ((True, False) if both else (True,)):
            chain += 1
            reqs.add(chain, res, c, _tr(unconstrained=True), profile_mixed=mixed)
    return chain


def _node(name, labels, cpu=8000, pods=4, gpu=None, taints=()):
    alloc = {"cpu": cpu, "memory": 64 << 30, "pods": pods, **({} if gpu is None else {"gpu": gpu})}
    return {"name": name, "labels": labels, "allocatable": alloc, "taints": list(taints)}


# ---------------------------------------------------------------------------------------------------------------------
# fixtures: name -> dict(topo, reqs, cap, claims, pairs); built once per session (the CPU and the GPU test share them)
# ---------------------------------------------------------------------------------------------------------------------
FIXTURES = {}


def fixture(*claims, pairs=None):
    def deco(f):
        FIXTURES[f.__name__] = (f, set(claims), pairs or {})
        return f
    return deco


@fixture("span512-lfc", "span512-bestfit", "cached-required", "unconstrained-lfc", "unconstrained-bestfit", "levels=3")
def cache_walk_hosts():
    """8,000 hosts at used=0.9 (many hosts hold no 60-cpu pod, so filter 2 skips them); unconstrained 60-cpu requests
    placing on 600, 1,500 and 3,000+ hosts walk the hostname level far beyond one cache fill, in both orders."""
    topo = tas.synth_topology(2, 4, 1000, seed=11, used=0.9)
    reqs = tas.TasRequests(topo)
    ch = _unconstrained(reqs, 0, {"cpu": 60_000}, [600, 1500, 3100])
    ch = _unconstrained(reqs, ch, {"cpu": 8000}, [5000])  # several pods per host: best_fit over the cached set at the end
    for c, key in [(1, tas.HOSTNAME), (40, tas.HOSTNAME), (300, topo.levels[1])]:
        for mixed in (True, False):
            ch += 1
            reqs.add(ch, {"cpu": 2000}, c, _tr(required=key), profile_mixed=mixed)
    return topo, _mixed(topo, 40, 21, reqs=reqs, chain0=ch).finalize()


@fixture("cached-required", "cached-preferred", "span512-lfc", "span512-bestfit", "levels=3")
def cache_walk_racks():
    """2,100 racks of 3 hosts: the rack level is itself a cached set; required / preferred rack requests fit there."""
    topo = _flat(_levels(3), [1, 2100, 3], seed=12, used=0.9)
    reqs = tas.TasRequests(topo)
    ch = _unconstrained(reqs, 0, {"cpu": 40_000}, [700, 2000])
    for c in (1, 2, 4, 5):
        for key in ("required", "preferred"):
            for mixed in (True, False):
                ch += 1
                reqs.add(ch, {"cpu": 30_000}, c, _tr(**{key: topo.levels[1]}), profile_mixed=mixed)
    return topo, reqs.finalize()


@fixture("slice-inner-0", "slice-inner-1", "slice-leaf", "slice-nondivisible", "slice-count-lt-size", "slice-only",
         "unconstrained-lfc", "unconstrained-bestfit", "levels=3")
def slices_3_levels():
    topo = _flat(_levels(3), [3, 6, 12], seed=13, used=0.5)
    reqs = tas.TasRequests(topo)
    ch = 0
    lv = topo.levels
    for tr, c in [(_tr(required=lv[0], sliceRequiredTopology=lv[1], sliceSize=8), 48), (_tr(preferred=lv[0], sliceRequiredTopology=lv[1], sliceSize=5), 37),
                  (_tr(required=lv[0], sliceRequiredTopology=lv[0], sliceSize=6), 30), (_tr(preferred=lv[1], sliceRequiredTopology=lv[2], sliceSize=3), 10),
                  (_tr(required=lv[1], sliceRequiredTopology=lv[1], sliceSize=7), 3), (_tr(sliceRequiredTopology=lv[1], sliceSize=4), 64),
                  (_tr(sliceRequiredTopology=lv[0], sliceSize=9), 200), (_tr(sliceRequiredTopology=lv[2], sliceSize=2), 41)]:
        for mixed in (True, False):
            ch += 1
            reqs.add(ch, {"cpu": 4000, "memory": 8 << 30}, c, tr, profile_mixed=mixed)
    return topo, _mixed(topo, 200, 31, max_pods=120, reqs=reqs, chain0=ch).finalize()


@fixture("slice-inner-0", "slice-inner-1", "slice-inner-2", "slice-inner-3", "slice-leaf", "slice-nondivisible", "slice-only", "levels=5")
def slices_5_levels():
    topo = _flat(_levels(5), [2, 3, (2, 4), (2, 5), (3, 8)], seed=14, used=0.4)
    reqs = tas.TasRequests(topo)
    ch = 0
    lv = topo.levels
    for a, b, ss, c in [(0, 0, 4, 24), (0, 0, 7, 50), (0, 1, 6, 60), (0, 2, 4, 30), (1, 3, 3, 10), (2, 3, 5, 22), (0, 4, 2, 9), (3, 3, 2, 5), (1, 2, 11, 33)]:
        for key in ("required", "preferred", None):
            for mixed in (True, False):
                ch += 1
                tr = _tr(**({key: lv[a]} if key else {}), sliceRequiredTopology=lv[b], sliceSize=ss)
                reqs.add(ch, {"cpu": 6000, "gpu": 1}, c, tr, profile_mixed=mixed)
    return topo, _mixed(topo, 300, 32, max_pods=80, chains=True, reqs=reqs, chain0=ch).finalize()


def _node_topology(seed, lowest="host"):
    """3 blocks x 4 racks x 5 hosts of node dicts: taints, a pool label, nodes without gpu, TAS and non-TAS usage."""
    rng = np.random.Generator(np.random.PCG64(seed))
    nodes, tas_usage, non_tas = [], {}, {}
    for b in range(3):
        for r in range(4):
            for h in range(5):
                name = f"b{b}-r{r}-h{h}"
                labels = {"cloud.com/block": f"b{b}", "cloud.com/rack": f"b{b}-r{r}", tas.HOSTNAME: name, "pool": "ab"[(r + h) % 2]}
                taints = [{"key": "dedicated", "value": "x", "effect": "NoSchedule"}] if (b + r + h) % 5 == 0 else []
                nodes.append(_node(name, labels, cpu=int(rng.integers(4, 17)) * 1000, pods=int(rng.integers(2, 7)),
                                   gpu=None if (r + h) % 4 == 3 else int(rng.integers(0, 5)), taints=taints))
                if rng.random() < 0.4:
                    tas_usage[name] = {"cpu": 3000, "pods": 1}
                if rng.random() < 0.2:
                    non_tas[name] = {"cpu": 1000}
    nodes.append(_node("not-ready", {"cloud.com/block": "b0", "cloud.com/rack": "b0-r0", tas.HOSTNAME: "not-ready"}) | {"ready": False})
    levels = ["cloud.com/block", "cloud.com/rack"] + ([tas.HOSTNAME] if lowest == "host" else [])
    return tas.TasTopology(levels, nodes, resources=["cpu", "gpu", "memory"], non_tas_usage=non_tas, tas_usage=tas_usage)


TOL = [{"key": "dedicated", "operator": "Equal", "value": "x", "effect": "NoSchedule"}]


@fixture("leaf-ok-filters", "missing-resource", "pair-leaf_ok", "pair-simulate_empty", "pair-slice_size", "pair-slice_level", "zero-request",
         "unconstrained-lfc", "unconstrained-bestfit", "levels=3",
         pairs={"leaf_ok": (0, 1), "simulate_empty": (2, 3), "slice_size": (4, 5), "slice_level": (6, 7)})
def node_dicts():
    topo = _node_topology(15)
    lv = topo.levels
    reqs = tas.TasRequests(topo)
    cpu = {"cpu": 2000}
    reqs.add(1, cpu, 12, _tr(required=lv[1]))                                      # taints exclude some hosts ...
    reqs.add(2, cpu, 12, _tr(required=lv[1]), tolerations=TOL)                      # ... unless tolerated
    reqs.add(3, cpu, 20, _tr(required=lv[0]))
    reqs.add(4, cpu, 20, _tr(required=lv[0]), simulate_empty=True)
    reqs.add(5, cpu, 6, _tr(required=lv[0], sliceRequiredTopology=lv[2], sliceSize=2), flavor_tolerations=TOL)
    reqs.add(6, cpu, 6, _tr(required=lv[0], sliceRequiredTopology=lv[2], sliceSize=3), flavor_tolerations=TOL)
    reqs.add(7, cpu, 8, _tr(required=lv[0], sliceRequiredTopology=lv[2], sliceSize=4), flavor_tolerations=TOL)
    reqs.add(8, cpu, 8, _tr(required=lv[0], sliceRequiredTopology=lv[1], sliceSize=4), flavor_tolerations=TOL)
    ch = 8
    for kw in [dict(node_selector={"pool": "a"}), dict(node_selector={"pool": "b"}, tolerations=TOL), dict(flavor_tolerations=TOL), {}]:
        for tr in (_tr(unconstrained=True), None, _tr(preferred=lv[1]), _tr(required=lv[0])):
            for mixed in (True, False):
                for req in ({"cpu": 1000, "gpu": 1}, {"cpu": 0, "gpu": 0}, {"cpu": 3000, "gpu": 0}):
                    ch += 1
                    reqs.add(ch, req, 5, tr, profile_mixed=mixed, **kw)
    return topo, reqs.finalize()


@fixture("multi-node-leaf", "levels=2", "unconstrained-lfc", "unconstrained-bestfit")
def rack_leaves():
    """The lowest level is the rack: each leaf holds five nodes' capacity."""
    topo = _node_topology(16, lowest="rack")
    return topo, _mixed(topo, 120, 33, max_pods=40, chains=True).finalize()


@fixture("levels=1", "unconstrained-lfc", "unconstrained-bestfit")
def one_level():
    topo = _flat([tas.HOSTNAME], [300], seed=17, used=0.6)
    return topo, _mixed(topo, 150, 34, max_pods=200, chains=True).finalize()


@fixture("levels=2", "unconstrained-lfc", "unconstrained-bestfit")
def two_levels():
    topo = _flat(_levels(2), [7, (1, 60)], seed=18, used=0.6)
    return topo, _mixed(topo, 200, 35, max_pods=150, chains=True).finalize()


@fixture("long-child-range", "span512-lfc", "span512-bestfit", "levels=3")
def ragged():
    """One rack of one host next to a rack of 3,000 hosts: per-parent walks longer than the CTA."""
    topo = _flat(_levels(3), [3, [1, 2, 3], [1, 3000, 40, 7, 200, 90]], seed=19, used=0.9)
    reqs = tas.TasRequests(topo)
    ch = _unconstrained(reqs, 0, {"cpu": 60_000}, [600, 1200])
    for c in (300, 900, 2000):
        for key in ("required", "preferred"):
            for mixed in (True, False):
                ch += 1
                reqs.add(ch, {"cpu": 20_000}, c, _tr(**{key: topo.levels[1]}), profile_mixed=mixed)
    return topo, _mixed(topo, 150, 36, max_pods=500, chains=True, reqs=reqs, chain0=ch).finalize()


@fixture("negative-leaf-state", "unconstrained-lfc", "unconstrained-bestfit", "emits-negative", "emits-more-leaves-than-count", "levels=3")
def over_used():
    """30 % of the leaves used at 130 %: negative leaf counts; counts from 1 to past the total capacity."""
    topo = _flat(_levels(3), [2, 4, 16], seed=20, used=0.5, over=0.3)
    reqs = tas.TasRequests(topo)
    ch = 0
    lv = topo.levels
    for c in (1, 2, 5, 17, 60, 150, 400, 900, 2000, 5000):
        for tr in (_tr(unconstrained=True), None, _tr(preferred=lv[1]), _tr(required=lv[0]), _tr(preferred=lv[0], sliceRequiredTopology=lv[1], sliceSize=2),
                   _tr(sliceRequiredTopology=lv[2], sliceSize=3)):
            for mixed in (True, False):
                ch += 1
                reqs.add(ch, {"cpu": 2000}, c, tr, profile_mixed=mixed)
    return topo, _mixed(topo, 150, 37, max_pods=300, chains=True, reqs=reqs, chain0=ch).finalize()


@fixture("negative-leaf-state", "levels=5")
def over_used_5_levels():
    topo = _flat(_levels(5), [2, 2, 3, (1, 4), (2, 6)], seed=21, used=0.5, over=0.25)
    return topo, _mixed(topo, 300, 38, max_pods=200, chains=True, sim_empty=True).finalize()


def _status_case(*rows, used=0.3):
    """Small topology of identical-capacity racks; rows = (chain, cpu, count, topology request[, profile_mixed])."""
    topo = _flat(_levels(3), [2, 3, 6], seed=22, used=used)
    reqs = tas.TasRequests(topo)
    for row in rows:
        reqs.add(row[0], {"cpu": row[1]}, row[2], row[3], profile_mixed=row[4] if len(row) > 4 else True)
    return topo, reqs.finalize()


LV3 = _levels(3)
BAD, NOFIT, STOP = abi.TAS_BAD_REQUEST, abi.TAS_NO_FIT, -1


@fixture(f"statuses={[BAD, 0]}")
def bad_missing_level():
    return _status_case((1, 8000, 2, _tr(required="example.com/missing")), (2, 8000, 2, None))


@fixture(f"statuses={[BAD, 0]}")
def bad_level_below_slice_level():
    return _status_case((1, 8000, 2, _tr(required=LV3[2], sliceRequiredTopology=LV3[1], sliceSize=2)), (2, 8000, 2, None))


@fixture(f"statuses={[BAD, 0]}")
def bad_slice_size_zero():
    return _status_case((1, 8000, 2, _tr(required=LV3[1], sliceRequiredTopology=LV3[2], sliceSize=0)), (2, 8000, 2, None))


@fixture(f"statuses={[NOFIT, STOP, STOP, 0]}")
def chain_stopped_by_first_podset():
    return _status_case((1, 8000, 500, _tr(required=LV3[2])), (1, 8000, 1, None), (1, 8000, 1, None), (2, 8000, 1, None))


@fixture(f"statuses={[0, NOFIT, STOP, 0]}")
def chain_stopped_by_middle_podset():
    return _status_case((1, 8000, 3, _tr(required=LV3[1])), (1, 8000, 10_000, None), (1, 8000, 1, None), (2, 8000, 1, None))


@fixture("chain-shared-leaf", f"statuses={[0] * 9}")
def chains_share_leaves():
    """Three podsets per chain on identical hosts: later podsets fill the hosts earlier ones left partly used (assumed)."""
    rows = [(ch, 10_000, 6 + 5 * k, _tr(required=LV3[1]), bool(ch % 2)) for ch in (1, 2) for k in range(3)]
    rows += [(3, 6000, 6, _tr(unconstrained=True), False) for _ in range(3)]
    return _status_case(*rows, used=0.0)


@fixture("mixed-simulate-empty-chain", "emits-negative", "levels=3")
def simulate_empty_then_not():
    """A simulate-empty podset followed by one that is not, on leaves that are not over-used: the first places against
    free capacity alone, so the second sees leaves whose usage plus assumed pods exceed free capacity."""
    topo = _flat(_levels(3), [2, 3, 8], seed=24, used=0.6)
    reqs = tas.TasRequests(topo)
    ch = 0
    for c1, c2 in [(200, 40), (400, 100), (120, 300)]:
        for tr in (_tr(unconstrained=True), None, _tr(required=LV3[0]), _tr(preferred=LV3[1])):
            for mixed in (True, False):
                ch += 1
                reqs.add(ch, {"cpu": 8000}, c1, tr, simulate_empty=True, profile_mixed=mixed)
                reqs.add(ch, {"cpu": 4000}, c2, tr, profile_mixed=mixed)
    return topo, reqs.finalize()


@fixture("negative-leaf-state", "span512-lfc", "span512-bestfit", "levels=3")
def over_used_cache_walk():
    """8,000 hosts, 5 % of them over-used: zero and negative keys crowd the cache fills of the hostname level."""
    topo = _flat(_levels(3), [2, 4, 1000], seed=23, used=0.9, over=0.05)
    reqs = tas.TasRequests(topo)
    ch = _unconstrained(reqs, 0, {"cpu": 60_000}, [600, 1500])
    ch = _unconstrained(reqs, ch, {"cpu": 8000}, [3000])
    return topo, _mixed(topo, 30, 39, max_pods=300, reqs=reqs, chain0=ch).finalize()


@fixture("span512-lfc", "span512-bestfit", "unconstrained-lfc", "unconstrained-bestfit", "levels=3")
def cfg5_topology():
    """The cfg5 topology (100,000 hosts) with 300 requests from tas.synth_requests and a few large unconstrained ones."""
    topo = tas.synth_topology(10, 100, 100)
    reqs = tas.synth_requests(topo, 300, seed=9, chains=True, max_pods=256, profile_mixed=None)
    ch = int(reqs.chain.max())
    _unconstrained(reqs, ch, {"cpu": 32_000}, [1000, 4000])
    return topo, reqs.finalize()


@functools.lru_cache(maxsize=None)
def build(name):
    f, claims, pairs = FIXTURES[name]
    topo, reqs = f()
    over = _negative_possible(topo)
    cap = int(np.clip(reqs.count, 0, None).sum()) + 16 + (topo.n_leaves * len(reqs.rows) if over else 0)
    return topo, reqs, cap, claims, pairs


def _negative_possible(topo):
    return bool((topo.free - topo.usage < 0).any() or (topo.free < 0).any())


# ---------------------------------------------------------------------------------------------------------------------
# facts about an output (host side) and invariants
# ---------------------------------------------------------------------------------------------------------------------
def _ancestors(topo):
    """anc[l][leaf] = the leaf's domain at level l."""
    L = len(topo.levels)
    leaf0 = int(topo.level_start[L - 1])
    anc = [None] * L
    anc[L - 1] = np.arange(leaf0, leaf0 + topo.n_leaves)
    for l in range(L - 2, -1, -1):
        anc[l] = topo.parent[anc[l + 1]]
    return anc


def _leaf_states(topo, reqs, q):
    """CountIn of request q on every leaf (no assumed usage), truncating like int32(cap / v)."""
    sim = bool(reqs.flags[q] & abi.TAS_SIMULATE_EMPTY)
    cap = topo.free - (0 if sim else topo.usage)
    mask = topo.cap_mask | (0 if sim else topo.usage_mask)
    st = np.full(topo.n_leaves, np.iinfo(np.int64).max)
    for k in range(len(topo.resources)):
        v = 1 if k == topo.pods_resource else int(reqs.pod_request[q, k])
        if k != topo.pods_resource and not (reqs.request_mask[q] >> k) & 1:
            continue
        if v == 0:
            continue
        c = np.trunc(cap[:, k] / v).astype(np.int64)
        c[(mask >> k) & 1 == 0] = 0
        st = np.minimum(st, c)
    return st


def facts(topo, reqs, out, pairs):
    L = len(topo.levels)
    sizes = np.diff(topo.level_start)
    leaf0 = int(topo.level_start[L - 1])
    n_children = np.bincount(topo.parent[leaf0:], minlength=1) if L > 1 else None  # children per parent of a leaf
    anc = _ancestors(topo)
    over = _negative_possible(topo)
    f = {f"levels={L}"}
    for q in range(len(reqs.rows)):
        st, fl = int(out.status[q]), int(reqs.flags[q])
        f.add({abi.TAS_OK: "status-ok", abi.TAS_NO_FIT: "status-nofit", abi.TAS_BAD_REQUEST: "status-bad", -1: "status-chain-stopped"}[st])
        if over and (_leaf_states(topo, reqs, q) < 0).any():
            f.add("negative-leaf-state")
        if st != abi.TAS_OK:
            continue
        asg = out.assignment(q)
        leaves = [lf for lf, _ in asg]
        counts = [c for _, c in asg]
        lfc = bool(fl & abi.TAS_UNCONSTRAINED) and bool(fl & abi.TAS_PROFILE_MIXED)
        lvl, ss, sl, cnt = int(reqs.level[q]), int(reqs.slice_size[q]), int(reqs.slice_level[q]), int(reqs.count[q])
        if len(leaves) > CACHE_KEYS and sizes[L - 1] > CACHE_MIN:
            f.add("span512-lfc" if lfc else "span512-bestfit")
        if fl & abi.TAS_UNCONSTRAINED:
            f.add("unconstrained-lfc" if lfc else "unconstrained-bestfit")
        if sizes[lvl] > CACHE_MIN and leaves and len(set(anc[lvl][leaves])) == 1:
            f.add("cached-required" if fl & abi.TAS_REQUIRED else "cached-preferred")
        if ss > 1:
            f.add(f"slice-inner-{sl}" if sl < L - 1 else "slice-leaf")
            if cnt % ss:
                f.add("slice-nondivisible")
            if cnt < ss:
                f.add("slice-count-lt-size")
            if lvl == 0 and fl & abi.TAS_UNCONSTRAINED:  # only a slice-only request is unconstrained at level 0 above the leaves
                f.add("slice-only")
        if any(c < 0 for c in counts):
            f.add("emits-negative")
        if len(leaves) > cnt:
            f.add("emits-more-leaves-than-count")
        if L > 1 and any(n_children[topo.parent[leaf0 + lf]] > CTA for lf in leaves):
            f.add("long-child-range")
        if topo.leaf_nodes and any(len(topo.leaf_nodes[lf]) > 1 for lf in leaves):
            f.add("multi-node-leaf")
        if reqs.leaf_ok is not None:
            ok = np.unpackbits(reqs.leaf_ok[q].view(np.uint8), bitorder="little")[:topo.n_leaves]
            if not ok.all():
                f.add("leaf-ok-filters")
        if reqs.rows[q]["requests"] and 0 in reqs.rows[q]["requests"].values():
            f.add("zero-request")
        wanted = [k for k in range(len(topo.resources)) if reqs.pod_request[q, k] > 0]
        have = topo.cap_mask | topo.usage_mask
        if any(((have >> k) & 1 == 0).any() for k in wanted):
            f.add("missing-resource")  # a requested resource some leaf does not list: CountIn gives it 0
    if len(reqs.rows) <= 12:
        f.add(f"statuses={out.status[:len(reqs.rows)].tolist()}")
    for q in range(1, len(reqs.rows)):
        if reqs.chain[q] == reqs.chain[q - 1] and (reqs.flags[q] ^ reqs.flags[q - 1]) & abi.TAS_SIMULATE_EMPTY:
            f.add("mixed-simulate-empty-chain")
    for kind, (a, b) in pairs.items():
        if out.status[a] != out.status[b] or out.assignment(a) != out.assignment(b):
            f.add(f"pair-{kind}")
    chain_leaves = {}
    for q in range(len(reqs.rows)):
        if out.status[q] == abi.TAS_OK:
            s = chain_leaves.setdefault(int(reqs.chain[q]), [])
            if any(set(lf for lf, _ in out.assignment(q)) & prev for prev in s):
                f.add("chain-shared-leaf")
            s.append(set(lf for lf, _ in out.assignment(q)))
    return f


def check_invariants(topo, reqs, out):
    L = len(topo.levels)
    anc = _ancestors(topo)
    over = _negative_possible(topo)
    # a simulate-empty podset places against free capacity alone, so a chain that mixes both is not bound by usage
    mixed_sim = {int(reqs.chain[q]) for q in range(1, len(reqs.rows))
                 if reqs.chain[q] == reqs.chain[q - 1] and (reqs.flags[q] ^ reqs.flags[q - 1]) & abi.TAS_SIMULATE_EMPTY}
    chain_use = {}
    for q in range(len(reqs.rows)):
        if out.status[q] != abi.TAS_OK:
            continue
        asg = out.assignment(q)
        leaves = np.array([lf for lf, _ in asg], np.int64)
        counts = np.array([c for _, c in asg], np.int64)
        cnt, ss, sl = int(reqs.count[q]), int(reqs.slice_size[q]), int(reqs.slice_level[q])
        assert counts.sum() == cnt // ss * ss, (q, int(counts.sum()), cnt, ss)
        assert (np.diff(leaves) > 0).all(), (q, "leaves not strictly ascending")
        assert (counts != 0).all()
        if len(leaves) and reqs.flags[q] & abi.TAS_REQUIRED:
            assert len(set(anc[int(reqs.level[q])][leaves].tolist())) == 1, (q, "leaves span several required domains")
        if len(leaves):
            per = {}
            for d, c in zip(anc[sl][leaves].tolist(), counts.tolist()):
                per[d] = per.get(d, 0) + c
            assert all(c % ss == 0 for c in per.values()), (q, "slice-level domain count not a multiple of the slice size", per)
        if not over and int(reqs.chain[q]) not in mixed_sim:
            # the pods of the chain so far fit each leaf's free capacity
            use = chain_use.setdefault(int(reqs.chain[q]), np.zeros_like(topo.free))
            for lf, c in zip(leaves.tolist(), counts.tolist()):
                use[lf] += reqs.pod_request[q] * c
                use[lf, topo.pods_resource] += c
            sim = bool(reqs.flags[q] & abi.TAS_SIMULATE_EMPTY)
            free = topo.free - (0 if sim else topo.usage)
            keys = [k for k in range(len(topo.resources)) if (reqs.request_mask[q] >> k) & 1 or k == topo.pods_resource]
            assert (use[leaves][:, keys] <= free[leaves][:, keys]).all(), (q, "chain exceeds a leaf's free capacity")


def _same(got, want):
    n = len(got.status) if len(want.status) else 0
    assert np.array_equal(got.status[:n], want.status[:n]), [(q, int(a), int(b)) for q, (a, b) in enumerate(zip(got.status, want.status)) if a != b][:10]
    assert np.array_equal(got.asg_start, want.asg_start), np.flatnonzero(got.asg_start != want.asg_start)[:10]
    m = int(want.asg_start[-1])
    assert np.array_equal(got.asg_leaf[:m], want.asg_leaf[:m]) and np.array_equal(got.asg_count[:m], want.asg_count[:m])


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ev():
    from kueue_b200 import native
    e = native.Evaluator(0)
    yield e
    e.close()


@pytest.mark.parametrize("name", list(FIXTURES))
def test_device_matches_oracle(ev, name):
    topo, reqs, cap, _, _ = build(name)
    want = oracle.tas_find(topo, reqs, cap)
    got = ev.tas_find(topo, reqs, cap)
    check_invariants(topo, reqs, got)
    _same(got, want)


def test_capacity_smaller_than_assignment(ev):
    """out.capacity < n_assigned: KB_ERR_CAPACITY, every status and asg_start complete, the first `capacity` pairs copied."""
    from kueue_b200 import native
    topo, reqs, cap, _, _ = build("chains_share_leaves")
    want = oracle.tas_find(topo, reqs, cap)
    n = int(want.asg_start[-1])
    assert n > 8
    small = n // 2
    out = tas.TasOut(reqs, small)
    rc = native.lib().kb_tas_find(ev._h, C.byref(topo.struct), C.byref(reqs.struct), C.byref(out.struct))
    assert rc == abi.KB_ERR_CAPACITY
    assert out.struct.n_assigned == n
    assert np.array_equal(out.status, want.status) and np.array_equal(out.asg_start, want.asg_start)
    assert np.array_equal(out.asg_leaf, want.asg_leaf[:small]) and np.array_equal(out.asg_count, want.asg_count[:small])


def test_output_regions_past_int32_are_refused(ev):
    """The per-request output regions are addressed with int32 offsets: a batch whose regions add up past 2^31 entries
    (32,769 requests of 65,536 pods over 65,536 hosts) is refused before anything is allocated, not wrapped."""
    from kueue_b200 import native
    topo = _flat([tas.HOSTNAME], [1 << 16], seed=25, used=0.0)
    reqs = tas.TasRequests(topo)
    for ch in range((1 << 15) + 1):
        reqs.add(ch, {"cpu": 1000}, 1 << 16, None)
    reqs.finalize()
    out = tas.TasOut(reqs, 16)
    rc = native.lib().kb_tas_find(ev._h, C.byref(topo.struct), C.byref(reqs.struct), C.byref(out.struct))
    assert rc == abi.KB_ERR_CAPACITY
    assert b"2^31" in native.lib().kb_last_error(ev._h)


def test_no_domains(ev):
    """No node of the flavor is schedulable (n_domains == 0): the first podset of every chain fails, bad requests as such."""
    topo = tas.TasTopology(_levels(3), [])
    assert topo.struct.n_domains == 0
    reqs = tas.TasRequests(topo)
    reqs.add(1, {}, 2, _tr(required=tas.HOSTNAME)); reqs.add(1, {}, 1, None)
    reqs.add(2, {}, 2, _tr(required="example.com/missing"))
    reqs.add(3, {}, 2, _tr(unconstrained=True), profile_mixed=False)
    reqs.add(4, {}, 2, _tr(required=tas.HOSTNAME, sliceRequiredTopology=_levels(3)[0], sliceSize=2))
    reqs.finalize()
    want = oracle.tas_find(topo, reqs)
    assert want.status.tolist() == [abi.TAS_NO_FIT, -1, abi.TAS_BAD_REQUEST, abi.TAS_NO_FIT, abi.TAS_BAD_REQUEST]
    _same(ev.tas_find(topo, reqs), want)


def test_calls_that_grow_and_shrink():
    """One evaluator, batches that grow and then shrink: the grow-only device buffer keeps what the last call left in
    n_out and assumed, so both must be cleared on every call."""
    from kueue_b200 import native
    e = native.Evaluator(0)
    try:
        for name in ("slices_3_levels", "over_used", "chains_share_leaves", "ragged", "bad_missing_level", "one_level", "over_used_5_levels",
                     "two_levels", "chains_share_leaves"):
            topo, reqs, cap, _, _ = build(name)
            _same(e.tas_find(topo, reqs, cap), oracle.tas_find(topo, reqs, cap))
    finally:
        e.close()
