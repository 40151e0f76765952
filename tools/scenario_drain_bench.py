"""kb_run_drain in event mode: the reference's baseline scheduler scenario to the end, and the cost of the event kernels.

1. The baseline scenario (synth.perf_scenario: 5 cohorts x 6 ClusterQueues, 15,000 workloads created at fixed intervals,
   each finishing its run time after admission, preemptions replayed) drained on the device until no event is left:
   cycles, simulated end time, device ms, mean (admit - create) per workload class and the minimum ClusterQueue usage
   (time-weighted mean over the drain, as a share of nominal).  The host definition (kueue_b200/drain.py) runs the
   same scenario on the CPU oracle in this process and the two are compared cycle by cycle.  The reference checks these
   quantities in configs/baseline/rangespec.yaml, but its values come from a live API server and a wall clock; the
   numbers here are context, not a parity target.
2. cfg3 at full size (1M pending workloads, 10k ClusterQueues) drained plain and with synth.add_events, alternating
   after a warm-up: device ms per cycle of each (median, min, max), i.e. what the event kernels cost.

Prints one JSON line with the card name and power limit read in the same call.

    python tools/scenario_drain_bench.py [--reps 3] [--warmup 1] [--max-cycles 60]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from afs_drain_bench import card  # noqa: E402


def usage_over_time(snap, out):
    """time-weighted mean of each ClusterQueue's cpu usage over [0, end_ns], from the admit / finish times (a row
    that was evicted is not counted: its workload's admit time is overwritten by the readmission)"""
    a = snap.arrays
    Q = snap.n_cq
    req = a["ps_req"].reshape(-1)
    fin = out.wl_finish_ns
    done = fin != np.iinfo(np.int64).max
    busy = np.zeros(Q)
    np.add.at(busy, a["wl_cq"][done], (fin[done] - out.wl_admit_ns[done]) * req[done])
    return busy / max(1, out.end_ns)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--max-cycles", type=int, default=60)
    args = ap.parse_args()
    import oracle
    from kueue_b200 import abi, native, synth
    from kueue_b200.drain import drain
    res = {"what": "kb_run_drain event mode: baseline scenario to the end; cfg3 plain vs with events", "card": card()}
    ev = native.Evaluator(0)
    # ---- 1. the baseline scenario, device and host definition
    snap = synth.perf_scenario(1.0)
    cap = 40 * snap.n_wl + 10000
    want = drain(snap, lambda s: oracle.run_cycle(s, cap), max_cycles=1_000_000)
    out = ev.run_drain(snap, abi.DrainOut(snap, max_cycles=1_000_000, trace_capacity=want.n_decisions))
    cyc = out.cycles()
    equal = (out.n_cycles == want.cycles and out.n_decisions == want.n_decisions and out.end_ns == want.end_ns and
             all(np.array_equal(cyc[k][0], want.heads[k]) and np.array_equal(cyc[k][1], want.decisions[k]) for k in range(want.cycles)) and
             np.array_equal(out.wl_admit_ns, want.wl_admit_ns) and np.array_equal(out.wl_finish_ns, want.wl_finish_ns) and
             np.array_equal(out.cq_usage, want.cq_usage))
    wait = (out.wl_admit_ns - snap.arrays["wl_create_ns"]) / 1e6
    nominal = snap.arrays["nominal"].reshape(-1)[:snap.n_cq]
    res["baseline"] = {
        "workloads": snap.n_wl, "cycles": out.n_cycles, "sim_end_s": out.end_ns / 1e9, "device_ms": out.gpu_ms,
        "admitted": out.n_admitted, "preemptions": out.n_evicted, "finished": out.n_finished,
        "mean_admit_wait_ms": {name: float(wait[snap.perf_class == c].mean()) for c, (name, *_) in enumerate(synth.PERF_CLASSES)},
        "min_cq_usage_share_of_nominal": float((usage_over_time(snap, out) / nominal).min()),
        "equals_host_definition": bool(equal)}
    # ---- 2. cfg3 at full size, plain and with events
    plain = synth.make_snapshot(3)
    events = synth.add_events(synth.make_snapshot(3), seed=7, span_ns=200_000, step_ns=2_000)
    legs = {"plain": native.pin_snapshot(plain), "events": native.pin_snapshot(events)}
    legs["events"].drain_cycle_ns = events.drain_cycle_ns  # a scalar of the header, not a table
    outs = {k: abi.DrainOut(s, max_cycles=args.max_cycles, trace=False) for k, s in legs.items()}
    for _ in range(args.warmup):
        for k, s in legs.items():
            ev.run_drain(s, outs[k])
    per_cycle = {k: [] for k in legs}
    for _ in range(args.reps):
        for k, s in legs.items():
            o = ev.run_drain(s, outs[k])
            per_cycle[k].append(o.gpu_ms / max(1, o.n_cycles))
    for k in legs:
        o = outs[k]
        res["cfg3_" + k] = {"cycles": o.n_cycles, "admitted": o.n_admitted, "finished": o.n_finished, "arrived": o.n_arrived,
                            "ms_per_cycle_median": statistics.median(per_cycle[k]), "ms_per_cycle_min": min(per_cycle[k]),
                            "ms_per_cycle_max": max(per_cycle[k])}
    res["cfg3_events_over_plain_per_cycle"] = res["cfg3_events"]["ms_per_cycle_median"] / res["cfg3_plain"]["ms_per_cycle_median"]
    res.update(reps=args.reps, warmup=args.warmup, max_cycles=args.max_cycles)
    ev.close()
    print(json.dumps(res))
    if not equal:
        sys.exit("the device drain differs from the host definition on the baseline scenario")


if __name__ == "__main__":
    main()
