"""kb_run_drain in event mode with stop / resume edits of spec.active (kb_snapshot.ac_*), each scenario with and without
the edits, in one process.

Pairs of legs, alternated after a warm-up:
  - baseline: the baseline scenario (synth.perf_scenario, 15,000 workloads, 1 ms cycles, run to the end), and the same
    with stops and resumes (perf_scenario(active=seed): 5% of the workloads stopped once, half of those resumed later);
  - cfg4: the hierarchical cfg4 at full size (evictable: adm_wl names every row) with synth.add_events, and with
    synth.add_active_changes, over --max-cycles;
  - cfg3: a cfg3 event drain (the flat route), and with synth.add_active_changes;
  - baseline_late: the baseline scenario with the same edits moved past its natural end, stopped after its natural
    cycles: the per-cycle cost of carrying the table; baseline_late_full runs it to the end, where the drain jumps to
    each edit (boundaries without a cycle): its gpu_ms beyond baseline_late's is the cost of those jumps.
Per leg: cycles, admissions, stops and resumes that changed the state, device ms per cycle (median / min / max) and the
queue layer's time (kernel_ms slot KB_K_DRAIN, k_drain_active included, with kb_set_profile).  Prints one JSON line with
the card name and power limit read in the same call.

    python tools/active_drain_bench.py [--reps 5] [--warmup 2] [--seed 3] [--max-cycles 2000]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=3, help="seed of the edits")
    ap.add_argument("--max-cycles", type=int, default=2000, help="cycles of the cfg3 / cfg4 legs")
    args = ap.parse_args()
    import numpy as np
    from afs_drain_bench import card
    from kueue_b200 import abi, native, synth

    def replay(s):
        if "adm_wl" not in s.arrays and s.n_adm == 0:
            s.set("adm_wl", np.zeros(0))
        return s

    base = synth.perf_scenario(1.0)
    probe = native.Evaluator(0)
    natural = probe.run_drain(base, abi.DrainOut(base, 1_000_000, trace=False))
    end, n_natural = natural.end_ns, natural.n_cycles
    probe.close()
    late = synth.perf_scenario(1.0, active=args.seed)
    late.set("ac_ns", late.arrays["ac_ns"] - late.arrays["ac_ns"].min() + end + 1)  # every edit after the natural end
    cfg4 = lambda: replay(synth.add_events(synth.make_snapshot(4, evictable=True), seed=1))  # noqa: E731
    cfg3 = lambda: replay(synth.add_events(synth.make_snapshot(3), seed=2))  # noqa: E731
    legs = {"baseline": (base, 1_000_000), "baseline_active": (synth.perf_scenario(1.0, active=args.seed), 1_000_000),
            "baseline_late": (late, n_natural), "baseline_late_full": (late, 1_000_000),
            "cfg4": (cfg4(), args.max_cycles), "cfg4_active": (synth.add_active_changes(cfg4(), seed=args.seed), args.max_cycles),
            "cfg3": (cfg3(), args.max_cycles), "cfg3_active": (synth.add_active_changes(cfg3(), seed=args.seed), args.max_cycles)}
    ev = native.Evaluator(0)
    outs = {k: abi.DrainOut(s, max_cycles=mc, trace=False) for k, (s, mc) in legs.items()}
    for _ in range(args.warmup):
        for k, (s, _) in legs.items():
            ev.run_drain(s, outs[k])
    per_cycle, total_ms, drain_ms = {k: [] for k in legs}, {k: [] for k in legs}, {k: [] for k in legs}
    for _ in range(args.reps):
        for k, (s, _) in legs.items():
            o = ev.run_drain(s, outs[k])
            per_cycle[k].append(o.gpu_ms / max(1, o.n_cycles))
            total_ms[k].append(o.gpu_ms)
    ev.set_profile(True)
    for k, (s, _) in legs.items():  # a profiled run of its own: the queue layer's share
        ev.run_drain(s, outs[k])
        drain_ms[k] = float(ev.stats().kernel_ms[13])
    ev.set_profile(False)
    res = {"what": "kb_run_drain event mode with and without stop / resume edits", "card": card(),
           "reps": args.reps, "warmup": args.warmup, "max_cycles": args.max_cycles}
    for k, (s, _) in legs.items():
        o = ev.run_drain(s, outs[k])
        res[k] = {"cycles": o.n_cycles, "admitted": o.n_admitted, "evicted": o.n_evicted, "end_s": o.end_ns / 1e9,
                  "edits": int(len(s.arrays["ac_ns"])) if "ac_ns" in s.arrays else 0, "stopped": o.n_stopped,
                  "resumed": o.n_resumed, "ms_per_cycle_median": statistics.median(per_cycle[k]),
                  "ms_per_cycle_min": min(per_cycle[k]), "ms_per_cycle_max": max(per_cycle[k]),
                  "gpu_ms_median": statistics.median(total_ms[k]),
                  "drain_layer_ms_profiled": drain_ms[k]}
    ev.close()
    res["late_jumps_ms"] = res["baseline_late_full"]["gpu_ms_median"] - res["baseline_late"]["gpu_ms_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
