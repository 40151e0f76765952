"""kb_run_drain in event mode with WaitForPodsReady (kb_snapshot.wl_pods_ready_ns), the baseline scenario with and
without the block, in one process.

Legs, alternated after a warm-up: the baseline scenario (synth.perf_scenario, 15,000 workloads, 1 ms cycles, run to the
end) without the block, with every delay 0 (the same schedule through the PodsReady path), and with PodsReady timeouts
(synth.perf_scenario(pods_ready=seed): delays of 0-50 ms, 10% of the workloads never ready, timeout 100 ms, backoff base
1 s, max 8 s, limit 2) and a 30 ms termination latency.  Per leg: cycles, simulated end time, timeouts, deactivations,
re-sorts, and device ms per cycle (the re-sorts included).  Prints one JSON line with the card name and power limit read
in the same call.

    python tools/pods_ready_drain_bench.py [--reps 5] [--warmup 2] [--seed 9]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=9, help="seed of the PodsReady delays and never-ready workloads")
    args = ap.parse_args()
    from afs_drain_bench import card
    from kueue_b200 import abi, native, synth

    zero = synth.perf_scenario(1.0)
    zero.set("wl_pods_ready_ns", np.zeros(zero.n_wl)); zero.set("wl_pods_ready_fail", np.zeros(zero.n_wl))
    legs = {"baseline": synth.perf_scenario(1.0), "baseline_pods_ready_zero": zero,
            "baseline_pods_ready": synth.perf_scenario(1.0, evict_ns=30_000_000, pods_ready=args.seed)}
    ev = native.Evaluator(0)
    outs = {k: abi.DrainOut(s, max_cycles=1_000_000, trace=False) for k, s in legs.items()}
    for _ in range(args.warmup):
        for k, s in legs.items():
            ev.run_drain(s, outs[k])
    per_cycle = {k: [] for k in legs}
    for _ in range(args.reps):
        for k, s in legs.items():
            o = ev.run_drain(s, outs[k])
            per_cycle[k].append(o.gpu_ms / max(1, o.n_cycles))
    res = {"what": "kb_run_drain event mode, baseline scenario with and without WaitForPodsReady", "card": card(),
           "reps": args.reps, "warmup": args.warmup, "cycle_ms": 1}
    for k, s in legs.items():
        o = ev.run_drain(s, outs[k])
        res[k] = {"cycles": o.n_cycles, "admitted": o.n_admitted, "finished": o.n_finished, "end_s": o.end_ns / 1e9,
                  "pods_ready_timeout": o.n_pods_ready_timeout, "pods_ready_deactivated": o.n_pods_ready_deactivated,
                  "resorts": o.n_resorts, "resort_ms_total": o.resort_ms,
                  "ms_per_cycle_median": statistics.median(per_cycle[k]), "ms_per_cycle_min": min(per_cycle[k]),
                  "ms_per_cycle_max": max(per_cycle[k])}
    ev.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
