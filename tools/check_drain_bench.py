"""kb_run_drain in event mode with admission checks (kb_snapshot.wl_check_ns), the baseline scenario with and without
checks, in one process.

Legs, alternated after a warm-up: the baseline scenario (synth.perf_scenario, 15,000 workloads, 1 ms cycles, run to the
end) without the check tables, with every delay 0 (the same schedule through the check path), and with checks on every
other ClusterQueue (synth.perf_scenario(checks=seed): delays of 20-200 ms, a share of failing attempts, backoff base 1 s,
max 8 s, limit 3).  Per leg: cycles, simulated end time, verdicts, re-sorts and device ms per re-sort, and device ms per
cycle (the re-sorts included).  Prints one JSON line with the card name and power limit read in the same call.

    python tools/check_drain_bench.py [--reps 5] [--warmup 2] [--seed 7]
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
    ap.add_argument("--seed", type=int, default=7, help="seed of the check delays and failures")
    args = ap.parse_args()
    from afs_drain_bench import card
    from kueue_b200 import abi, native, synth

    zero = synth.perf_scenario(1.0)
    zero.set("wl_check_ns", np.zeros(zero.n_wl)); zero.set("wl_check_fail", np.zeros(zero.n_wl))
    legs = {"baseline": synth.perf_scenario(1.0), "baseline_checks_zero": zero, "baseline_checks": synth.perf_scenario(1.0, checks=args.seed)}
    ev = native.Evaluator(0)
    outs = {k: abi.DrainOut(s, max_cycles=1_000_000, trace=False) for k, s in legs.items()}
    for _ in range(args.warmup):
        for k, s in legs.items():
            ev.run_drain(s, outs[k])
    per_cycle = {k: [] for k in legs}
    per_resort = []
    for _ in range(args.reps):
        for k, s in legs.items():
            o = ev.run_drain(s, outs[k])
            per_cycle[k].append(o.gpu_ms / max(1, o.n_cycles))
            if k == "baseline_checks" and o.n_resorts:
                per_resort.append(o.resort_ms / o.n_resorts)
    res = {"what": "kb_run_drain event mode, baseline scenario with and without admission checks", "card": card(),
           "reps": args.reps, "warmup": args.warmup, "cycle_ms": 1}
    for k, s in legs.items():
        o = ev.run_drain(s, outs[k])
        res[k] = {"cycles": o.n_cycles, "admitted": o.n_admitted, "finished": o.n_finished, "end_s": o.end_ns / 1e9,
                  "check_ready": o.n_check_ready, "check_retry": o.n_check_retry, "check_rejected": o.n_check_rejected,
                  "resorts": o.n_resorts, "resort_ms_total": o.resort_ms,
                  "ms_per_cycle_median": statistics.median(per_cycle[k]), "ms_per_cycle_min": min(per_cycle[k]),
                  "ms_per_cycle_max": max(per_cycle[k])}
    if per_resort:
        res["baseline_checks"]["ms_per_resort_median"] = statistics.median(per_resort)
    ev.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
