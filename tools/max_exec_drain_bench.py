"""kb_run_drain in event mode with MaximumExecutionTimeSeconds (kb_snapshot.wl_max_exec_s), the baseline scenario with
and without the block, in one process.

Legs, alternated after a warm-up: the baseline scenario (synth.perf_scenario, 15,000 workloads, 1 ms cycles, run to the
end) without the block, with every limit nil (the same schedule through the block's paths), and with limits and a 30 ms
termination latency (synth.perf_scenario(evict_ns=30 ms, max_exec=seed): half of the workloads limited to 1 s, a fifth
of those starting with 0-2 s accumulated).  Per leg: cycles, simulated end time, evictions, deactivations, records with
an accumulated time and its total in seconds, and device ms per cycle.  Prints one JSON line with the card name and
power limit read in the same call.

    python tools/max_exec_drain_bench.py [--reps 5] [--warmup 2] [--seed 3]
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
    ap.add_argument("--seed", type=int, default=3, help="seed of the limits and starting accumulated times")
    args = ap.parse_args()
    from afs_drain_bench import card
    from kueue_b200 import abi, native, synth

    nil = synth.perf_scenario(1.0)
    nil.set("wl_max_exec_s", np.zeros(nil.n_wl)); nil.set("adm_exec_since_ns", np.zeros(0))
    legs = {"baseline": synth.perf_scenario(1.0), "baseline_max_exec_nil": nil,
            "baseline_max_exec": synth.perf_scenario(1.0, evict_ns=30_000_000, max_exec=args.seed)}
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
    res = {"what": "kb_run_drain event mode, baseline scenario with and without MaximumExecutionTimeSeconds", "card": card(),
           "reps": args.reps, "warmup": args.warmup, "cycle_ms": 1}
    for k, s in legs.items():
        o = ev.run_drain(s, outs[k])
        acc = outs[k].wl_exec_acc_s_out if "wl_max_exec_s" in s.arrays else np.full(s.n_wl, -1)
        res[k] = {"cycles": o.n_cycles, "admitted": o.n_admitted, "finished": o.n_finished, "end_s": o.end_ns / 1e9,
                  "evicted": o.n_evicted, "evict_done": o.n_evict_done, "max_exec_deactivated": o.n_max_exec_deactivated,
                  "records_with_acc": int((acc >= 0).sum()), "acc_s_total": int(acc[acc >= 0].sum()),
                  "ms_per_cycle_median": statistics.median(per_cycle[k]), "ms_per_cycle_min": min(per_cycle[k]),
                  "ms_per_cycle_max": max(per_cycle[k])}
    ev.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
