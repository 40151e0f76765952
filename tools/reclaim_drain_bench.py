"""kb_run_drain in event mode with reclaim steps (kb_snapshot.wl_rc_start, rc_*), each scenario with and without the
steps, in one process.

Pairs of legs, alternated after a warm-up:
  - baseline: the baseline scenario with one pod per cpu (synth.perf_scenario(reclaim=seed) without its step tables: the
    medium and large classes are 5- and 20-pod Jobs), and the same with the steps (a third of the multi-pod workloads
    give back pods up to 3 times within their run), both run to the end;
  - cfg4: the hierarchical cfg4 at full size (evictable) with 2-pod podsets and synth.add_events, and the same with
    synth.add_reclaims, over --max-cycles.
Per leg: cycles, admissions, steps applied (n_reclaims), device ms per cycle (median / min / max) and the queue layer's
time (kernel_ms slot KB_K_DRAIN, with kb_set_profile).  Prints one JSON line with the card name and power limit read in
the same call.

    python tools/reclaim_drain_bench.py [--reps 5] [--warmup 2] [--seed 3] [--max-cycles 2000]
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
    ap.add_argument("--seed", type=int, default=3, help="seed of the steps")
    ap.add_argument("--max-cycles", type=int, default=2000, help="cycles of the cfg4 legs")
    args = ap.parse_args()
    import numpy as np
    from afs_drain_bench import card
    from kueue_b200 import abi, native, synth

    def without_steps(s):
        for k in abi.RECLAIM_FIELDS:
            s.arrays.pop(k, None)
        s.__dict__["_struct"] = None
        return s

    def cfg4():
        s = synth.make_snapshot(4, evictable=True)
        s.set("ps_count", np.full(s.n_podset, 2)); s.set("ps_req", s.arrays["ps_req"] * 2)
        s.flags &= ~abi.F_PARTIAL_ADMISSION
        s = synth.add_events(s, seed=1)
        if "adm_wl" not in s.arrays and s.n_adm == 0:
            s.set("adm_wl", np.zeros(0))
        return s

    legs = {"baseline": (without_steps(synth.perf_scenario(1.0, reclaim=args.seed)), 1_000_000),
            "baseline_reclaim": (synth.perf_scenario(1.0, reclaim=args.seed), 1_000_000),
            "cfg4": (cfg4(), args.max_cycles), "cfg4_reclaim": (synth.add_reclaims(cfg4(), seed=args.seed), args.max_cycles)}
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
    res = {"what": "kb_run_drain event mode with and without reclaim steps", "card": card(),
           "reps": args.reps, "warmup": args.warmup, "max_cycles": args.max_cycles}
    for k, (s, _) in legs.items():
        o = ev.run_drain(s, outs[k])
        res[k] = {"cycles": o.n_cycles, "admitted": o.n_admitted, "evicted": o.n_evicted, "end_s": o.end_ns / 1e9,
                  "steps": int(len(s.arrays["rc_after_ns"])) if "rc_after_ns" in s.arrays else 0, "reclaims": o.n_reclaims,
                  "ms_per_cycle_median": statistics.median(per_cycle[k]), "ms_per_cycle_min": min(per_cycle[k]),
                  "ms_per_cycle_max": max(per_cycle[k]), "gpu_ms_median": statistics.median(total_ms[k]),
                  "drain_layer_ms_profiled": drain_ms[k]}
    ev.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
