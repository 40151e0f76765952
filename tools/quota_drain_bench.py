"""kb_run_drain in event mode with planned ClusterQueue / Cohort quota changes (kb_snapshot.qc_*), each scenario with
and without the edits, in one process.

Pairs of legs, alternated after a warm-up:
  - baseline: the baseline scenario (synth.perf_scenario, 15,000 workloads, 1 ms cycles, run to the end), and the same
    with a capacity dip (perf_scenario(quota=seed): every ClusterQueue of a cohort drops to half its nominal quota at
    one time and gets it back later, some lending limits, some no-op edits);
  - cfg4: the hierarchical cfg4 at full size with synth.add_events, and with synth.add_quota_changes, over --max-cycles;
  - cfg3: a cfg3 event drain (the flat route and its tree-local tables), and with synth.add_quota_changes;
  - baseline_late: the baseline scenario with the same edits moved past its natural end: the cost of carrying the table
    (the drain then jumps to every edit before it ends).
Per leg: cycles, admissions, edits applied, device ms per cycle (median / min / max) and the queue layer's time
(kernel_ms slot KB_K_DRAIN, k_drain_quota included, with kb_set_profile).  Prints one JSON line with the card name and
power limit read in the same call.

    python tools/quota_drain_bench.py [--reps 5] [--warmup 2] [--seed 3] [--max-cycles 2000]
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
    from afs_drain_bench import card
    from kueue_b200 import abi, native, synth

    base = synth.perf_scenario(1.0)
    probe = native.Evaluator(0)
    end = probe.run_drain(base, abi.DrainOut(base, 1_000_000, trace=False)).end_ns
    probe.close()
    late = synth.perf_scenario(1.0, quota=args.seed)
    late.set("qc_ns", late.arrays["qc_ns"] - late.arrays["qc_ns"].min() + end + 1)  # every edit after the natural end
    cfg4 = lambda: synth.add_events(synth.make_snapshot(4), seed=1)  # noqa: E731
    cfg3 = lambda: synth.add_events(synth.make_snapshot(3), seed=2)  # noqa: E731
    legs = {"baseline": (base, 1_000_000), "baseline_quota": (synth.perf_scenario(1.0, quota=args.seed), 1_000_000),
            "baseline_late": (late, 1_000_000),
            "cfg4": (cfg4(), args.max_cycles), "cfg4_quota": (synth.add_quota_changes(cfg4(), seed=args.seed), args.max_cycles),
            "cfg3": (cfg3(), args.max_cycles), "cfg3_quota": (synth.add_quota_changes(cfg3(), seed=args.seed), args.max_cycles)}
    ev = native.Evaluator(0)
    outs = {k: abi.DrainOut(s, max_cycles=mc, trace=False) for k, (s, mc) in legs.items()}
    for _ in range(args.warmup):
        for k, (s, _) in legs.items():
            ev.run_drain(s, outs[k])
    per_cycle, drain_ms = {k: [] for k in legs}, {k: [] for k in legs}
    for _ in range(args.reps):
        for k, (s, _) in legs.items():
            o = ev.run_drain(s, outs[k])
            per_cycle[k].append(o.gpu_ms / max(1, o.n_cycles))
    ev.set_profile(True)
    for k, (s, _) in legs.items():  # a profiled run of its own: the queue layer's share
        ev.run_drain(s, outs[k])
        drain_ms[k] = float(ev.stats().kernel_ms[13])
    ev.set_profile(False)
    res = {"what": "kb_run_drain event mode with and without ClusterQueue / Cohort quota changes", "card": card(),
           "reps": args.reps, "warmup": args.warmup, "max_cycles": args.max_cycles}
    for k, (s, _) in legs.items():
        o = ev.run_drain(s, outs[k])
        res[k] = {"cycles": o.n_cycles, "admitted": o.n_admitted, "evicted": o.n_evicted, "end_s": o.end_ns / 1e9,
                  "edits": int(len(s.arrays["qc_ns"])) if "qc_ns" in s.arrays else 0, "edits_applied": o.n_quota_changes,
                  "ms_per_cycle_median": statistics.median(per_cycle[k]), "ms_per_cycle_min": min(per_cycle[k]),
                  "ms_per_cycle_max": max(per_cycle[k]), "drain_layer_ms_profiled": drain_ms[k]}
    ev.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
