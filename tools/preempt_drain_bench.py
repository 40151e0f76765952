"""kb_run_drain on cfg4 with and without eviction replay (kb_snapshot.adm_wl), in one process.

The same cfg4 snapshot (1M pending workloads, 10k ClusterQueues in a depth-4 cohort forest, preemption policies) is
drained as it is and with every admitted workload evictable (synth.make_snapshot(evictable=True): a pending record per
admitted workload plus adm_wl), alternating after a warm-up.  Without replay the targets of a Preempting entry keep
their quota; with it they leave the admitted tables and return to their queues, so the two drains run different numbers
of cycles and the comparison is per cycle: device ms per cycle (kb_drain_out.gpu_ms / cycles; median, min, max), and
from one more run of each with per-kernel events the queue layer's share (KB_K_DRAIN, which holds the eviction,
requeue and compaction kernels) and the single-cell target searches' (k_search_cells).  Prints one JSON line with the
card name and power limit read in the same call.

    python tools/preempt_drain_bench.py [--reps 3] [--warmup 1] [--max-cycles 100]
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

from afs_drain_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--max-cycles", type=int, default=100)
    args = ap.parse_args()
    from kueue_b200 import abi, native, synth
    legs = {"no_replay": native.pin_snapshot(synth.make_snapshot(4)),
            "replay": native.pin_snapshot(synth.make_snapshot(4, evictable=True))}
    ev = native.Evaluator(0)
    outs = {k: abi.DrainOut(s, max_cycles=args.max_cycles, trace=False) for k, s in legs.items()}
    for _ in range(args.warmup):
        for k, s in legs.items():
            ev.run_drain(s, outs[k])
    per_cycle = {k: [] for k in legs}
    for _ in range(args.reps):
        for k, s in legs.items():
            o = ev.run_drain(s, outs[k])
            per_cycle[k].append(o.gpu_ms / max(1, o.n_cycles))
    res = {"what": "kb_run_drain cfg4, without vs with eviction replay (adm_wl)", "card": card(), "reps": args.reps,
           "warmup": args.warmup, "max_cycles": args.max_cycles}
    ev.set_profile(True)
    for k, s in legs.items():
        o = ev.run_drain(s, outs[k])
        kms = list(ev.stats().kernel_ms)
        tot = sum(kms) or 1.0
        res[k] = {"cycles": o.n_cycles, "ended_before_max_cycles": o.n_cycles < args.max_cycles, "decisions": o.n_decisions,
                  "admitted": o.n_admitted, "evicted": o.n_evicted,
                  "ms_per_cycle_median": statistics.median(per_cycle[k]), "ms_per_cycle_min": min(per_cycle[k]),
                  "ms_per_cycle_max": max(per_cycle[k]),
                  "k_drain_share_profiled": kms[abi.KERNEL_NAMES.index("k_drain")] / tot,
                  "k_search_cells_share_profiled": kms[abi.KERNEL_NAMES.index("k_search_cells")] / tot}
    ev.set_profile(False)
    ev.close()
    res["replay_over_no_replay_per_cycle"] = res["replay"]["ms_per_cycle_median"] / res["no_replay"]["ms_per_cycle_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
