"""kb_run_drain with and without the sticky-workload table (kb_snapshot.cq_sticky, every slot -1 at the start), in one
process.

Pairs, each run with and without the table, alternated after a warm-up: the baseline scenario (synth.perf_scenario,
15,000 workloads, 1 ms cycles, run to the end) with a termination latency of --baseline-ms, the same without latency, the
same with a termination latency of --long-ms, and cfg4 at full size with events (synth.add_events) and latencies drawn in
[--cfg4-lo, --cfg4-hi] cycles (synth.add_evict_latency) over --max-cycles cycles.  Per leg: cycles, admissions,
evictions issued and completed, the end time, per-class mean admit wait (baseline: last admission - creation, over the
workloads admitted), device ms per cycle (median / min / max), and the queue layer's share of the device time
(KB_K_DRAIN, from one more run of each with per-kernel events).  Per pair: the ratio of the median ms per cycle with the
table to without.  Prints one JSON line with the card name and power limit read in the same call.

    python tools/sticky_drain_bench.py [--reps 5] [--warmup 2] [--max-cycles 300]
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
    ap.add_argument("--max-cycles", type=int, default=300, help="cycles of the cfg4 legs (the baseline runs to the end)")
    ap.add_argument("--baseline-ms", type=int, default=30, help="termination latency of the baseline scenario, ms")
    ap.add_argument("--long-ms", type=int, default=150, help="a second, longer termination latency of the baseline, ms")
    ap.add_argument("--cfg4-lo", type=int, default=5, help="smallest cfg4 latency, in cycles")
    ap.add_argument("--cfg4-hi", type=int, default=40, help="largest cfg4 latency, in cycles")
    args = ap.parse_args()
    from afs_drain_bench import card
    from kueue_b200 import abi, native, synth
    ms = 1_000_000

    def cfg4():
        snap = synth.add_events(synth.make_snapshot(4, evictable=True), seed=3)
        step = snap.drain_cycle_ns
        return synth.add_evict_latency(snap, (args.cfg4_lo * step, args.cfg4_hi * step), seed=4)
    pairs = {
        f"baseline_latency_{args.baseline_ms}ms": (lambda: synth.perf_scenario(1.0, evict_ns=args.baseline_ms * ms), 1_000_000),
        "baseline_no_latency": (lambda: synth.perf_scenario(1.0), 1_000_000),
        f"baseline_latency_{args.long_ms}ms": (lambda: synth.perf_scenario(1.0, evict_ns=args.long_ms * ms), 1_000_000),
        f"cfg4_latency_{args.cfg4_lo}_{args.cfg4_hi}_cycles": (cfg4, args.max_cycles),
    }
    legs = {}
    for k, (make, mc) in pairs.items():
        legs[f"{k}/without"] = (make(), mc)
        snap = make()
        snap.set("cq_sticky", np.full(snap.n_cq, -1))
        legs[f"{k}/with"] = (snap, mc)
    ev = native.Evaluator(0)
    outs = {k: abi.DrainOut(s, max_cycles=mc, trace=False) for k, (s, mc) in legs.items()}
    for _ in range(args.warmup):
        for k, (s, _) in legs.items():
            ev.run_drain(s, outs[k])
    per_cycle = {k: [] for k in legs}
    for _ in range(args.reps):
        for k, (s, _) in legs.items():
            o = ev.run_drain(s, outs[k])
            per_cycle[k].append(o.gpu_ms / max(1, o.n_cycles))
    res = {"what": "kb_run_drain with and without the sticky-workload table", "card": card(), "reps": args.reps,
           "warmup": args.warmup, "max_cycles_cfg4": args.max_cycles, "baseline_cycle_ms": 1,
           "cfg4_cycle_ns": legs[f"cfg4_latency_{args.cfg4_lo}_{args.cfg4_hi}_cycles/without"][0].drain_cycle_ns}
    ev.set_profile(True)
    slot = abi.KERNEL_NAMES.index("k_drain")
    for k, (s, _) in legs.items():
        o = ev.run_drain(s, outs[k])
        st = ev.stats()
        leg = {"cycles": o.n_cycles, "admitted": o.n_admitted, "finished": o.n_finished, "evictions_issued": o.n_evicted,
               "evictions_completed": o.n_evict_done, "end_s": o.end_ns / 1e9,
               "ms_per_cycle_median": statistics.median(per_cycle[k]), "ms_per_cycle_min": min(per_cycle[k]),
               "ms_per_cycle_max": max(per_cycle[k]),
               "k_drain_share_profiled": st.kernel_ms[slot] / max(1e-9, o.gpu_ms)}
        if k.startswith("baseline"):
            admitted = o.wl_admit_ns != abi.KB_TS_UNSET
            wait = (o.wl_admit_ns - s.arrays["wl_create_ns"]) / 1e6
            leg["mean_admit_wait_ms"] = {name: float(wait[admitted & (s.perf_class == c)].mean())
                                         for c, (name, *_rest) in enumerate(synth.PERF_CLASSES)}
        res[k] = leg
    ev.set_profile(False)
    ev.close()
    for k in pairs:
        res[f"{k}/cost_ratio_with_over_without"] = res[f"{k}/with"]["ms_per_cycle_median"] / res[f"{k}/without"]["ms_per_cycle_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
