"""kb_run_drain in event mode on cfg3 with AdmissionFairSharing, with and without the decay tables, in one process.

The same snapshot (1M pending workloads, 10k ClusterQueues, 8 LocalQueues each: synth.add_afs, events: synth.add_events)
is drained without the decay tables and with them (synth.add_afs_decay: a sample every --sampling cycles, a half-life
of --half-life cycles), alternating after a warm-up.  The two drains admit different workloads, so the comparison is
per cycle: device ms per cycle, the queue layer's share (KB_K_DRAIN, from one more run of each with per-kernel events),
cycles, admissions and decay samples.  Prints one JSON line with the card name and power limit read in the same call.

    python tools/afs_decay_drain_bench.py [--reps 5] [--warmup 2] [--max-cycles 300]
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
    ap.add_argument("--lq", type=int, default=8)
    ap.add_argument("--sampling", type=int, default=20, help="sampling interval in cycles")
    ap.add_argument("--half-life", type=int, default=100, help="half-life in cycles")
    ap.add_argument("--max-cycles", type=int, default=300)
    args = ap.parse_args()
    from afs_drain_bench import card
    from kueue_b200 import abi, native, synth
    plain = synth.add_events(synth.make_snapshot(3, afs=args.lq), seed=1)
    decay = synth.add_events(synth.make_snapshot(3, afs=args.lq), seed=1)
    step = decay.drain_cycle_ns
    synth.add_afs_decay(decay, seed=2, half_life_ns=args.half_life * step, sampling_ns=args.sampling * step)
    ev = native.Evaluator(0)
    legs = {"no_decay": plain, "decay": decay}
    outs = {k: abi.DrainOut(s, max_cycles=args.max_cycles, trace=False) for k, s in legs.items()}
    for _ in range(args.warmup):
        for k, s in legs.items():
            ev.run_drain(s, outs[k])
    per_cycle = {k: [] for k in legs}
    for _ in range(args.reps):
        for k, s in legs.items():
            o = ev.run_drain(s, outs[k])
            per_cycle[k].append(o.gpu_ms / max(1, o.n_cycles))
    res = {"what": "kb_run_drain cfg3 event mode with AFS, without vs with the decay tables", "local_queues_per_cq": args.lq,
           "sampling_cycles": args.sampling, "half_life_cycles": args.half_life, "card": card(), "reps": args.reps,
           "warmup": args.warmup, "max_cycles": args.max_cycles}
    ev.set_profile(True)
    slot = abi.KERNEL_NAMES.index("k_drain")
    for k, s in legs.items():
        o = ev.run_drain(s, outs[k])
        st = ev.stats()
        res[k] = {"cycles": o.n_cycles, "admitted": o.n_admitted, "finished": o.n_finished, "afs_samples": o.n_afs_samples,
                  "kernel_launches": st.kernel_launches,
                  "ms_per_cycle_median": statistics.median(per_cycle[k]), "ms_per_cycle_min": min(per_cycle[k]),
                  "ms_per_cycle_max": max(per_cycle[k]), "k_drain_ms_per_cycle_profiled": st.kernel_ms[slot] / max(1, o.n_cycles)}
    ev.set_profile(False)
    ev.close()
    res["decay_over_no_decay_per_cycle"] = res["decay"]["ms_per_cycle_median"] / res["no_decay"]["ms_per_cycle_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
