"""kb_run_drain on cfg3 with and without AdmissionFairSharing tables, in one process.

The same snapshot (1M pending workloads, 10k ClusterQueues in flat cohorts) is drained plain and with 8 LocalQueues per
ClusterQueue (synth.add_afs), alternating after a warm-up.  The two drains admit different workloads and run different
numbers of cycles, so the comparison is per cycle: device ms per cycle (kb_drain_out.gpu_ms / cycles) and the queue
layer's share (KB_K_DRAIN, from one more run of each with per-kernel events).  Prints one JSON line with the card name
and power limit read in the same call.

    python tools/afs_drain_bench.py [--reps 5] [--warmup 2] [--lq 8] [--max-cycles 1000]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """name and power limit of GPU 0 (read-only query)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001 — no nvidia-smi: report what is known
        return {"name": None, "power_limit": None, "error": type(e).__name__}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lq", type=int, default=8)
    ap.add_argument("--max-cycles", type=int, default=1000)
    args = ap.parse_args()
    from kueue_b200 import abi, native, synth
    plain = native.pin_snapshot(synth.make_snapshot(3))
    afs = native.pin_snapshot(synth.make_snapshot(3, afs=args.lq))
    ev = native.Evaluator(0)
    legs = {"plain": plain, "afs": afs}
    outs = {k: abi.DrainOut(s, max_cycles=args.max_cycles, trace=False) for k, s in legs.items()}
    for _ in range(args.warmup):
        for k, s in legs.items():
            ev.run_drain(s, outs[k])
    per_cycle = {k: [] for k in legs}
    gpu_ms = {k: [] for k in legs}
    for _ in range(args.reps):
        for k, s in legs.items():
            o = ev.run_drain(s, outs[k])
            gpu_ms[k].append(o.gpu_ms)
            per_cycle[k].append(o.gpu_ms / max(1, o.n_cycles))
    res = {"what": "kb_run_drain cfg3, plain vs AdmissionFairSharing tables", "local_queues_per_cq": args.lq,
           "card": card(), "reps": args.reps, "warmup": args.warmup}
    ev.set_profile(True)
    drain_slot = abi.KERNEL_NAMES.index("k_drain")
    for k, s in legs.items():
        o = ev.run_drain(s, outs[k])
        st = ev.stats()
        kms = list(st.kernel_ms)
        res[k] = {"cycles": o.n_cycles, "decisions": o.n_decisions, "admitted": o.n_admitted,
                  "gpu_ms_median": statistics.median(gpu_ms[k]), "ms_per_cycle_median": statistics.median(per_cycle[k]),
                  "ms_per_cycle_min": min(per_cycle[k]), "ms_per_cycle_max": max(per_cycle[k]),
                  "queue_layer_ms_per_cycle_profiled": kms[drain_slot] / max(1, o.n_cycles),
                  "k_cycle_flat_ms_per_cycle_profiled": kms[abi.KERNEL_NAMES.index("k_cycle_flat")] / max(1, o.n_cycles)}
    ev.set_profile(False)
    ev.close()
    res["afs_over_plain_per_cycle"] = res["afs"]["ms_per_cycle_median"] / res["plain"]["ms_per_cycle_median"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
