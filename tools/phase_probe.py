"""Phase times of the fused cfg3 kernel (thread 0 of CTA 0, cycles): python tools/phase_probe.py [cold]
cold = a 512 MiB buffer is written between cycles (L2 flushed, like bench.py's timed steps)."""
import sys; sys.path.insert(0,'.')
from kueue_b200 import abi, native, synth
cold = len(sys.argv) > 1 and sys.argv[1] == "cold"
snap = synth.compact_to_heads(synth.make_snapshot(3, heads="one_per_cq"))
ev = native.Evaluator(0); ev.upload(snap); ev.set_profile(True)
if cold:
    import torch
    flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
for _ in range(4):
    if cold:
        flush.zero_(); torch.cuda.synchronize()
    ev.cycle_resident()
st = ev.stats(); print("cold" if cold else "warm", "cycle ms", st.last_cycle_gpu_ms, [ (abi.KERNEL_NAMES[i], round(st.kernel_ms[i],4)) for i in range(16) if st.kernel_ms[i]>0])
print("phase cycles (k_cycle_flat: stage A, entries+records+tree+stage B, nominate+keys+requests, rank+thresholds, ordered loop+publish, publish tail):", list(st.search_stat)[:6])
