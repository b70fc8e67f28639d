"""Per-phase cycle profile of K1's node-mode map path on the bench workload (needs the GPU).
usage: k1_profile.py [config] [frames] [repeats]

Runs the bench step, then K1 of that step again as its profiling build (erasor_profile_k1): lane 0 of every warp adds the
SM cycles between consecutive phase boundaries to the warp's counters.  A phase ends at the instruction that waits for its
results, so a load's exposed latency lands in "scan" and shared-memory back-pressure in whichever phase issues the next
shared access.  Prints each phase's share of the map warps' cycles, cycles per dense row, and the spread of the CTAs'
times; the product kernel's own time (CUDA events, same step) is printed beside it, with the card and its power limit."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import bench  # noqa: E402
from erasor_b200 import capi  # noqa: E402

PHASES = ["scan", "compact", "bin", "table", "lists", "flush"]

config = sys.argv[1] if len(sys.argv) > 1 else "seq05"
frames = int(sys.argv[2]) if len(sys.argv) > 2 else bench.FRAMES_PER_PASS
repeats = int(sys.argv[3]) if len(sys.argv) > 3 else 5

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip().splitlines()
print("card:", card[0] if card else "unknown")

p, map_world, poses, qs = bench.load_workload(config, 0, 1, frames)
qo = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint64)
Q = np.concatenate(qs)
m = capi.Map(map_world)
h = capi.Handle(p)
h.attach_map(m)
for _ in range(3):
    h.process_nodes(poses, Q, qo)
h.reset_kernel_times(True)
for _ in range(20):
    h.process_nodes(poses, Q, qo)
k1_ms, k1_n = h.kernel_time_ms(1)
h.reset_kernel_times(False)
h.process_nodes(poses, Q, qo)
print(f"product K1: {k1_ms / k1_n:.4f} ms per launch (CUDA events, {k1_n} launches)")

runs = np.stack([h.k1_profile() for _ in range(repeats)]).astype(np.float64)   # [repeat, chunk, warp, slot]
prof = np.median(runs, axis=0)
rows = runs[0, :, :, 7]
is_map = ~(runs[0, :, 0, 7] == 0xFFFFFFFF)
pm = prof[is_map]                                   # map chunks: [chunk, warp, slot]
tot_phase = pm[:, :, :6].sum(axis=(0, 1))
n_rows = rows[is_map].sum()
print(f"{int(is_map.sum())} map chunks x {prof.shape[1]} warps, {int((~is_map).sum())} query chunks; "
      f"{int(n_rows)} dense rows; profiling-build kernel median of {repeats}")
print("phase shares of the map warps' cycles (cycles per dense row):")
for k, name in enumerate(PHASES):
    print(f"  {name:8s} {tot_phase[k] / tot_phase.sum():6.3f}  ({tot_phase[k] / max(n_rows, 1):8.1f})")
cta_map = pm[:, :, 6].max(axis=1)
print("map CTA time, cycles (max over its warps): min %d  median %d  max %d  (max / median %.2f)"
      % (cta_map.min(), np.median(cta_map), cta_map.max(), cta_map.max() / np.median(cta_map)))
work = pm[:, :, :6].sum(axis=2) - pm[:, :, 5]       # a warp's cycles before its CTA barrier
print("map warp time before the barrier, cycles: min %d  median %d  max %d; dense rows per warp: min %d  median %d  max %d"
      % (work.min(), np.median(work), work.max(), rows[is_map].min(), np.median(rows[is_map]), rows[is_map].max()))
if (~is_map).any():
    cq = prof[~is_map][:, :, 6].max(axis=1)
    print("query CTA time, cycles: min %d  median %d  max %d" % (cq.min(), np.median(cq), cq.max()))
h.close()
m.close()
