"""The Scan Ratio Test sweep (erasor_process_nodes_sweep, DESIGN.md section 8.5) against plain node-mode passes on bench.py's seq 05
twin: the README's five thresholds (0.10 .. 0.30), 20 nodes per call, 1 and 4 lanes (handles sharing one map; 4 lanes take 80 nodes).
First the masks: each sweep mask must equal the map's keep mask after plain passes with that threshold.  Then per lane count the
wall time (ending in a synchronise) of one sweep over the nodes against five plain passes, median of REPS after a warm-up; the
union-flagged bins and R-GPF points of the sweep against the default setting (0.30, seq_05.yaml); PR / RR / F1 per threshold with
the initial map as GT (capi.Evaluator, voxelsize 0.2).  The card's name and power limit are read in the same run.  Prints one JSON
line.
usage: srt_sweep_timing.py [reps]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from erasor_b200 import capi, params, synth  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 10
THRESHOLDS = (0.10, 0.15, 0.20, 0.25, 0.30)
PER_CALL = 20


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def median_s(fn):
    fn()
    times = []
    for _ in range(REPS):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return float(np.median(times))


def main():
    p = params.preset("seq_05").replace(skip_voxelize=1)
    w = synth.make_frames(seed=5, n_frames=4 * PER_CALL, preset_max_range=p.max_range, n_map_nodes=161, n_beams=64, n_az=1800, length=160.0,
                          n_dynamic=12, query_voxel=0.2, map_stride=2)
    map_world = w["map_world"]
    n = len(map_world)
    poses = np.stack([w["scene"].pose7(f[2]) for f in w["frames"]]).astype(np.float64)
    qs = [f[1] for f in w["frames"]]
    groups = []
    for g in range(4):
        sl = slice(g * PER_CALL, (g + 1) * PER_CALL)
        Q = np.concatenate(qs[sl])
        groups.append(dict(poses=np.ascontiguousarray(poses[sl]), qo=np.cumsum([0] + [len(q) for q in qs[sl]]).astype(np.uint64),
                           dQ=torch.from_numpy(Q).cuda()))
    variants = [dict(scan_ratio_threshold=t) for t in THRESHOLDS]
    V = len(variants)
    m = capi.Map(map_world)
    sweep_h = [capi.Handle(p) for _ in range(4)]
    plain_h = [[capi.Handle(p.replace(**v)) for _ in range(4)] for v in variants]
    for h in sweep_h + [h for row in plain_h for h in row]:
        h.attach_map(m)
    keep = torch.empty(V * n, dtype=torch.uint8, device="cuda")
    out = dict(gpu=gpu_info(), workload=f"seq05 twin, {n} map points, {PER_CALL} nodes per call", thresholds=THRESHOLDS, reps=REPS)

    def sweep(lanes):
        sweep_h[0].reset_keep_mask(keep.data_ptr(), V * n)
        sweep_h[0].synchronize()
        for k in range(4):                     # 1 lane: the four calls back to back on one handle; 4 lanes: one call per handle
            h, g = sweep_h[k % lanes], groups[k]
            h.process_nodes_sweep(g["poses"], g["dQ"].data_ptr(), g["qo"], variants, keep.data_ptr(), asynchronous=True)
            if lanes == 1:
                h.wait()
        for h in sweep_h[:lanes]:
            h.wait()

    def plain(lanes, v):
        m.reset_keep()
        for k in range(4):
            h, g = plain_h[v][k % lanes], groups[k]
            h.process_nodes_ptr(g["poses"], g["dQ"].data_ptr(), g["qo"], 0.0, 0, 0, capi.PTR_DEVICE, asynchronous=True)
            if lanes == 1:
                h.wait()
        for h in plain_h[v][:lanes]:
            h.wait()

    # masks first
    for lanes in (1, 4):
        sweep(lanes)
        got = keep.reshape(V, n).cpu().numpy()
        for v in range(V):
            plain(lanes, v)
            if not np.array_equal(got[v], m.get_keep()):
                raise SystemExit(f"{lanes} lanes, threshold {THRESHOLDS[v]}: the sweep mask differs from the plain pass")
    out["masks_equal"] = True
    for lanes in (1, 4):
        t_sweep = median_s(lambda: sweep(lanes))
        t_plain = median_s(lambda: [plain(lanes, v) for v in range(V)])
        out[f"lanes{lanes}"] = dict(sweep_ms=1e3 * t_sweep, five_plain_ms=1e3 * t_plain, speedup=t_plain / t_sweep)
    # union-flagged bins and R-GPF points of one call against the default setting (0.30)
    g = groups[0]
    sweep_h[0].reset_keep_mask(keep.data_ptr(), V * n)
    sweep_h[0].process_nodes_sweep(g["poses"], g["dQ"].data_ptr(), g["qo"], variants, keep.data_ptr())
    _, uf, _ = sweep_h[0].node_stats()
    upts, _ = sweep_h[0].rgpf_profile()
    d = plain_h[V - 1][0]
    d.process_nodes_ptr(g["poses"], g["dQ"].data_ptr(), g["qo"], 0.0, 0, 0, capi.PTR_DEVICE)
    _, df, _ = d.node_stats()
    dpts, _ = d.rgpf_profile()
    out["union_vs_default"] = dict(flagged_bins=int(uf.sum()), default_flagged_bins=int(df.sum()), rgpf_points=int(upts.sum()),
                                   default_rgpf_points=int(dpts.sum()))
    # quality per threshold over all 80 nodes
    sweep(4)
    with capi.Evaluator() as ev:
        out["quality"] = [dict(scan_ratio_threshold=t, **{k: ev.evaluate_ptr(m.points_ptr, n, m.points_ptr, n, keep.data_ptr() + v * n)[k]
                                                           for k in ("PR", "RR", "F1")}) for v, t in enumerate(THRESHOLDS)]
    for h in sweep_h + [h for row in plain_h for h in row]:
        h.close()
    m.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
