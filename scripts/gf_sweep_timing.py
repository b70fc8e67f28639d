"""The Scan Ratio Test and ground-filter sweep (erasor_process_nodes_sweep_ex, DESIGN.md section 8.6) on bench.py's seq 05 twin: the
README's five thresholds (0.10 .. 0.30) x gf_dist_thr {0.075, 0.15, 0.25} (the values of the reference's configs), 20 nodes per call,
1 and 4 lanes (handles sharing one map; 4 lanes take 80 nodes).  First the masks: each mask of the sweep must equal the map's keep
mask after plain passes with that setting, and the three Scan Ratio Test sweeps (one per gf_dist_thr) must give the same masks.  Then
per lane count the wall time (ending in a synchronise), median of REPS after a warm-up, of
  - one 15-setting sweep, against 15 plain passes (the sum of the per-setting medians: each setting's four handles exist only
    while it is timed) and against three process_nodes_sweep calls, one per gf_dist_thr;
  - process_nodes_sweep and the one-group process_nodes_sweep_ex on the five thresholds, timed alternately in the same run.
Also: union-flagged bins, R-GPF points and fits of one call, and PR / RR / F1 per setting with the initial map as GT (capi.Evaluator,
voxelsize 0.2).  The card's name and power limit are read in the same run.  Prints one JSON line.
usage: gf_sweep_timing.py [reps]"""
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
DIST_THR = (0.075, 0.15, 0.25)
PER_CALL = 20


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def time_s(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def median_s(fn):
    fn()
    return float(np.median([time_s(fn) for _ in range(REPS)]))


def main():
    p = params.preset("seq_05").replace(skip_voxelize=1)
    w = synth.make_frames(seed=5, n_frames=4 * PER_CALL, preset_max_range=p.max_range, n_map_nodes=161, n_beams=64, n_az=1800, length=160.0,
                          n_dynamic=12, query_voxel=0.2, map_stride=2)
    map_world = w["map_world"]
    n = len(map_world)
    poses = np.stack([w["scene"].pose7(f[2]) for f in w["frames"]]).astype(np.float64)
    qs = [f[1] for f in w["frames"]]
    calls = []
    for g in range(4):
        sl = slice(g * PER_CALL, (g + 1) * PER_CALL)
        calls.append(dict(poses=np.ascontiguousarray(poses[sl]), qo=np.cumsum([0] + [len(q) for q in qs[sl]]).astype(np.uint64),
                          dQ=torch.from_numpy(np.concatenate(qs[sl])).cuda()))
    settings = [dict(scan_ratio_threshold=t, gf_dist_thr=d) for t in THRESHOLDS for d in DIST_THR]
    variants = [dict(scan_ratio_threshold=t) for t in THRESHOLDS]
    V, T = len(settings), len(THRESHOLDS)
    m = capi.Map(map_world)
    sweep_h = [capi.Handle(p) for _ in range(4)]
    srt_h = [[capi.Handle(p.replace(gf_dist_thr=d)) for _ in range(4)] for d in DIST_THR]
    for h in sweep_h + [h for row in srt_h for h in row]:
        h.attach_map(m)
    keep = torch.empty(V * n, dtype=torch.uint8, device="cuda")
    keep_srt = torch.empty(V * n, dtype=torch.uint8, device="cuda")      # [gf_dist_thr][threshold][n]
    out = dict(gpu=gpu_info(), workload=f"seq05 twin, {n} map points, {PER_CALL} nodes per call", thresholds=THRESHOLDS, gf_dist_thr=DIST_THR,
               reps=REPS)

    def run(handles, lanes, submit):
        for k in range(4):                     # 1 lane: the four calls back to back on one handle; 4 lanes: one call per handle
            h, c = handles[k % lanes], calls[k]
            submit(h, c)
            if lanes == 1:
                h.wait()
        for h in handles[:lanes]:
            h.wait()

    def sweep_ex(lanes, ss=settings, buf=keep):
        sweep_h[0].reset_keep_mask(buf.data_ptr(), len(ss) * n)
        sweep_h[0].synchronize()
        run(sweep_h, lanes, lambda h, c: h.process_nodes_sweep_ex(c["poses"], c["dQ"].data_ptr(), c["qo"], ss, buf.data_ptr(), asynchronous=True))

    def sweep_srt(lanes):
        sweep_h[0].reset_keep_mask(keep.data_ptr(), T * n)
        sweep_h[0].synchronize()
        run(sweep_h, lanes, lambda h, c: h.process_nodes_sweep(c["poses"], c["dQ"].data_ptr(), c["qo"], variants, keep.data_ptr(), asynchronous=True))

    def three_srt(lanes):
        sweep_h[0].reset_keep_mask(keep_srt.data_ptr(), V * n)
        sweep_h[0].synchronize()
        for i in range(len(DIST_THR)):
            run(srt_h[i], lanes, lambda h, c: h.process_nodes_sweep(c["poses"], c["dQ"].data_ptr(), c["qo"], variants,
                                                                      keep_srt.data_ptr() + i * T * n, asynchronous=True))

    def plain_handles(v):
        hs = [capi.Handle(p.replace(**settings[v])) for _ in range(4)]
        for h in hs:
            h.attach_map(m)
        return hs

    def plain(handles, lanes):
        m.reset_keep()
        run(handles, lanes, lambda h, c: h.process_nodes_ptr(c["poses"], c["dQ"].data_ptr(), c["qo"], 0.0, 0, 0, capi.PTR_DEVICE, asynchronous=True))

    # masks first: the sweep against plain passes, and against the three Scan Ratio Test sweeps
    for lanes in (1, 4):
        sweep_ex(lanes)
        got = keep.reshape(V, n).cpu().numpy()
        for v in range(V):
            hs = plain_handles(v)
            plain(hs, lanes)
            for h in hs:
                h.close()
            if not np.array_equal(got[v], m.get_keep()):
                raise SystemExit(f"{lanes} lanes, {settings[v]}: the sweep mask differs from the plain pass")
        three_srt(lanes)
        srt = keep_srt.reshape(len(DIST_THR), T, n).cpu().numpy()
        for v, s in enumerate(settings):
            if not np.array_equal(got[v], srt[DIST_THR.index(s["gf_dist_thr"]), THRESHOLDS.index(s["scan_ratio_threshold"])]):
                raise SystemExit(f"{lanes} lanes, {s}: the sweep mask differs from the Scan Ratio Test sweep")
    out["masks_equal"] = True
    for lanes in (1, 4):
        t_sweep = median_s(lambda: sweep_ex(lanes))
        t_three = median_s(lambda: three_srt(lanes))
        t_plain = 0.0
        for v in range(V):
            hs = plain_handles(v)
            t_plain += median_s(lambda: plain(hs, lanes))
            for h in hs:
                h.close()
        # process_nodes_sweep against the one-group process_nodes_sweep_ex (the handle's gf_dist_thr), alternately
        sweep_srt(lanes)
        sweep_ex(lanes, variants)
        srt_t, one_t = [], []
        for _ in range(REPS):
            srt_t.append(time_s(lambda: sweep_srt(lanes)))
            one_t.append(time_s(lambda: sweep_ex(lanes, variants)))
        out[f"lanes{lanes}"] = dict(sweep15_ms=1e3 * t_sweep, plain15_ms=1e3 * t_plain, three_srt_sweeps_ms=1e3 * t_three,
                                    speedup_vs_plain=t_plain / t_sweep, speedup_vs_three_srt=t_three / t_sweep,
                                    srt_sweep5_ms=1e3 * float(np.median(srt_t)), one_group_sweep_ex5_ms=1e3 * float(np.median(one_t)))
    # union-flagged bins, R-GPF points and fits of one call (flags grow with the threshold, so each gf_dist_thr group fits the
    # bins its 0.30 setting flags)
    c = calls[0]
    sweep_h[0].reset_keep_mask(keep.data_ptr(), V * n)
    sweep_h[0].process_nodes_sweep_ex(c["poses"], c["dQ"].data_ptr(), c["qo"], settings, keep.data_ptr())
    _, uf, _ = sweep_h[0].node_stats()
    nf, _ = sweep_h[0].sweep_stats()
    upts, _ = sweep_h[0].rgpf_profile()
    top = [settings.index(dict(scan_ratio_threshold=THRESHOLDS[-1], gf_dist_thr=d)) for d in DIST_THR]
    out["per_call"] = dict(union_flagged_bins=int(uf.sum()), rgpf_points=int(upts.sum()), fits=int(sum(nf[v].sum() for v in top)),
                           plain_fits=int(nf.sum()))
    # quality per setting over all 80 nodes
    sweep_ex(4)
    with capi.Evaluator() as ev:
        out["quality"] = [dict(**s, **{k: ev.evaluate_ptr(m.points_ptr, n, m.points_ptr, n, keep.data_ptr() + v * n)[k] for k in ("PR", "RR", "F1")})
                          for v, s in enumerate(settings)]
    for h in sweep_h + [h for row in srt_h for h in row]:
        h.close()
    m.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
