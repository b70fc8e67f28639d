"""The geometry sweep (erasor_process_nodes_tune, DESIGN.md section 8.7) on bench.py's seq 05 twin: the three KITTI geometries
(15 x 60 @ 60 m, 15 x 108 @ 60 m, 20 x 108 @ 80 m) x the five thresholds 0.10 .. 0.30, 20 nodes per call, device-resident queries,
an 80 m VoI radius.  First the masks: every arm must give the masks of 15 plain passes.  Then per lane count (1: four calls back to
back on one handle; 4: four handles sharing the map, one call each) the wall time ending in a synchronise, median of REPS after a
warm-up, of
  - one tune call (the geometries packed into K1 launches of at most 56 KB of tables);
  - the same tune call with one geometry per K1 launch (ERASOR_B200_TUNE_UNPACKED=1 on its handles);
  - one process_nodes_sweep_ex per geometry, on three handles of those geometries sharing the map;
  - 15 plain passes.
The card's name and power limit are read in the same run.  Prints one JSON line.
usage: geo_sweep_timing.py [reps]"""
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
KITTI = (dict(max_range=60.0, num_rings=15, num_sectors=60), dict(max_range=60.0, num_rings=15, num_sectors=108),
         dict(max_range=80.0, num_rings=20, num_sectors=108))
PER_CALL, LANES, VOI = 20, 4, 80.0


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def median_ms(fn):
    fn()
    ts = []
    for _ in range(REPS):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


def handle(p, m, unpacked=False):
    os.environ["ERASOR_B200_TUNE_UNPACKED"] = "1" if unpacked else "0"
    h = capi.Handle(p)
    os.environ.pop("ERASOR_B200_TUNE_UNPACKED")
    h.attach_map(m)
    return h


def main():
    p = params.preset("seq_05").replace(skip_voxelize=1)
    w = synth.make_frames(seed=5, n_frames=LANES * PER_CALL, preset_max_range=p.max_range, n_map_nodes=161, n_beams=64, n_az=1800,
                          length=160.0, n_dynamic=12, query_voxel=0.2, map_stride=2)
    n = len(w["map_world"])
    poses = np.stack([w["scene"].pose7(f[2]) for f in w["frames"]]).astype(np.float64)
    qs = [f[1] for f in w["frames"]]
    calls = []
    for c in range(LANES):
        sl = slice(c * PER_CALL, (c + 1) * PER_CALL)
        q = np.concatenate(qs[sl])
        calls.append((poses[sl], torch.from_numpy(np.ascontiguousarray(q)).cuda(), np.cumsum([0] + [len(x) for x in qs[sl]]).astype(np.uint64)))
    settings = [dict(g, scan_ratio_threshold=t) for g in KITTI for t in THRESHOLDS]
    V = len(settings)
    m = capi.Map(w["map_world"])
    keep = torch.empty(V * n, dtype=torch.uint8, device="cuda")
    tune_h = [handle(p, m) for _ in range(LANES)]
    unp_h = [handle(p, m, unpacked=True) for _ in range(LANES)]
    ex_h = [[handle(p.replace(**g), m) for g in KITTI] for _ in range(LANES)]
    plain_h = [[handle(p.replace(**s), m) for s in settings] for _ in range(LANES)]
    plain_keep = [torch.empty(n, dtype=torch.uint8, device="cuda") for _ in range(V)]

    def tune(hs, lanes):
        for i in range(lanes if lanes > 1 else LANES):
            h = hs[i if lanes > 1 else 0]
            P, dq, qo = calls[i]
            h.process_nodes_tune(P, dq.data_ptr(), qo, settings, keep.data_ptr(), voi_max_range=VOI, asynchronous=True)
            if lanes == 1:
                h.wait()
        for h in hs[:lanes]:
            h.wait()

    def ex(lanes):
        for i in range(lanes if lanes > 1 else LANES):
            for g, h in enumerate(ex_h[i if lanes > 1 else 0]):
                P, dq, qo = calls[i]
                h.process_nodes_sweep_ex(P, dq.data_ptr(), qo, settings[5 * g:5 * g + 5], keep.data_ptr() + 5 * g * n,
                                         voi_max_range=VOI, asynchronous=True)
                if lanes == 1:
                    h.wait()
        for hs in ex_h[:lanes]:
            for h in hs:
                h.wait()

    def plain(lanes):
        for i in range(lanes if lanes > 1 else LANES):
            for v, h in enumerate(plain_h[i if lanes > 1 else 0]):
                P, dq, qo = calls[i]
                h.process_nodes_ptr(P, dq.data_ptr(), qo, VOI, 0, 0, capi.PTR_DEVICE, asynchronous=True)
                if lanes == 1:
                    h.wait()
        for hs in plain_h[:lanes]:
            for h in hs:
                h.wait()

    # masks of the first call: every arm against the plain passes
    for v in range(V):
        h = plain_h[0][v]
        m.reset_keep()
        P, dq, qo = calls[0]
        h.process_nodes_ptr(P, dq.data_ptr(), qo, VOI, 0, plain_keep[v].data_ptr(), capi.PTR_DEVICE)
    ref = torch.stack(plain_keep).cpu().numpy()
    arms = {"tune": lambda hs=tune_h: hs[0].process_nodes_tune(*calls[0][:1], calls[0][1].data_ptr(), calls[0][2], settings, keep.data_ptr(), voi_max_range=VOI),
            "tune_unpacked": lambda hs=unp_h: hs[0].process_nodes_tune(*calls[0][:1], calls[0][1].data_ptr(), calls[0][2], settings, keep.data_ptr(), voi_max_range=VOI),
            "sweep_ex_per_geometry": lambda: [h.process_nodes_sweep_ex(calls[0][0], calls[0][1].data_ptr(), calls[0][2], settings[5 * g:5 * g + 5],
                                                                       keep.data_ptr() + 5 * g * n, voi_max_range=VOI) for g, h in enumerate(ex_h[0])]}
    for name, fn in arms.items():
        tune_h[0].reset_keep_mask(keep.data_ptr(), V * n)
        tune_h[0].synchronize()
        fn()
        torch.cuda.synchronize()
        assert np.array_equal(keep.reshape(V, n).cpu().numpy(), ref), name
    out = {"gpu": gpu_info(), "workload": f"bench seq05 twin, {PER_CALL} nodes per call, {V} settings (3 KITTI geometries x 5 thresholds), "
                                          f"device queries, VoI {VOI} m", "n_map": n, "reps": REPS, "masks_equal": True}
    for lanes in (1, LANES):
        out[f"lanes{lanes}_ms"] = {"tune": median_ms(lambda: tune(tune_h, lanes)), "tune_unpacked": median_ms(lambda: tune(unp_h, lanes)),
                                   "sweep_ex_per_geometry": median_ms(lambda: ex(lanes)), "plain_15": median_ms(lambda: plain(lanes))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
