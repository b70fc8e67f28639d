"""PR/RR on the device (capi.Evaluator, erasor_evaluate) against erasor_b200/evaluate.py (sklearn kd-tree, one host core) in
the same call, at two sizes.  Prints one JSON line.
  twin:    bench.py's seq 05 twin (337 k-point map), 20 nodes in node mode, the map's keep mask scored in place
  config4: a config-4-sized cloud built on the device as scripts/config4_largescale.py builds it (50 M points, seed 5) with a
           seeded 90 % keep mask; the sklearn arm scores a seeded 1 M-point GT subset, which the device also scores on its own
Device times: CUDA events around warmed, repeated synchronous calls on device pointers; the upload of the inputs from pinned host
memory is timed separately (and the host-pointer call, which includes it, is given for the twin).  The sklearn arm is warmed
(import and one small fit + query) before any timing; its best of several calls is reported, with every call's time.
usage: eval_timing.py [n_points] [reps]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from erasor_b200 import capi, synth  # noqa: E402
from erasor_b200 import evaluate as E  # noqa: E402

N_TARGET = int(sys.argv[1]) if len(sys.argv) > 1 else 50_000_000
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
KEYS4 = ("gt_static", "gt_dynamic", "preserved_static", "preserved_dynamic")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        out = f"nvidia-smi unavailable: {e}"
    return out


def events_ms(fn, reps):
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()                       # synchronous: each call ends when its stream has drained
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def h2d_ms(arrays, reps):
    pinned = [torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in arrays]
    dev = [torch.empty_like(p, device="cuda") for p in pinned]
    def copy():
        for d, p in zip(dev, pinned):
            d.copy_(p, non_blocking=True)
    return events_ms(copy, reps)


def sklearn_warm():
    """evaluate.evaluate imports sklearn inside the call: import it, and run the kd-tree once, outside every timed window"""
    rng = np.random.default_rng(0)
    c = rng.uniform(-5, 5, (2000, 4)).astype(np.float32)
    E.evaluate(c, c[::2])


def sklearn_s(gt, est, reps):
    """(result, best and every wall time of `reps` calls) -- sklearn warmed by sklearn_warm()"""
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = E.evaluate(gt, est)
        times.append(time.perf_counter() - t0)
    return r, min(times), [round(t, 3) for t in times]


def twin(ev):
    import bench
    p, map_world, poses, qs = bench.load_workload("seq05", 0, 1, 20)
    gm = capi.Map(map_world, device=0)
    h = capi.Handle(p, device=0)
    h.attach_map(gm)
    keep, _ = h.process_nodes(poses, np.concatenate(qs), np.cumsum([0] + [len(q) for q in qs]).astype(np.uint64))
    dev_ms = events_ms(lambda: ev.evaluate_map(gm), REPS)
    d = ev.evaluate_map(gm)
    c = ev.last_counts()
    host_ptr_ms = events_ms(lambda: ev.evaluate(map_world, map_world, keep=keep), REPS)
    r, sk, sk_runs = sklearn_s(map_world, map_world[keep.astype(bool)], 3)
    h.close(); gm.close()
    return {"n_gt": len(map_world), "n_est": int(keep.sum()), "device_ms": round(dev_ms, 3),
            "h2d_ms": round(h2d_ms([map_world, keep], REPS), 3), "host_pointer_call_ms": round(host_ptr_ms, 3),
            "sklearn_s": round(sk, 3), "sklearn_runs_s": sk_runs, "speedup_vs_sklearn": round(1000 * sk / dev_ms, 1),
            "counts_equal": all(d[k] == r[k] for k in KEYS4), "dict_equal": d == r,
            "inliers": c["inliers"], "ambiguous_ties": c["ambiguous_ties"], "PR": d["PR"], "RR": d["RR"]}


def config4(ev):
    w = synth.make_frames(seed=5, n_frames=6, preset_max_range=80.0, n_map_nodes=41, n_beams=32, n_az=900)
    base = w["frames"][2][0]
    base = base[(base[:, 0].astype(np.float64) ** 2 + base[:, 1].astype(np.float64) ** 2) < 82.0 ** 2]
    reps = int(np.ceil(N_TARGET / len(base)))
    g = torch.Generator(device="cuda").manual_seed(5)
    M = torch.from_numpy(base).cuda().repeat(reps, 1)
    M[:, :3] += (torch.rand((M.shape[0], 3), device="cuda", generator=g) - 0.5) * torch.tensor([0.19, 0.19, 0.02], device="cuda")
    N = M.shape[0]
    K = (torch.rand(N, device="cuda", generator=g) < 0.9).to(torch.uint8)
    torch.cuda.synchronize()       # the evaluator runs on a stream of its own
    dev_ms = events_ms(lambda: ev.evaluate_ptr(M.data_ptr(), N, M.data_ptr(), N, K.data_ptr(), 0.2, capi.PTR_DEVICE), REPS)
    d_full = ev.evaluate_ptr(M.data_ptr(), N, M.data_ptr(), N, K.data_ptr(), 0.2, capi.PTR_DEVICE)
    c_full = ev.last_counts()
    host = M.cpu().numpy()
    keep = K.cpu().numpy().astype(bool)
    h2d = h2d_ms([host, keep.view(np.uint8)], 2)
    rng = np.random.default_rng(5)
    sub = host[np.sort(rng.choice(N, 1_000_000, replace=False))]
    S = torch.from_numpy(sub).cuda()
    torch.cuda.synchronize()
    sub_ms = events_ms(lambda: ev.evaluate_ptr(S.data_ptr(), len(sub), M.data_ptr(), N, K.data_ptr(), 0.2, capi.PTR_DEVICE), REPS)
    d = ev.evaluate_ptr(S.data_ptr(), len(sub), M.data_ptr(), N, K.data_ptr(), 0.2, capi.PTR_DEVICE)
    c = ev.last_counts()
    r, sk, sk_runs = sklearn_s(sub, host[keep], 2)
    return {"n_gt": int(N), "n_est": int(keep.sum()), "device_ms": round(dev_ms, 3), "h2d_ms": round(h2d, 3),
            "full_inliers": c_full["inliers"], "full_ambiguous_ties": c_full["ambiguous_ties"], "full_PR": d_full["PR"], "full_RR": d_full["RR"],
            "subset_n_gt": len(sub), "subset_device_ms": round(sub_ms, 3), "subset_sklearn_s": round(sk, 3), "subset_sklearn_runs_s": sk_runs,
            "subset_speedup_vs_sklearn": round(1000 * sk / sub_ms, 1),
            "subset_counts_equal": all(d[k] == r[k] for k in KEYS4), "subset_dict_equal": d == r,
            "subset_inliers": c["inliers"], "subset_ambiguous_ties": c["ambiguous_ties"]}


def main():
    torch.cuda.init()
    sklearn_warm()
    ev = capi.Evaluator(device=0)
    line = {"what": "PR/RR: device evaluator (erasor_evaluate) vs erasor_b200/evaluate.py (sklearn kd-tree) in the same call",
            "gpu": gpu_info(), "reps": REPS, "twin_337k_node_mode": twin(ev), "config4_50M": config4(ev)}
    ev.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
