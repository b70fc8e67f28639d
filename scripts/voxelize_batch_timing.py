"""Timing of erasor_voxelize_batch (DESIGN.md section 8.3) on synthetic HDL-64 scans (64 beams x 1800 azimuths, ~115 k points).

  prepare    20 raw scans -> 20 body-frame queries (leaf 0.2, seq-05 lidar2body) in one call: scans in device memory, and in pinned
             host memory (the call uploads them); CUDA events on the handle's stream around each call
  updater    the same 20 scans through 20 erasor_updater_voxelize calls (host scans; one cooperative launch and one read-back each)
  oracle     the same 20 scans through the CPU oracle's voxelize_preserving_labels on one core
  nodes      node mode end to end in the bench's pattern: 4 lanes (a handle and a host thread each) sharing one resident map, batches
             of 20 nodes; raw scans (device-resident, or pinned host) prepared by voxelize_batch then erasor_process_nodes on the device
             queries, against the same lanes fed queries prepared ahead of time (device-resident)
The arms alternate within every repetition; outputs are compared bit for bit first.  Prints one JSON object; the card's name and power
limit are read in the same run.
  usage: python scripts/voxelize_batch_timing.py [--reps 20] [--batches 40]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from erasor_b200 import capi, synth  # noqa: E402
from erasor_b200 import params as P  # noqa: E402

L2B = [0.0, 0.0, 1.73, 0.0, 0.0, 0.0, 1.0]


class Events:
    """CUDA events recorded on a given stream (the runtime the library loaded)."""

    def __init__(self):
        capi.lib()
        self.rt = ctypes.CDLL("libcudart.so.12")
        self.a, self.b = ctypes.c_void_p(), ctypes.c_void_p()
        self.rt.cudaEventCreate(ctypes.byref(self.a))
        self.rt.cudaEventCreate(ctypes.byref(self.b))

    def time_ms(self, stream: int, fn) -> float:
        self.rt.cudaEventRecord(self.a, ctypes.c_void_p(stream))
        fn()
        self.rt.cudaEventRecord(self.b, ctypes.c_void_p(stream))
        self.rt.cudaEventSynchronize(self.b)
        ms = ctypes.c_float()
        self.rt.cudaEventElapsedTime(ctypes.byref(ms), self.a, self.b)
        return float(ms.value)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def stats(v):
    v = np.asarray(v, dtype=np.float64)
    return {"median_ms": round(float(np.median(v)), 3), "min_ms": round(float(v.min()), 3), "max_ms": round(float(v.max()), 3), "n": int(len(v))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batches", type=int, default=40)
    a = ap.parse_args()
    import torch
    from oracle import oracle_py

    sc = synth.Scene(seed=5, length=160.0, n_nodes=161, n_dynamic=12)
    ks = list(range(0, 160, 8))
    scans = [sc.scan(k) for k in ks]
    off = np.cumsum([0] + [len(s) for s in scans]).astype(np.uint64)
    raw = np.concatenate(scans)
    raw_pin = torch.from_numpy(raw).pin_memory()
    raw_dev = torch.from_numpy(raw).cuda()
    ep, up = P.preset("seq_05"), P.updater_preset("seq_05")
    h = capi.Handle(ep)
    ev = Events()
    mw = sc.build_map(range(0, 161, 2), voxel=0.2, n_beams=64, n_az=1800)
    u = capi.Updater(up, ep, mw[:10])
    u_stream = int(capi.lib().erasor_stream(capi.lib().erasor_updater_erasor(u.h)) or 0)

    # the same bits from every arm
    vox, oo = h.voxelize_batch(raw, off, 0.2, pose7=L2B)
    for i, s in enumerate(scans):
        want = oracle_py.transform(oracle_py.voxelize(s, 0.2), oracle_py.pose_to_matrix(L2B))
        assert np.array_equal(vox[int(oo[i]):int(oo[i + 1])].view(np.uint32), want.view(np.uint32)), f"scan {i}"
        assert np.array_equal(u.voxelize(s, 0.2).view(np.uint32), oracle_py.voxelize(s, 0.2).view(np.uint32))

    arms = {"prepare_device": [], "prepare_pinned": [], "updater_20_calls": []}
    run = {
        "prepare_device": (h.stream, lambda: h.voxelize_batch_ptr(raw_dev.data_ptr(), off, 0.2, 0, L2B, capi.PTR_DEVICE)),
        "prepare_pinned": (h.stream, lambda: h.voxelize_batch_ptr(raw_pin.data_ptr(), off, 0.2, 0, L2B, capi.PTR_HOST)),
        "updater_20_calls": (u_stream, lambda: [u.voxelize(s, 0.2) for s in scans]),
    }
    for _ in range(3):                                     # warm-up of every shape
        for name, (st, fn) in run.items():
            ev.time_ms(st, fn)
    launches0 = h.kernel_launch_count()
    h.voxelize_batch_ptr(raw_dev.data_ptr(), off, 0.2, 0, L2B, capi.PTR_DEVICE)
    launches = h.kernel_launch_count() - launches0
    for _ in range(a.reps):
        for name, (st, fn) in run.items():
            arms[name].append(ev.time_ms(st, fn))
    t0 = time.perf_counter()
    for s in scans:
        oracle_py.voxelize(s, 0.2)
    oracle_ms = (time.perf_counter() - t0) * 1e3

    # node mode, 4 lanes over one resident map
    m = capi.Map(mw)
    lanes = [capi.Handle(ep.replace(version=up.version)) for _ in range(4)]
    for x in lanes:
        x.attach_map(m)
    poses = np.ascontiguousarray(np.stack([sc.pose7(k) for k in ks]), dtype=np.float64)
    qv, qo = h.voxelize_batch(raw, off, up.query_voxel_size, pose7=up.lidar2body)
    q_dev = torch.from_numpy(qv).cuda()
    torch.cuda.synchronize()

    def lane_raw(x, src_ptr, kind, n):
        for _ in range(n):
            d, o = x.voxelize_batch_ptr(src_ptr, off, up.query_voxel_size, 0, up.lidar2body, kind)
            x.process_nodes_ptr(poses, d, o, up.max_range, 0, 0, capi.PTR_DEVICE)

    def lane_prepared(x, n):
        for _ in range(n):
            x.process_nodes_ptr(poses, q_dev.data_ptr(), qo, up.max_range, 0, 0, capi.PTR_DEVICE)

    def four_lanes(target):
        per = a.batches // 4
        th = [threading.Thread(target=target, args=(x, per)) for x in lanes]
        t = time.perf_counter()
        for t_ in th:
            t_.start()
        for t_ in th:
            t_.join()
        for x in lanes:
            x.synchronize()
        return 4 * per * len(ks) / (time.perf_counter() - t)

    node_arms = {"raw_device": lambda x, n: lane_raw(x, raw_dev.data_ptr(), capi.PTR_DEVICE, n),
                 "raw_pinned": lambda x, n: lane_raw(x, raw_pin.data_ptr(), capi.PTR_HOST, n),
                 "prepared_device": lane_prepared}
    for f in node_arms.values():
        four_lanes(f)
    rates = {k: [] for k in node_arms}
    for _ in range(5):
        for k, f in node_arms.items():
            rates[k].append(four_lanes(f))
    out = {
        "card": card(),
        "scans": len(scans), "raw_points": int(len(raw)), "voxels": int(oo[-1]),
        "launches_per_prepare": int(launches),
        "prepare_20_scans": {k: stats(v) for k, v in arms.items()},
        "oracle_one_core_20_scans_ms": round(oracle_ms, 1),
        "node_mode_scans_per_s_4_lanes": {k: {"median": round(float(np.median(v))), "min": round(float(min(v))), "max": round(float(max(v)))}
                                          for k, v in rates.items()},
    }
    print(json.dumps(out))
    for x in lanes:
        x.close()
    m.close(); u.close(); h.close()


if __name__ == "__main__":
    main()
