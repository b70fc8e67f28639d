"""Times erasor_bag_index / erasor_bag_load (DESIGN.md section 12.2) on a synthetic bag shaped like the seq 05 twin: 161 nodes (+ the
duplicated first frame) of N points in pcl::toROSMsg's 32-byte PointXYZI layout, each frame also carrying /tf, /debug/pc_raw and
/debug/pc_label as kitti2node writes them.  Reports, best of R calls after a warm-up:
  - the host index;
  - a load of every node from a pageable and from a pinned file buffer (host clock around the synchronous call);
  - a plain host-to-device copy of the same number of bytes from pinned memory, i.e. the H2D share of the load;
  - the numpy model reader (tests/bag_model.py) on the same host.
Prints one JSON line, and writes it to --out when given.  Needs a CUDA device.
  usage: python scripts/bag_timing.py [--points 60000] [--repeats 5] [--out result.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bag_model as M  # noqa: E402
from erasor_b200 import capi  # noqa: E402


def best(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=60000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import torch
    rng = np.random.default_rng(5)
    nodes = []
    for k in range(161):
        c = (rng.normal(size=(a.points, 4)) * 20).astype(np.float32)
        nodes.append((2350 + 2 * k, np.r_[rng.normal(size=3), 0, 0, 0, 1], c))
    data = M.write_bag(M.kitti2node_messages(nodes), chunk_bytes=768 * 1024)
    pin = torch.empty(len(data), dtype=torch.uint8, pin_memory=True)
    pin.numpy()[:] = np.frombuffer(data, np.uint8)
    out = torch.empty((161 * a.points, 4), dtype=torch.float32, device="cuda")
    res = {"file_bytes": len(data), "nodes": 161, "points_per_node": a.points}
    with capi.PcdCodec() as codec:
        res["index_ms"] = best(lambda: codec.bag_index(data), a.repeats)
        info = codec.bag_index(data)
        _, _, _, clouds = codec.bag_meta()
        blob = sum(c["data_len"] for c in clouds)
        res["selected_blob_bytes"] = blob
        off = np.zeros(162, np.uint64)
        op = off.ctypes.data_as(capi.POINTER(capi.c_uint64))

        def load():
            assert codec.L.erasor_bag_load(codec.h, 0, 161, capi.c_void_p(out.data_ptr()), out.shape[0], capi.PTR_DEVICE, op) == 0
        res["load_pageable_ms"] = best(load, a.repeats)
        codec.bag_index(pin)
        res["load_pinned_ms"] = best(load, a.repeats)
        assert int(off[-1]) == info["total_points"]
    src = torch.empty(blob, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(blob, dtype=torch.uint8, device="cuda")

    def h2d():
        dst.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
    res["h2d_pinned_same_bytes_ms"] = best(h2d, a.repeats)
    res["h2d_share_of_pinned_load"] = res["h2d_pinned_same_bytes_ms"] / res["load_pinned_ms"]
    res["numpy_model_reader_ms"] = best(lambda: M.read_bag(data), 1)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res["gpu"] = q.stdout.strip()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
