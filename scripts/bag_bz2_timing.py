"""Times erasor_bag_index / erasor_bag_load on a bag with bz2 chunks (DESIGN.md section 12.2.2): the synthetic seq 05 bag of
scripts/bag_timing.py (161 nodes of N points, /tf and the two debug clouds per frame, 768 KB chunks), written with every chunk a
bzip2 stream at level 9 (what `rosbag record -j` writes) and at level 1.  Two arms: random floats in the 32-byte PointXYZI layout
(--values 0), and a compressible arm (--values K: every value one of K floats, 16-byte points).  Reports, best of R calls after a
warm-up (host clock around the synchronous calls):
  - the file sizes;
  - erasor_bag_index (pinned file) and erasor_bag_load of every node;
  - the device ms of each stage group (erasor_bag_bz2_stats: scan + walk + chain, decode, inverse BWT, RLE1 + CRC), blocks,
    candidates per block and the peak scratch;
  - the same chunks through Python's bz2.decompress (libbz2) on one host core, and on every host core (a process pool).
Prints one JSON line, and writes it to --out when given.  Needs a CUDA device.
  usage: python scripts/bag_bz2_timing.py [--points 60000] [--values 0] [--repeats 3] [--out result.json]"""
import argparse
import bz2
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bag_model as M  # noqa: E402
import bz2_model as B  # noqa: E402
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
    ap.add_argument("--values", type=int, default=0, help="distinct values per coordinate (0: random floats, 32-byte layout)")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import torch
    rng = np.random.default_rng(5)
    nodes = []
    for k in range(161):
        c = (rng.normal(size=(a.points, 4)) * 20).astype(np.float32)
        if a.values:
            c = (rng.integers(0, a.values, size=(a.points, 4)) * 0.25).astype(np.float32)
        nodes.append((2350 + 2 * k, np.r_[rng.normal(size=3), 0, 0, 0, 1], c))
    plain = M.write_bag(M.kitti2node_messages(nodes, layout="packed" if a.values else "pcl_xyzi"), chunk_bytes=768 * 1024)
    res = {"nodes": 161, "points_per_node": a.points, "values": a.values, "plain_bytes": len(plain)}
    out = torch.empty((161 * a.points, 4), dtype=torch.float32, device="cuda")
    off = np.zeros(162, np.uint64)
    op = off.ctypes.data_as(capi.POINTER(capi.c_uint64))
    with capi.PcdCodec() as codec:
        def load():
            assert codec.L.erasor_bag_load(codec.h, 0, 161, capi.c_void_p(out.data_ptr()), out.shape[0], capi.PTR_DEVICE, op) == 0
        for level in (9, 1):
            streams = []
            twin = B.bz2_twin(plain, lambda d: streams.append(bz2.compress(d, level)) or streams[-1])
            pin = torch.empty(len(twin), dtype=torch.uint8, pin_memory=True)
            pin.numpy()[:] = np.frombuffer(twin, np.uint8)
            r = {"bz2_bytes": len(twin), "chunks": len(streams)}
            r["index_pinned_ms"] = best(lambda: codec.bag_index(pin), a.repeats)
            codec.bag_index(pin)
            r["load_ms"] = best(load, a.repeats)
            st = codec.bag_bz2_stats()
            r["stats"] = st
            r["candidates_per_block"] = st["candidates"] / max(st["blocks"], 1)
            r["device_stage_ms_total"] = st["scan_ms"] + st["decode_ms"] + st["bwt_ms"] + st["rle_ms"]
            r["libbz2_single_core_ms"] = best(lambda: [bz2.decompress(s) for s in streams], 1)
            workers = os.cpu_count() or 1
            with ProcessPoolExecutor(workers) as ex:
                r["libbz2_all_cores_ms"] = best(lambda: list(ex.map(bz2.decompress, streams, chunksize=4)), 1)
            r["host_cores"] = workers
            res[f"level{level}"] = r
            del pin
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res["gpu"] = q.stdout.strip()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
