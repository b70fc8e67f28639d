"""Times erasor_bag_index / erasor_bag_load on a bag with lz4 chunks (DESIGN.md section 12.2.1) against its uncompressed twin: the
synthetic seq 05 bag of scripts/bag_timing.py (161 nodes + the duplicated first frame of N points in the 32-byte PointXYZI layout,
with /tf and the two debug clouds per frame, 768 KB chunks), written uncompressed and with every chunk an LZ4 frame (the host
build's greedy encoder, block max id --bsid, content checksum as roslz4 writes it).  Reports, best of R calls after a warm-up
(host clock around the synchronous calls):
  - the file sizes and the compression ratio (random floats compress poorly: the ratio is part of the result);
  - erasor_bag_index and erasor_bag_load of every node, both bags, pageable and pinned files;
  - the bytes each call copies host to device;
  - the decode and checksum kernels' device time (CUDA events, erasor_bag_lz4_stats) and the decoded bytes per second;
  - a single-core liblz4 decode of the same chunks, when ctypes can load a system liblz4.
--values K draws every coordinate and intensity from K distinct floats and packs points in 16 bytes (no padding), so the frames
hold many short matches and the sequence decoder, not the stored-block copy, does the work; 0 (the default) keeps random floats
in the 32-byte layout, which do not compress.
Prints one JSON line, and writes it to --out when given.  Needs a CUDA device and liberasor_b200_hostcheck.so.
  usage: python scripts/bag_lz4_timing.py [--points 60000] [--values 0] [--bsid 6] [--repeats 5] [--out result.json]"""
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
import lz4_model as Z  # noqa: E402
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
    ap.add_argument("--bsid", type=int, default=6, help="LZ4 block max id: 4 (64 KB) .. 7 (4 MB)")
    ap.add_argument("--repeats", type=int, default=5)
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
    frames = []
    twin = Z.lz4_twin(plain, lambda d: frames.append(Z.hc_frame(d, a.bsid, False, True)) or frames[-1])
    res = {"nodes": 161, "points_per_node": a.points, "values": a.values, "bsid": a.bsid, "plain_bytes": len(plain), "lz4_bytes": len(twin),
           "ratio": len(plain) / len(twin)}
    out = torch.empty((161 * a.points, 4), dtype=torch.float32, device="cuda")
    off = np.zeros(162, np.uint64)
    op = off.ctypes.data_as(capi.POINTER(capi.c_uint64))
    with capi.PcdCodec() as codec:
        def load():
            assert codec.L.erasor_bag_load(codec.h, 0, 161, capi.c_void_p(out.data_ptr()), out.shape[0], capi.PTR_DEVICE, op) == 0
        for name, data in (("plain", plain), ("lz4", twin)):
            pin = torch.empty(len(data), dtype=torch.uint8, pin_memory=True)
            pin.numpy()[:] = np.frombuffer(data, np.uint8)
            for kind, buf in (("pageable", data), ("pinned", pin)):
                res[f"{name}_index_{kind}_ms"] = best(lambda: codec.bag_index(buf), a.repeats)
                codec.bag_index(buf)
                res[f"{name}_load_{kind}_ms"] = best(load, a.repeats)
            st = codec.bag_lz4_stats()
            _, _, _, clouds = codec.bag_meta()
            blob = sum(c["data_len"] for c in clouds)
            res[f"{name}_h2d_index_bytes"] = st["compressed_bytes"]
            res[f"{name}_h2d_load_bytes"] = 0 if name == "lz4" else blob
            if name == "lz4":
                res["lz4_stats"] = st
                res["decoded_GBps"] = st["decoded_bytes"] / (st["decode_ms"] * 1e6)
                res["decode_and_checksum_GBps"] = st["decoded_bytes"] / ((st["decode_ms"] + st["checksum_ms"]) * 1e6)
            del pin
    L = Z.liblz4()
    if L is not None:
        sizes = [r[4] for r in Z.top_records(plain) if r[2]["op"][1][0] == 5]

        def serial():
            for f, n in zip(frames, sizes):
                Z.lib_decompress(L, f, n)
        res["liblz4_single_core_all_chunks_ms"] = best(serial, 1)
        res["liblz4_all_chunks_decoded_bytes"] = sum(sizes)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    res["gpu"] = q.stdout.strip()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
