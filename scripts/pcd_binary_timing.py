"""Binary and binary_compressed PCD reading on the device (capi.PcdCodec.load_bytes over erasor_pcd_load).  Prints one JSON line.
  twin:     bench.py's seq 05 twin map (337 k points)
  labelled: a seeded 1 M-point labelled cloud
  config4:  a 50 M-point config-4-sized cloud built as scripts/pcd_io_timing.py builds it
each in two layouts (xyzi: PointXYZI; wide: tests/pcd_binary_model.py's WIDE, 50 bytes per point with "_" padding, U2 / U4 / U1 x 4
fields and COUNT 3 normals around x y z intensity) and both modes.  The compressed files use the greedy encoder of
tests/pcd_binary_model.py (its C++ build in liberasor_b200_hostcheck.so).
Per file: its bytes and, compressed, the stream's; the device load (file in device memory -> float4 in device memory) from CUDA
events around warmed synchronous calls; the H2D copy of the file from pinned memory on its own; for binary, the bytes the pass
must move (the body read once, 16 bytes written per point) over the load time against the H100 SXM data sheet's 3.35 TB/s; and a
host arm: numpy's structured-dtype read for binary, and for binary_compressed a serial liblzf-style decoder (the hostcheck build,
-O2) on the stream alone.
usage: pcd_binary_timing.py [n_points_config4] [reps]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pcd_binary_model as M  # noqa: E402
from erasor_b200 import capi, synth  # noqa: E402

N_TARGET = int(sys.argv[1]) if len(sys.argv) > 1 else 50_000_000
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 5
HBM_PEAK = 3.35e12


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


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


def wall_s(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return min(times)


def one_file(codec, spec, rec, mode, cloud):
    data = M.write_pcd(spec, rec, mode, compress=M.hc_lzf_compress)
    n = len(rec)
    dfile = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()
    out = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    import ctypes
    size, info = ctypes.c_size_t(0), capi.PcdLoadInfoC()

    def load():
        rc = codec.L.erasor_pcd_load(codec.h, ctypes.c_void_p(dfile.data_ptr()), dfile.numel(), capi.PTR_DEVICE, ctypes.c_void_p(out.data_ptr()),
                                     n, capi.PTR_DEVICE, ctypes.byref(size), ctypes.byref(info))
        assert rc == 0, codec.L.erasor_pcd_last_error(codec.h)

    load()
    r = {"file_bytes": len(data), "equal": bool(np.array_equal(out.cpu().numpy().view(np.uint32), cloud.view(np.uint32)))}
    r["device_load_ms"] = round(events_ms(load, REPS), 3)
    pinned = torch.empty(len(data), dtype=torch.uint8).pin_memory()
    r["h2d_file_ms"] = round(events_ms(lambda: dfile.copy_(pinned, non_blocking=True), REPS), 3)
    if mode == "binary":
        moved = n * M.point_step(spec) + 16 * n
        r["moved_bytes"] = moved
        r["hbm_share_of_3_35_TBps"] = round(moved / (r["device_load_ms"] * 1e-3) / HBM_PEAK, 3)
        r["host_numpy_read_s"] = round(wall_s(lambda: M.read_reference(data), 2), 4)
    else:
        r["compressed_bytes"] = int(info.compressed_size)
        r["uncompressed_bytes"] = int(info.uncompressed_size)
        r["lzf_tokens"] = int(info.lzf_tokens)
        off = int(info.data_offset)
        stream = data[off + 8: off + 8 + int(info.compressed_size)]
        r["host_serial_lzf_decode_s"] = round(wall_s(lambda: M.hc_lzf_serial(stream, int(info.uncompressed_size)), 2), 4)
    del dfile, out, pinned
    torch.cuda.empty_cache()
    return r


def workload(codec, cloud):
    res = {"points": len(cloud)}
    for lname, spec in (("xyzi", M.XYZI), ("wide", M.WIDE)):
        rec = M.random_records(spec, len(cloud), seed=7, xyzi=cloud)
        for mode in ("binary", "binary_compressed"):
            res[f"{lname}_{mode}"] = one_file(codec, spec, rec, mode, cloud)
        del rec
    return res


def config4_cloud():
    w = synth.make_frames(seed=5, n_frames=6, preset_max_range=80.0, n_map_nodes=41, n_beams=32, n_az=900)
    base = w["frames"][2][0]
    base = base[(base[:, 0].astype(np.float64) ** 2 + base[:, 1].astype(np.float64) ** 2) < 82.0 ** 2]
    reps = int(np.ceil(N_TARGET / len(base)))
    g = torch.Generator(device="cuda").manual_seed(5)
    m = torch.from_numpy(base).cuda().repeat(reps, 1)
    m[:, :3] += (torch.rand((m.shape[0], 3), device="cuda", generator=g) - 0.5) * torch.tensor([0.19, 0.19, 0.02], device="cuda")
    return m.cpu().numpy()


def main():
    torch.cuda.init()
    import bench
    codec = capi.PcdCodec(0)
    rng = np.random.default_rng(1)
    n = 1_000_000
    lab = rng.choice(np.array([0, 40, 44, 48, 50, 70, 252, 253, 254, 255, 256, 257, 258, 259], dtype=np.float32), n)
    labelled = np.concatenate([rng.uniform(-80, 80, (n, 3)).astype(np.float32), lab[:, None]], axis=1).astype(np.float32)
    _, map_world, _, _ = bench.load_workload("seq05", 0, 1, 20)
    line = {"what": "binary / binary_compressed PCD read on the device (erasor_pcd_load) vs numpy and a serial liblzf-style decoder",
            "gpu": gpu_info(), "reps": REPS}
    line["twin"] = workload(codec, np.ascontiguousarray(map_world, dtype=np.float32))
    line["labelled_1M"] = workload(codec, labelled)
    line["config4_50M"] = workload(codec, np.ascontiguousarray(config4_cloud(), dtype=np.float32))
    codec.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
