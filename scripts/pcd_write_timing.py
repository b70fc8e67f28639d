"""Binary and binary_compressed PCD writing on the device (erasor_pcd_format, capi.PcdCodec.format / write).  Prints one JSON line.
  twin:     bench.py's seq 05 twin map (337 k points)
  labelled: a seeded 1 M-point labelled cloud
  config4:  a 50 M-point config-4-sized cloud, built as scripts/pcd_binary_timing.py builds it
Per workload and mode: the device format (cloud in device memory -> file in device memory) from CUDA events around warmed
synchronous calls; the D2H copy of the file into pinned memory on its own; the wall time of codec.write from a device cloud to a
file under the system's temporary directory; for binary_compressed the stream's size and ratio next to the ratio of
tests/pcd_binary_model.py's unsegmented greedy encoder (its C++ build) on the same SoA, and the serial host encoder of the same
segmented rule (the hostcheck build, -O2); for binary numpy's tobytes of the cloud.  The card's name and power limit are read in
the same run.
usage: pcd_write_timing.py [n_points_config4] [reps]"""
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import lzf_encode_model as E  # noqa: E402
import pcd_binary_model as M  # noqa: E402
from erasor_b200 import capi, synth  # noqa: E402

N_TARGET = int(sys.argv[1]) if len(sys.argv) > 1 else 50_000_000
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 5


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


def one_mode(codec, cloud, dev, mode, tmpdir):
    n, m = len(cloud), capi.PCD_MODES[mode]
    size, info = ctypes.c_size_t(0), capi.PcdFormatInfoC()
    L = codec.L
    assert L.erasor_pcd_format(codec.h, ctypes.c_void_p(dev.data_ptr()), n, capi.PTR_DEVICE, m, None, 0, capi.PTR_DEVICE, ctypes.byref(size),
                               ctypes.byref(info)) == 0
    out = torch.empty(size.value, dtype=torch.uint8, device="cuda")

    def fmt():
        rc = L.erasor_pcd_format(codec.h, ctypes.c_void_p(dev.data_ptr()), n, capi.PTR_DEVICE, m, ctypes.c_void_p(out.data_ptr()), size.value,
                                 capi.PTR_DEVICE, ctypes.byref(size), ctypes.byref(info))
        assert rc == 0, L.erasor_pcd_last_error(codec.h)

    fmt()
    r = {"file_bytes": size.value, "device_format_ms": round(events_ms(fmt, REPS), 3)}
    pinned = torch.empty(size.value, dtype=torch.uint8).pin_memory()
    r["d2h_file_ms"] = round(events_ms(lambda: pinned.copy_(out, non_blocking=True), REPS), 3)
    back = codec.load_bytes(out, device_out=True)
    r["reads_back_equal"] = bool(torch.equal(back.view(torch.int32), dev.view(torch.int32)))
    del back
    path = os.path.join(tmpdir, f"w_{mode}.pcd")
    r["codec_write_s"] = round(wall_s(lambda: codec.write(path, dev, mode=mode), 2), 4)
    os.remove(path)
    if mode == "binary":
        r["host_numpy_tobytes_s"] = round(wall_s(lambda: cloud.tobytes(), 2), 4)
    else:
        raw = E.soa(cloud)
        r.update(segments=int(info.segments), lzf_tokens=int(info.lzf_tokens), compressed_bytes=int(info.compressed_size),
                 uncompressed_bytes=int(info.uncompressed_size), ratio=round(info.uncompressed_size / max(info.compressed_size, 1), 4))
        t0 = time.perf_counter()
        stream, _, _ = E.hc_encode(raw)
        r["host_serial_segmented_encode_s"] = round(time.perf_counter() - t0, 4)
        r["host_equals_device"] = bool(len(stream) == info.compressed_size and
                                       out[size.value - len(stream):].cpu().numpy().tobytes() == stream)
        del stream
        t0 = time.perf_counter()
        greedy = M.hc_lzf_compress(raw)
        r["host_greedy_unsegmented_encode_s"] = round(time.perf_counter() - t0, 4)
        r["greedy_unsegmented_bytes"] = len(greedy)
        r["greedy_unsegmented_ratio"] = round(len(raw) / max(len(greedy), 1), 4)
        del greedy, raw
    del out, pinned
    torch.cuda.empty_cache()
    return r


def workload(codec, cloud, tmpdir):
    cloud = np.ascontiguousarray(cloud, dtype=np.float32)
    dev = torch.from_numpy(cloud).cuda()
    res = {"points": len(cloud)}
    for mode in ("binary", "binary_compressed"):
        res[mode] = one_mode(codec, cloud, dev, mode, tmpdir)
    del dev
    torch.cuda.empty_cache()
    return res


def config4_cloud():
    w = synth.make_frames(seed=5, n_frames=6, preset_max_range=80.0, n_map_nodes=41, n_beams=32, n_az=900)
    base = w["frames"][2][0]
    base = base[(base[:, 0].astype(np.float64) ** 2 + base[:, 1].astype(np.float64) ** 2) < 82.0 ** 2]
    reps = int(np.ceil(N_TARGET / len(base)))
    g = torch.Generator(device="cuda").manual_seed(5)
    m = torch.from_numpy(base).cuda().repeat(reps, 1)[:N_TARGET]
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
    line = {"what": "binary / binary_compressed PCD write on the device (erasor_pcd_format) vs numpy and the serial host encoder",
            "gpu": gpu_info(), "reps": REPS, "segment_bytes": E.SEG}
    with tempfile.TemporaryDirectory() as tmpdir:
        line["twin"] = workload(codec, map_world, tmpdir)
        line["labelled_1M"] = workload(codec, labelled, tmpdir)
        line["config4_50M"] = workload(codec, config4_cloud(), tmpdir)
    codec.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
