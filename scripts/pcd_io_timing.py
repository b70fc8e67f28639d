"""ASCII PCD reading and writing: the device codec (capi.PcdCodec, erasor_pcd_parse_ascii / erasor_pcd_format_ascii) against the
host reader and writer (evaluate.read_pcd_ascii / write_pcd_ascii: np.loadtxt / np.savetxt).  Prints one JSON line.
  twin:     bench.py's seq 05 twin map (337 k points)
  labelled: a seeded 1 M-point labelled cloud
  config4:  a config-4-sized cloud built as scripts/eval_timing.py builds it (50 M points, seed 5); its file is written by the
            device formatter (the same bytes), and the host reader and writer are timed on a seeded 1 M-point subset only
Per workload: the file's bytes; host read and write (wall, file in the page cache, best of a few); device parse (text in device
memory -> float4 in device memory) and format (size query + fetch into device memory), each from CUDA events around warmed
synchronous calls; the H2D copy of the text and the D2H copy of the formatted text from pinned memory, timed on their own; and the
wall time of the whole codec.read(path) (bytes in the page cache -> numpy float32) and codec.write(path, cloud).
usage: pcd_io_timing.py [n_points] [reps]"""
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from erasor_b200 import capi, synth  # noqa: E402
from erasor_b200 import evaluate as E  # noqa: E402

N_TARGET = int(sys.argv[1]) if len(sys.argv) > 1 else 50_000_000
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 5


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


def wall_s(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return min(times)


def copy_ms(dst, src, reps):
    return events_ms(lambda: dst.copy_(src, non_blocking=True), reps)


def device_format(codec, x):
    """size query + fetch into device memory; returns the device text"""
    L, size = codec.L, ctypes.c_size_t(0)
    assert L.erasor_pcd_format_ascii(codec.h, x.data_ptr(), x.shape[0], capi.PTR_DEVICE, None, 0, capi.PTR_DEVICE, ctypes.byref(size)) == 0
    out = torch.empty(size.value, dtype=torch.uint8, device="cuda")
    assert L.erasor_pcd_format_ascii(codec.h, x.data_ptr(), x.shape[0], capi.PTR_DEVICE, out.data_ptr(), size.value, capi.PTR_DEVICE,
                                     ctypes.byref(size)) == 0
    return out


def host_arm(cloud, d, reps):
    path = os.path.join(d, "host.pcd")
    w = wall_s(lambda: E.write_pcd_ascii(path, cloud), reps)
    r = wall_s(lambda: E.read_pcd_ascii(path), reps)
    return {"host_points": len(cloud), "host_bytes": os.path.getsize(path), "host_read_s": round(r, 3), "host_write_s": round(w, 3)}


def workload(codec, cloud, d, host_subset=None):
    x = torch.from_numpy(np.ascontiguousarray(cloud, dtype=np.float32)).cuda()
    text = device_format(codec, x)
    path = os.path.join(d, "dev.pcd")
    raw = text.cpu().numpy()
    with open(path, "wb") as f:
        f.write(memoryview(raw))
    out = {"points": len(cloud), "bytes": int(text.numel())}
    sub = cloud if host_subset is None else host_subset
    h = host_arm(sub, d, 3 if len(sub) <= 2_000_000 else 1)
    if host_subset is None:
        out["file_equal_to_write_pcd_ascii"] = open(os.path.join(d, "host.pcd"), "rb").read() == raw.tobytes()
    out.update(h)
    parsed = codec.parse(text, device_out=True)
    out["parse_equal_to_read_pcd_ascii"] = bool(np.array_equal(parsed.cpu().numpy().view(np.uint32),
                                                              E.read_pcd_ascii(path).view(np.uint32))) if host_subset is None else None
    torch.cuda.synchronize()
    out["device_parse_ms"] = round(events_ms(lambda: codec.parse(text, device_out=True), REPS), 3)
    out["device_format_ms"] = round(events_ms(lambda: device_format(codec, x), REPS), 3)
    pinned = torch.empty(text.numel(), dtype=torch.uint8).pin_memory()
    out["h2d_text_ms"] = round(copy_ms(text, pinned, REPS), 3)
    out["d2h_text_ms"] = round(copy_ms(pinned, text, REPS), 3)
    out["codec_read_wall_s"] = round(wall_s(lambda: codec.read(path), 3), 3)
    out["codec_write_wall_s"] = round(wall_s(lambda: codec.write(os.path.join(d, "w.pcd"), cloud), 3), 3)
    out["slow_tokens"] = codec.last_info()["slow_tokens"]
    for f in ("dev.pcd", "host.pcd", "w.pcd"):
        if os.path.exists(os.path.join(d, f)):
            os.remove(os.path.join(d, f))
    return out


def config4_cloud():
    w = synth.make_frames(seed=5, n_frames=6, preset_max_range=80.0, n_map_nodes=41, n_beams=32, n_az=900)
    base = w["frames"][2][0]
    base = base[(base[:, 0].astype(np.float64) ** 2 + base[:, 1].astype(np.float64) ** 2) < 82.0 ** 2]
    reps = int(np.ceil(N_TARGET / len(base)))
    g = torch.Generator(device="cuda").manual_seed(5)
    M = torch.from_numpy(base).cuda().repeat(reps, 1)
    M[:, :3] += (torch.rand((M.shape[0], 3), device="cuda", generator=g) - 0.5) * torch.tensor([0.19, 0.19, 0.02], device="cuda")
    return M.cpu().numpy()


def main():
    torch.cuda.init()
    import bench
    codec = capi.PcdCodec(0)
    rng = np.random.default_rng(1)
    n = 1_000_000
    lab = rng.choice(np.array([0, 40, 44, 48, 50, 70, 252, 253, 254, 255, 256, 257, 258, 259], dtype=np.float32), n)
    labelled = np.concatenate([rng.uniform(-80, 80, (n, 3)).astype(np.float32), lab[:, None]], axis=1).astype(np.float32)
    _, map_world, _, _ = bench.load_workload("seq05", 0, 1, 20)
    line = {"what": "ASCII PCD I/O: device codec (erasor_pcd_parse_ascii / erasor_pcd_format_ascii) vs read_pcd_ascii / write_pcd_ascii",
            "gpu": gpu_info(), "reps": REPS}
    with tempfile.TemporaryDirectory() as d:
        line["twin"] = workload(codec, map_world, d)
        line["labelled_1M"] = workload(codec, labelled, d)
        big = config4_cloud()
        sub = big[np.sort(np.random.default_rng(5).choice(len(big), 1_000_000, replace=False))]
        line["config4_50M"] = workload(codec, big, d, host_subset=sub)
    codec.close()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
