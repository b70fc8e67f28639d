"""GPU: binary and binary_compressed PCD files read on the device (capi.PcdCodec.load over erasor_pcd_load) against the numpy
reference of tests/pcd_binary_model.py, bit for bit, through every pointer-kind combination; the same cloud read from its ASCII,
binary and compressed files; streams and bodies past the 32-bit byte range; malformed streams; and the callers that read through
load: the evaluator, `python -m erasor_b200.analysis` and the C++ driver."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

import pcd_binary_model as M
from erasor_b200 import capi, synth
from erasor_b200 import evaluate as E
from test_gpu_cpp_driver import BIN, YAML

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def codec():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    with capi.PcdCodec(0) as c:
        yield c


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def check_kinds(codec, data, ref):
    """load == ref through host / device file x host / device cloud"""
    import torch
    assert same_bits(codec.load_bytes(data), ref)
    assert same_bits(codec.load_bytes(data, device_out=True).cpu().numpy(), ref)
    dfile = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    assert same_bits(codec.load_bytes(dfile), ref)
    assert same_bits(codec.load_bytes(dfile, device_out=True).cpu().numpy(), ref)


def nan_records(spec, n, seed):
    """random records whose x, y, z, intensity hold NaNs with payloads, infinities and signed zeros at some points"""
    rec = M.random_records(spec, n, seed=seed)
    specials = np.array([0x7FC01234, 0xFFBFFFFF, 0x7F800001, 0x80000000, 0x7F800000, 0x00000001], dtype=np.uint32).view(np.float32)
    for name in ("x", "y", "z", "intensity"):
        for f in spec:
            if f[0] == name and f[1:] == ("F", 4, 1):
                col = rec[name].copy()
                col[::7][:len(specials)] = specials[:len(col[::7])]
                rec[name] = col
    return rec


@pytest.mark.parametrize("mode", ["binary", "binary_compressed"])
@pytest.mark.parametrize("layout", sorted(M.LAYOUTS))
def test_layouts_bit_exact(codec, layout, mode):
    spec = M.LAYOUTS[layout]
    for n, head in ((5000, {}), (4096 + 13, {"comment": " x"}), (64 * 9, {"width": 64, "height": 9, "comment": " organized"}), (1, {})):
        rec = nan_records(spec, n, seed=n)
        data = M.write_pcd(spec, rec, mode, compress=M.hc_lzf_compress, **head)
        ref, flag = M.read_reference(data, decompress=lambda s, u: M.hc_lzf_serial(s, u)[1])
        check_kinds(codec, data, ref)
        info = codec.last_load_info()
        assert info["intensity_zero_filled"] == flag and info["points"] == n
        assert info["data_mode"] == (1 if mode == "binary" else 2)


def test_empty_cloud(codec):
    for mode in ("binary", "binary_compressed"):
        assert codec.load_bytes(M.header(M.XYZI, 0, mode)).shape == (0, 4)


def test_ascii_binary_and_compressed_files_agree(codec, tmp_path):
    sc = synth.Scene(seed=12, length=30.0, n_nodes=4, n_dynamic=3)
    p = str(tmp_path / "a.pcd")
    E.write_pcd_ascii(p, sc.scan(2, n_beams=16, n_az=400))
    c = E.read_pcd_ascii(p)                            # the floats the ASCII file parses to
    rec = M.random_records(M.WIDE, len(c), seed=1, xyzi=c)
    got = [codec.load(p)]
    assert codec.last_load_info()["data_mode"] == 0 and codec.last_load_info()["ascii"]["rows"] == len(c)
    for spec, r in ((M.XYZI, M.random_records(M.XYZI, len(c), xyzi=c)), (M.WIDE, rec)):
        for mode in ("binary", "binary_compressed"):
            got.append(codec.load_bytes(M.write_pcd(spec, r, mode, compress=M.hc_lzf_compress)))
    for g in got:
        assert same_bits(g, c)


def labelled_cloud(n, seed=1):
    rng = np.random.default_rng(seed)
    lab = rng.choice(np.array([0, 40, 44, 48, 50, 70, 252, 253, 254, 255, 256, 257, 258, 259], dtype=np.float32), n)
    return np.concatenate([rng.uniform(-80, 80, (n, 3)).astype(np.float32), lab[:, None]], axis=1).astype(np.float32)


def test_greedy_compressed_labelled_map(codec):
    c = labelled_cloud(1_000_000)
    data = M.write_pcd(M.XYZI, M.random_records(M.XYZI, len(c), xyzi=c), "binary_compressed", compress=M.hc_lzf_compress)
    assert same_bits(codec.load_bytes(data, device_out=True).cpu().numpy(), c)
    info = codec.last_load_info()
    assert info["compressed_size"] < info["uncompressed_size"] == 16 * len(c)


def test_stream_near_the_uint32_limit(codec):
    import torch
    n = (2 ** 32 - 1) // 16                          # uncompressed_size 4294967280
    pts = np.array([[1.5, -2.25, 3.0, 7.0], [np.nan, 1e30, -0.0, 255.0]], dtype=np.float32)
    soa = pts.T.reshape(-1)                            # not SoA across n points: the stream repeats a 32-byte period instead
    prefix = soa.tobytes()
    stream = M.periodic_stream(prefix, 16 * n)
    data = M.header(M.XYZI, n, "binary_compressed") + struct.pack("<II", len(stream), 16 * n) + stream
    out = codec.load_bytes(data, device_out=True)
    info = codec.last_load_info()
    assert info["uncompressed_size"] == 16 * n and info["lzf_tokens"] > 16_000_000
    period = np.frombuffer(prefix, dtype=np.uint32)
    idx = np.unique(np.concatenate([np.arange(8), np.random.default_rng(0).integers(0, n, 4000), n - 1 - np.arange(8)]))
    got = out[torch.from_numpy(idx).cuda()].cpu().numpy().view(np.uint32)
    for s in range(4):                                 # point i, slot s = the decompressed word at (s n + i) mod 8
        assert np.array_equal(got[:, s], period[(s * n + idx) % 8])
    del out
    torch.cuda.empty_cache()


def test_binary_body_above_4gib_from_device(codec):
    import torch
    n = 2 ** 32 // 16 + 4099
    head = M.header(M.XYZI, n, "binary", comment=" odd")
    assert len(head) % 16 != 0
    buf = torch.empty(len(head) + 16 * n, dtype=torch.uint8, device="cuda")
    buf[:len(head)] = torch.frombuffer(bytearray(head), dtype=torch.uint8).cuda()
    body = torch.arange(4 * n, dtype=torch.int32, device="cuda")
    buf[len(head):] = body.view(torch.uint8)
    del body
    out = codec.load_bytes(buf, device_out=True)
    del buf
    idx = np.unique(np.concatenate([np.arange(4), np.random.default_rng(1).integers(0, n, 4000), n - 1 - np.arange(4)]))
    got = out[torch.from_numpy(idx).cuda()].cpu().numpy().view(np.int32)
    assert np.array_equal(got, 4 * idx[:, None] + np.arange(4)[None, :])
    del out
    torch.cuda.empty_cache()


@pytest.mark.parametrize("kind", ["host", "device"])
def test_malformed_streams_are_rejected_and_the_handle_stays_usable(codec, kind):
    import torch
    from test_pcd_binary_model import malformed
    good = M.write_pcd(M.XYZI, M.random_records(M.XYZI, 300), "binary_compressed")
    good_ref, _ = M.read_reference(good)
    for name, (stream, usize) in sorted(malformed().items()):
        n = -(-usize // 16)
        data = M.header(M.XYZI, n, "binary_compressed") + struct.pack("<II", len(stream), 16 * n) + stream
        arg = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda() if kind == "device" else data
        with pytest.raises(capi.ErasorError) as ei:
            codec.load_bytes(arg, device_out=kind == "device")
        assert ei.value.code == capi.E_INVALID, name
        assert same_bits(codec.load_bytes(good), good_ref)


def test_evaluator_on_device_loaded_clouds(codec, tmp_path):
    import torch
    gt = labelled_cloud(60_000, seed=3)
    rng = np.random.default_rng(4)
    est = gt[rng.random(len(gt)) < 0.8].copy()
    est[:, :3] += rng.normal(0, 0.03, (len(est), 3)).astype(np.float32)
    pa, pb = str(tmp_path / "gt.pcd"), str(tmp_path / "est.pcd")
    E.write_pcd_ascii(pa, gt)
    E.write_pcd_ascii(pb, est)
    ga, ea = E.read_pcd_ascii(pa), E.read_pcd_ascii(pb)
    gd = codec.load_bytes(M.write_pcd(M.WIDE, M.random_records(M.WIDE, len(ga), xyzi=ga), "binary_compressed", compress=M.hc_lzf_compress), device_out=True)
    ed = codec.load_bytes(M.write_pcd(M.XYZI, M.random_records(M.XYZI, len(ea), xyzi=ea), "binary"), device_out=True)
    with capi.Evaluator(0) as ev:
        want = ev.evaluate(ga, ea)
        got = ev.evaluate_ptr(gd.data_ptr(), gd.shape[0], ed.data_ptr(), ed.shape[0])
        torch.cuda.synchronize()
    assert got == want


def test_analysis_cli_on_compressed_files(tmp_path):
    gt = labelled_cloud(20_000, seed=5)
    est = gt[np.random.default_rng(6).random(len(gt)) < 0.7]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    outs = []
    for kind in ("ascii", "compressed"):
        d = tmp_path / kind
        d.mkdir()
        for name, c in (("gt.pcd", gt), ("est.pcd", est)):
            if kind == "ascii":
                E.write_pcd_ascii(str(d / name), c)
            else:
                c = E.read_pcd_ascii(str(tmp_path / "ascii" / name))
                (d / name).write_bytes(M.write_pcd(M.XYZI, M.random_records(M.XYZI, len(c), xyzi=c), "binary_compressed",
                                                   compress=M.hc_lzf_compress))
        outs.append(subprocess.run([sys.executable, "-m", "erasor_b200.analysis", "--gt", "gt.pcd", "--est", "est.pcd"], cwd=d, env=env,
                                   check=True, capture_output=True, text=True).stdout)
    assert outs[1] == outs[0] and "gt.pcd" in outs[0]


def run_driver(tmp_path, name, gt_map, scans, poses, map_mode, scan_modes):
    data, save = tmp_path / name / "data", tmp_path / name / "out"
    (data / "pcds").mkdir(parents=True)
    save.mkdir()

    def write(path, c, mode):
        if mode == "ascii":
            E.write_pcd_ascii(path, c)
        else:
            spec = M.WIDE if mode == "binary_compressed" else M.XYZI
            open(path, "wb").write(M.write_pcd(spec, M.random_records(spec, len(c), xyzi=c), mode, compress=M.hc_lzf_compress))

    write(str(data / "dense_global_map.pcd"), gt_map, map_mode)
    with open(data / "poses_lidar2body.csv", "w") as f:
        f.write("index,time,x,y,z,qx,qy,qz,qw\n")
        for k, (s, p) in enumerate(zip(scans, poses)):
            write(str(data / "pcds" / f"{k:06d}.pcd"), s, scan_modes[k % len(scan_modes)])
            f.write(f"{k},{k * 0.1}," + ",".join(f"{v:.9g}" for v in p) + "\n")
    cfg = tmp_path / name / "seq_05.yaml"
    cfg.write_text(YAML.format(save=str(save)))
    r = subprocess.run([BIN, str(cfg), str(data)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:] + r.stdout[-2000:]
    return open(save / "05_result.pcd", "rb").read()


def test_cpp_driver_reads_every_data_mode(tmp_path):
    assert os.path.exists(BIN), "build with erasor_b200/csrc/build.sh"
    sc = synth.Scene(seed=43, length=40.0, n_nodes=12, n_dynamic=6)
    kw = dict(n_beams=24, n_az=480)
    nodes = list(range(12))
    p = str(tmp_path / "round.pcd")
    E.write_pcd_ascii(p, sc.build_map(nodes, voxel=0.2, **kw))
    gt_map = E.read_pcd_ascii(p)
    scans, poses = [], []
    for k in nodes:
        E.write_pcd_ascii(p, sc.scan(k, seed_offset=9, **kw))
        scans.append(E.read_pcd_ascii(p))
        poses.append(sc.pose7(k))
    ascii_only = run_driver(tmp_path, "ascii", gt_map, scans, poses, "ascii", ["ascii"])
    mixed = run_driver(tmp_path, "mixed", gt_map, scans, poses, "binary_compressed", ["binary_compressed", "ascii", "binary"])
    assert len(E.read_pcd_ascii(str(tmp_path / "mixed" / "out" / "05_result.pcd"))) > 0
    assert mixed == ascii_only
