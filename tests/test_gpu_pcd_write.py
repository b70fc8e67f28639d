"""GPU: binary and binary_compressed PCD files written on the device (erasor_pcd_format, capi.PcdCodec.format / write) against
the host build of the same writer and the Python model of tests/lzf_encode_model.py, byte for byte; every host / device
combination of input and output; read back by erasor_pcd_load bit for bit; and the callers: the C++ PcdCodec::write,
pipeline.run_sequence(pcd_mode=...) and `python -m erasor_b200.analysis`."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import lzf_encode_model as E
import pcd_binary_model as M
from erasor_b200 import capi

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("binary", "binary_compressed")


@pytest.fixture(scope="module")
def codec():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    with capi.PcdCodec(0) as c:
        yield c


def labelled_cloud(n, seed=1):
    rng = np.random.default_rng(seed)
    lab = rng.choice(np.array([0, 40, 44, 48, 50, 70, 252, 253, 254, 255, 256, 257, 258, 259], dtype=np.float32), n)
    return np.concatenate([rng.uniform(-80, 80, (n, 3)).astype(np.float32), lab[:, None]], axis=1).astype(np.float32)


def special_cloud(n=5000, seed=8):
    bits = np.array([0x7FC01234, 0xFFBFFFFF, 0x7F800001, 0xFF800000, 0x7F800000, 0x80000000, 0x00000000, 0x00000001, 0x807FFFFF,
                     0x00400000, 0x3F800000, 0xFFFFFFFF, 0x7FFFFFFF], dtype=np.uint32)
    return bits[np.random.default_rng(seed).integers(0, len(bits), (n, 4))].view(np.float32)


def twin_map():
    import bench
    _, map_world, _, _ = bench.load_workload("seq05", 0, 1, 20)
    return np.ascontiguousarray(map_world, dtype=np.float32)


SEG_PTS = E.SEG // 16                 # points whose SoA fills one segment
CLOUDS = {
    "n0": lambda: np.zeros((0, 4), np.float32),
    "n1": lambda: labelled_cloud(1, seed=2),
    "n2": lambda: labelled_cloud(2, seed=3),
    "soa_3_segments": lambda: labelled_cloud(3 * SEG_PTS, seed=4),              # SoA of exactly 3 S bytes
    "soa_3_segments_and_a_point": lambda: labelled_cloud(3 * SEG_PTS + 1, seed=5),   # 16 bytes over (a point is 16 bytes)
    "specials": special_cloud,
    "labelled_1M": lambda: labelled_cloud(1_000_000),
    "twin_map": twin_map,
}
_cache = {}


def cloud(name):
    if name not in _cache:
        _cache[name] = CLOUDS[name]()
    return _cache[name]


def fmt(codec, x, n, in_kind, mode, out_kind):
    """erasor_pcd_format straight through the C ABI: size query, then fetch; (bytes, info dict)"""
    import torch
    L = codec.L
    size, info = ctypes.c_size_t(0), capi.PcdFormatInfoC()
    m = capi.PCD_MODES[mode]
    assert L.erasor_pcd_format(codec.h, x, n, in_kind, m, None, 0, capi.PTR_HOST, ctypes.byref(size), ctypes.byref(info)) == 0
    if out_kind == capi.PTR_HOST:
        out = np.zeros(max(size.value, 1), np.uint8)
        ptr = out.ctypes.data
    else:
        out = torch.zeros(max(size.value, 1), dtype=torch.uint8, device="cuda")
        ptr = out.data_ptr()
    assert L.erasor_pcd_format(codec.h, x, n, in_kind, m, ctypes.c_void_p(ptr), size.value, out_kind, ctypes.byref(size),
                               ctypes.byref(info)) == 0, L.erasor_pcd_last_error(codec.h)
    data = out[:size.value].tobytes() if out_kind == capi.PTR_HOST else out[:size.value].cpu().numpy().tobytes()
    return data, {name: int(getattr(info, name)) for name, _ in capi.PcdFormatInfoC._fields_}


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", sorted(CLOUDS))
def test_device_bytes_equal_the_host_build(codec, name, mode):
    import torch
    c = cloud(name)
    rc, want, hinfo = E.hc_format(c, mode)
    assert rc == 0
    if len(c) <= 3 * SEG_PTS + 1 or name == "specials":        # the Python model too, where it is quick
        assert want == E.write_file(c, mode)
    host = c if len(c) else np.zeros((1, 4), np.float32)
    dev = torch.from_numpy(host).cuda()
    for in_kind, x in ((capi.PTR_HOST, host.ctypes.data), (capi.PTR_DEVICE, dev.data_ptr())):
        for out_kind in (capi.PTR_HOST, capi.PTR_DEVICE):
            got, info = fmt(codec, ctypes.c_void_p(x), len(c), in_kind, mode, out_kind)
            assert got == want, (in_kind, out_kind)
            assert info == hinfo
    assert codec.format(c, mode=mode) == want
    assert codec.format(dev[:len(c)], mode=mode) == want
    if mode == "binary_compressed":
        _, tok, seg = E.hc_encode(E.soa(c))
        assert (hinfo["lzf_tokens"], hinfo["segments"], hinfo["compressed_size"]) == (tok, seg, len(E.stream_of(want)))
    # read back on the device, bit for bit, from host and device memory
    assert bits_equal(codec.load_bytes(want), c)
    dfile = torch.frombuffer(bytearray(want), dtype=torch.uint8).cuda()
    assert bits_equal(codec.load_bytes(dfile, device_out=True).cpu().numpy(), c)
    li = codec.last_load_info()
    assert li["data_mode"] == capi.PCD_MODES[mode] and li["points"] == len(c)
    if mode == "binary_compressed" and len(c):
        assert li["lzf_tokens"] == hinfo["lzf_tokens"]


def test_ascii_mode_is_format_ascii(codec):
    c = special_cloud(777)
    want = codec.format(c)                                      # erasor_pcd_format_ascii's text
    got, info = fmt(codec, ctypes.c_void_p(c.ctypes.data), len(c), capi.PTR_HOST, "ascii", capi.PTR_HOST)
    assert got == want and info["data_mode"] == 0 and info["header_bytes"] == len(M.header(M.XYZI, len(c), "ascii"))
    assert codec.format(c, mode="ascii") == want


def test_one_cache_serves_every_mode(codec):
    """a size query in one mode followed by a fetch in another formats again, in the fetch's mode"""
    L = codec.L
    c = labelled_cloud(5000, seed=9)
    want = {m: E.hc_format(c, m)[1] for m in MODES}
    want["ascii"] = codec.format(c)
    for first in ("ascii",) + MODES:
        for second in ("ascii",) + MODES:
            size, info = ctypes.c_size_t(0), capi.PcdFormatInfoC()
            assert L.erasor_pcd_format(codec.h, ctypes.c_void_p(c.ctypes.data), len(c), capi.PTR_HOST, capi.PCD_MODES[first], None, 0,
                                       capi.PTR_HOST, ctypes.byref(size), ctypes.byref(info)) == 0
            assert size.value == len(want[first])
            buf = np.zeros(len(want[second]), np.uint8)
            assert L.erasor_pcd_format(codec.h, ctypes.c_void_p(c.ctypes.data), len(c), capi.PTR_HOST, capi.PCD_MODES[second],
                                       ctypes.c_void_p(buf.ctypes.data), len(buf), capi.PTR_HOST, ctypes.byref(size), ctypes.byref(info)) == 0
            assert buf.tobytes() == want[second] and info.data_mode == capi.PCD_MODES[second]
    # too small a buffer: ERASOR_E_CAPACITY with the exact size
    small = np.zeros(10, np.uint8)
    assert L.erasor_pcd_format(codec.h, ctypes.c_void_p(c.ctypes.data), len(c), capi.PTR_HOST, 2, ctypes.c_void_p(small.ctypes.data), 10,
                               capi.PTR_HOST, ctypes.byref(size), None) == capi.E_CAPACITY
    assert size.value == len(want["binary_compressed"])


def test_errors(codec):
    import torch
    L = codec.L
    size = ctypes.c_size_t(0)
    c = labelled_cloud(64)
    for bad in (3, -1, 7):
        assert L.erasor_pcd_format(codec.h, ctypes.c_void_p(c.ctypes.data), len(c), capi.PTR_HOST, bad, None, 0, capi.PTR_HOST,
                                   ctypes.byref(size), None) == capi.E_INVALID
    with pytest.raises(ValueError):
        codec.format(c, mode="compressed")
    # a device cloud 4 bytes off its 16-byte alignment: refused before anything is read (and every byte of n points lies inside)
    d = torch.zeros(65 * 4, dtype=torch.float32, device="cuda")
    for mode in MODES:
        assert L.erasor_pcd_format(codec.h, ctypes.c_void_p(d.data_ptr() + 4), 64, capi.PTR_DEVICE, capi.PCD_MODES[mode], None, 0,
                                   capi.PTR_HOST, ctypes.byref(size), None) == capi.E_INVALID
    # the handle is still usable
    assert codec.format(c, mode="binary_compressed") == E.hc_format(c, "binary_compressed")[1]


CPP = r'''
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "erasor/offline_map_updater.hpp"
using namespace erasor_b200;
int main(int argc, char** argv) {
    FILE* f = std::fopen(argv[1], "rb");
    std::vector<float> v;
    float x;
    while (std::fread(&x, 4, 1, f) == 1) v.push_back(x);
    std::fclose(f);
    PointCloud c(v.size() / 4);
    std::memcpy(c.data(), v.data(), v.size() * 4);
    PcdCodec codec;
    codec.write(argv[2], c, std::atoi(argv[3]));
    return 0;
}
'''


def test_cpp_pcdcodec_write(codec, tmp_path):
    src, exe = tmp_path / "w.cpp", tmp_path / "w"
    src.write_text(CPP)
    lib = os.path.join(ROOT, "erasor_b200", "_lib")
    subprocess.run(["g++", "-std=c++17", "-O1", "-include", "cstring", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include",
                    str(src), "-o", str(exe), "-L" + lib, "-lerasor_b200", "-Wl,-rpath," + lib, "-L/usr/local/cuda/lib64",
                    "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"], check=True, capture_output=True, text=True)
    c = special_cloud(3000, seed=11)
    (tmp_path / "c.bin").write_bytes(c.tobytes())
    for mode in ("ascii",) + MODES:
        out = tmp_path / f"{mode}.pcd"
        r = subprocess.run([str(exe), str(tmp_path / "c.bin"), str(out), str(capi.PCD_MODES[mode])], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        py = tmp_path / f"{mode}_py.pcd"
        codec.write(str(py), c, mode=mode)
        assert out.read_bytes() == py.read_bytes()


def _pipeline_case():
    from erasor_b200 import params as P
    from test_mapgen import _nodes
    nodes = _nodes(n_nodes=12, seed=7)
    ep, up = P.preset("seq_05"), P.updater_preset("seq_05")
    up.removal_interval = 2
    up.map_voxel_size = 0.2
    return nodes, up, ep


def test_run_sequence_writes_binary_compressed(codec, tmp_path):
    from erasor_b200 import pipeline
    nodes, up, ep = _pipeline_case()
    res = pipeline.run_sequence(nodes, up, ep, out_dir=str(tmp_path), pcd_mode="binary_compressed")
    name = getattr(up, "data_name", "seq")
    for fname, arr in ((f"{name}_naive_map.pcd", res["naive_map"]), (f"{name}_result.pcd", res["static_map"])):
        data = (tmp_path / fname).read_bytes()
        assert b"\nDATA binary_compressed\n" in data[:400]
        assert bits_equal(codec.load(str(tmp_path / fname)), arr)
    with pytest.raises(ValueError):
        pipeline.run_sequence(nodes, up, ep, pcd_mode="binary_compressed", make_updater=lambda u, e, m: None)


def test_analysis_cli_reads_binary_compressed_files(codec, tmp_path):
    gt = labelled_cloud(20_000, seed=5)
    est = gt[np.random.default_rng(6).random(len(gt)) < 0.7]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    outs = []
    for mode in ("ascii", "binary_compressed"):
        d = tmp_path / mode
        d.mkdir()
        for name, c in (("gt.pcd", gt), ("est.pcd", est)):
            if mode != "ascii":
                c = codec.load(str(tmp_path / "ascii" / name))          # the floats the ASCII file holds
            codec.write(str(d / name), c, mode=mode)
        outs.append(subprocess.run([sys.executable, "-m", "erasor_b200.analysis", "--gt", "gt.pcd", "--est", "est.pcd"], cwd=d, env=env,
                                   check=True, capture_output=True, text=True).stdout)
    assert outs[1] == outs[0] and "gt.pcd" in outs[0]
