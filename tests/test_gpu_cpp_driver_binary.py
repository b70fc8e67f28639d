"""GPU: the C++ driver (examples/offline_map_updater_main) on a layout that mixes ASCII and binary scans.  ASCII scans are parsed
on the device; binary ones, which the device codec leaves to load_pcd, are read on the host and uploaded.  With every binary
scan holding exactly the floats its ASCII twin parses to, the saved static map must be byte-identical to the all-ASCII run's."""
import os
import subprocess

import numpy as np
import pytest

from erasor_b200 import evaluate as E
from erasor_b200 import synth
from test_gpu_cpp_driver import BIN, YAML

pytestmark = pytest.mark.gpu


def write_pcd_binary(path, xyzi):
    """the layout pcl::io::savePCDFileBinary writes for PointXYZI (x y z intensity, four floats per point)"""
    n = len(xyzi)
    head = ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\nTYPE F F F F\n"
            f"COUNT 1 1 1 1\nWIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA binary\n")
    with open(path, "wb") as f:
        f.write(head.encode())
        f.write(np.ascontiguousarray(xyzi, dtype="<f4").tobytes())


def run_driver(tmp_path, name, gt_map, scans, poses, binary_scans):
    data, save = tmp_path / name / "data", tmp_path / name / "out"
    (data / "pcds").mkdir(parents=True)
    save.mkdir()
    E.write_pcd_ascii(str(data / "dense_global_map.pcd"), gt_map)
    with open(data / "poses_lidar2body.csv", "w") as f:
        f.write("index,time,x,y,z,qx,qy,qz,qw\n")
        for k, (s, p) in enumerate(zip(scans, poses)):
            path = str(data / "pcds" / f"{k:06d}.pcd")
            if k in binary_scans:
                write_pcd_binary(path, s)
            else:
                E.write_pcd_ascii(path, s)
            f.write(f"{k},{k * 0.1}," + ",".join(f"{v:.9g}" for v in p) + "\n")
    cfg = tmp_path / name / "seq_05.yaml"
    cfg.write_text(YAML.format(save=str(save)))
    r = subprocess.run([BIN, str(cfg), str(data)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:] + r.stdout[-2000:]
    return open(save / "05_result.pcd", "rb").read()


def test_cpp_driver_reads_binary_scans(tmp_path):
    assert os.path.exists(BIN), "build with erasor_b200/csrc/build.sh"
    sc = synth.Scene(seed=43, length=40.0, n_nodes=15, n_dynamic=6)
    kw = dict(n_beams=24, n_az=480)
    nodes = list(range(15))
    gt_map = sc.build_map(nodes, voxel=0.2, **kw)
    scans, poses = [], []
    for k in nodes:
        p = str(tmp_path / "round.pcd")
        E.write_pcd_ascii(p, sc.scan(k, seed_offset=9, **kw))
        scans.append(E.read_pcd_ascii(p))           # the floats an ASCII scan file parses to
        poses.append(sc.pose7(k))
    ascii_only = run_driver(tmp_path, "ascii", gt_map, scans, poses, binary_scans=set())
    mixed = run_driver(tmp_path, "mixed", gt_map, scans, poses, binary_scans={0, 1, 4, 7, 8, 14})
    assert len(E.read_pcd_ascii(str(tmp_path / "mixed" / "out" / "05_result.pcd"))) > 0
    assert mixed == ascii_only
