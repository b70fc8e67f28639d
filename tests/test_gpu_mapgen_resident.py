"""GPU: the resident map generator (erasor_mapgen_*, capi.MapGen, DESIGN.md section 8.2) against the oracle's restatement of the
reference's mapgen (src/mapgen/mapgen.hpp:198-305), bit for bit via view(np.uint32): every node's cloud_curr and cloud_map, both
saved clouds, large-scale parking at the true period, edge cases, device scans, buffer regrowth, the per-node launch and
synchronisation counts, the error paths, and the C++ driver (examples/mapgen_main) end to end into offline_map_updater_main."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from erasor_b200 import capi, kitti, mapgen
from erasor_b200 import evaluate as E
from erasor_b200 import params as P
from test_mapgen import _nodes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "erasor_b200", "_lib")


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _run_both(oracle_mod, nodes, leafsize, large_scale, check_every_node=True, gen=None):
    own = gen is None
    gen = gen or capi.MapGen(leafsize, large_scale)
    o = oracle_mod.OracleMapGen(leafsize, large_scale)
    for k, odom, cloud in nodes:
        gen.accum(odom, cloud)
        o.accum(odom, cloud)
        if check_every_node:
            assert _same(gen.cloud(gen.CLOUD_CURR), o.cloud(o.CLOUD_CURR)), f"node {k}: cloud_curr"
            assert _same(gen.cloud(gen.CLOUD_MAP), o.cloud(o.CLOUD_MAP)), f"node {k}: cloud_map"
    assert _same(gen.cloud(gen.CLOUD_MAP), o.cloud(o.CLOUD_MAP))
    orig, vox = gen.save_naive_map()
    assert _same(orig, o.cloud(o.SAVED_ORIGINAL)), "SAVED_ORIGINAL"
    assert _same(vox, o.cloud(o.SAVED_VOXELIZED)), "SAVED_VOXELIZED"
    o.close()
    if own:
        gen.close()
    return orig, vox


@pytest.mark.parametrize("large_scale", [False, True])
def test_resident_mapgen_matches_the_oracle_node_by_node(oracle_mod, large_scale):
    orig, vox = _run_both(oracle_mod, _nodes(), 0.2, large_scale)
    assert len(vox) > 1000 and len(vox) < len(orig)


def _small_nodes(n_nodes, n_pts=300, seed=21):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_nodes):
        r = rng.uniform(0.5, 35.0, n_pts); th = rng.uniform(-np.pi, np.pi, n_pts)
        scan = np.stack([r * np.cos(th), r * np.sin(th), rng.normal(-1.7, 0.2, n_pts), rng.choice([40.0, 48.0, 252.0], n_pts)], axis=1)
        yaw = 0.002 * k
        odom = np.array([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2)])
        out.append((k, odom, np.ascontiguousarray(scan, dtype=np.float32)))
    return out


def test_long_large_scale_run_parks_at_the_true_period(oracle_mod):
    """1100 nodes: parking fires at the 2nd, 502nd and 1002nd node (mapgen.hpp:248); 3 extra launches"""
    nodes = _small_nodes(1100)
    gen = capi.MapGen(0.2, True)
    o = oracle_mod.OracleMapGen(0.2, True)
    launches = []
    for k, odom, cloud in nodes:
        before = gen.counters()["launches"]
        gen.accum(odom, cloud)
        o.accum(odom, cloud)
        launches.append(gen.counters()["launches"] - before)
        if k in (0, 1, 2, 500, 501, 502, 1000, 1001, 1002, 1099):
            assert _same(gen.cloud(gen.CLOUD_CURR), o.cloud(o.CLOUD_CURR)), f"node {k}: cloud_curr"
            assert _same(gen.cloud(gen.CLOUD_MAP), o.cloud(o.CLOUD_MAP)), f"node {k}: cloud_map"
    assert [k for k, c in enumerate(launches) if c == 2] == [1, 501, 1001]
    assert all(c in (1, 2) for c in launches)
    assert _same(gen.cloud(gen.SAVED_ORIGINAL), o.cloud(o.SAVED_ORIGINAL))
    assert _same(gen.cloud(gen.SAVED_VOXELIZED), o.cloud(o.SAVED_VOXELIZED))
    gen.close(); o.close()


@pytest.mark.parametrize("large_scale", [False, True])
def test_edge_cases(oracle_mod, large_scale):
    """an empty first node, a node wholly inside 2.7 m, an empty node later on, the cut's float/double edge"""
    r = np.float32(2.7)
    edge = np.array([[r, 0, 0, 1], [np.nextafter(r, np.float32(0)), 0, 0, 2], [np.nextafter(r, np.float32(9)), 0, 0, 3],
                     [1.0, 1.0, 0.5, 4], [30.0, -4.0, -1.2, 5], [-1.9091883, 1.9091883, 0.1, 6], [0, 0, 0, 7]], dtype=np.float32)
    inside = np.array([[1.0, 0.5, -1.0, 40], [-2.0, 1.0, -1.5, 48], [0.0, 2.6, 0.0, 252]], dtype=np.float32)
    base = _nodes(4, seed=8)
    ident = np.array([0, 0, 0, 0, 0, 0, 1.0])
    seq = [(0, ident, np.zeros((0, 4), dtype=np.float32)), (1, ident, edge), (2, base[1][1], inside), (3, base[2][1], base[2][2]),
           (5, ident, np.zeros((0, 4), dtype=np.float32)), (6, base[3][1], base[3][2])]
    _run_both(oracle_mod, seq, 0.2, large_scale)


def test_device_scans_equal_host_scans(oracle_mod):
    import torch
    nodes = _nodes(6, seed=3)
    host = capi.MapGen(0.2, True)
    dev = capi.MapGen(0.2, True)
    keep = []
    for _, odom, cloud in nodes:
        host.accum(odom, cloud)
        t = torch.from_numpy(cloud).cuda()
        keep.append(t)                       # read asynchronously: alive until the next call that returns data
        dev.accum_ptr(odom, t.data_ptr(), len(cloud), capi.PTR_DEVICE)
    for which in range(4):
        assert _same(dev.cloud(which), host.cloud(which)), which
    p, n = dev.device_cloud(dev.SAVED_ORIGINAL)
    assert n == len(host.cloud(host.SAVED_ORIGINAL)) and p != 0
    out = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    nn = ctypes.c_size_t(0)
    dev._ck(dev.L.erasor_mapgen_get_cloud(dev.h, dev.SAVED_ORIGINAL, ctypes.c_void_p(out.data_ptr()), n, capi.PTR_DEVICE, ctypes.byref(nn)))
    assert _same(out.cpu().numpy(), host.cloud(host.SAVED_ORIGINAL))
    host.close(); dev.close()


def test_buffer_growth_gives_the_same_map(oracle_mod):
    """scans that double in size: the map buffer (64 Ki points at first) and the scratch buffers regrow several times"""
    rng = np.random.default_rng(4)
    nodes = []
    for k, n in enumerate([5000, 20000, 40000, 80000, 160000, 1000, 200000]):
        r = rng.uniform(3.0, 60.0, n); th = rng.uniform(-np.pi, np.pi, n)
        scan = np.stack([r * np.cos(th), r * np.sin(th), rng.uniform(-2.0, 4.0, n), rng.choice([40.0, 252.0], n)], axis=1).astype(np.float32)
        nodes.append((k, np.array([2.0 * k, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]), scan))
    gen = capi.MapGen(0.1, False)
    _run_both(oracle_mod, nodes, 0.1, False, gen=gen)
    assert gen.counters()["regrowths"] >= 6
    gen.close()


def test_counters_one_launch_and_no_sync_per_node():
    nodes = _small_nodes(40, n_pts=2000, seed=2)
    gen = capi.MapGen(0.2, True)
    prev = gen.counters()
    steady = 0
    for k, odom, cloud in nodes:
        gen.accum(odom, cloud)
        c = gen.counters()
        d = {key: c[key] - prev[key] for key in c}
        prev = c
        if k == 1:
            assert d["launches"] == 2, d                 # the 2nd node parks
        elif d["regrowths"] == 0:
            assert d["launches"] == 1 and d["host_syncs"] == 0, (k, d)
            steady += 1
        else:
            assert d["launches"] == 1 and d["host_syncs"] <= 1, (k, d)      # one read-back of the size, then the regrowths
    assert steady >= 30
    gen.close()


def test_error_paths():
    L = capi.lib()
    h = ctypes.c_void_p()
    bad = capi.MapGenParamsC(0.0, 0)
    assert L.erasor_mapgen_create(ctypes.byref(bad), 0, ctypes.byref(h)) == capi.E_INVALID
    assert L.erasor_mapgen_create(None, 0, ctypes.byref(h)) == capi.E_INVALID
    assert L.erasor_mapgen_last_error(None)
    gen = capi.MapGen(0.2, False)
    odom = np.array([0, 0, 0, 0, 0, 0, 1.0])
    pts = _nodes(2)[1][2]
    od = odom.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    assert L.erasor_mapgen_accum(None, od, pts.ctypes.data, len(pts), capi.PTR_HOST) == capi.E_INVALID
    assert L.erasor_mapgen_accum(gen.h, None, pts.ctypes.data, len(pts), capi.PTR_HOST) == capi.E_INVALID
    assert L.erasor_mapgen_accum(gen.h, od, None, len(pts), capi.PTR_HOST) == capi.E_INVALID
    assert L.erasor_mapgen_accum(gen.h, od, pts.ctypes.data, len(pts), capi.PTR_HOST | capi.PTR_QUERY_XYZ) == capi.E_INVALID
    assert b"intensity" in L.erasor_mapgen_last_error(gen.h)
    assert L.erasor_mapgen_accum(gen.h, od, pts.ctypes.data, 1 << 31, capi.PTR_HOST) == capi.E_CAPACITY
    gen.accum(odom, pts)
    n = ctypes.c_size_t(0)
    assert L.erasor_mapgen_get_cloud(gen.h, 0, None, 0, capi.PTR_HOST, None) == capi.E_INVALID
    assert L.erasor_mapgen_get_cloud(gen.h, 7, None, 0, capi.PTR_HOST, ctypes.byref(n)) == capi.E_INVALID
    assert L.erasor_mapgen_get_cloud(gen.h, 0, None, 0, capi.PTR_HOST, ctypes.byref(n)) == capi.OK and n.value > 0
    small = np.empty((n.value - 1, 4), dtype=np.float32)
    assert L.erasor_mapgen_get_cloud(gen.h, 0, small.ctypes.data, n.value - 1, capi.PTR_HOST, ctypes.byref(n)) == capi.E_CAPACITY
    p = ctypes.c_void_p()
    assert L.erasor_mapgen_device_cloud(gen.h, 0, None, ctypes.byref(n)) == capi.E_INVALID
    assert L.erasor_mapgen_device_cloud(gen.h, 1, ctypes.byref(p), None) == capi.E_INVALID
    assert L.erasor_mapgen_get_counters(None, None, None, None) == capi.E_INVALID
    assert L.erasor_mapgen_synchronize(None) == capi.E_INVALID
    # the handle is still usable after the failed calls
    o = mapgen.NaiveMapGenerator(mapgen.device_voxelizer(), leafsize=0.2)
    o.accum_point_cloud(odom, pts)
    assert _same(gen.cloud(gen.CLOUD_MAP), o.cloud_map)
    gen.close()


def test_build_map_uses_the_resident_generator(oracle_mod):
    nodes = _nodes(7, seed=5)
    for large_scale in (False, True):
        orig, vox = mapgen.build_map(nodes, leafsize=0.2, is_large_scale=large_scale)
        o = oracle_mod.OracleMapGen(0.2, large_scale)
        for _, odom, cloud in nodes:
            o.accum(odom, cloud)
        assert _same(orig, o.cloud(o.SAVED_ORIGINAL)) and _same(vox, o.cloud(o.SAVED_VOXELIZED))
        o.close()


YAML = """
erasor:
    max_range: 60.0
    num_rings: 15
    num_sectors: 60
    min_h: -1.3
    max_h: 3.2
    th_bin_max_h: 0.05
    scan_ratio_threshold: 0.3
    minimum_num_pts: 10
    rejection_ratio: 0
    gf_dist_thr: 0.15
    gf_iter: 3
    gf_num_lpr: 10
    gf_th_seeds_height: 0.5
    version: 3

MapUpdater:
    data_name: "05"
    initial_map_path: "unused"
    env: "outdoor"
    save_path: "{save}"
    query_voxel_size: 0.2
    map_voxel_size: 0.05
    removal_interval: 2

tf:
     lidar2body: [0.0, 0.0, 1.73, 0, 0.0, 0.0, 1.0]

verbose: false
"""


@pytest.mark.parametrize("large_scale", [False, True])
def test_cpp_mapgen_driver_end_to_end(tmp_path, oracle_mod, large_scale):
    """nodes -> export_env_layout -> mapgen_main: both files byte-identical to write_pcd_ascii of the oracle's saved clouds, under
    the reference's names; then offline_map_updater_main on the produced map equals the oracle's updater pass"""
    binm = os.path.join(LIB, "mapgen_main")
    binu = os.path.join(LIB, "offline_map_updater_main")
    assert os.path.exists(binm) and os.path.exists(binu), "build with erasor_b200/csrc/build.sh"
    nodes = _nodes(10, seed=6)
    data = tmp_path / "data"
    kitti.export_env_layout(nodes, str(data))
    save = tmp_path / "maps"
    save.mkdir()
    target = "05_0_to_18_w_interval_2_node.bag"
    r = subprocess.run([binm, str(data), target, str(save), "0.2", "true" if large_scale else "false"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:] + r.stdout[-2000:]
    stem = f"05_0_to_18_w_interval2_voxel_{float(np.float32(0.2)):f}"
    assert stem == "05_0_to_18_w_interval2_voxel_0.200000"
    # the oracle fed what the driver read: the scans as written to the files, the poses exactly (%.17g, stod)
    scans = [E.read_pcd_ascii(str(data / "pcds" / f"{i:06d}.pcd")) for i in range(len(nodes))]
    o = oracle_mod.OracleMapGen(0.2, large_scale)
    for (_, odom, _), s in zip(nodes, scans):
        o.accum(odom, s)
    for suffix, which in (("_original.pcd", o.SAVED_ORIGINAL), (".pcd", o.SAVED_VOXELIZED)):
        ref = tmp_path / ("ref" + suffix)
        E.write_pcd_ascii(str(ref), o.cloud(which))
        assert (save / (stem + suffix)).read_bytes() == ref.read_bytes(), suffix
    naive = o.cloud(o.SAVED_VOXELIZED)
    o.close()
    # stage 2 on the produced map, as test_gpu_cpp_driver checks it
    (data / "dense_global_map.pcd").write_bytes((save / (stem + ".pcd")).read_bytes())
    out = tmp_path / "out"
    out.mkdir()
    cfg = tmp_path / "seq_05.yaml"
    cfg.write_text(YAML.format(save=str(out)))
    r = subprocess.run([binu, str(cfg), str(data)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:] + r.stdout[-2000:]
    result = E.read_pcd_ascii(str(out / "05_result.pcd"))
    ep, up = P.preset("seq_05"), P.updater_preset("seq_05")
    up.removal_interval = 2
    m0 = E.read_pcd_ascii(str(data / "dense_global_map.pcd"))
    assert np.allclose(m0, naive, rtol=2e-7, atol=1e-7)
    ou = oracle_mod.OracleUpdater(up, ep, m0)
    for i, (_, odom, _) in enumerate(nodes):
        ou.callback_node(i, np.array([np.float32(v) for v in odom], dtype=np.float64), scans[i])     # stof() in that driver
    ref = ou.save_static_map(0.2)
    assert result.shape == ref.shape
    assert np.allclose(result, ref, rtol=2e-7, atol=1e-7)
    a, b = E.evaluate(m0, result), E.evaluate(m0, ref)
    assert abs(a["PR"] - b["PR"]) < 1e-9 and abs(a["RR"] - b["RR"]) < 1e-9
