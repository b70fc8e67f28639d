"""GPU parity of erasor_voxelize_batch (voxelize_batch.cu) against the oracle, bit for bit, cloud by cloud: prepared queries
(oracle.transform(oracle.voxelize(scan, leaf), T_lidar2body)) over batch sizes, leaves, edge clouds, a 2.6 M-point cloud, host and
device inputs and three lidar2body poses; agreement with the updater's query VoI; the keep mask; node mode fed prepared queries;
saving node mode's static map; run_frame_independent; launch counts; and the fences."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

from erasor_b200 import params as P  # noqa: E402
from erasor_b200 import synth  # noqa: E402
from test_voxelize_batch_model import batch_of, mixed_clouds  # noqa: E402

pytestmark = pytest.mark.gpu

L2B = {"identity": [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0],
       "seq05": [0.0, 0.0, 1.73, 0.0, 0.0, 0.0, 1.0],
       "tilted": [0.31, -0.12, 1.73, 0.0436, -0.0262, 0.0087, 0.9986]}


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.fixture(scope="module")
def scene():
    return synth.Scene(seed=17, length=120.0, n_nodes=61, n_dynamic=10)


@pytest.fixture(scope="module")
def handle():
    from erasor_b200 import capi
    h = capi.Handle(P.preset("seq_05"))
    yield h
    h.close()


def _prepared(oracle_mod, cloud, leaf, pose7):
    v = oracle_mod.voxelize(cloud, leaf)
    return v if pose7 is None else oracle_mod.transform(v, oracle_mod.pose_to_matrix(pose7))


def _check(oracle_mod, h, clouds, leaf, pose7=None, device=False, keep=None):
    import torch
    xyzi, off = batch_of(clouds)
    if device:
        t = torch.from_numpy(xyzi).cuda()
        k = torch.from_numpy(keep).cuda() if keep is not None else None
        d, oo = h.voxelize_batch_ptr(t.data_ptr() if len(xyzi) else 0, off, leaf, k.data_ptr() if k is not None else 0, pose7, 1)
        from erasor_b200.capi import _memcpy_from_device
        out = np.empty((int(oo[-1]), 4), dtype=np.float32)
        _memcpy_from_device(out, d)
    else:
        out, oo = h.voxelize_batch(xyzi, off, leaf, keep=keep, pose7=pose7)
    o = off.astype(np.int64)
    for c, cloud in enumerate(clouds):
        sel = cloud if keep is None else cloud[keep[o[c]:o[c + 1]] != 0]
        want = _prepared(oracle_mod, sel, leaf, pose7)
        got = out[int(oo[c]):int(oo[c + 1])]
        assert _same(got, want), f"cloud {c} of {len(clouds)} (n={len(cloud)}) leaf={leaf}: {got.shape} vs {want.shape}"


@pytest.mark.parametrize("F", [1, 2, 7, 20, 64, 300])
def test_prepared_queries_batch_sizes(oracle_mod, scene, handle, F):
    kw = dict(n_beams=64, n_az=1800) if F <= 20 else dict(n_beams=16, n_az=360)      # HDL-64 (~115 k points) up to 20 scans
    clouds = [scene.scan(k % 61, seed_offset=k // 61, **kw) for k in range(F)]
    _check(oracle_mod, handle, clouds, 0.2, L2B["seq05"], device=(F % 2 == 0))


@pytest.mark.parametrize("leaf", [0.1, 0.2, 0.5, 1.0])
@pytest.mark.parametrize("pose", ["identity", "seq05", "tilted"])
def test_prepared_queries_leaves_and_poses(oracle_mod, scene, handle, leaf, pose):
    clouds = [scene.scan(k, n_beams=64, n_az=1800) for k in (5, 30)] + mixed_clouds(seed=4)
    _check(oracle_mod, handle, clouds, leaf, L2B[pose], device=(pose == "tilted"))


@pytest.mark.parametrize("device", [False, True])
def test_edge_clouds(oracle_mod, handle, device):
    """empty, 1-point and 2-point clouds, one voxel, duplicates with different labels, voxel faces and +-1 ulp, an overflowing
    cloud between normal ones (with a duplicate of another label inside), no pose and a pose"""
    cl = mixed_clouds(seed=9)
    cl.insert(3, np.array([[0.5, 0.5, 0.5, 3.0], [0.5, 0.5, 0.5, 4.0]], np.float32))
    for leaf in (0.2, 1.0):
        _check(oracle_mod, handle, cl, leaf, None, device=device)
        _check(oracle_mod, handle, cl, leaf, L2B["tilted"], device=device)


def test_large_cloud_in_a_batch_of_small_ones(oracle_mod, scene, handle):
    rng = np.random.default_rng(11)
    big = np.zeros((2_600_000, 4), np.float32)
    big[:, :2] = rng.uniform(-60, 60, (len(big), 2))
    big[:, 2] = rng.uniform(-3, 3, len(big))
    big[:, 3] = rng.integers(0, 260, len(big))
    big[1_000_000:1_300_000] = big[:300_000]
    big[1_000_000:1_300_000, 3] += 1.0                          # duplicates far apart, other labels: ties to the lowest index
    ovf = np.zeros((30_000, 4), np.float32)
    ovf[:, :3] = rng.uniform(-4000, 4000, (len(ovf), 3))
    ovf[20_000:] = ovf[:10_000]
    ovf[20_000:, 3] = 9.0
    small = [scene.scan(k, n_beams=16, n_az=360) for k in range(6)]
    clouds = small[:3] + [big] + small[3:5] + [ovf] + small[5:]
    _check(oracle_mod, handle, clouds, 0.3, None, device=True)
    _check(oracle_mod, handle, clouds, 0.3, L2B["seq05"], device=False)


def test_keep_mask_selects_points_and_the_1nn(oracle_mod, scene, handle):
    clouds = [scene.scan(k, n_beams=64, n_az=1800) for k in (2, 9, 40)] + mixed_clouds(seed=5)
    xyzi, _ = batch_of(clouds)
    rng = np.random.default_rng(2)
    keep = (rng.random(len(xyzi)) < 0.5).astype(np.uint8)
    # a deselected exact duplicate in front of a selected point, with another label: the 1-NN must not see it
    xyzi_dup = [c.copy() for c in clouds]
    _check(oracle_mod, handle, xyzi_dup, 0.2, None, keep=keep)
    _check(oracle_mod, handle, xyzi_dup, 0.2, L2B["seq05"], keep=keep, device=True)
    dup = np.array([[1.0, 1.0, 1.0, 200.0], [1.0, 1.0, 1.0, 7.0], [1.05, 1.0, 1.0, 8.0]], np.float32)
    _check(oracle_mod, handle, [dup], 0.2, None, keep=np.array([0, 1, 1], np.uint8))


def test_agrees_with_the_updater_query_voi(scene, handle):
    from erasor_b200 import capi
    ep, up = P.preset("seq_05"), P.updater_preset("seq_05")
    up.removal_interval = 1
    mw = scene.build_map(range(0, 61, 6), voxel=0.2, n_beams=32, n_az=720)
    u = capi.Updater(up, ep, mw)
    scans = [scene.scan(k, n_beams=64, n_az=1800, seed_offset=3) for k in (4, 11, 27)]
    out, oo = handle.voxelize_batch(*batch_of(scans), up.query_voxel_size, pose7=up.lidar2body)
    for i, k in enumerate((4, 11, 27)):
        assert u.process_node(k, scene.pose7(k), scans[i])
        assert _same(out[int(oo[i]):int(oo[i + 1])], u.cloud(u.QUERY_VOI)), f"scan {k}"
    u.close()


@pytest.mark.parametrize("n_nodes", [20, 160])
def test_node_mode_on_prepared_queries(oracle_mod, scene, n_nodes):
    """process_scans (raw scans -> device queries -> node mode) against node mode fed the oracle's prepared queries: keep mask,
    frame_keep and node stats byte-identical.  160 nodes exceed the 150-node records split."""
    from erasor_b200 import capi
    ep, up = P.preset("seq_05"), P.updater_preset("seq_05")
    mw = scene.build_map(range(0, 61, 3), voxel=0.2, n_beams=32, n_az=720)
    ks = [k % 61 for k in range(n_nodes)]
    kw = dict(n_beams=64, n_az=1800) if n_nodes <= 20 else dict(n_beams=32, n_az=600)
    scans = [scene.scan(k, seed_offset=7 + i // 61, **kw) for i, k in enumerate(ks)]
    poses = np.stack([scene.pose7(k) for k in ks])
    raw, off = batch_of(scans)
    res = []
    for prepared_by_oracle in (False, True):
        m = capi.Map(mw)
        h = capi.Handle(ep.replace(version=up.version))
        h.attach_map(m)
        if prepared_by_oracle:
            qs = [_prepared(oracle_mod, s, up.query_voxel_size, up.lidar2body) for s in scans]
            q, qo = batch_of(qs)
            keep, fk = h.process_nodes(poses, q, qo, voi_max_range=up.max_range, want_frame_keep=True)
        else:
            keep, fk = h.process_scans(poses, raw, off, up.query_voxel_size, up.lidar2body, voi_max_range=up.max_range, want_frame_keep=True)
        res.append((keep, fk, h.node_stats()))
        h.close(); m.close()
    (k0, f0, s0), (k1, f1, s1) = res
    assert np.array_equal(k0, k1) and np.array_equal(f0, f1)
    for a, b in zip(s0, s1):
        assert np.array_equal(a, b)
    assert (k0 == 0).any()


def test_save_static_map(oracle_mod, scene, handle):
    from erasor_b200 import capi
    rng = np.random.default_rng(4)
    twin = scene.build_map(range(0, 61, 2), voxel=0.2, n_beams=32, n_az=900)
    big = np.zeros((2_700_000, 4), np.float32)
    big[:, :2] = rng.uniform(-80, 80, (len(big), 2))
    big[:, 2] = rng.uniform(-2, 6, len(big))
    big[:, 3] = rng.integers(0, 260, len(big))
    for mw, voxel in ((twin, 0.2), (twin, 0.05), (big, 0.2)):
        m = capi.Map(mw)
        keep = (rng.random(len(mw)) < 0.8).astype(np.uint8)
        import torch
        tk = torch.from_numpy(keep).cuda()
        import ctypes
        ctypes.CDLL("libcudart.so.12").cudaMemcpy(ctypes.c_void_p(m.keep_ptr), ctypes.c_void_p(tk.data_ptr()), ctypes.c_size_t(len(keep)), 3)
        got = handle.save_static_map(m, voxel)
        want = oracle_mod.voxelize(mw[keep != 0], voxel)
        assert _same(got, want), f"n={len(mw)} voxel={voxel}"
        m.close()


def test_run_frame_independent_matches_oracle_prepared(oracle_mod, scene, tmp_path):
    from erasor_b200 import evaluate, pipeline
    ep, up = P.preset("seq_05"), P.updater_preset("seq_05")
    up.removal_interval = 2
    mw = scene.build_map(range(0, 61, 3), voxel=0.2, n_beams=32, n_az=720)
    nodes = [(k, scene.pose7(k), scene.scan(k, n_beams=64, n_az=1800, seed_offset=2)) for k in range(0, 40)]

    def oracle_prepare(raw, off):
        o = off.astype(np.int64)
        return batch_of([_prepared(oracle_mod, raw[o[c]:o[c + 1]], up.query_voxel_size, up.lidar2body) for c in range(len(o) - 1)])

    a = pipeline.run_frame_independent(nodes, mw, up, ep, batch=7, save_voxel_size=0.2)
    b = pipeline.run_frame_independent(nodes, mw, up, ep, batch=20, save_voxel_size=0.2, prepare=oracle_prepare)
    assert a["processed_scans"] == b["processed_scans"] == 20 and a["nodes"] == 40
    assert np.array_equal(a["keep"], b["keep"]) and _same(a["static_map"], b["static_map"])
    assert _same(a["static_map"], oracle_mod.voxelize(mw[a["keep"] != 0], 0.2))
    pa, pb = tmp_path / "a.pcd", tmp_path / "b.pcd"
    evaluate.write_pcd_ascii(str(pa), a["static_map"])
    evaluate.write_pcd_ascii(str(pb), b["static_map"])
    assert pa.read_bytes() == pb.read_bytes()


def test_launch_count_does_not_depend_on_the_batch(scene, handle):
    scans = [scene.scan(k % 61, n_beams=16, n_az=360, seed_offset=k // 61) for k in range(64)]
    counts = []
    for F in (1, 64, 64, 2):
        n0 = handle.kernel_launch_count()
        handle.voxelize_batch(*batch_of(scans[:F]), 0.2, pose7=L2B["seq05"])
        counts.append(handle.kernel_launch_count() - n0)
    assert len(set(counts)) == 1, counts
    n0 = handle.kernel_launch_count()
    handle.voxelize_batch(*batch_of(scans * 5), 0.2)             # 320 clouds: a second cloud-index digit, one more radix pass
    assert handle.kernel_launch_count() - n0 == counts[0] + 3


def test_fences_and_recovery(oracle_mod, scene, handle):
    from erasor_b200 import capi
    clouds = [scene.scan(k, n_beams=16, n_az=360) for k in range(3)]
    xyzi, off = batch_of(clouds)

    def code(*a, **k):
        with pytest.raises(capi.ErasorError) as e:
            handle.voxelize_batch_ptr(*a, **k)
        return e.value.code, str(e.value)

    bad = xyzi.copy()
    bad[int(off[1]) + 5, 1] = np.nan
    c, msg = code(bad.ctypes.data, off, 0.2)
    assert c == capi.E_INVALID and "point 5 of cloud 1" in msg
    bad[int(off[1]) + 5, 1] = np.inf
    keep = np.ones(len(bad), np.uint8)
    keep[int(off[1]) + 5] = 0
    out, _ = handle.voxelize_batch(bad, off, 0.2, keep=keep)            # a deselected non-finite point is not looked at
    assert code(xyzi.ctypes.data, np.array([0, 10, 5, len(xyzi)], np.uint64), 0.2)[0] == capi.E_INVALID
    assert code(xyzi.ctypes.data, np.array([3, len(xyzi)], np.uint64), 0.2)[0] == capi.E_INVALID
    assert code(xyzi.ctypes.data, np.array([0], np.uint64), 0.2)[0] == capi.E_INVALID
    assert code(xyzi.ctypes.data, off, 0.0)[0] == capi.E_INVALID
    assert code(xyzi.ctypes.data, np.array([0, 1 << 31], np.uint64), 0.2)[0] == capi.E_CAPACITY
    assert code(xyzi.ctypes.data, np.array([0, (1 << 31) - 1, (1 << 32) - 2, (1 << 32) - 1], np.uint64), 0.2)[0] == capi.E_CAPACITY
    _check(oracle_mod, handle, clouds, 0.2, L2B["seq05"])             # the handle still works


def test_static_map_nodes_driver(oracle_mod, tmp_path):
    """examples/static_map_nodes_main on the file layout, scans in ASCII and binary: its file equals run_frame_independent with the
    oracle's prepared queries, followed by write_pcd_ascii, byte for byte."""
    import subprocess
    from erasor_b200 import evaluate as E
    from erasor_b200 import pipeline
    from test_gpu_cpp_driver import YAML
    from test_gpu_cpp_driver_binary import write_pcd_binary
    binary = os.path.join(os.path.dirname(HERE), "erasor_b200", "_lib", "static_map_nodes_main")
    assert os.path.exists(binary), "build with erasor_b200/csrc/build.sh"
    sc = synth.Scene(seed=43, length=60.0, n_nodes=25, n_dynamic=6)
    kw = dict(n_beams=32, n_az=720)
    data, save = tmp_path / "data", tmp_path / "out"
    (data / "pcds").mkdir(parents=True)
    save.mkdir()
    E.write_pcd_ascii(str(data / "dense_global_map.pcd"), sc.build_map(range(25), voxel=0.2, **kw))
    gt_map = E.read_pcd_ascii(str(data / "dense_global_map.pcd"))
    nodes = []
    with open(data / "poses_lidar2body.csv", "w") as f:
        f.write("index,time,x,y,z,qx,qy,qz,qw\n")
        for k in range(25):
            path = str(data / "pcds" / f"{k:06d}.pcd")
            E.write_pcd_ascii(path, sc.scan(k, seed_offset=9, **kw))
            scan = E.read_pcd_ascii(path)
            if k % 3 == 1:
                write_pcd_binary(path, scan)
            pose = np.float32(sc.pose7(k)).astype(np.float64)            # the driver reads the csv as floats
            f.write(f"{k},{k * 0.1}," + ",".join(f"{v:.9g}" for v in pose) + "\n")
            nodes.append((k, pose, scan))
    cfg = tmp_path / "seq_05.yaml"
    cfg.write_text(YAML.format(save=str(save)))
    r = subprocess.run([binary, str(cfg), str(data), "0", "5"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:] + r.stdout[-2000:]
    ep, up = P.load_yaml(str(cfg))

    def oracle_prepare(raw, off):
        o = off.astype(np.int64)
        return batch_of([_prepared(oracle_mod, raw[o[c]:o[c + 1]], up.query_voxel_size, up.lidar2body) for c in range(len(o) - 1)])

    res = pipeline.run_frame_independent(nodes, gt_map, up, ep, batch=20, save_voxel_size=0.2, prepare=oracle_prepare)
    assert res["processed_scans"] == 12 and (res["keep"] == 0).any()
    E.write_pcd_ascii(str(tmp_path / "want.pcd"), res["static_map"])
    assert (save / "05_result.pcd").read_bytes() == (tmp_path / "want.pcd").read_bytes()
