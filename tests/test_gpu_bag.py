"""GPU: erasor/node bags read on the device (erasor_bag_index / erasor_bag_load, DESIGN.md section 12.2).  Decoded clouds must equal
the numpy model of tests/bag_model.py bit for bit, from pinned and pageable file buffers, into host and device outputs; the fences
must leave the handle usable; and the drivers and pipeline.run_bag fed from a bag must give exactly what the same nodes give
through the existing paths."""
import glob
import os
import subprocess

import numpy as np
import pytest

import bag_model as M
from erasor_b200 import capi, params, pipeline, synth
from test_gpu_cpp_driver import YAML
from test_gpu_cpp_driver_binary import write_pcd_binary

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "erasor_b200", "_lib")


def bits(a):
    a = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    return np.ascontiguousarray(a).view(np.uint32)


def rand_nodes(n_nodes, n_pts, seed, big=None, empty=(), nan=False):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_nodes):
        m = 0 if k in empty else (big if k == n_nodes // 2 and big else n_pts + (k * 37) % 101)
        c = (rng.normal(size=(m, 4)) * 30).astype(np.float32)
        c[:, 3] = rng.integers(0, 1 << 22, m).astype(np.float32)
        if nan and m:
            c.view(np.uint32)[::7, 1] = 0x7FA00000 + np.uint32(k)
        q = rng.normal(size=4)
        out.append((2 * k, np.r_[rng.normal(size=3) * 50, q / np.linalg.norm(q)], c))
    return out


def pinned(data):
    import torch
    t = torch.empty(len(data), dtype=torch.uint8, pin_memory=True)
    t.numpy()[:] = np.frombuffer(data, np.uint8)
    return t


def check_loads(codec, data, want, sizes=(1, 20, None)):
    for buf in (data, pinned(data)):
        info = codec.bag_index(buf)
        assert info["nodes"] == len(want)
        for size in sizes:
            count = len(want) if size is None else min(size, len(want))
            first = (len(want) - count) // 2
            for dev in (False, True):
                xyzi, off = codec.bag_load(first, count, device_out=dev)
                sub = want[first:first + count]
                assert np.array_equal(off, np.cumsum([0] + [len(w["cloud"]) for w in sub]).astype(np.uint64))
                ref = np.concatenate([w["cloud"] for w in sub]) if sub else np.zeros((0, 4), np.float32)
                assert np.array_equal(bits(xyzi), ref.view(np.uint32))
        seq, stamp, odom, clouds = codec.bag_meta()
        assert [int(s) for s in seq] == [w["seq"] for w in want]
        assert [int(s) for s in stamp] == [w["stamp_ns"] for w in want]
        assert np.array_equal(odom.view(np.uint64), np.stack([w["odom"] for w in want]).view(np.uint64))
        assert clouds == [w["layout"] for w in want]


@pytest.mark.parametrize("layout", [k for k in M.LAYOUTS if k != "x_float64"])
def test_layouts_bit_identical_to_the_model(layout):
    nodes = rand_nodes(30, 700, seed=len(layout), empty=(3, 17), nan=True)
    data = M.write_bag(M.kitti2node_messages(nodes, layout=layout, frame_ids=["f" * k for k in range(16)]), chunk_bytes=100000)
    with capi.PcdCodec() as codec:
        check_loads(codec, data, M.read_bag(data))


def test_organised_clouds_with_row_padding():
    rng = np.random.default_rng(4)
    msgs = []
    for k, (h, pad, lay) in enumerate([(2, 0, "packed"), (64, 12, "odd_step"), (16, 3, "pcl_xyzi"), (1, 7, "i_uint16"), (128, 40, "odd_step")]):
        c = rng.normal(size=(h * 1000, 4)).astype(np.float32)
        d, pc = M.pack_cloud(c, M.LAYOUTS[lay], height=h, row_pad=pad, seed=k)
        msgs.append((M.TOPIC, (10 + k, 0), M.node_payload(k, (10 + k, 0), np.arange(7.0), pc, d)))
    data = M.write_bag(msgs)
    with capi.PcdCodec() as codec:
        check_loads(codec, data, M.read_bag(data), sizes=(1, 2, None))


def test_wide_points_take_the_unstaged_path():
    c = np.arange(4000 * 4, dtype=np.float32).reshape(-1, 4)
    wide = dict(fields=[("x", 0, 7, 1), ("y", 9000, 7, 1), ("z", 17000, 7, 1), ("intensity", 20000, 7, 1)], point_step=20008)
    d, pc = M.pack_cloud(c[:300], wide)
    d2, pc2 = M.pack_cloud(c, M.LAYOUTS["packed"])
    msgs = [(M.TOPIC, (1, k), M.node_payload(k, (1, k), np.arange(7.0), *((pc, d) if k % 2 else (pc2, d2)))) for k in range(5)]
    data = M.write_bag(msgs, chunk_bytes=1 << 24)
    with capi.PcdCodec() as codec:
        check_loads(codec, data, M.read_bag(data), sizes=(1, 3, None))


def test_seq05_twin_with_a_large_cloud():
    """161 node messages plus the debug clouds, one 2.6 M-point cloud among small ones"""
    nodes = rand_nodes(161, 4000, seed=5, big=2_600_000)
    data = M.write_bag(M.kitti2node_messages(nodes), chunk_bytes=768 * 1024)
    want = M.read_bag(data)
    assert len(want) == 161 and max(len(w["cloud"]) for w in want) == 2_600_000
    with capi.PcdCodec() as codec:
        check_loads(codec, data, want)
        info = codec.bag_index(data)
        assert info["messages"] == 4 * 162 and info["selected"] == 162
        got = list(codec.bag_nodes(batch=20))
        assert [g[0] for g in got] == [s for s, _, _ in nodes]
        for (s, o, c), (_, o2, c2) in zip(got, nodes):
            assert np.array_equal(o, o2) and np.array_equal(bits(c), c2.view(np.uint32))
        sel = list(range(1, 161, 8))
        xyzi, off = codec.bag_load(nodes=sel, device_out=True)
        assert np.array_equal(bits(xyzi), np.concatenate([want[i]["cloud"] for i in sel]).view(np.uint32))


def test_fences_leave_the_handle_usable():
    good = M.write_bag(M.kitti2node_messages(rand_nodes(5, 100, seed=1)))
    want = M.read_bag(good)
    bad = {
        "version": (M.write_bag(M.kitti2node_messages(rand_nodes(2, 10, 2)), version=b"1.2"), capi.E_UNSUPPORTED),
        "bz2": (M.write_bag(M.kitti2node_messages(rand_nodes(2, 10, 2)), compression="bz2"), capi.E_UNSUPPORTED),
        "type": (M.write_bag(M.kitti2node_messages(rand_nodes(2, 10, 2)), types={M.TOPIC: "x/y"}), capi.E_UNSUPPORTED),
        "x_float64": (M.write_bag(M.kitti2node_messages(rand_nodes(2, 10, 2), layout="x_float64")), capi.E_UNSUPPORTED),
        "truncated": (good[:len(good) // 2], capi.E_INVALID),
    }
    with capi.PcdCodec() as codec:
        with pytest.raises(capi.ErasorError) as e:
            codec.bag_load(0, 1)
        assert e.value.code == capi.E_STATE
        for name, (data, code) in bad.items():
            with pytest.raises(capi.ErasorError) as e:
                codec.bag_index(data)
            assert e.value.code == code, name
            with pytest.raises(capi.ErasorError):
                codec.bag_load(0, 1)
            check_loads(codec, good, want, sizes=(2,))
        codec.bag_index(good)
        with pytest.raises(capi.ErasorError) as e:
            codec.bag_load(3, 5)
        assert e.value.code == capi.E_INVALID
        off = np.zeros(3, np.uint64)
        out = np.zeros((1, 4), np.float32)
        rc = codec.L.erasor_bag_load(codec.h, 0, 2, out.ctypes.data, 1, capi.PTR_HOST, off.ctypes.data_as(capi.POINTER(capi.c_uint64)))
        assert rc == capi.E_CAPACITY
        check_loads(codec, good, want, sizes=(5,))
        # the PCD entry points on the same handle are unaffected
        assert len(codec.load_bytes(b"# .PCD\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\nWIDTH 1\nHEIGHT 1\nPOINTS 1\nDATA ascii\n1 2 3\n")) == 1


# ---- drivers and the pipeline, end to end ----------------------------------------------------------------------------------------
def scene_nodes(n=15):
    sc = synth.Scene(seed=43, length=40.0, n_nodes=n, n_dynamic=6)
    kw = dict(n_beams=24, n_az=480)
    nodes = [(100 + k, sc.pose7(k), sc.scan(k, seed_offset=9, **kw)) for k in range(n)]
    return sc, nodes, sc.build_map(list(range(n)), voxel=0.2, **kw)


def write_config(tmp_path, map_path, save):
    cfg = tmp_path / "seq_05.yaml"
    cfg.write_text(YAML.format(save=str(save)).replace('initial_map_path: "unused"', f'initial_map_path: "{map_path}"'))
    return str(cfg)


def run(args):
    r = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:] + r.stdout[-2000:]
    return r


@pytest.fixture(scope="module")
def bag_case(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("bag")
    sc, nodes, gt_map = scene_nodes()
    bag = tmp / "05_0_to_15_w_interval_1_node.bag"
    bag.write_bytes(M.write_bag(M.kitti2node_messages(nodes), chunk_bytes=300000))
    with capi.PcdCodec() as codec:
        codec.write(str(tmp / "map.pcd"), gt_map)
        initial = codec.load(str(tmp / "map.pcd"))
    return tmp, nodes, str(bag), initial


def test_mapgen_main_from_a_bag_equals_the_env_layout(bag_case):
    tmp, nodes, bag, _ = bag_case
    data, out_a, out_b = tmp / "env", tmp / "mg_env", tmp / "mg_bag"
    (data / "pcds").mkdir(parents=True)
    out_a.mkdir()
    out_b.mkdir()
    with open(data / "poses_lidar2body.csv", "w") as f:
        f.write("index,time,x,y,z,qx,qy,qz,qw\n")
        for i, (seq, odom, cloud) in enumerate(nodes):
            f.write(f"{i},{seq}," + ",".join(f"{v:.17g}" for v in odom) + "\n")
            write_pcd_binary(str(data / "pcds" / f"{i:06d}.pcd"), cloud)
    binm = os.path.join(LIB, "mapgen_main")
    run([binm, str(data), os.path.basename(bag), str(out_a), "0.2"])
    run([binm, bag, str(out_b), "0.2"])
    fa, fb = sorted(glob.glob(str(out_a / "*.pcd"))), sorted(glob.glob(str(out_b / "*.pcd")))
    assert len(fa) == 2 and [os.path.basename(x) for x in fa] == [os.path.basename(x) for x in fb]
    for a, b in zip(fa, fb):
        assert open(a, "rb").read() == open(b, "rb").read()


def test_offline_map_updater_main_from_a_bag_equals_run_offline(bag_case):
    tmp, nodes, bag, initial = bag_case
    save = tmp / "upd"
    save.mkdir()
    cfg = write_config(tmp, tmp / "map.pcd", save)
    run([os.path.join(LIB, "offline_map_updater_main"), cfg, bag])
    ep, up = params.load_yaml(cfg)
    res = pipeline.run_offline(nodes, initial, up, ep, save_voxel_size=0.2)
    with capi.PcdCodec() as codec:
        ref = codec.format(res["static_map"])
    assert res["processed_scans"] > 0 and open(save / "05_result.pcd", "rb").read() == ref


def test_static_map_nodes_main_from_a_bag_equals_run_frame_independent(bag_case):
    tmp, nodes, bag, initial = bag_case
    save = tmp / "nodes"
    save.mkdir()
    cfg = write_config(tmp, tmp / "map.pcd", save)
    run([os.path.join(LIB, "static_map_nodes_main"), cfg, bag, "0", "3"])
    ep, up = params.load_yaml(cfg)
    res = pipeline.run_frame_independent(nodes, initial, up, ep, batch=3, save_voxel_size=0.2)
    with capi.PcdCodec() as codec:
        ref = codec.format(res["static_map"])
    assert open(save / "05_result.pcd", "rb").read() == ref


@pytest.mark.parametrize("frame_independent", [False, True])
def test_run_bag_equals_run_sequence(bag_case, frame_independent):
    tmp, nodes, bag, _ = bag_case
    cfg = write_config(tmp, tmp / "map.pcd", tmp)
    got = pipeline.run_bag(bag, cfg, frame_independent=frame_independent)
    ep, up = params.load_yaml(cfg)
    want = pipeline.run_sequence(nodes, up, ep, frame_independent=frame_independent)
    assert got.keys() == want.keys()
    for k in want:
        if isinstance(want[k], np.ndarray):
            assert np.array_equal(bits(got[k]) if want[k].dtype == np.float32 else got[k], bits(want[k]) if want[k].dtype == np.float32 else want[k]), k
        else:
            assert got[k] == want[k], k
