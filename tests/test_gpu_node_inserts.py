"""GPU checks of node-mode inserts (erasor_set_node_inserts): every node's inserted points and offsets against the oracle model
(tests/node_inserts_model.py), bit for bit in values and order; the masks and counters unchanged by the switch; sub-batches,
the late class-C run, two lanes on one map, the packed-xyz refusal, the saved map and the pipeline."""
import numpy as np
import pytest

from erasor_b200 import params as P

import node_inserts_model as NI

pytestmark = pytest.mark.gpu

IDENTITY = np.array([0, 0, 0, 0, 0, 0, 1], dtype=np.float64)


@pytest.fixture(scope="module")
def capi():
    from erasor_b200 import capi as C
    return C


def _nodes(small_workload, picks):
    scene = small_workload["scene"]
    poses = np.stack([scene.pose7(small_workload["frames"][i][2]) for i in picks]).astype(np.float64)
    return poses, [small_workload["frames"][i][1] for i in picks]


def _off(qs):
    return np.cumsum([0] + [len(q) for q in qs]).astype(np.uint64)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("name", ["seq_05", "seq_00", "synthetic_40x360"])
@pytest.mark.parametrize("version,skip", [(3, 0), (3, 1), (2, 1)])
def test_inserts_equal_oracle(capi, oracle_mod, small_workload, name, version, skip):
    import torch
    p = P.preset(name).replace(version=version, skip_voxelize=skip)
    mw = small_workload["map_world"]
    poses, qs = _nodes(small_workload, range(6))
    Q, qo = np.concatenate(qs), _off(qs)
    ref, ref_off, ref_fk = NI.node_inserts(oracle_mod, p, mw, poses, qs)
    m = capi.Map(mw)
    h = capi.Handle(p)
    h.attach_map(m)
    keep0, fk0 = h.process_nodes(poses, Q, qo, want_frame_keep=True)
    st0 = h.node_stats()
    launches_off = h.kernel_launch_count()
    h.process_nodes(poses, Q, qo)
    launches_off = h.kernel_launch_count() - launches_off
    h.set_node_inserts(True)
    for rep in range(2):                      # second call: the captured graph replays
        m.reset_keep()
        keep, fk = h.process_nodes(poses, Q, qo, want_frame_keep=True)
        ins, off = h.node_inserts()
        assert np.array_equal(off, ref_off), f"{name} v{version}: offsets {off} != {ref_off}"
        assert np.array_equal(_bits(ins), _bits(ref)), f"{name} v{version}: inserts differ in {np.count_nonzero((_bits(ins) != _bits(ref)).any(1))} points"
        assert np.array_equal(fk, fk0) and np.array_equal(keep, keep0) and np.array_equal(fk, ref_fk)
        for a, b in zip(h.node_stats(), st0):
            assert np.array_equal(a, b)
    # device queries, asynchronous
    m.reset_keep()
    dq = torch.from_numpy(np.ascontiguousarray(Q)).cuda()
    h.process_nodes_ptr(np.ascontiguousarray(poses), dq.data_ptr(), qo, 0.0, 0, 0, capi.PTR_DEVICE, asynchronous=True)
    h.wait()
    ins, off = h.node_inserts()
    assert np.array_equal(off, ref_off) and np.array_equal(_bits(ins), _bits(ref))
    # switched off again: the launches of inserts off
    h.set_node_inserts(False)
    n0 = h.kernel_launch_count()
    h.process_nodes(poses, Q, qo)
    assert h.kernel_launch_count() - n0 == launches_off
    with pytest.raises(capi.ErasorError):
        h.node_inserts()
    h.close(); m.close()


def test_sub_batches_keep_every_frame(capi, oracle_mod):
    """150 nodes at 40 x 360 bins: more flagged-bin records than one submission holds, so the call is split; every node's inserts
    survive, in node order."""
    from test_gpu_parity import _crafted_bin_frame
    p = P.preset("synthetic_40x360").replace(skip_voxelize=1)
    rng = np.random.default_rng(77)
    mw, q = _crafted_bin_frame(rng, 300, "rough")
    qs = [q[np.sort(rng.choice(len(q), int(rng.integers(1, len(q) + 1)), replace=False))] for _ in range(150)]
    poses = np.tile(IDENTITY, (150, 1))
    ref, ref_off, _ = NI.node_inserts(oracle_mod, p, mw, poses, qs)
    m = capi.Map(mw)
    h = capi.Handle(p)
    h.attach_map(m)
    h.set_node_inserts(True)
    h.process_nodes(poses, np.concatenate(qs), _off(qs))
    ins, off = h.node_inserts()
    assert np.array_equal(off, ref_off) and np.array_equal(_bits(ins), _bits(ref))
    h.close(); m.close()


@pytest.mark.parametrize("version,skip", [(3, 1), (3, 0)])
def test_late_class_c(capi, oracle_mod, version, skip):
    """A bin beyond class B's capacity met while class C is off: erasor_wait runs the class and rebuilds the inserts, which equal
    those of the run that launches class C up front (and the oracle's)."""
    from test_gpu_parity import _crafted_bin_frame
    p = P.preset("seq_05").replace(version=version, skip_voxelize=skip)
    rng = np.random.default_rng(5)
    small = _crafted_bin_frame(rng, 200, "rough")
    big = _crafted_bin_frame(rng, 5000, "rough")
    h = capi.Handle(p)
    h.set_node_inserts(True)
    got = []
    for tag, (mw, q) in (("small", small), ("small, class C off", small), ("big, late class C", big), ("big, class C up front", big)):
        m = capi.Map(mw)
        h.attach_map(m)
        h.process_nodes(IDENTITY[None], q, _off([q]))
        ins, off = h.node_inserts()
        ref, ref_off, _ = NI.node_inserts(oracle_mod, p, mw, IDENTITY[None], [q])
        assert np.array_equal(off, ref_off) and np.array_equal(_bits(ins), _bits(ref)), tag
        got.append(ins)
        h.attach_map(None)
        m.close()
    assert np.array_equal(_bits(got[2]), _bits(got[3]))
    h.close()


def test_two_lanes_one_map_and_save(capi, oracle_mod, small_workload):
    """Two handles on one map appending in node order save what one handle saves, and what the oracle saves; packed x y z
    queries are refused while inserts are on, and the handle stays usable."""
    p = P.preset("seq_05")
    mw = small_workload["map_world"]
    poses, qs = _nodes(small_workload, range(6))
    ref, _, ref_fk = NI.node_inserts(oracle_mod, p, mw, poses, qs)
    ref_map = NI.saved_map(oracle_mod, mw, ref_fk.min(axis=0), ref, p.map_voxel_size)
    m1 = capi.Map(mw)
    h = capi.Handle(p)
    h.attach_map(m1)
    assert len(h.save_static_map(m1, p.map_voxel_size)) == len(oracle_mod.voxelize(mw, p.map_voxel_size))
    h.set_node_inserts(True)
    with pytest.raises(capi.ErasorError):
        h.process_nodes(poses, np.concatenate(qs), _off(qs), packed_xyz=True)
    h.process_nodes(poses, np.concatenate(qs), _off(qs))
    m1.append_inserts(h)
    one = h.save_static_map(m1, p.map_voxel_size)
    assert np.array_equal(_bits(m1.inserts()), _bits(ref))
    assert np.array_equal(_bits(one), _bits(ref_map))
    m2 = capi.Map(mw)
    a, b = capi.Handle(p), capi.Handle(p)
    for x in (a, b):
        x.attach_map(m2); x.set_node_inserts(True)
    q1, q2 = np.concatenate(qs[:3]), np.concatenate(qs[3:])          # alive until the waits
    a.process_nodes_ptr(np.ascontiguousarray(poses[:3]), q1.ctypes.data, _off(qs[:3]), 0.0, 0, 0, capi.PTR_HOST, asynchronous=True)
    b.process_nodes_ptr(np.ascontiguousarray(poses[3:]), q2.ctypes.data, _off(qs[3:]), 0.0, 0, 0, capi.PTR_HOST, asynchronous=True)
    a.wait(); b.wait()
    m2.append_inserts(a); m2.append_inserts(b)
    assert np.array_equal(_bits(a.save_static_map(m2, p.map_voxel_size)), _bits(one))
    m2.clear_inserts()
    assert len(m2.inserts()) == 0
    for x in (a, b, h):
        x.close()
    m1.close(); m2.close()


def test_pipeline_inserts_equal_oracle_chain(capi, oracle_mod, small_workload):
    """run_frame_independent(inserts=True) with the queries prepared on the host == the oracle chain: kept map + every node's
    inserts, voxelised."""
    scene, mw = small_workload["scene"], small_workload["map_world"]
    ep = P.preset("seq_05")
    up = P.UpdaterParams(removal_interval=1, version=3, max_range=ep.max_range, map_voxel_size=0.05)
    frames = small_workload["frames"]
    nodes = [(i, scene.pose7(f[2]), f[1]) for i, f in enumerate(frames)]
    from erasor_b200 import pipeline
    res = pipeline.run_frame_independent(nodes, mw, up, ep, batch=4, prepare=lambda raw, off: (raw, off), inserts=True)
    poses = np.stack([n[1] for n in nodes]).astype(np.float64)
    p = ep.replace(version=up.version)
    ref, _, fk = NI.node_inserts(oracle_mod, p, mw, poses, [n[2] for n in nodes], up.max_range)
    assert np.array_equal(res["keep"], fk.min(axis=0))
    assert np.array_equal(_bits(res["static_map"]), _bits(NI.saved_map(oracle_mod, mw, fk.min(axis=0), ref, up.map_voxel_size)))


def test_golden_frames_as_nodes(capi, oracle_mod):
    """each golden frame as one node (its map VoI as the map, identity pose): inserts equal the model"""
    from test_node_inserts_model import GOLDEN, golden_node
    for path in GOLDEN:
        p, mw, pose, q = golden_node(path)
        ref, ref_off, _ = NI.node_inserts(oracle_mod, p, mw, pose[None], [q])
        m, h = capi.Map(mw), capi.Handle(p)
        h.attach_map(m)
        h.set_node_inserts(True)
        h.process_nodes(pose[None], q, _off([q]))
        ins, off = h.node_inserts()
        assert np.array_equal(off, ref_off) and np.array_equal(_bits(ins), _bits(ref)), path
        h.close(); m.close()


@pytest.mark.parametrize("skip", [0, 1])
def test_several_frames_past_the_shared_memory_caps(capi, oracle_mod, skip):
    """Three nodes in one submission, each holding bins past K4b's shared-memory cap (version 3 voxelises them per frame in
    global scratch, regions keyed by (frame, bin)) and one R-GPF bin past class C's cap: every frame's inserts equal the model."""
    import bin_cases as C
    p = P.preset("seq_05").replace(version=3, skip_voxelize=skip, map_voxel_size=0.2)
    specs = list(C.K4B_FRAMES[0.2]) + [C.Bin(2, 50, C.K4_C_CAP + 2, "rough")]
    mw, q = C.flagged_bins(p, specs, seed=11)
    rng = np.random.default_rng(3)
    qs = [q] + [q[np.sort(rng.choice(len(q), int(0.8 * len(q)), replace=False))] for _ in range(2)]
    poses = np.tile(IDENTITY, (3, 1))
    ref, ref_off, ref_fk = NI.node_inserts(oracle_mod, p, mw, poses, qs)
    m, h = capi.Map(mw), capi.Handle(p)
    h.attach_map(m)
    h.set_node_inserts(True)
    _, fk = h.process_nodes(poses, np.concatenate(qs), _off(qs), want_frame_keep=True)
    ins, off = h.node_inserts()
    assert np.array_equal(fk, ref_fk)
    assert np.array_equal(off, ref_off) and np.array_equal(_bits(ins), _bits(ref))
    h.close(); m.close()


def test_static_map_nodes_driver_with_inserts(oracle_mod, tmp_path):
    """examples/static_map_nodes_main with inserts on (its fifth argument): the file equals run_frame_independent(inserts=True)
    on the oracle's prepared queries, then write_pcd_ascii, byte for byte -- the C++ class's inserts, appends and save."""
    import os
    import subprocess
    from erasor_b200 import evaluate as E
    from erasor_b200 import pipeline, synth
    from test_gpu_cpp_driver import YAML
    from test_gpu_voxelize_batch import _prepared, batch_of
    binary = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "erasor_b200", "_lib", "static_map_nodes_main")
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
            pose = np.float32(sc.pose7(k)).astype(np.float64)            # the driver reads the csv as floats
            f.write(f"{k},{k * 0.1}," + ",".join(f"{v:.9g}" for v in pose) + "\n")
            nodes.append((k, pose, E.read_pcd_ascii(path)))
    cfg = tmp_path / "seq_05.yaml"
    cfg.write_text(YAML.format(save=str(save)))
    ep, up = P.load_yaml(str(cfg))

    def oracle_prepare(raw, off):
        o = off.astype(np.int64)
        return batch_of([_prepared(oracle_mod, raw[o[c]:o[c + 1]], up.query_voxel_size, up.lidar2body) for c in range(len(o) - 1)])

    plain = pipeline.run_frame_independent(nodes, gt_map, up, ep, batch=5, save_voxel_size=0.2, prepare=oracle_prepare)
    res = pipeline.run_frame_independent(nodes, gt_map, up, ep, batch=5, save_voxel_size=0.2, prepare=oracle_prepare, inserts=True)
    assert len(res["static_map"]) > len(plain["static_map"])
    E.write_pcd_ascii(str(tmp_path / "want.pcd"), res["static_map"])
    r = subprocess.run([binary, str(cfg), str(data), "0", "5", "1"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:] + r.stdout[-2000:]
    assert (save / "05_result.pcd").read_bytes() == (tmp_path / "want.pcd").read_bytes()


def test_other_submissions_end_the_inserts(capi, small_workload):
    """the inserts of a node call are gone after a later submission of another kind with the same frame count"""
    p = P.preset("seq_05")
    poses, qs = _nodes(small_workload, [0])
    m, h = capi.Map(small_workload["map_world"]), capi.Handle(p)
    h.attach_map(m)
    h.set_node_inserts(True)
    h.process_nodes(poses, qs[0], _off(qs))
    h.node_inserts()
    voi, q, _, _ = small_workload["frames"][0]
    h.process_frames(voi, np.array([0, len(voi)], np.uint64), q, np.array([0, len(q)], np.uint64))
    with pytest.raises(capi.ErasorError):
        h.node_inserts()
    with pytest.raises(capi.ErasorError):
        m.append_inserts(h)
    h.close(); m.close()
