"""GPU checks of the node-mode re-test (DESIGN.md section 8.4.1): the device re-test map (erasor_map_create_retest) against the
model's M2 and extents (tests/node_retest_model.py), the compaction on a 2^25-point map, erasor_process_nodes_retest against the
oracle model and against single-node calls on fresh prefix maps, the same mask from every batching, query kind, lane layout,
sub-batch split and graph replay, the refusals, the pipeline and the C++ driver -- every comparison bit for bit."""
import ctypes

import numpy as np
import pytest

from erasor_b200 import params as P

import node_inserts_model as NI
import node_retest_model as NR

pytestmark = pytest.mark.gpu

FAR = np.array([5000.0, 0, 0, 0, 0, 0, 1], dtype=np.float64)     # a pose whose VoI holds no map point: v3 inserts nothing there


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
    return np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 4).view(np.uint32)


def _points(capi, m):
    out = np.empty((m.size, 4), dtype=np.float32)
    capi._memcpy_from_device(out, m.points_ptr)
    return out


def _set_keep(capi, m, keep):
    """the map's keep mask <- keep (host bytes)"""
    keep = np.ascontiguousarray(keep, dtype=np.uint8)
    capi._memcpy_from_device(np.zeros(0, np.uint8), 0)             # loads the runtime capi copies with
    assert capi._CUDART.cudaMemcpy(m.keep_ptr, keep.ctypes.data, keep.nbytes, 1) == 0


def _pass1(capi, p, mw, poses, qs, batches=None):
    """device pass 1 with inserts on, appended in node order -> (map, its keep mask)"""
    m, h = capi.Map(mw), capi.Handle(p)
    h.attach_map(m)
    h.set_node_inserts(True)
    for b0, b1 in batches or [(0, len(qs))]:
        h.process_nodes(poses[b0:b1], np.concatenate(qs[b0:b1]), _off(qs[b0:b1]))
        m.append_inserts(h)
    h.close()
    return m, m.get_keep()


def _model(oracle_mod, p, mw, poses, qs):
    ins, off, fk = NI.node_inserts(oracle_mod, p, mw, poses, qs)
    keep1 = fk.min(axis=0)
    M2, ext = NR.retest_map(mw, keep1, [ins[int(off[j]):int(off[j + 1])] for j in range(len(qs))])
    return keep1, M2, ext


@pytest.mark.parametrize("name,version,skip", [("seq_05", 3, 0), ("seq_05", 3, 1), ("seq_00", 2, 1)])
def test_retest_map_and_keep_equal_model(capi, oracle_mod, small_workload, name, version, skip):
    p = P.preset(name).replace(version=version, skip_voxelize=skip)
    mw = small_workload["map_world"]
    poses, qs = _nodes(small_workload, range(6))
    keep1, M2, ext = _model(oracle_mod, p, mw, poses, qs)
    m, k1 = _pass1(capi, p, mw, poses, qs, [(0, 2), (2, 3), (3, 6)])
    assert np.array_equal(k1, keep1)
    store = m.inserts()
    r = m.create_retest()
    assert np.array_equal(m.get_keep(), k1) and np.array_equal(_bits(m.inserts()), _bits(store)), "the source map changed"
    assert r.size == len(M2) and np.array_equal(_bits(_points(capi, r)), _bits(M2))
    assert (r.get_keep() == 1).all() and len(r.inserts()) == 0
    assert np.array_equal(r.retest_extents(), ext)
    with pytest.raises(capi.ErasorError):
        m.retest_extents()
    # pass 2 against the oracle model
    want = NR.retest_keep(oracle_mod, p, M2, ext, poses, qs)
    h = capi.Handle(p)
    h.attach_map(r)
    keep2 = h.process_nodes_retest(poses, np.concatenate(qs), _off(qs), 0)
    assert np.array_equal(keep2, want), f"{np.count_nonzero(keep2 != want)} points differ"
    # ... and against single-node plain calls on fresh maps holding each node's prefix
    anded = np.ones(len(M2), dtype=np.uint8)
    for j in range(len(qs)):
        e = int(ext[j])
        fm = capi.Map(M2[:e])
        g = capi.Handle(p)
        g.attach_map(fm)
        kj, _ = g.process_nodes(poses[j:j + 1], qs[j], _off(qs[j:j + 1]))
        anded[:e] &= kj
        g.close(); fm.close()
    assert np.array_equal(keep2, anded)
    h.close(); r.close(); m.close()


@pytest.mark.parametrize("case", ["empty store", "nodes without inserts", "all rejected"])
def test_retest_map_edge_cases(capi, oracle_mod, small_workload, case):
    p = P.preset("seq_05").replace(version=3, skip_voxelize=1)
    mw = small_workload["map_world"]
    poses, qs = _nodes(small_workload, range(4))
    if case == "empty store":                     # no node appended: no nodes, the kept points alone
        m = capi.Map(mw)
        k1 = (np.arange(len(mw)) % 3 != 0).astype(np.uint8)
        _set_keep(capi, m, k1)
        r = m.create_retest()
        assert r.size == int(k1.sum()) and len(r.retest_extents()) == 0
        assert np.array_equal(_bits(_points(capi, r)), _bits(mw[k1 != 0]))
        h = capi.Handle(p)
        h.attach_map(r)
        with pytest.raises(capi.ErasorError):
            h.process_nodes_retest(poses[:1], qs[0], _off(qs[:1]), 0)
        # attached to plain erasor_process_nodes it is a plain map
        keep, _ = h.process_nodes(poses, np.concatenate(qs), _off(qs))
        _, _, fk = NI.node_inserts(oracle_mod, p, mw[k1 != 0], poses, qs)
        assert np.array_equal(keep, fk.min(axis=0))
        h.close(); r.close(); m.close()
        return
    if case == "nodes without inserts":
        poses = poses.copy()
        poses[1] = poses[2] = FAR
    ins, off, fk = NI.node_inserts(oracle_mod, p, mw, poses, qs)
    keep1 = fk.min(axis=0)
    m, _ = _pass1(capi, p, mw, poses, qs)
    if case == "all rejected":
        keep1 = np.zeros(len(mw), np.uint8)
        _set_keep(capi, m, keep1)
    M2, ext = NR.retest_map(mw, keep1, [ins[int(off[j]):int(off[j + 1])] for j in range(len(qs))])
    if case == "all rejected":
        assert ext[0] == 0 and len(M2) == len(ins) > 0
    else:
        assert (np.diff(ext.astype(np.int64)) == 0).any()
    r = m.create_retest()
    assert np.array_equal(_bits(_points(capi, r)), _bits(M2)) and np.array_equal(r.retest_extents(), ext)
    assert (r.get_keep() == 1).all()
    h = capi.Handle(p)
    h.attach_map(r)
    keep2 = h.process_nodes_retest(poses, np.concatenate(qs), _off(qs), 0)
    assert np.array_equal(keep2, NR.retest_keep(oracle_mod, p, M2, ext, poses, qs))
    h.close(); r.close(); m.close()


def test_compaction_of_a_large_map(capi):
    """2^25 + 77 points, a random keep mask, no store: the re-test map is numpy's points[keep != 0]"""
    rng = np.random.default_rng(9)
    n = (1 << 25) + 77
    mw = rng.standard_normal((n, 4), dtype=np.float32)
    keep = (rng.random(n) < 0.6).astype(np.uint8)
    keep[:4096] = 0                                   # a whole tile rejected
    keep[4096:8192] = 1                               # a whole tile kept
    m = capi.Map(mw)
    _set_keep(capi, m, keep)
    r = m.create_retest()
    got = _points(capi, r)
    assert r.size == int(keep.sum()) and np.array_equal(_bits(got), _bits(mw[keep != 0]))
    assert len(r.retest_extents()) == 0
    r.close(); m.close()


def test_same_keep_from_every_submission_form(capi, oracle_mod, small_workload):
    """batches of 1, 3 and all nodes; host, device and packed x y z queries; two lanes sharing the map asynchronously; graph replay
    (every batching twice): one mask, the model's"""
    import torch
    p = P.preset("seq_05").replace(version=3, skip_voxelize=1)
    mw = small_workload["map_world"]
    poses, qs = _nodes(small_workload, range(6))
    keep1, M2, ext = _model(oracle_mod, p, mw, poses, qs)
    want = NR.retest_keep(oracle_mod, p, M2, ext, poses, qs)
    m, _ = _pass1(capi, p, mw, poses, qs)
    r = m.create_retest()
    h = capi.Handle(p)
    h.attach_map(r)
    for size in (1, 3, 6):
        for rep in range(2):                          # the second round replays the captured graphs
            r.reset_keep()
            for b0 in range(0, 6, size):
                keep = h.process_nodes_retest(poses[b0:b0 + size], np.concatenate(qs[b0:b0 + size]), _off(qs[b0:b0 + size]), b0)
            assert np.array_equal(keep, want), f"batches of {size}, round {rep}"
    r.reset_keep()
    assert np.array_equal(h.process_nodes_retest(poses, np.concatenate(qs), _off(qs), 0, packed_xyz=True), want)
    # device queries, asynchronous; packed x y z from the device
    Q = np.ascontiguousarray(np.concatenate(qs))
    for packed in (False, True):
        r.reset_keep()
        dq = torch.from_numpy(np.ascontiguousarray(Q[:, :3]) if packed else Q).cuda()
        dkeep = torch.empty(r.size, dtype=torch.uint8, device="cuda")
        P7, qo = np.ascontiguousarray(poses), _off(qs)
        h.process_nodes_retest_ptr(P7, dq.data_ptr(), qo, 0, 0.0, dkeep.data_ptr(), capi.PTR_DEVICE | (capi.PTR_QUERY_XYZ if packed else 0),
                                   asynchronous=True)
        h.wait()
        assert np.array_equal(dkeep.cpu().numpy(), want)
    # two lanes on one re-test map
    r.reset_keep()
    a, b = capi.Handle(p), capi.Handle(p)
    for x in (a, b):
        x.attach_map(r)
    q1, q2 = np.concatenate(qs[:3]), np.concatenate(qs[3:])
    pa, pb, oa, ob = np.ascontiguousarray(poses[:3]), np.ascontiguousarray(poses[3:]), _off(qs[:3]), _off(qs[3:])
    a.process_nodes_retest_ptr(pa, q1.ctypes.data, oa, 0, 0.0, 0, capi.PTR_HOST, asynchronous=True)
    b.process_nodes_retest_ptr(pb, q2.ctypes.data, ob, 3, 0.0, 0, capi.PTR_HOST, asynchronous=True)
    a.wait(); b.wait()
    assert np.array_equal(r.get_keep(), want)
    a.close(); b.close()
    h.close(); r.close(); m.close()


def test_sub_batches_by_scratch_budget(capi, small_workload, monkeypatch):
    """ERASOR_B200_NODE_SCRATCH_GB=1 on a re-test map of 8 M points: sub-batches of two nodes, the mask of one submission"""
    p = P.preset("seq_05").replace(version=3, skip_voxelize=1)
    base = small_workload["map_world"]
    filler = np.concatenate([base + np.array([3000.0 + 500.0 * t, 0, 0, 0], dtype=np.float32) for t in range(63)])
    mw = np.concatenate([base, filler])
    assert (1 << 30) // (46 * (len(mw) + 20000)) == 2
    poses, qs = _nodes(small_workload, range(6))
    m, _ = _pass1(capi, p, mw, poses, qs)
    r = m.create_retest()
    assert (1 << 30) // (46 * r.size) == 2
    outs = []
    for split in (False, True):
        if split:
            monkeypatch.setenv("ERASOR_B200_NODE_SCRATCH_GB", "1")
        else:
            monkeypatch.delenv("ERASOR_B200_NODE_SCRATCH_GB", raising=False)
        r.reset_keep()
        h = capi.Handle(p)
        h.attach_map(r)
        outs.append(h.process_nodes_retest(poses, np.concatenate(qs), _off(qs), 0))
        h.close()
    monkeypatch.delenv("ERASOR_B200_NODE_SCRATCH_GB", raising=False)
    assert (outs[0] == 0).any() and np.array_equal(outs[0], outs[1])
    r.close(); m.close()


def test_refusals_leave_the_handle_usable(capi, oracle_mod, small_workload):
    p = P.preset("seq_05").replace(version=3, skip_voxelize=1)
    mw = small_workload["map_world"]
    poses, qs = _nodes(small_workload, range(3))
    Q, qo = np.ascontiguousarray(np.concatenate(qs), dtype=np.float32), _off(qs)
    m, _ = _pass1(capi, p, mw, poses, qs)
    r = m.create_retest()
    h = capi.Handle(p)
    P7 = np.ascontiguousarray(poses)

    def rc(first, frames=3):
        return h.L.erasor_process_nodes_retest(h.h, P7.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), Q.ctypes.data,
                                               qo.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)), frames, first, 0.0, None, capi.PTR_HOST)

    assert rc(0) == capi.E_STATE                                     # no map attached
    h.attach_map(m)
    assert rc(0) == capi.E_INVALID                                   # not a re-test map
    h.attach_map(r)
    assert rc(-1) == capi.E_INVALID and rc(1) == capi.E_INVALID      # first_node < 0, first_node + n_frames > n_nodes
    h.set_node_inserts(True)
    assert rc(0) == capi.E_INVALID                                   # node inserts on
    h.set_node_inserts(False)
    h.process_nodes_retest_ptr(P7, Q.ctypes.data, qo, 0, 0.0, 0, capi.PTR_HOST, asynchronous=True)
    assert rc(0) == capi.E_STATE                                     # a submission pending
    h.wait()
    r.reset_keep()
    keep1, M2, ext = _model(oracle_mod, p, mw, poses, qs)
    assert np.array_equal(h.process_nodes_retest(poses, Q, qo, 0), NR.retest_keep(oracle_mod, p, M2, ext, poses, qs))
    h.close(); r.close(); m.close()


def test_pipeline_retest_equals_oracle_chain(capi, oracle_mod, small_workload):
    """run_frame_independent(inserts=True, retest=True) with host-prepared queries == the oracle chain: pass 1, the re-test map,
    pass 2, then the saved map of M2 under keep2"""
    from erasor_b200 import pipeline
    scene, mw = small_workload["scene"], small_workload["map_world"]
    ep = P.preset("seq_00")
    up = P.UpdaterParams(removal_interval=1, version=2, max_range=ep.max_range, map_voxel_size=0.05)
    nodes = [(i, scene.pose7(f[2]), f[1]) for i, f in enumerate(small_workload["frames"])]
    with pytest.raises(ValueError):
        pipeline.run_frame_independent(nodes, mw, up, ep, retest=True)
    res = pipeline.run_frame_independent(nodes, mw, up, ep, batch=4, prepare=lambda raw, off: (raw, off), inserts=True, retest=True)
    poses = np.stack([n[1] for n in nodes]).astype(np.float64)
    qs = [n[2] for n in nodes]
    p = ep.replace(version=up.version)
    ins, off, fk = NI.node_inserts(oracle_mod, p, mw, poses, qs, up.max_range)
    keep1 = fk.min(axis=0)
    M2, ext = NR.retest_map(mw, keep1, [ins[int(off[j]):int(off[j + 1])] for j in range(len(qs))])
    keep2 = NR.retest_keep(oracle_mod, p, M2, ext, poses, qs, up.max_range)
    assert np.array_equal(res["keep"], keep1) and res["retest_size"] == len(M2)
    assert np.array_equal(res["retest_keep"], keep2) and (keep2 == 0).any()
    want = NI.saved_map(oracle_mod, M2, keep2, np.zeros((0, 4), np.float32), up.map_voxel_size)
    assert np.array_equal(_bits(res["static_map"]), _bits(want))


def test_static_map_nodes_driver_with_retest(oracle_mod, tmp_path):
    """examples/static_map_nodes_main with inserts = 2: the file equals run_frame_independent(inserts=True, retest=True) on the
    oracle's prepared queries, then write_pcd_ascii, byte for byte"""
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

    res = pipeline.run_frame_independent(nodes, gt_map, up, ep, batch=5, save_voxel_size=0.2, prepare=oracle_prepare, inserts=True, retest=True)
    E.write_pcd_ascii(str(tmp_path / "want.pcd"), res["static_map"])
    r = subprocess.run([binary, str(cfg), str(data), "0", "5", "2"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:] + r.stdout[-2000:]
    assert (save / "05_result.pcd").read_bytes() == (tmp_path / "want.pcd").read_bytes()
