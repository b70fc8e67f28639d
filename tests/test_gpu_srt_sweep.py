"""GPU: the Scan Ratio Test sweep (erasor_process_nodes_sweep, DESIGN.md section 8.5).  Every mask and every sweep counter must
equal, bit for bit, a separate erasor_process_nodes run with that setting's parameters on a fresh map: over the bench twin, seq 00,
version 2 th_bin_max_h settings and minimum_num_pts settings (a negative one included), V = 1, 5 and 32 and duplicates, host,
device and packed-xyz queries, sub-batch splits, class-C bins that turn up late, lanes sharing one mask buffer, graph replay, and
the AND of two half sweeps.  Also: a plain erasor_process_nodes after a sweep is unchanged, every refusal, and
pipeline.sweep_frame_independent and its command line against run_frame_independent + capi.Evaluator."""
import os
import subprocess
import sys

import numpy as np
import pytest

from erasor_b200 import params as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THRESHOLDS = (0.10, 0.15, 0.20, 0.25, 0.30)


@pytest.fixture(scope="module")
def capi():
    from erasor_b200 import capi as C
    return C


@pytest.fixture(scope="module")
def twin():
    """bench.py's seq 05 twin, 20 nodes"""
    from erasor_b200 import synth
    w = synth.make_frames(seed=5, n_frames=20, preset_max_range=60.0, n_map_nodes=161, n_beams=64, n_az=1800, length=160.0, n_dynamic=12,
                          query_voxel=0.2, map_stride=2)
    poses = np.stack([w["scene"].pose7(f[2]) for f in w["frames"]]).astype(np.float64)
    return w["map_world"], poses, [f[1] for f in w["frames"]]


def small(small_workload):
    scene = small_workload["scene"]
    poses = np.stack([scene.pose7(f[2]) for f in small_workload["frames"]]).astype(np.float64)
    return small_workload["map_world"], poses, [f[1] for f in small_workload["frames"]]


def offsets(qs):
    return np.cumsum([0] + [len(q) for q in qs]).astype(np.uint64)


def separate(capi, p, map_world, poses, qs, variants, voi_max_range=0.0):
    """V plain erasor_process_nodes runs: masks [V, n], flagged [V, F], rejected [V, F], voi [F]"""
    keeps, nfs, nrs = [], [], []
    Q, qo = np.concatenate(qs), offsets(qs)
    for var in variants:
        m = capi.Map(map_world)
        h = capi.Handle(p.replace(**var))
        h.attach_map(m)
        keep, _ = h.process_nodes(poses, Q, qo, voi_max_range=voi_max_range)
        nv, nf, nr = h.node_stats()
        keeps.append(keep); nfs.append(nf); nrs.append(nr)
        h.close(); m.close()
    return np.stack(keeps), np.stack(nfs), np.stack(nrs), nv


def sweep(capi, h, n, poses, qs, variants, kind="host", keep=None, reset=True, asynchronous=False, voi_max_range=0.0):
    import torch
    V = len(variants)
    if keep is None:
        keep = torch.empty(V * n, dtype=torch.uint8, device="cuda")
    if reset:
        h.reset_keep_mask(keep.data_ptr(), V * n)
    Q, qo = np.concatenate(qs), offsets(qs)
    if kind == "host":
        h.process_nodes_sweep(poses, Q, qo, variants, keep.data_ptr(), voi_max_range=voi_max_range, asynchronous=asynchronous)
    elif kind == "packed":
        h.process_nodes_sweep(poses, Q, qo, variants, keep.data_ptr(), voi_max_range=voi_max_range, packed_xyz=True, asynchronous=asynchronous)
    else:
        dQ = torch.from_numpy(np.ascontiguousarray(Q)).cuda()
        h._dq = dQ
        h.process_nodes_sweep(poses, dQ.data_ptr(), qo, variants, keep.data_ptr(), voi_max_range=voi_max_range, asynchronous=asynchronous)
    return keep


def check(capi, p, map_world, poses, qs, variants, kinds=("host",), voi_max_range=0.0):
    ref_k, ref_f, ref_r, ref_v = separate(capi, p, map_world, poses, qs, variants, voi_max_range)
    assert (ref_k == 0).any(), "the workload must reject something"
    n = len(map_world)
    m = capi.Map(map_world)
    h = capi.Handle(p)
    h.attach_map(m)
    for kind in kinds:
        keep = sweep(capi, h, n, poses, qs, variants, kind, voi_max_range=voi_max_range)
        got = keep.reshape(len(variants), n).cpu().numpy()
        for v in range(len(variants)):
            assert np.array_equal(got[v], ref_k[v]), f"{kind} {variants[v]}: {np.count_nonzero(got[v] != ref_k[v])} points differ"
        nf, nr = h.sweep_stats()
        assert np.array_equal(nf, ref_f) and np.array_equal(nr, ref_r), kind
        nv, uf, ur = h.node_stats()
        assert np.array_equal(nv, ref_v) and (uf >= ref_f.max(axis=0)).all() and (ur >= ref_r.max(axis=0)).all()
        assert np.all(m.get_keep() == 1), "a sweep leaves the map's keep mask alone"
    h.close(); m.close()
    return ref_k


def test_bench_twin_v3_thresholds(capi, twin):
    map_world, poses, qs = twin
    p = P.preset("seq_05").replace(skip_voxelize=1)
    ks = check(capi, p, map_world, poses, qs, [dict(scan_ratio_threshold=t) for t in THRESHOLDS], kinds=("host", "device", "packed"))
    assert len({k.tobytes() for k in ks}) > 1


@pytest.mark.parametrize("V", [1, 5, 32])
def test_seq00_v3_variant_counts(capi, small_workload, V):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_00").replace(skip_voxelize=1)
    grid = [dict(scan_ratio_threshold=t, minimum_num_pts=k) for k in (0, 3, 6, 10, 20, -1) for t in (0.05,) + THRESHOLDS][:32]
    variants = grid[:V] if V > 1 else [dict(scan_ratio_threshold=0.2)]
    check(capi, p, map_world, poses, qs, variants, kinds=("host", "device"))


def test_v2_th_bin_max_h_and_duplicates(capi, small_workload):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1, version=2)
    variants = [dict(th_bin_max_h=h) for h in (-1.0, 0.0, 0.05, 0.5, 1.5)] + [dict(th_bin_max_h=0.05), dict(th_bin_max_h=0.05, scan_ratio_threshold=0.1)]
    check(capi, p, map_world, poses, qs, variants, kinds=("host", "packed"))


def test_minimum_num_pts_including_negative(capi, small_workload):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    ks = check(capi, p, map_world, poses, qs, [dict(minimum_num_pts=k) for k in (-5, -1, 0, 1, 10, 40)], voi_max_range=0.8 * p.max_range)
    assert np.all(ks[0] == 1) and np.all(ks[1] == 1), "a negative minimum_num_pts flags nothing"


def test_sub_batch_split(capi, small_workload):
    """150 nodes on 40 x 360 bins: more than one submission's work queue holds (2^21 / 14400 = 145 frames)"""
    map_world, poses, qs = small(small_workload)
    idx = [i % len(qs) for i in range(150)]
    p = P.preset("synthetic_40x360").replace(skip_voxelize=1)
    check(capi, p, map_world, poses[idx], [qs[i] for i in idx], [dict(scan_ratio_threshold=t) for t in (0.1, 0.3)])


def test_class_c_bins_turning_up_late(capi):
    """a sweep that meets bins beyond 2560 points while class C is off: erasor_wait runs the class and folds into the variant masks"""
    import torch
    from test_gpu_parity import _crafted_bin_frame
    p = P.preset("seq_05").replace(skip_voxelize=1)
    rng = np.random.default_rng(5)
    small_f, big_f = _crafted_bin_frame(rng, 200, "rough"), _crafted_bin_frame(rng, 3500, "rough")
    pose = np.array([[0, 0, 0, 0, 0, 0, 1.0]])
    variants = [dict(scan_ratio_threshold=t) for t in THRESHOLDS]
    h = capi.Handle(p)
    for tag, (mw, q) in (("small", small_f), ("small again", small_f), ("big (fix-up)", big_f), ("big", big_f), ("small", small_f)):
        ref_k, ref_f, ref_r, _ = separate(capi, p, mw, pose, [q], variants)
        m = capi.Map(mw)
        h.attach_map(m)
        keep = sweep(capi, h, len(mw), pose, [q], variants)
        assert np.array_equal(keep.reshape(len(variants), -1).cpu().numpy(), ref_k), tag
        nf, nr = h.sweep_stats()
        assert np.array_equal(nf, ref_f) and np.array_equal(nr, ref_r), tag
        assert (ref_k == 0).any()
        h.attach_map(None); m.close()
    torch.cuda.synchronize()
    h.close()


def test_lanes_share_one_mask_graph_replay_and_sharding(capi, twin):
    import torch
    map_world, poses, qs = twin
    p = P.preset("seq_05").replace(skip_voxelize=1)
    variants = [dict(scan_ratio_threshold=t) for t in THRESHOLDS]
    V, n = len(variants), len(map_world)
    ref_k = separate(capi, p, map_world, poses, qs, variants)[0]
    m = capi.Map(map_world)
    lanes = [capi.Handle(p) for _ in range(2)]
    for h in lanes:
        h.attach_map(m)
    halves = [(poses[:10], qs[:10]), (poses[10:], qs[10:])]
    shared = torch.empty(V * n, dtype=torch.uint8, device="cuda")
    launches = []
    for rep in range(3):                       # the first call captures a graph per lane, the next ones replay it
        lanes[0].reset_keep_mask(shared.data_ptr(), V * n)
        lanes[0].synchronize()
        for h, (ps, q) in zip(lanes, halves):
            sweep(capi, h, n, ps, q, variants, "device", keep=shared, reset=False, asynchronous=True)
        for h in lanes:
            h.wait()
        assert np.array_equal(shared.reshape(V, n).cpu().numpy(), ref_k), rep
        launches.append(lanes[0].kernel_launch_count())
    assert launches[2] - launches[1] == launches[1] - launches[0]
    # another variant set on the same pointers: a new graph, not the replay of the old one
    other = [dict(scan_ratio_threshold=0.12)]
    ref_o = separate(capi, p, map_world, poses, qs, other)[0]
    k1 = sweep(capi, lanes[0], n, poses, qs, other, "device")
    assert np.array_equal(k1.cpu().numpy(), ref_o[0])
    # sharding: two half-node sweeps AND-ed through erasor_and_keep_masks == the whole sweep
    both = torch.empty((2, V * n), dtype=torch.uint8, device="cuda")
    for r, (h, (ps, q)) in enumerate(zip(lanes, halves)):
        sweep(capi, h, n, ps, q, variants, "host", keep=both[r])
    out = torch.empty(V * n, dtype=torch.uint8, device="cuda")
    lanes[0].and_keep_masks(both.data_ptr(), 2, V * n, out.data_ptr())
    lanes[0].synchronize()
    assert np.array_equal(out.reshape(V, n).cpu().numpy(), ref_k)
    for h in lanes:
        h.close()
    m.close()


def test_plain_process_nodes_after_a_sweep_is_unchanged(capi, small_workload):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    Q, qo = np.concatenate(qs), offsets(qs)
    m = capi.Map(map_world)
    h = capi.Handle(p)
    h.attach_map(m)
    keep0, fk0 = h.process_nodes(poses, Q, qo, want_frame_keep=True)
    l0 = h.kernel_launch_count()
    keep0b, _ = h.process_nodes(poses, Q, qo, want_frame_keep=True)
    per_call = h.kernel_launch_count() - l0
    stats0 = h.node_stats()
    sweep(capi, h, len(map_world), poses, qs, [dict(scan_ratio_threshold=t) for t in THRESHOLDS])
    m.reset_keep()
    l1 = h.kernel_launch_count()
    keep1, fk1 = h.process_nodes(poses, Q, qo, want_frame_keep=True)
    assert h.kernel_launch_count() - l1 == per_call
    assert np.array_equal(keep1, keep0) and np.array_equal(fk1, fk0)
    assert all(np.array_equal(a, b) for a, b in zip(h.node_stats(), stats0))
    with pytest.raises(capi.ErasorError) as e:
        h.sweep_stats()
    assert e.value.code == capi.E_STATE
    h.close(); m.close()


def test_refusals(capi, small_workload):
    import torch
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    Q, qo = np.concatenate(qs), offsets(qs)
    n = len(map_world)
    keep = torch.ones(33 * n, dtype=torch.uint8, device="cuda")
    h = capi.Handle(p)
    one = [dict(scan_ratio_threshold=0.2)]

    def code(fn):
        with pytest.raises(capi.ErasorError) as e:
            fn()
        return e.value.code
    h._map = capi.Map(map_world)                       # sizes only: not attached yet
    assert code(lambda: h.process_nodes_sweep(poses, Q, qo, one, keep.data_ptr())) == capi.E_INVALID          # no map attached
    h.attach_map(h._map)
    assert code(lambda: h.process_nodes_sweep(poses, Q, qo, [], keep.data_ptr())) == capi.E_INVALID
    assert code(lambda: h.process_nodes_sweep(poses, Q, qo, one * 33, keep.data_ptr())) == capi.E_INVALID
    assert code(lambda: h.process_nodes_sweep(poses, Q, qo, one, 0)) == capi.E_INVALID
    arr, _ = h.sweep_variants(one)
    rc = h.L.erasor_process_nodes_sweep(h.h, poses.ctypes.data_as(capi.POINTER(capi.c_double)), Q.ctypes.data,
                                        qo.ctypes.data_as(capi.POINTER(capi.c_uint64)), len(qs), 0.0, None, 1, keep.data_ptr(), capi.PTR_HOST)
    assert rc == capi.E_INVALID
    h.set_node_inserts(True)
    assert code(lambda: h.process_nodes_sweep(poses, Q, qo, one, keep.data_ptr())) == capi.E_INVALID
    h.set_node_inserts(False)
    h.process_nodes_sweep(poses, Q, qo, one, keep.data_ptr(), asynchronous=True)
    assert code(lambda: h.process_nodes_sweep(poses, Q, qo, one, keep.data_ptr())) == capi.E_STATE
    h.wait()
    h.process_nodes_sweep(poses, Q, qo, one * 32, keep.data_ptr())       # usable afterwards, 32 accepted
    h.close()
    h._map.close()


def _bag_nodes_and_config(tmp_path, capi):
    from erasor_b200 import mapgen, pipeline
    from test_gpu_cpp_driver import YAML
    nodes = pipeline.read_bag_nodes(os.path.join(ROOT, "tests", "golden", "node_tiny.bag"))
    _, naive = mapgen.build_map(nodes, leafsize=0.2)
    with capi.PcdCodec() as codec:
        codec.write(str(tmp_path / "map.pcd"), naive)
        initial = codec.load(str(tmp_path / "map.pcd"))
    cfg = tmp_path / "seq_05.yaml"
    cfg.write_text(YAML.format(save=str(tmp_path)).replace('initial_map_path: "unused"', f'initial_map_path: "{tmp_path / "map.pcd"}"')
                   .replace("removal_interval: 2", "removal_interval: 1"))
    return nodes, initial, str(cfg)


def test_sweep_frame_independent_rows_and_cli(capi, tmp_path):
    from erasor_b200 import params, pipeline, sweep as cli
    nodes, initial, cfg = _bag_nodes_and_config(tmp_path, capi)
    ep, up = params.load_yaml(cfg)
    variants = cli.variants_of([0.1, 0.2, 0.3], [0, 10])
    rows = pipeline.sweep_frame_independent(nodes, initial, up, ep, variants, batch=2)
    assert len(rows) == 6
    with capi.Evaluator() as ev:
        for var, row in zip(variants, rows):
            res = pipeline.run_frame_independent(nodes, initial, up, ep.replace(**var), batch=2)
            q = ev.evaluate(initial, res["static_map"], voxelsize=0.2)
            want = dict(PR=q["PR"], RR=q["RR"], F1=q["F1"], kept=int(np.count_nonzero(res["keep"])), saved=len(res["static_map"]))
            assert {k: row[k] for k in want} == want, var
            assert row["scan_ratio_threshold"] == var["scan_ratio_threshold"] and row["minimum_num_pts"] == var["minimum_num_pts"]
    best = tmp_path / "best.pcd"
    r = subprocess.run([sys.executable, "-m", "erasor_b200.sweep", cfg, os.path.join(ROOT, "tests", "golden", "node_tiny.bag"),
                        "--scan-ratio", "0.1,0.2,0.3", "--min-pts", "0,10", "--batch", "2", "--save-best", str(best)],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    assert r.stdout == cli.format_rows(rows)
    with capi.PcdCodec() as codec:
        saved = codec.load(str(best))
    assert len(saved) == rows[cli.best_row(rows)]["saved"]
    with pytest.raises(ValueError):
        pipeline.sweep_frame_independent(nodes, initial, up, ep, [dict(gf_iter=2)])
