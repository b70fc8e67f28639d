"""GPU: the geometry and height-window sweep (erasor_process_nodes_tune, DESIGN.md section 8.7).  Every mask and every sweep counter
must equal, bit for bit, a separate erasor_process_nodes run with p.replace(**setting) on a fresh map and the same explicit
voi_max_range: the three KITTI geometries x five thresholds on the bench twin with host, device and packed-xyz queries, min_h /
max_h pairs and an ERASOR max_range below the VoI radius, the handle's own geometry among others, a 40 x 360 geometry next to small
ones (two K1 launches, both thread counts), 32 geometries, ground-filter groups inside a geometry, a sub-batched call, graph replay
and a new graph on a geometry change.  Also: the call with the handle's geometry alone is process_nodes_sweep_ex, plain calls and
sweeps after a geometry sweep are unchanged, every refusal, and pipeline.tune_frame_independent and its command line against
run_frame_independent + capi.Evaluator."""
import os
import subprocess
import sys

import numpy as np
import pytest

from erasor_b200 import params as P
from test_gpu_srt_sweep import THRESHOLDS, _bag_nodes_and_config, capi, offsets, separate, small, twin  # noqa: F401 (fixtures)
from test_gpu_srt_sweep import sweep as srt_sweep
from test_gpu_gf_sweep import sweep_ex

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VOI = 80.0                                             # the VoI radius every call passes (/MapUpdater/max_range)
KITTI = (dict(max_range=60.0, num_rings=15, num_sectors=60), dict(max_range=60.0, num_rings=15, num_sectors=108),
         dict(max_range=80.0, num_rings=20, num_sectors=108))


def tune(h, n, poses, qs, settings, kind="host", keep=None, voi=VOI):
    import torch
    V = len(settings)
    if keep is None:
        keep = torch.empty(V * n, dtype=torch.uint8, device="cuda")
    h.reset_keep_mask(keep.data_ptr(), V * n)
    Q, qo = np.concatenate(qs), offsets(qs)
    if kind == "device":
        dQ = torch.from_numpy(np.ascontiguousarray(Q)).cuda()
        h._dq = dQ
        h.process_nodes_tune(poses, dQ.data_ptr(), qo, settings, keep.data_ptr(), voi_max_range=voi)
    else:
        h.process_nodes_tune(poses, Q, qo, settings, keep.data_ptr(), voi_max_range=voi, packed_xyz=(kind == "packed"))
    return keep


def check(capi, p, map_world, poses, qs, settings, kinds=("host",)):
    ref_k, ref_f, ref_r, ref_v = separate(capi, p, map_world, poses, qs, settings, voi_max_range=VOI)
    assert (ref_k == 0).any(), "the workload must reject something"
    n = len(map_world)
    m = capi.Map(map_world)
    h = capi.Handle(p)
    h.attach_map(m)
    for kind in kinds:
        got = tune(h, n, poses, qs, settings, kind).reshape(len(settings), n).cpu().numpy()
        for v in range(len(settings)):
            assert np.array_equal(got[v], ref_k[v]), f"{kind} {settings[v]}: {np.count_nonzero(got[v] != ref_k[v])} points differ"
        nf, nr = h.sweep_stats()
        assert np.array_equal(nf, ref_f) and np.array_equal(nr, ref_r), kind
        nv, uf, _ = h.node_stats()
        geo0 = [v for v in range(len(settings)) if all(settings[v].get(f) == settings[0].get(f) for f in capi.GEOMETRY_SWEEP_FIELDS)]
        assert np.array_equal(nv, ref_v) and (uf >= ref_f[geo0].max(axis=0)).all()
        assert np.all(m.get_keep() == 1), "a sweep leaves the map's keep mask alone"
    h.close(); m.close()
    return ref_k


def test_bench_twin_kitti_geometries_x_thresholds(capi, twin):
    map_world, poses, qs = twin
    p = P.preset("seq_05").replace(skip_voxelize=1)
    settings = [dict(g, scan_ratio_threshold=t) for g in KITTI for t in THRESHOLDS]
    ks = check(capi, p, map_world, poses, qs, settings, kinds=("host", "device", "packed"))
    assert len({ks[5 * g + 2].tobytes() for g in range(3)}) == 3, "every geometry must matter"


def test_height_window_and_short_max_range(capi, small_workload):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    settings = [dict(min_h=lo, max_h=hi) for lo, hi in ((-1.3, 3.2), (-1.3, 1.5), (-1.3, 1.0), (-2.0, 4.0), (-1.6, 2.5))]
    settings += [dict(max_range=30.0), dict(max_range=45.0, scan_ratio_threshold=0.3)]
    ks = check(capi, p, map_world, poses, qs, settings, kinds=("host", "device"))
    assert len({k.tobytes() for k in ks}) == len(ks)


def test_own_geometry_among_others_and_ground_filter_groups(capi, small_workload):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    settings = [dict(gf_dist_thr=d, scan_ratio_threshold=t) for d in (0.075, 0.25) for t in (0.1, 0.3)]
    settings += [dict(s, num_rings=20, num_sectors=108) for s in settings] + [dict(gf_iter=1, num_sectors=90)]
    check(capi, p, map_world, poses, qs, settings)
    check(capi, p, map_world, poses, qs, settings[4:] + settings[:4])


def test_own_geometry_alone_is_process_nodes_sweep_ex(capi, twin):
    map_world, poses, qs = twin
    p = P.preset("seq_05").replace(skip_voxelize=1)
    n = len(map_world)
    own = {f: getattr(p, f) for f in capi.GEOMETRY_SWEEP_FIELDS}
    settings = [dict(scan_ratio_threshold=t, gf_dist_thr=d) for t in (0.1, 0.3) for d in (0.075, 0.25)]
    m = capi.Map(map_world)
    h = capi.Handle(p)
    h.attach_map(m)
    sweep_ex(h, n, poses, qs, settings)                   # the handle's first call also launches class C
    out = []
    for call in ("ex", "tune", "ex", "tune"):
        l0 = h.kernel_launch_count()
        if call == "ex":
            keep = sweep_ex(h, n, poses, qs, settings)
        else:
            keep = tune(h, n, poses, qs, [dict(s, **own) for s in settings], voi=0.0)
        out.append((keep.cpu().numpy(), h.sweep_stats(), h.node_stats(), h.kernel_launch_count() - l0))
    for (k0, s0, n0, l0), (k1, s1, n1, l1) in zip(out[0::2], out[1::2]):
        assert np.array_equal(k0, k1) and l0 == l1
        assert all(np.array_equal(a, b) for a, b in zip(s0 + n0, s1 + n1))
    h.close(); m.close()


def test_big_geometry_next_to_small_ones(capi, small_workload):
    """40 x 360 bins (173 KB of K1 tables: a 32-warp launch of its own) and two small geometries packed into an 8-warp one"""
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    settings = [dict(num_rings=40, num_sectors=360, max_range=80.0, scan_ratio_threshold=t) for t in (0.1, 0.3)]
    settings += [dict(g, scan_ratio_threshold=0.2) for g in KITTI[:2]]
    check(capi, p, map_world, poses, qs, settings, kinds=("host", "device"))
    check(capi, p, map_world, poses, qs, settings[2:] + settings[:2])


def test_32_geometries(capi, small_workload):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    settings = [dict(num_rings=8 + i % 8, num_sectors=40 + 4 * (i // 8), max_range=40.0 + i) for i in range(32)]
    check(capi, p, map_world, poses, qs, settings, kinds=("host", "device"))


def test_sub_batches(capi, small_workload):
    """150 nodes under a 40 x 360 geometry: kMaxRecords / B = 145 frames, so the call runs in two sub-batches"""
    map_world, poses, qs = small(small_workload)
    reps = -(-150 // len(qs))
    poses, qs = np.concatenate([poses] * reps)[:150], (qs * reps)[:150]
    p = P.preset("seq_05").replace(skip_voxelize=1)
    check(capi, p, map_world, poses, qs, [dict(num_rings=40, num_sectors=360, max_range=80.0), dict(num_rings=20, num_sectors=108)])


def test_graph_replay_and_new_graph_on_a_geometry_change(capi, twin):
    import torch
    map_world, poses, qs = twin
    p = P.preset("seq_05").replace(skip_voxelize=1)
    n = len(map_world)
    a = [dict(KITTI[1], scan_ratio_threshold=t) for t in (0.1, 0.3)]
    b = [dict(KITTI[2], scan_ratio_threshold=t) for t in (0.1, 0.3)]
    ref_a = separate(capi, p, map_world, poses, qs, a, voi_max_range=VOI)[0]
    ref_b = separate(capi, p, map_world, poses, qs, b, voi_max_range=VOI)[0]
    assert not np.array_equal(ref_a, ref_b)
    m = capi.Map(map_world)
    h = capi.Handle(p)
    h.attach_map(m)
    dQ = torch.from_numpy(np.ascontiguousarray(np.concatenate(qs))).cuda()
    keep = torch.empty(2 * n, dtype=torch.uint8, device="cuda")
    launches = []
    for tag, s, ref in (("a", a, ref_a), ("a replay", a, ref_a), ("b", b, ref_b), ("a again", a, ref_a), ("b replay", b, ref_b)):
        h.reset_keep_mask(keep.data_ptr(), 2 * n)
        l0 = h.kernel_launch_count()
        h.process_nodes_tune(poses, dQ.data_ptr(), offsets(qs), s, keep.data_ptr(), voi_max_range=VOI)
        launches.append(h.kernel_launch_count() - l0)
        assert np.array_equal(keep.reshape(2, n).cpu().numpy(), ref), tag
    assert len(set(launches)) == 1
    h.close(); m.close()


def test_plain_call_and_sweeps_after_a_geometry_sweep(capi, small_workload):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    Q, qo = np.concatenate(qs), offsets(qs)
    n = len(map_world)
    variants = [dict(scan_ratio_threshold=t) for t in THRESHOLDS]
    gf = [dict(gf_dist_thr=d) for d in (0.075, 0.25)]
    m = capi.Map(map_world)
    h = capi.Handle(p)
    h.attach_map(m)

    def others():
        m.reset_keep()
        l0 = h.kernel_launch_count()
        keep, fk = h.process_nodes(poses, Q, qo, want_frame_keep=True)
        plain = (keep, fk, h.node_stats(), h.kernel_launch_count() - l0)
        srt = (srt_sweep(capi, h, n, poses, qs, variants).cpu().numpy(), h.sweep_stats(), h.node_stats())
        ex = (sweep_ex(h, n, poses, qs, gf).cpu().numpy(), h.sweep_stats(), h.node_stats())
        return plain, srt, ex
    others()                                              # the handle's first call also launches class C
    before = others()
    tune(h, n, poses, qs, [dict(g, scan_ratio_threshold=0.2) for g in KITTI] + [dict(num_rings=40, num_sectors=360)])
    after = others()
    (kb, fb, sb, lb), *rb = before
    (ka, fa, sa, la), *ra = after
    assert np.array_equal(ka, kb) and np.array_equal(fa, fb) and la == lb
    assert all(np.array_equal(x, y) for x, y in zip(sa, sb))
    for (vb, wb, ub), (va, wa, ua) in zip(rb, ra):
        assert np.array_equal(va, vb) and all(np.array_equal(x, y) for x, y in zip(wa + ua, wb + ub))
    h.close(); m.close()


def test_refusals(capi, small_workload):
    import torch
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    Q, qo = np.concatenate(qs), offsets(qs)
    n = len(map_world)
    keep = torch.ones(33 * n, dtype=torch.uint8, device="cuda")
    h = capi.Handle(p)
    one = [dict(num_rings=20)]

    def code(settings, voi=VOI, ptr=None):
        with pytest.raises(capi.ErasorError) as e:
            h.process_nodes_tune(poses, Q, qo, settings, keep.data_ptr() if ptr is None else ptr, voi_max_range=voi)
        return e.value.code
    h._map = capi.Map(map_world)
    assert code(one) == capi.E_INVALID                                          # no map attached
    h.attach_map(h._map)
    assert code([]) == capi.E_INVALID
    assert code(one * 33) == capi.E_INVALID
    assert code(one, ptr=0) == capi.E_INVALID
    assert code(one + [dict(gf_iter=9)]) == capi.E_UNSUPPORTED
    arr, _ = h.tune_settings(one)
    rc = h.L.erasor_process_nodes_tune(h.h, poses.ctypes.data_as(capi.POINTER(capi.c_double)), Q.ctypes.data,
                                       qo.ctypes.data_as(capi.POINTER(capi.c_uint64)), len(qs), VOI, None, 1, keep.data_ptr(), capi.PTR_HOST)
    assert rc == capi.E_INVALID
    assert code([dict(num_rings=0)]) == capi.E_INVALID
    assert code([dict(num_rings=300, num_sectors=300)]) == capi.E_INVALID                # beyond 65534 bins
    assert code([dict(num_rings=100, num_sectors=600)]) == capi.E_UNSUPPORTED            # tables beyond the shared memory
    assert code([dict(max_range=-1.0)]) == capi.E_INVALID                                # build_bin_tables refuses it
    assert code([dict(max_range=60.0), dict(max_range=80.0)], voi=0.0) == capi.E_INVALID
    h.set_node_inserts(True)
    assert code(one) == capi.E_INVALID
    h.set_node_inserts(False)
    h.process_nodes_tune(poses, Q, qo, one, keep.data_ptr(), voi_max_range=VOI, asynchronous=True)
    assert code(one) == capi.E_STATE
    h.wait()
    h.process_nodes_tune(poses, Q, qo, [dict(max_range=60.0 + i) for i in range(32)], keep.data_ptr(), voi_max_range=VOI)
    h.process_nodes_tune(poses, Q, qo, [dict(max_range=70.0), dict(max_range=70.0, num_rings=10)], keep.data_ptr(), voi_max_range=0.0)
    h.close()
    h._map.close()


def test_tune_frame_independent_rows_and_cli(capi, tmp_path):
    from erasor_b200 import params, pipeline, sweep as cli
    nodes, initial, cfg = _bag_nodes_and_config(tmp_path, capi)
    ep, up = params.load_yaml(cfg)
    settings = cli.variants_of([0.1, 0.3], None, None, num_rings=[10, 20], max_h=[1.5, 3.0])
    rows = pipeline.tune_frame_independent(nodes, initial, up, ep, settings, batch=2)
    assert len(rows) == 8
    with capi.Evaluator() as ev:
        for s, row in zip(settings, rows):
            res = pipeline.run_frame_independent(nodes, initial, up, ep.replace(**s), batch=2)
            q = ev.evaluate(initial, res["static_map"], voxelsize=0.2)
            want = dict(PR=q["PR"], RR=q["RR"], F1=q["F1"], kept=int(np.count_nonzero(res["keep"])), saved=len(res["static_map"]))
            assert {k: row[k] for k in want} == want, s
            assert all(row[f] == s.get(f, getattr(ep, f)) for f in capi.SRT_SWEEP_FIELDS + capi.GF_SWEEP_FIELDS + capi.GEOMETRY_SWEEP_FIELDS), s
    best = tmp_path / "best.pcd"
    r = subprocess.run([sys.executable, "-m", "erasor_b200.sweep", cfg, os.path.join(ROOT, "tests", "golden", "node_tiny.bag"),
                        "--scan-ratio", "0.1,0.3", "--num-rings", "10,20", "--max-h", "1.5,3.0", "--batch", "2", "--save-best", str(best)],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    assert r.stdout == cli.format_rows(rows, ("num_rings", "max_h"))
    with capi.PcdCodec() as codec:
        saved = codec.load(str(best))
    assert len(saved) == rows[cli.best_row(rows)]["saved"]
    with pytest.raises(ValueError):
        pipeline.tune_frame_independent(nodes, initial, up, ep, [dict(num_rings=10, cov_mode=1)])
