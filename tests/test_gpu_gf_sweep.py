"""GPU: the Scan Ratio Test and ground-filter sweep (erasor_process_nodes_sweep_ex, DESIGN.md section 8.6).  Every mask and every
sweep counter must equal, bit for bit, a separate erasor_process_nodes run with p.replace(**setting) on a fresh map: thresholds x
gf_dist_thr on the bench twin, gf_num_lpr x num_lowest_pts on seq 00, gf_th_seeds_height, gf_iter (0 included), version 2, 32
settings in 32 ground-filter groups and duplicates, host, device and packed-xyz queries, and crafted bins of every R-GPF size class
(class C in shared memory and beyond it, turning up late).  Also: the one-group call is process_nodes_sweep, graph replay and a new
graph when only a ground-filter field changes, lanes sharing one mask, plain calls and Scan Ratio Test sweeps after a ground-filter
sweep, every refusal, and pipeline.tune_frame_independent and its command line against run_frame_independent + capi.Evaluator."""
import os
import subprocess
import sys

import numpy as np
import pytest

from erasor_b200 import params as P
from test_gpu_srt_sweep import THRESHOLDS, _bag_nodes_and_config, capi, offsets, separate, small, twin  # noqa: F401 (fixtures)
from test_gpu_srt_sweep import sweep as srt_sweep

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIST_THR = (0.075, 0.15, 0.25)


def sweep_ex(h, n, poses, qs, settings, kind="host", keep=None, reset=True, asynchronous=False):
    import torch
    V = len(settings)
    if keep is None:
        keep = torch.empty(V * n, dtype=torch.uint8, device="cuda")
    if reset:
        h.reset_keep_mask(keep.data_ptr(), V * n)
    Q, qo = np.concatenate(qs), offsets(qs)
    if kind == "device":
        dQ = torch.from_numpy(np.ascontiguousarray(Q)).cuda()
        h._dq = dQ
        h.process_nodes_sweep_ex(poses, dQ.data_ptr(), qo, settings, keep.data_ptr(), asynchronous=asynchronous)
    else:
        h.process_nodes_sweep_ex(poses, Q, qo, settings, keep.data_ptr(), packed_xyz=(kind == "packed"), asynchronous=asynchronous)
    return keep


def check(capi, p, map_world, poses, qs, settings, kinds=("host",)):
    ref_k, ref_f, ref_r, ref_v = separate(capi, p, map_world, poses, qs, settings)
    assert (ref_k == 0).any(), "the workload must reject something"
    n = len(map_world)
    m = capi.Map(map_world)
    h = capi.Handle(p)
    h.attach_map(m)
    for kind in kinds:
        got = sweep_ex(h, n, poses, qs, settings, kind).reshape(len(settings), n).cpu().numpy()
        for v in range(len(settings)):
            assert np.array_equal(got[v], ref_k[v]), f"{kind} {settings[v]}: {np.count_nonzero(got[v] != ref_k[v])} points differ"
        nf, nr = h.sweep_stats()
        assert np.array_equal(nf, ref_f) and np.array_equal(nr, ref_r), kind
        nv, uf, _ = h.node_stats()
        assert np.array_equal(nv, ref_v) and (uf >= ref_f.max(axis=0)).all()
        assert np.all(m.get_keep() == 1), "a sweep leaves the map's keep mask alone"
    h.close(); m.close()
    return ref_k


def test_bench_twin_thresholds_x_dist_thr(capi, twin):
    map_world, poses, qs = twin
    p = P.preset("seq_05").replace(skip_voxelize=1)
    settings = [dict(scan_ratio_threshold=t, gf_dist_thr=d) for t in THRESHOLDS for d in DIST_THR]
    ks = check(capi, p, map_world, poses, qs, settings, kinds=("host", "device", "packed"))
    assert len({ks[v].tobytes() for v in range(3)}) > 1, "gf_dist_thr must matter"


def test_seq00_num_lpr_x_num_lowest_pts(capi, small_workload):
    """num_lowest_pts 600 is beyond every class-A bin (its LPR is 0 there) but not beyond the larger bins"""
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_00").replace(skip_voxelize=1)
    check(capi, p, map_world, poses, qs, [dict(gf_num_lpr=k, num_lowest_pts=l) for k in (5, 10, 20) for l in (0, 1, 5, 600)], kinds=("host", "device"))


def test_seeds_height_and_gf_iter(capi, small_workload):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    settings = [dict(gf_th_seeds_height=s, scan_ratio_threshold=t) for s in (0.1, 0.5, 1.5) for t in (0.1, 0.3)]
    settings += [dict(gf_iter=k) for k in (0, 1, 3, 8)]
    check(capi, p, map_world, poses, qs, settings)


def test_v2(capi, small_workload):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1, version=2)
    check(capi, p, map_world, poses, qs, [dict(th_bin_max_h=h, gf_dist_thr=d) for h in (0.0, 0.5) for d in DIST_THR], kinds=("host", "packed"))


def test_32_groups_and_duplicates(capi, small_workload):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    check(capi, p, map_world, poses, qs, [dict(gf_dist_thr=0.02 + 0.01 * i, scan_ratio_threshold=(0.1, 0.2, 0.3)[i % 3]) for i in range(32)],
          kinds=("host", "device"))
    dup = [dict(gf_dist_thr=0.1), dict(gf_dist_thr=0.1), dict(gf_dist_thr=0.1, scan_ratio_threshold=0.3), dict(gf_iter=1), dict(gf_dist_thr=0.1)]
    ks = check(capi, p, map_world, poses, qs, dup)
    assert np.array_equal(ks[0], ks[1]) and np.array_equal(ks[0], ks[4])


def test_crafted_bins_of_every_class_and_late_class_c(capi):
    """one flagged bin of 200 (class A), 1500 and 2300 (class B, the second on the radix path), 5000 (class C in shared memory)
    and 9000 points (class C in global scratch); the class-C bins turn up while class C is off, so erasor_wait runs it late"""
    import torch
    from test_gpu_parity import _crafted_bin_frame
    p = P.preset("seq_05").replace(skip_voxelize=1)
    rng = np.random.default_rng(7)
    frame = {n: _crafted_bin_frame(rng, n - 60, "rough") for n in (200, 1500, 2300, 5000, 9000)}
    settings = [dict(scan_ratio_threshold=t, gf_dist_thr=d) for t in (0.1, 0.3) for d in (0.02, 0.075, 0.25)]
    settings += [dict(gf_iter=0), dict(num_lowest_pts=600), dict(gf_th_seeds_height=0.05, gf_num_lpr=3)]
    pose = np.array([[0, 0, 0, 0, 0, 0, 1.0]])
    h = capi.Handle(p)
    for n in (200, 1500, 2300, 9000, 9000, 200, 5000, 5000):
        mw, q = frame[n]
        ref_k, ref_f, ref_r, _ = separate(capi, p, mw, pose, [q], settings)
        m = capi.Map(mw)
        h.attach_map(m)
        keep = sweep_ex(h, len(mw), pose, [q], settings)
        assert np.array_equal(keep.reshape(len(settings), -1).cpu().numpy(), ref_k), n
        nf, nr = h.sweep_stats()
        assert np.array_equal(nf, ref_f) and np.array_equal(nr, ref_r), n
        assert len({k.tobytes() for k in ref_k}) > 1, n
        h.attach_map(None); m.close()
    torch.cuda.synchronize()
    h.close()


def test_one_group_is_process_nodes_sweep(capi, twin):
    map_world, poses, qs = twin
    p = P.preset("seq_05").replace(skip_voxelize=1)
    n = len(map_world)
    variants = [dict(scan_ratio_threshold=t) for t in THRESHOLDS]
    same_gf = [dict(v, gf_dist_thr=p.gf_dist_thr, gf_iter=p.gf_iter) for v in variants]
    m = capi.Map(map_world)
    h = capi.Handle(p)
    h.attach_map(m)
    srt_sweep(capi, h, n, poses, qs, variants)             # the handle's first call also launches class C (nothing seen yet)
    out = []
    for rep in range(2):
        for call in ("srt", "ex"):
            l0 = h.kernel_launch_count()
            if call == "srt":
                keep = srt_sweep(capi, h, n, poses, qs, variants)
            else:
                keep = sweep_ex(h, n, poses, qs, same_gf if rep else variants)
            out.append((call, keep.cpu().numpy(), h.sweep_stats(), h.node_stats(), h.kernel_launch_count() - l0))
    for (_, k0, s0, n0, l0), (_, k1, s1, n1, l1) in zip(out[0::2], out[1::2]):
        assert np.array_equal(k0, k1) and l0 == l1
        assert all(np.array_equal(a, b) for a, b in zip(s0, s1)) and all(np.array_equal(a, b) for a, b in zip(n0, n1))
    h.close(); m.close()


def test_graph_replay_and_new_graph_on_a_ground_filter_change(capi, twin):
    """device queries and one mask buffer: the same pointers every call, so the second call of a setting list replays its graph and
    a call that changes only gf_dist_thr must capture its own"""
    import torch
    map_world, poses, qs = twin
    p = P.preset("seq_05").replace(skip_voxelize=1)
    n = len(map_world)
    a = [dict(scan_ratio_threshold=t, gf_dist_thr=0.075) for t in (0.1, 0.3)]
    b = [dict(scan_ratio_threshold=t, gf_dist_thr=0.25) for t in (0.1, 0.3)]
    ref_a, ref_b = separate(capi, p, map_world, poses, qs, a)[0], separate(capi, p, map_world, poses, qs, b)[0]
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
        h.process_nodes_sweep_ex(poses, dQ.data_ptr(), offsets(qs), s, keep.data_ptr())
        got = keep.reshape(2, n).cpu().numpy()
        launches.append(h.kernel_launch_count() - l0)
        assert np.array_equal(got, ref), tag
    assert len(set(launches[1:])) == 1            # (the handle's first call also launches class C)
    h.close(); m.close()


def test_lanes_share_one_mask(capi, twin):
    import torch
    map_world, poses, qs = twin
    p = P.preset("seq_05").replace(skip_voxelize=1)
    settings = [dict(scan_ratio_threshold=t, gf_dist_thr=d) for t in (0.1, 0.2) for d in DIST_THR]
    V, n = len(settings), len(map_world)
    ref_k = separate(capi, p, map_world, poses, qs, settings)[0]
    m = capi.Map(map_world)
    lanes = [capi.Handle(p) for _ in range(2)]
    for h in lanes:
        h.attach_map(m)
    shared = torch.empty(V * n, dtype=torch.uint8, device="cuda")
    for rep in range(2):
        lanes[0].reset_keep_mask(shared.data_ptr(), V * n)
        lanes[0].synchronize()
        for h, sl in zip(lanes, (slice(0, 10), slice(10, 20))):
            sweep_ex(h, n, poses[sl], qs[sl], settings, "device", keep=shared, reset=False, asynchronous=True)
        for h in lanes:
            h.wait()
        assert np.array_equal(shared.reshape(V, n).cpu().numpy(), ref_k), rep
    for h in lanes:
        h.close()
    m.close()


def test_plain_call_and_srt_sweep_after_a_ground_filter_sweep(capi, small_workload):
    map_world, poses, qs = small(small_workload)
    p = P.preset("seq_05").replace(skip_voxelize=1)
    Q, qo = np.concatenate(qs), offsets(qs)
    n = len(map_world)
    variants = [dict(scan_ratio_threshold=t) for t in THRESHOLDS]
    m = capi.Map(map_world)
    h = capi.Handle(p)
    h.attach_map(m)

    def plain_and_srt():
        m.reset_keep()
        l0 = h.kernel_launch_count()
        keep, fk = h.process_nodes(poses, Q, qo, want_frame_keep=True)
        plain = (keep, fk, h.node_stats(), h.kernel_launch_count() - l0)
        srt = (srt_sweep(capi, h, n, poses, qs, variants).cpu().numpy(), h.sweep_stats(), h.node_stats())
        return plain, srt
    plain_and_srt()                                     # the handle's first call also launches class C
    before = plain_and_srt()
    sweep_ex(h, n, poses, qs, [dict(gf_dist_thr=d, gf_iter=k) for d in DIST_THR for k in (0, 1, 8)])
    after = plain_and_srt()
    (kb, fb, sb, lb), (vb, wb, ub) = before
    (ka, fa, sa, la), (va, wa, ua) = after
    assert np.array_equal(ka, kb) and np.array_equal(fa, fb) and la == lb
    assert all(np.array_equal(x, y) for x, y in zip(sa, sb))
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
    one = [dict(gf_dist_thr=0.1)]

    def code(fn):
        with pytest.raises(capi.ErasorError) as e:
            fn()
        return e.value.code
    h._map = capi.Map(map_world)                       # sizes only: not attached yet
    assert code(lambda: h.process_nodes_sweep_ex(poses, Q, qo, one, keep.data_ptr())) == capi.E_INVALID          # no map attached
    h.attach_map(h._map)
    assert code(lambda: h.process_nodes_sweep_ex(poses, Q, qo, [], keep.data_ptr())) == capi.E_INVALID
    assert code(lambda: h.process_nodes_sweep_ex(poses, Q, qo, one * 33, keep.data_ptr())) == capi.E_INVALID
    assert code(lambda: h.process_nodes_sweep_ex(poses, Q, qo, one, 0)) == capi.E_INVALID
    assert code(lambda: h.process_nodes_sweep_ex(poses, Q, qo, one + [dict(gf_iter=9)], keep.data_ptr())) == capi.E_UNSUPPORTED
    rc = h.L.erasor_process_nodes_sweep_ex(h.h, poses.ctypes.data_as(capi.POINTER(capi.c_double)), Q.ctypes.data,
                                           qo.ctypes.data_as(capi.POINTER(capi.c_uint64)), len(qs), 0.0, None, 1, keep.data_ptr(), capi.PTR_HOST)
    assert rc == capi.E_INVALID
    h.set_node_inserts(True)
    assert code(lambda: h.process_nodes_sweep_ex(poses, Q, qo, one, keep.data_ptr())) == capi.E_INVALID
    h.set_node_inserts(False)
    h.process_nodes_sweep_ex(poses, Q, qo, one, keep.data_ptr(), asynchronous=True)
    assert code(lambda: h.process_nodes_sweep_ex(poses, Q, qo, one, keep.data_ptr())) == capi.E_STATE
    h.wait()
    h.process_nodes_sweep_ex(poses, Q, qo, [dict(gf_iter=8, gf_dist_thr=0.01 * i) for i in range(32)], keep.data_ptr())   # usable, 32 accepted
    h.close()
    h._map.close()


def test_tune_frame_independent_rows_and_cli(capi, tmp_path):
    from erasor_b200 import params, pipeline, sweep as cli
    nodes, initial, cfg = _bag_nodes_and_config(tmp_path, capi)
    ep, up = params.load_yaml(cfg)
    settings = cli.variants_of([0.1, 0.3], None, None, gf_dist_thr=[0.05, 0.2], gf_iter=[1, 3])
    rows = pipeline.tune_frame_independent(nodes, initial, up, ep, settings, batch=2)
    assert len(rows) == 8
    with capi.Evaluator() as ev:
        for s, row in zip(settings, rows):
            res = pipeline.run_frame_independent(nodes, initial, up, ep.replace(**s), batch=2)
            q = ev.evaluate(initial, res["static_map"], voxelsize=0.2)
            want = dict(PR=q["PR"], RR=q["RR"], F1=q["F1"], kept=int(np.count_nonzero(res["keep"])), saved=len(res["static_map"]))
            assert {k: row[k] for k in want} == want, s
            assert all(row[f] == s.get(f, getattr(ep, f)) for f in capi.SRT_SWEEP_FIELDS + capi.GF_SWEEP_FIELDS), s
    best = tmp_path / "best.pcd"
    r = subprocess.run([sys.executable, "-m", "erasor_b200.sweep", cfg, os.path.join(ROOT, "tests", "golden", "node_tiny.bag"),
                        "--scan-ratio", "0.1,0.3", "--gf-dist-thr", "0.05,0.2", "--gf-iter", "1,3", "--batch", "2", "--save-best", str(best)],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    assert r.stdout == cli.format_rows(rows, ("gf_dist_thr", "gf_iter"))
    with capi.PcdCodec() as codec:
        saved = codec.load(str(best))
    assert len(saved) == rows[cli.best_row(rows)]["saved"]
    with pytest.raises(ValueError):
        pipeline.tune_frame_independent(nodes, initial, up, ep, [dict(cov_mode=1)])
    with pytest.raises(ValueError):
        pipeline.sweep_frame_independent(nodes, initial, up, ep, [dict(gf_dist_thr=0.1)])
