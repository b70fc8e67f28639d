"""The device PR/RR evaluator (capi.Evaluator, erasor_evaluate) against erasor_b200.evaluate (sklearn), the reference script's
golden table, and per point against the numpy model of tests/test_eval_grid_model.py."""
import json

import numpy as np
import pytest

from erasor_b200 import capi
from erasor_b200 import evaluate as E
from erasor_b200 import params as P
from test_eval_grid_model import ADV, NO_MATCH, model_eval, seed41_pass, sq_dist, thr_of

pytestmark = pytest.mark.gpu

KEYS4 = ("gt_static", "gt_dynamic", "preserved_static", "preserved_dynamic")


@pytest.fixture(scope="module")
def ev():
    e = capi.Evaluator(device=0)
    yield e
    e.close()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _device_call(ev, gt, est, keep, vs):
    """the same call with device pointers; returns (counts, match)"""
    import torch
    g, e = _dev(np.asarray(gt, np.float32).reshape(-1, 4)), _dev(np.asarray(est, np.float32).reshape(-1, 4))
    k = _dev(np.asarray(keep).astype(np.uint8)) if keep is not None else None
    m = torch.empty(len(g), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()                             # the evaluator runs on a stream of its own
    d = ev.evaluate_ptr(g.data_ptr() if len(g) else 0, len(g), e.data_ptr() if len(e) else 0, len(e), k.data_ptr() if k is not None and len(k) else 0,
                        vs, capi.PTR_DEVICE, m.data_ptr() if len(g) else 0)
    c = ev.last_counts()
    assert d == E.rates(*(c[x] for x in KEYS4))
    return c, m.cpu().numpy().view(np.uint32)


def _check_against_model(ev, gt, est, keep=None, vs=0.2):
    want, want_m = model_eval(gt, est, keep, vs)
    d = ev.evaluate(gt, est, keep, vs, want_match=True)
    got = ev.last_counts()
    m = got.pop("match")
    assert got == want, (got, want)
    assert np.array_equal(m, want_m)
    assert d == E.rates(*(want[x] for x in KEYS4))
    got_d, m_d = _device_call(ev, gt, est, keep, vs)
    assert got_d == want and np.array_equal(m_d, want_m)
    return want


# ---- the device counts equal the host evaluator's ------------------------------------------------------------------------
def test_seed41_pass_equals_host_and_golden_table(ev, oracle_mod):
    from test_evaluate import REF_TABLE
    gt, est = seed41_pass(oracle_mod)
    d = ev.evaluate(gt, est)
    assert ev.last_counts()["ambiguous_ties"] == 0
    assert d == E.evaluate(gt, est)
    t = json.load(open(REF_TABLE))["table"]
    assert tuple(d[x] for x in KEYS4) == (t["gt_S"], t["gt_D"], t["kept_S"], t["kept_D"])


def test_node_mode_final_map_scored_in_place(ev):
    """bench.py's seq 05 twin: 20 nodes against the resident map, then the map's keep mask scored where it lives -- the
    estimate bench.py's final_map_quality builds on the host"""
    import bench
    p, map_world, poses, qs = bench.load_workload("seq05", 0, 1, 20)
    gm = capi.Map(map_world, device=0)
    h = capi.Handle(p, device=0)
    h.attach_map(gm)
    keep, _ = h.process_nodes(poses, np.concatenate(qs), np.cumsum([0] + [len(q) for q in qs]).astype(np.uint64))
    assert 0 < int((keep == 0).sum()) < len(keep)
    d = ev.evaluate_map(gm)
    assert ev.last_counts()["ambiguous_ties"] == 0
    assert d == E.evaluate(map_world, map_world[keep.astype(bool)])
    assert d == ev.evaluate(map_world, map_world, keep=keep)
    h.close()
    gm.close()


def test_sequential_updater_static_map(ev):
    from erasor_b200 import synth
    sc = synth.Scene(seed=41, length=40.0, n_nodes=17, n_dynamic=6)
    kw = dict(n_beams=24, n_az=480)
    m = sc.build_map(list(range(17)), voxel=0.2, **kw)
    ep, up = P.preset("seq_05"), P.updater_preset("seq_05")
    up.removal_interval = 2
    u = capi.Updater(up, ep, m, device=0)
    for k in range(17):
        u.process_node(k, sc.pose7(k), sc.scan(k, seed_offset=3, **kw))
    est = u.save_static_map(0.2)
    u.close()
    d = ev.evaluate(m, est)
    assert ev.last_counts()["ambiguous_ties"] == 0
    assert d == E.evaluate(m, est)


def test_run_sequence_scores_on_the_device(ev):
    """pipeline.run_sequence with the device updater scores through capi.Evaluator: the same call on its output has no
    ambiguous tie, gives run_sequence's dict and equals the host evaluator"""
    from erasor_b200 import pipeline
    from test_mapgen import _nodes
    nodes = _nodes(n_nodes=12, seed=7)
    ep, up = P.preset("seq_05"), P.updater_preset("seq_05")
    up.removal_interval = 2
    up.map_voxel_size = 0.2
    res = pipeline.run_sequence(nodes, up, ep)
    d = ev.evaluate(res["naive_map"], res["static_map"], voxelsize=0.2)
    assert ev.last_counts()["ambiguous_ties"] == 0
    assert d == res["quality"] == E.evaluate(res["naive_map"], res["static_map"], voxelsize=0.2)


# ---- per point, on the adversarial sets -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(ADV))
def test_adversarial_sets_equal_the_model(ev, name):
    gt, est, keep, vs = ADV[name]
    c = _check_against_model(ev, gt, est, keep, vs)
    assert c["inliers"] > 0


# ---- input handling ------------------------------------------------------------------------------------------------------------
def test_keep_masks(ev):
    gt, est, _, _ = ADV["10km"]
    rng = np.random.default_rng(3)
    for keep in (np.zeros(len(est), np.uint8), np.ones(len(est), np.uint8), (rng.random(len(est)) < 0.5).astype(np.uint8),
                 (rng.integers(0, 256, len(est))).astype(np.uint8)):
        _check_against_model(ev, gt, est, keep)
    assert ev.evaluate(gt, est, keep=np.zeros(len(est), np.uint8)) == E.rates(*(model_eval(gt, est[:0])[0][x] for x in KEYS4))


def test_empty_clouds(ev):
    gt, est, _, _ = ADV["ties"]
    c = _check_against_model(ev, gt, est[:0])
    assert c["inliers"] == 0 and c["gt_static"] + c["gt_dynamic"] == len(gt)
    c = _check_against_model(ev, gt[:0], est)
    assert all(v == 0 for v in c.values())
    c = _check_against_model(ev, gt[:0], est[:0])
    assert all(v == 0 for v in c.values())


@pytest.mark.parametrize("which", ["gt", "est"])
def test_non_finite_coordinates_are_rejected(ev, which):
    gt, est, _, _ = ADV["ties"]
    gt, est = gt.copy(), est.copy()
    (gt if which == "gt" else est)[7, 1] = np.nan
    with pytest.raises(capi.ErasorError) as ei:
        ev.evaluate(gt, est)
    assert ei.value.code == capi.E_INVALID and "non-finite" in str(ei.value)
    if which == "est":                                   # a dropped point may be anything
        keep = np.ones(len(est), np.uint8)
        keep[7] = 0
        _check_against_model(ev, gt, est, keep)
    # the handle stays usable
    _check_against_model(ev, *ADV["ties"][:2])


def test_one_handle_serves_growing_and_shrinking_sizes(ev):
    names = ["labels", "10km", "ties", "far", "10km", "thr_ulps", "cell_faces", "labels"]
    rng = np.random.default_rng(9)
    big = rng.uniform(-30, 30, (300000, 4)).astype(np.float32)
    big[:, 3] = rng.choice([40.0, 252.0], len(big))
    calls = [(ADV[n][0], ADV[n][1], ADV[n][2], ADV[n][3]) for n in names]
    calls.insert(3, (big[:50000], big, None, 0.2))
    calls.insert(6, (big[:1000], big[:2000], None, 0.2))
    for gt, est, keep, vs in calls:
        d = ev.evaluate(gt, est, keep, vs, want_match=True)
        c = ev.last_counts()
        with capi.Evaluator() as fresh:
            assert fresh.evaluate(gt, est, keep, vs, want_match=True) == d
            f = fresh.last_counts()
        assert np.array_equal(c.pop("match"), f.pop("match")) and c == f


# ---- a 20 M-point cloud -----------------------------------------------------------------------------------------------------
def test_20m_point_cloud(ev):
    import torch
    from scipy.spatial import cKDTree
    n, n_sub = 20_000_000, 200_000
    g = torch.Generator(device="cuda").manual_seed(20)
    est = torch.rand((n, 4), device="cuda", generator=g)
    est[:, :3] = est[:, :3] * torch.tensor([400.0, 400.0, 8.0], device="cuda") - torch.tensor([200.0, 200.0, 4.0], device="cuda")
    est[:, 3] = torch.where(est[:, 3] < 0.2, 252.0, 40.0)
    torch.cuda.synchronize()                             # the evaluator runs on a stream of its own
    # size-independent: the cloud against itself -- every point is its own nearest point
    d_self = ev.evaluate_ptr(est.data_ptr(), n, est.data_ptr(), n, 0, 0.2, capi.PTR_DEVICE)
    c = ev.last_counts()
    assert c["inliers"] == n and c["gt_static"] + c["gt_dynamic"] == n and c["ambiguous_ties"] == 0
    assert d_self["PR"] == 100.0 and d_self["RR"] == 0.0
    # a seeded 200 k GT subset, jittered, scored as a separate call
    host = est.cpu().numpy()
    rng = np.random.default_rng(20)
    gt = host[rng.choice(n, n_sub, replace=False)].copy()
    gt[:, :3] += rng.normal(0, 0.1, (n_sub, 3)).astype(np.float32)
    gt[:, 3] = rng.choice([40.0, 252.0], n_sub)
    gt_d = _dev(gt)
    m = torch.empty(n_sub, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ev.evaluate_ptr(gt_d.data_ptr(), n_sub, est.data_ptr(), n, 0, 0.2, capi.PTR_DEVICE, m.data_ptr())
    got = ev.last_counts()
    match = m.cpu().numpy().view(np.uint32)
    want, want_m = model_eval(gt, host)
    assert got == want
    assert np.array_equal(match, want_m)
    assert 0.2 * n_sub < want["inliers"] < 0.9 * n_sub
    # the match against a kd-tree radius query resolved to the lowest index among the equally nearest
    thr = thr_of(0.2)
    tree = cKDTree(host[:, :3].astype(np.float64))
    cand = tree.query_ball_point(gt[:, :3].astype(np.float64), r=thr * (1 + 1e-9))
    ref = np.full(n_sub, NO_MATCH, dtype=np.uint32)
    for i, js in enumerate(cand):
        if not js:
            continue
        js = np.sort(np.asarray(js))
        d2 = sq_dist(gt[i][None, :], host[js])
        b = d2.min()
        if np.sqrt(b) < thr:
            ref[i] = js[np.argmax(d2 == b)]
    assert np.array_equal(match, ref)
