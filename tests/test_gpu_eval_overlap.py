"""The device overlap report (capi.Evaluator.overlap / report, erasor_eval_overlap) against sklearn's kneighbors distances
(erasor_b200.evaluate), numpy's percentiles, the numpy model of tests/test_eval_overlap_model.py and the reference script's stdout."""
import os
import subprocess
import sys

import numpy as np
import pytest

from erasor_b200 import capi
from erasor_b200 import evaluate as E
from test_eval_grid_model import seed41_pass, sq_dist
from test_eval_overlap_model import GOLDEN_STDOUT, OSETS, ROOT, brute_overlap, jittered_estimate, model_overlap, write_pair

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ev():
    e = capi.Evaluator(device=0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def golden_pairs(oracle_mod):
    gt, est = seed41_pass(oracle_mod)
    return {"seed41": (gt, est), "seed41_jittered": (gt, jittered_estimate(est))}


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def sklearn_dist(gt, est, keep=None):
    sel = np.ones(len(est), bool) if keep is None else np.asarray(keep).astype(bool)
    d = np.full(len(est), np.nan)
    if sel.any():
        d[sel] = E.overlap_distances(gt, est[sel])
    return d


def check(ev, gt, est, keep=None, vs=0.2, want=None):
    """host and device pointers give the same distances, equal to `want` (default: sklearn's), and the same dict, equal to
    evaluate.overlap on the selected points; the order statistics and counts agree with the distances.  Returns the counts."""
    import torch
    gt, est = np.asarray(gt, np.float32), np.asarray(est, np.float32)
    if want is None:
        want = sklearn_dist(gt, est, keep)
    r, d = ev.overlap(gt, est, keep, vs, want_dist=True)
    c = ev.last_overlap()
    assert np.array_equal(d, want, equal_nan=True)
    sel = ~np.isnan(want)
    assert c["n"] == sel.sum()
    s_, d_ = E.est_counts(est[sel])
    assert (c["est_static"], c["est_dynamic"]) == (s_, d_)
    ds = want[sel]
    if len(ds):
        host = E.overlap(gt, est[sel], vs)
        assert r == host
        assert c["max"] == ds.max()
        srt = np.sort(ds)
        ranks = E.overlap_ranks(len(ds))
        assert r == E.overlap_from_ranks(len(ds), srt[ranks], srt[-1], tuple(int((ds < t).sum()) for t in (0.5 * vs, vs, 2 * vs)), vs)
    # device pointers, with the distances written to device memory
    g, e = _dev(gt.reshape(-1, 4)), _dev(est.reshape(-1, 4))
    k = _dev(np.asarray(keep).astype(np.uint8)) if keep is not None else None
    dd = torch.empty(len(est), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    r2 = ev.overlap_ptr(g.data_ptr() if len(gt) else 0, len(gt), e.data_ptr() if len(est) else 0, len(est),
                        k.data_ptr() if k is not None and len(k) else 0, vs, capi.PTR_DEVICE, dd.data_ptr() if len(est) else 0)
    assert r2 == r and ev.last_overlap() == c
    assert np.array_equal(dd.cpu().numpy(), want, equal_nan=True)
    return c


# ---- real clouds ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(GOLDEN_STDOUT))
def test_golden_pairs_equal_sklearn(ev, golden_pairs, name):
    gt, est = golden_pairs[name]
    c = check(ev, gt, est)
    assert (c["far_points"] > 0) == (name == "seed41_jittered")
    keep = (np.random.default_rng(4).random(len(est)) < 0.7).astype(np.uint8)
    check(ev, gt, est, keep)


@pytest.mark.parametrize("shift", [50.0, 5000.0])
def test_misaligned_clouds_take_the_far_path(ev, golden_pairs, shift):
    gt, est = golden_pairs["seed41"]
    moved = est.copy()
    moved[:, 0] += np.float32(shift)
    moved[:, 2] += np.float32(shift / 10)
    c = check(ev, gt, moved)
    assert c["far_points"] > 0.5 * len(est)


def test_node_mode_map_scored_in_place(ev):
    import bench
    p, map_world, poses, qs = bench.load_workload("seq05", 0, 1, 20)
    gm = capi.Map(map_world, device=0)
    h = capi.Handle(p, device=0)
    h.attach_map(gm)
    keep, _ = h.process_nodes(poses, np.concatenate(qs), np.cumsum([0] + [len(q) for q in qs]).astype(np.uint64))
    r = ev.overlap_map(gm)
    c = ev.last_overlap()
    assert r == E.overlap(map_world, map_world[keep.astype(bool)]) and c["n"] == keep.sum()
    assert r == ev.overlap(map_world, map_world, keep=keep)
    rep = ev.report_map(gm)
    assert rep == E.report(map_world, map_world[keep.astype(bool)])
    check(ev, map_world, map_world, keep)
    h.close()
    gm.close()


def test_sequential_updater_static_map(ev):
    from erasor_b200 import params as P
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
    check(ev, m, est)
    assert ev.report(m, est) == E.report(m, est)


# ---- adversarial sets, per point, also against the model -------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(OSETS))
def test_adversarial_sets(ev, name):
    gt, est, keep, vs = OSETS[name]
    want = brute_overlap(gt, est, keep)
    c = check(ev, gt, est, keep, vs, want)
    d, far = model_overlap(gt, est, keep, vs)
    assert np.array_equal(d, want, equal_nan=True) and c["far_points"] == far.sum()


# ---- the report and the CLI ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(GOLDEN_STDOUT))
def test_report_and_cli_reproduce_the_runner(ev, tmp_path, golden_pairs, name):
    write_pair(tmp_path, *golden_pairs[name])
    gt, est = E.read_pcd_ascii(str(tmp_path / "gt.pcd")), E.read_pcd_ascii(str(tmp_path / "est.pcd"))
    r = ev.report(gt, est)
    assert r == E.report(gt, est)
    golden = open(GOLDEN_STDOUT[name]).read()
    assert E.format_report(r, 0.2, "gt.pcd", "est.pcd") == golden
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    out = subprocess.run([sys.executable, "-m", "erasor_b200.analysis", "--gt", "gt.pcd", "--est", "est.pcd"], cwd=tmp_path, env=env,
                         check=True, capture_output=True, text=True).stdout
    assert out == golden


# ---- input handling ---------------------------------------------------------------------------------------------------------------------
def test_empty_inputs(ev):
    gt, est, _, _ = OSETS["subset_dups"]
    assert ev.overlap(gt, est[:0]) is None and ev.last_overlap()["n"] == 0
    assert ev.overlap(gt, est, keep=np.zeros(len(est), np.uint8)) is None and ev.last_overlap()["n"] == 0
    r, d = ev.overlap(gt[:0], est, want_dist=True)
    assert np.all(np.isinf(d)) and ev.last_overlap()["n"] == len(est) and r["max"] == np.inf and r["frac_two"] == 0.0
    assert ev.overlap(gt[:0], est[:0]) is None


def test_invalid_inputs(ev):
    gt, est, _, _ = OSETS["subset_dups"]
    for which in ("gt", "est"):
        g, e = gt.copy(), est.copy()
        (g if which == "gt" else e)[7, 1] = np.nan
        with pytest.raises(capi.ErasorError) as ei:
            ev.overlap(g, e)
        assert ei.value.code == capi.E_INVALID and "non-finite" in str(ei.value)
    keep = np.ones(len(est), np.uint8)
    keep[7] = 0
    e = est.copy()
    e[7, 1] = np.inf
    check(ev, gt, e, keep)                               # a dropped point may be anything
    with pytest.raises(capi.ErasorError):
        ev.overlap(gt, est, voxelsize=0.0)
    # a rank at n is invalid
    o = capi.EvalOverlapC()
    ranks = np.array([0, len(est)], np.uint64)
    vals = np.empty(2)
    g, e = capi._cloud(gt), capi._cloud(est)
    rc = ev.L.erasor_eval_overlap(ev.h, g.ctypes.data, len(g), e.ctypes.data, len(e), None, 0.2, capi.PTR_HOST, ranks.ctypes.data, 2,
                                  vals.ctypes.data, None, o)
    assert rc == capi.E_INVALID
    check(ev, gt, est)                                   # the handle stays usable


def test_handle_reuse_and_interleaving_with_evaluate(ev, golden_pairs):
    names = ["far_octants", "subset_dups", "10km_extent", "single_gt", "cell_faces", "far_octants"]
    gt41, est41 = golden_pairs["seed41"]
    for i, n in enumerate(names):
        gt, est, keep, vs = OSETS[n]
        want = ev.evaluate(gt, est, keep, vs)
        check(ev, gt, est, keep, vs, brute_overlap(gt, est, keep))
        assert ev.evaluate(gt, est, keep, vs) == want
        if i == 2:
            check(ev, gt41, est41)
            assert ev.evaluate(gt41, est41) == E.evaluate(gt41, est41)


# ---- a 20 M-point GT -----------------------------------------------------------------------------------------------------------------
def test_20m_point_gt(ev):
    import torch
    from scipy.spatial import cKDTree
    n, n_sub = 20_000_000, 200_000
    g = torch.Generator(device="cuda").manual_seed(21)
    gt = torch.rand((n, 4), device="cuda", generator=g)
    gt[:, :3] = gt[:, :3] * torch.tensor([400.0, 400.0, 8.0], device="cuda") - torch.tensor([200.0, 200.0, 4.0], device="cuda")
    gt[:, 3] = torch.where(gt[:, 3] < 0.2, 252.0, 40.0)
    host = gt.cpu().numpy()
    rng = np.random.default_rng(21)
    est = host[rng.choice(n, n_sub, replace=False)].copy()
    est[:, :3] += rng.normal(0, 0.5, (n_sub, 3)).astype(np.float32)
    est[:1000, :3] += np.float32(300.0)                  # a few far away
    e = _dev(est)
    dd = torch.empty(n_sub, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    r = ev.overlap_ptr(gt.data_ptr(), n, e.data_ptr(), n_sub, 0, 0.2, capi.PTR_DEVICE, dd.data_ptr())
    c = ev.last_overlap()
    d = dd.cpu().numpy()
    tree = cKDTree(host[:, :3].astype(np.float64))
    _, idx = tree.query(est[:, :3].astype(np.float64))
    want = np.sqrt(sq_dist(est, host[idx]))
    assert np.array_equal(d, want)
    assert c["far_points"] >= 1000
    srt = np.sort(d)
    assert r == E.overlap_from_ranks(n_sub, srt[E.overlap_ranks(n_sub)], srt[-1], tuple(int((d < t).sum()) for t in (0.1, 0.2, 0.4)))
    assert r["median"] == float(np.median(d)) and r["p99"] == float(np.percentile(d, 99))
