"""CPU: the boundary shells of tests/pose_cases.py cover what they claim at every pose, and the oracle's cut predicates --
fetch_VoI's radius, set_submap's square, mapgen's 2.7 m body cut -- decide them exactly as the reference's double expressions,
ties excluded and non-finite coordinates included.  The host pose arithmetic of the node mode (pose_math.h, through the host
build) equals the oracle's at every pose, -q and scaled quaternions included."""
import ctypes
import os

import numpy as np
import pytest

import pose_cases as pc
from erasor_b200 import params as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTCHECK = os.path.join(ROOT, "erasor_b200", "_lib", "liberasor_b200_hostcheck.so")
POSE_IDS = [n for n, _ in pc.POSES]


def _shell_at(pose, r, oracle_mod, nonfinite=False, seed=0):
    px, py = pc.criterion(pose, oracle_mod)
    xy, cls = pc.shell(px, py, r, seed=seed, nonfinite=nonfinite)
    return px, py, xy, cls


def test_pose_list_covers_the_data_like_cases():
    P7 = np.stack([p for _, p in pc.POSES])
    qn = np.linalg.norm(P7[:, 3:], axis=1)
    assert {0.5, 1.0, 2.0} <= set(np.round(qn, 12))
    assert (P7[:, 6] < 0).any() and (P7[:, 5] < 0).any() and (np.abs(P7[:, 5]) == np.abs(qn)).any()   # qw < 0, qz < 0, |qz| == |q|
    assert np.abs(P7[:, :2]).max() == 20000 and np.abs(P7[:, 2]).max() == 50
    tilt = np.abs(np.arcsin(np.clip(2 * (P7[:, 6] * P7[:, 4] - P7[:, 5] * P7[:, 3]) / qn ** 2, -1, 1)))
    assert 0 < np.rad2deg(tilt).max() <= 5.01
    assert any("30 deg" in n for n, _ in pc.POSES)


@pytest.mark.parametrize("pose", [p for _, p in pc.POSES], ids=POSE_IDS)
def test_shells_cover_every_class(oracle_mod, pose):
    for r in pc.RADII:
        px, py, xy, cls = _shell_at(pose, r, oracle_mod)
        truth = pc.voi_truth(xy[:, 0], xy[:, 1], px, py, r)
        assert truth.any() and (~truth).any(), f"r={r}: both sides of the limit"
        tie = cls == pc.TIE
        assert tie.sum() >= 1, f"r={r}: no exact tie"
        d2 = (xy[tie, 0].astype(np.float64) - px) ** 2 + (xy[tie, 1].astype(np.float64) - py) ** 2
        assert np.all(d2 == r * r) and not truth[tie].any(), f"r={r}: a tie is inside"
        lo, hi = pc.band(r)
        v = pc.d2f(xy[:, 0], xy[:, 1], px, py)
        assert int(((v >= lo) & (v <= hi)).sum()) >= 100, f"r={r}: fewer than 100 points in the float band"
        # the walk crosses the limit at the ulp scale: its points fall on both sides
        w = truth[cls == pc.WALK]
        assert w.any() and (~w).any()


@pytest.mark.parametrize("pose", [p for _, p in pc.POSES], ids=POSE_IDS)
def test_oracle_fetch_voi_is_the_double_expression(oracle_mod, pose):
    rng = np.random.default_rng(7)
    for r in pc.RADII:
        px, py, xy, _ = _shell_at(pose, r, oracle_mod, nonfinite=True)
        fill = np.stack([px + rng.uniform(-2 * r, 2 * r, 500), py + rng.uniform(-2 * r, 2 * r, 500)], 1).astype(np.float32)
        xy = np.concatenate([xy, fill])
        cloud = pc.with_z(xy, rng)
        _, idx = oracle_mod.fetch_voi(cloud, pose, r)
        expect = np.flatnonzero(pc.voi_truth(xy[:, 0], xy[:, 1], px, py, r)).astype(np.uint32)
        assert np.array_equal(idx, expect), f"r={r}: {len(idx)} vs {len(expect)}"


def _submap_complement(oracle_mod, pose, submap_size, cloud):
    """set_submap through the oracle's caller loop: the first large-scale node splits the initial map into the submap and its
    complement around the node; the complement is untouched by the rest of the node."""
    ep = P.preset("seq_05").replace(skip_voxelize=1)
    up = P.updater_preset("seq_05")
    up.is_large_scale, up.submap_size, up.removal_interval = True, submap_size, 1
    rng = np.random.default_rng(3)
    scan = pc.with_z(rng.uniform(-20, 20, (200, 2)).astype(np.float32), rng, -1.8, 1.0)
    o = oracle_mod.OracleUpdater(up, ep, cloud)
    assert o.callback_node(0, pose, scan)
    _, src = o.cloud(o.SUBMAP_COMPLEMENT)
    o.close()
    return src


@pytest.mark.parametrize("pose", [p for _, p in pc.POSES[::3]], ids=POSE_IDS[::3])
def test_oracle_set_submap_is_the_double_expression(oracle_mod, pose):
    rng = np.random.default_rng(11)
    cx, cy = pc.criterion(pose, oracle_mod)
    for s in (0.5, 9.5, 80.0):
        xy = pc.square_shell(cx, cy, s, seed=5, nonfinite=True)
        fill = np.stack([cx + rng.uniform(-2 * s, 2 * s, 300), cy + rng.uniform(-2 * s, 2 * s, 300)], 1).astype(np.float32)
        xy = np.concatenate([xy, fill])
        inside = pc.submap_truth(xy[:, 0], xy[:, 1], cx, cy, s)
        assert inside.any() and (~inside).any()
        # exact ties on the edges are outside (strict <)
        on_edge = (np.abs(xy[:, 0].astype(np.float64) - cx) == s) & (np.abs(xy[:, 1].astype(np.float64) - cy) < s)
        assert on_edge.any() and not inside[on_edge].any()
        src = _submap_complement(oracle_mod, pose, s, pc.with_z(xy, rng))
        assert np.array_equal(src, np.flatnonzero(~inside).astype(np.uint32)), f"s={s}"


def test_oracle_body_cut_is_the_double_expression(oracle_mod):
    """mapgen's body cut on shells around 2.7 m: every point gets its own z (0.5 m apart), so each kept point is alone in its
    0.2 m voxel and cloud_curr holds exactly the kept points, lifted by 1.73 m."""
    xy = pc.body_cut_shell(seed=4)
    kept = pc.body_cut_kept(xy[:, 0], xy[:, 1])
    assert kept.any() and (~kept).any()
    # points straddling the float limit: the double distance of some is within one float ulp of it on either side
    d2 = xy[:, 0].astype(np.float64) ** 2 + xy[:, 1].astype(np.float64) ** 2
    lim = float(pc.F32(pc.BODY_CUT ** 2))
    assert ((d2 < lim) & (d2 > lim * (1 - 1e-7))).any() and ((d2 >= lim) & (d2 < lim * (1 + 1e-7))).any()
    cloud = np.zeros((len(xy), 4), dtype=np.float32)
    cloud[:, :2] = xy
    cloud[:, 2] = 0.5 * np.arange(len(xy))
    cloud[:, 3] = 1.0
    g = oracle_mod.OracleMapGen(0.2, False)
    g.accum(np.array([0, 0, 0, 0, 0, 0, 1.0]), cloud)
    curr = g.cloud(g.CLOUD_CURR)
    g.close()
    lifted_z = (cloud[:, 2] + np.float32(1.73)).astype(np.float32)
    got = np.zeros(len(xy), dtype=bool)
    pos = np.searchsorted(lifted_z, curr[:, 2])
    assert np.array_equal(lifted_z[pos], curr[:, 2])
    got[pos] = True
    assert np.array_equal(curr[:, :2].view(np.uint32), cloud[pos, :2].view(np.uint32))
    assert np.array_equal(got, kept), f"{int((got != kept).sum())} points decided differently"


def test_host_node_pose_is_the_oracles_at_every_pose(oracle_mod):
    L = ctypes.CDLL(HOSTCHECK)
    for name, odom in pc.POSES:
        odom = np.ascontiguousarray(odom, dtype=np.float64)
        for r in pc.RADII:
            ppl = np.zeros(3); T12 = np.zeros(12, dtype=np.float32); g4 = np.zeros(4, dtype=np.float32)
            assert L.erasor_hostcheck_node_pose(odom.ctypes.data_as(ctypes.c_void_p), ctypes.c_double(r), ppl.ctypes.data_as(ctypes.c_void_p),
                                                T12.ctypes.data_as(ctypes.c_void_p), g4.ctypes.data_as(ctypes.c_void_p)) == 0
            T = oracle_mod.pose_to_matrix(odom)
            Tinv = oracle_mod.invert4(T)
            assert np.array_equal(T12.view(np.uint32), Tinv[:3].reshape(-1).view(np.uint32)), name
            assert ppl[0] == float(T[0, 3]) and ppl[1] == float(T[1, 3]) and ppl[2] == r * r, name
            assert g4[0] == T[0, 3] and g4[1] == T[1, 3], name
            lo, hi = pc.band(r)                                  # the generators aim at the band the device uses
            assert g4[2] == lo and g4[3] == hi, name
        # -q and 0.5 q / 2 q give the same matrix as q (geoPose2eigen divides by |q|^2; the products are exact scalings)
        base = np.concatenate([odom[:3], odom[3:] / np.linalg.norm(odom[3:])])
        Tb = oracle_mod.pose_to_matrix(base)
        assert np.allclose(oracle_mod.pose_to_matrix(odom), Tb, rtol=0, atol=1e-6 * max(1.0, np.abs(odom[:3]).max())), name
