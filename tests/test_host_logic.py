"""CPU suite: host-side logic of the product -- exact binning thresholds (binning.h compiled for the host),
parameter / yaml mirror, and that the C-ABI library loads and exports every symbol the header declares."""
import ctypes
import os
import re

import numpy as np
import pytest

from erasor_b200 import params as P
from erasor_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTCHECK = os.path.join(ROOT, "erasor_b200", "_lib", "liberasor_b200_hostcheck.so")


def _host_bins(p, pts):
    L = ctypes.CDLL(HOSTCHECK)
    pc = p.to_c()
    n = len(pts)
    bins = np.empty(n, np.int32)
    st = np.zeros(3, np.uint64)
    qe, eps = ctypes.c_double(), ctypes.c_double()
    rc = L.erasor_hostcheck_bin_points(ctypes.byref(pc), pts.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(n),
                                       bins.ctypes.data_as(ctypes.c_void_p), st.ctypes.data_as(ctypes.c_void_p),
                                       ctypes.byref(qe), ctypes.byref(eps))
    assert rc == 0
    return bins, st, qe.value, eps.value


# the edges of the legal geometry range (seq_05 otherwise): one ring or sector, 19 000 of either, a grid past node mode's K1
# limit, a tiny and a huge max_range, a height window with no float32 inside it
GEOMETRY_EDGES = {
    "1x1": dict(num_rings=1, num_sectors=1), "1x2": dict(num_rings=1, num_sectors=2), "2x1": dict(num_rings=2, num_sectors=1),
    "3x3": dict(num_rings=3, num_sectors=3), "7x9": dict(num_rings=7, num_sectors=9), "1x19000": dict(num_rings=1, num_sectors=19000),
    "19000x1": dict(num_rings=19000, num_sectors=1), "120x160": dict(num_rings=120, num_sectors=160),
    "range0.5": dict(max_range=0.5), "range5000": dict(max_range=5000.0, num_rings=20),
    "z_one_ulp": dict(min_h=0.0, max_h=float(np.nextafter(np.float32(0), np.float32(1)))),
}


@pytest.mark.parametrize("name", list(P.PRESETS) + list(GEOMETRY_EDGES))
def test_exact_thresholds_match_oracle(oracle_mod, name):
    from test_erasor_float64_reference import pi_sliver
    p = (P.preset(name) if name in P.PRESETS else P.preset("seq_05").replace(**GEOMETRY_EDGES[name])).replace(skip_voxelize=1)
    pts = synth.adversarial_points(p, n_random=400000, seed=21)
    s = pi_sliver()
    z = np.float32(0.5 * (p.min_h + p.max_h))
    pts = np.concatenate([pts, np.stack([s[:, 0], s[:, 1], np.full(len(s), z), np.ones(len(s))], 1).astype(np.float32)])
    b, st, qerr, eps = _host_bins(p, pts)
    o = oracle_mod.Oracle(p)
    o.run(pts, pts[:0])
    assert np.array_equal(b, o.bin_of_point(0))
    assert st[1] == 0, "ambiguous sector decisions"
    if name in P.PRESETS:
        assert st[2] > 0, "the adversarial set must exercise the exact sector path"
    assert qerr < 0.5 * eps, f"float sector coordinate error {qerr} too close to the guard band {eps}"


def test_threshold_tables_are_tight(oracle_mod):
    """ring_thr[k] is the first double s with ring(s) >= k; s_max the last with r <= max_r."""
    L = ctypes.CDLL(HOSTCHECK)
    p = P.preset("seq_00")
    pc = p.to_c()
    thr = np.zeros(p.num_rings + 1)
    smax, zlo, zhi, sop = ctypes.c_double(), ctypes.c_float(), ctypes.c_float(), ctypes.c_int()
    assert L.erasor_hostcheck_tables(ctypes.byref(pc), thr.ctypes.data_as(ctypes.c_void_p), ctypes.byref(smax), ctypes.byref(zlo),
                                     ctypes.byref(zhi), ctypes.byref(sop)) == 0
    ring_size = p.max_range / p.num_rings
    for k in range(1, p.num_rings):
        s = thr[k]
        assert int(np.sqrt(s) / ring_size) >= k and int(np.sqrt(np.nextafter(s, -np.inf)) / ring_size) < k
    assert np.sqrt(smax.value) <= p.max_range < np.sqrt(np.nextafter(smax.value, np.inf))
    assert np.float64(zhi.value) >= p.max_h > np.float64(np.nextafter(np.float32(zhi.value), np.float32(-np.inf)))
    assert np.float64(zlo.value) <= p.min_h < np.float64(np.nextafter(np.float32(zlo.value), np.float32(np.inf)))
    assert sop.value == min(int(np.arctan2(0.0, -1.0) / (2 * 3.1415926535 / p.num_sectors)), p.num_sectors - 1)


@pytest.mark.parametrize("name", ["seq_05", "seq_00", "synthetic_40x360"])
def test_float_guard_bands_never_contradict_the_exact_thresholds(name):
    """K1's fast path decides ring and range from sf = float(x^2 + y^2) against thresholds widened by the float error (binning_tables.cpp).
    On points packed around every ring boundary and around max_range: whenever the float test is sure, the exact double test agrees."""
    p = P.preset(name)
    L = ctypes.CDLL(HOSTCHECK)
    pc = p.to_c()
    R = p.num_rings
    thr = np.zeros(R + 1); smax = ctypes.c_double(); zlo = ctypes.c_float(); zhi = ctypes.c_float(); sop = ctypes.c_int()
    assert L.erasor_hostcheck_tables(ctypes.byref(pc), thr.ctypes.data_as(ctypes.c_void_p), ctypes.byref(smax), ctypes.byref(zlo), ctypes.byref(zhi), ctypes.byref(sop)) == 0
    guard = np.zeros(2 * (R + 1), dtype=np.float32); sm = np.zeros(2, dtype=np.float32)
    assert L.erasor_hostcheck_guards(ctypes.byref(pc), guard.ctypes.data_as(ctypes.c_void_p), sm.ctypes.data_as(ctypes.c_void_p)) == 0
    up, dn = guard[0::2], guard[1::2]
    rng = np.random.default_rng(3)
    bounds = list(thr[1:R]) + [smax.value]
    n_sure = 0
    for T in bounds:
        r = np.sqrt(T) * (1.0 + rng.uniform(-3e-6, 3e-6, 200000))
        th = rng.uniform(0, 2 * np.pi, r.size)
        x, y = (r * np.cos(th)).astype(np.float32), (r * np.sin(th)).astype(np.float32)
        s = x.astype(np.float64) ** 2 + y.astype(np.float64) ** 2                     # exact: 24-bit mantissas squared, one rounding
        for sf in ((y * y + x * x).astype(np.float32), np.float32(1) * (x * x + y * y)):   # two float evaluation orders (fma differs by < 1 ulp more)
            if T == smax.value:
                assert np.all(s[sf <= sm[0]] <= T) and np.all(s[sf > sm[1]] > T)
                n_sure += int((sf <= sm[0]).sum() + (sf > sm[1]).sum())
            else:
                k = bounds.index(T) + 1
                assert np.all(s[sf >= up[k]] >= T) and np.all(s[sf < dn[k]] < T)
                n_sure += int((sf >= up[k]).sum() + (sf < dn[k]).sum())
    assert n_sure > 0.5 * 2 * 200000 * len(bounds)          # the bands are narrow: most of even these adversarial points are decided in float
    assert up[0] == -np.inf and dn[R] == np.inf


def test_node_pose_matches_the_oracle(oracle_mod):
    """Host side of erasor_process_nodes (pose_math.h): the origin -> body rows, the criterion point and the squared radius are the
    oracle's (geoPose2eigen -> float 4x4 -> cofactor inverse, OfflineMapUpdater.cpp:219,246-247,434), bit for bit; the float guard
    band of the radius pre-test brackets the limit."""
    L = ctypes.CDLL(HOSTCHECK)
    rng = np.random.default_rng(9)
    for _ in range(200):
        q = rng.normal(size=4); q /= np.linalg.norm(q)
        odom = np.concatenate([rng.normal(0, 300, 3), q])
        rng_m = float(rng.choice([9.5, 20.0, 60.0, 80.0]))
        ppl = np.zeros(3); T12 = np.zeros(12, dtype=np.float32); g4 = np.zeros(4, dtype=np.float32)
        assert L.erasor_hostcheck_node_pose(odom.ctypes.data_as(ctypes.c_void_p), ctypes.c_double(rng_m), ppl.ctypes.data_as(ctypes.c_void_p),
                                            T12.ctypes.data_as(ctypes.c_void_p), g4.ctypes.data_as(ctypes.c_void_p)) == 0
        T = oracle_mod.pose_to_matrix(odom)
        Tinv = oracle_mod.invert4(T)
        assert np.array_equal(T12.view(np.uint32), Tinv[:3].reshape(-1).view(np.uint32))
        assert ppl[0] == float(T[0, 3]) and ppl[1] == float(T[1, 3]) and ppl[2] == rng_m ** 2
        assert g4[0] == T[0, 3] and g4[1] == T[1, 3]
        assert float(g4[2]) < ppl[2] < float(g4[3]) and (float(g4[3]) - float(g4[2])) / ppl[2] < 2.5e-6


def test_capi_exports_every_declared_symbol():
    from erasor_b200 import capi
    hdr = open(os.path.join(ROOT, "include", "erasor_b200.h")).read()
    declared = set(re.findall(r"\b(erasor_[a-z_0-9]+)\s*\(", hdr))
    declared.discard("erasor_ctx")
    assert declared == set(capi.EXPORTS), declared ^ set(capi.EXPORTS)
    L = ctypes.CDLL(capi.LIB_PATH)          # loads without a GPU (no compute call is made)
    for s in sorted(declared):
        assert hasattr(L, s), s
    assert L.erasor_abi_version() == 2


def test_create_fails_loudly_without_cuda():
    from erasor_b200 import capi
    from conftest import has_cuda
    if has_cuda():
        pytest.skip("a CUDA device is present")
    with pytest.raises(capi.ErasorError) as e:
        capi.Handle(P.preset("seq_05"))
    assert e.value.code == capi.E_CUDA and "no CPU path" in str(e.value)


REFERENCE_STYLE_YAML = """
idx: 450
erasor:
    max_range: 80.0
    num_rings: 20
    num_sectors: 108
    min_h: -1.3
    max_h: 3.0
    th_bin_max_h: 0.2
    scan_ratio_threshold: 0.2
    minimum_num_pts: 6
    rejection_ratio: 0
    gf_dist_thr: 0.25
    gf_iter: 3
    gf_num_lpr: 20
    gf_th_seeds_height: 0.5
    map_voxel_size: 0.2
    version: 3
MapUpdater:
    data_name: "00"
    initial_map_path: "/x/y.pcd"
    env: "outdoor"
    save_path: "/x/out"
    query_voxel_size: 0.2
    map_voxel_size: 0.2
    voxelization_interval: 2
    removal_interval: 4
tf:
     lidar2body: [0.0, 0.0, 1.73, 0, 0.0, 0.0, 1.0]
verbose: true
"""


def test_reference_yaml_keys(tmp_path):
    f = tmp_path / "large_scale_05.yaml"
    f.write_text(REFERENCE_STYLE_YAML)
    ep, up = P.load_yaml(str(f))
    assert (ep.max_range, ep.num_rings, ep.num_sectors, ep.gf_num_lpr, ep.gf_dist_thr) == (80.0, 20, 108, 20, 0.25)
    assert ep.num_lowest_pts == 5 and ep.version == 3                      # defaults of erasor.h:54 / OfflineMapUpdater.cpp:81
    assert (up.removal_interval, up.query_voxel_size, up.data_name, up.max_range) == (4, 0.2, "00", 80.0)
    assert up.lidar2body == [0.0, 0.0, 1.73, 0.0, 0.0, 0.0, 1.0]
    for name in P.PRESETS:
        assert P.preset(name).num_bins <= 65534
