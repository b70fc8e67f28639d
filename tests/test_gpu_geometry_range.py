"""Every mode across the legal polar-geometry range, against the oracle bit for bit and the float64 reference's bin candidates.

erasor_create takes any 1 <= R * S <= 65534 whose K1 tables fit the device's shared memory; the code that depends on the geometry
is tested here at its edges: one ring or one sector (sector tables that are always / never true for one y branch, odd S), R > S
(the Scan Ratio Test's neighbour wrap by num_rings lands out of range and is fenced), S slightly above R (the wrap lands on a wrong
but valid sector, as the reference does), 720 rings or sectors, both sides of K1's 8 / 32-warp switch at 56 KB of tables
(1 x 4777: exactly 57 344 bytes), tiny and huge max_range, a height window with no float32 inside it, and the largest grid node
mode's K1 can launch.  An empty height window (min_h >= max_h) is refused with ERASOR_E_INVALID, by erasor_create and by tune.  Every geometry's scenes hold flagged bins of every R-GPF size class and MERGE bins whose neighbour across
the sector wrap is CURR_HIGH, and run through cloud mode (v2 and v3), process_frames, process_nodes (identity and a rotated
far-from-origin pose, with and without inserts), the tune path and, at three geometries, the sequential updater.

Node mode's K1 keeps a 32 KB VoI ring in static shared memory, so it reaches fewer bins than erasor_create admits: between the
two limits node mode, sweeps and tune must refuse with ERASOR_E_UNSUPPORTED before enqueuing anything, and leave the handle and
the thread's other handles working."""
import math

import numpy as np
import pytest

import bin_cases as BC
import node_inserts_model as NI
from erasor_b200 import params as P
from test_erasor_float64_reference import _assert_bins, edge_points, polar, xy_in_bin

pytestmark = pytest.mark.gpu

F32 = np.float32
BASE = P.preset("seq_05").replace(skip_voxelize=1)
LIMIT_R = 100                                         # the ring count at which the shared-memory limits are found
GEOMETRIES = [
    ("1x1", dict(num_rings=1, num_sectors=1)),
    ("1x2", dict(num_rings=1, num_sectors=2)),
    ("2x1", dict(num_rings=2, num_sectors=1)),
    ("1x3", dict(num_rings=1, num_sectors=3)),
    ("3x3", dict(num_rings=3, num_sectors=3)),
    ("15x2", dict(num_rings=15, num_sectors=2)),      # R > S: the wrapped neighbour index is out of range
    ("40x3", dict(num_rings=40, num_sectors=3)),
    ("7x5", dict(num_rings=7, num_sectors=5)),
    ("7x9", dict(num_rings=7, num_sectors=9)),        # S slightly above R: the wrap lands on a wrong but valid sector
    ("12x13", dict(num_rings=12, num_sectors=13)),
    ("1x720", dict(num_rings=1, num_sectors=720)),
    ("720x1", dict(num_rings=720, num_sectors=1)),
    ("1x4777", dict(num_rings=1, num_sectors=4777)),  # 57 344 bytes of K1 tables: the 8-warp kernel
    ("1x4778", dict(num_rings=1, num_sectors=4778)),  # 16 bytes more: the 32-warp kernel
    ("range0.5", dict(max_range=0.5, num_rings=4, num_sectors=12)),
    ("range5000", dict(max_range=5000.0, num_rings=20, num_sectors=30)),
    ("z_one_ulp", dict(min_h=0.5, max_h=float(np.nextafter(F32(0.5), F32(1))))),   # no float32 strictly inside the window
    ("largest", None),                                # LIMIT_R x the most sectors node mode's K1 launches (node_limit)
]
IDS = [g[0] for g in GEOMETRIES]
RGPF_SIZES = (60, 200, 300, 700, 1500, 2600)          # R-GPF's size classes: networks to 128 / 256 / 512, radix, class B, class C
MERGE, CURR_HIGH = 0.25, 1.0


def k1_table_bytes(R, S):
    """kernels.cu k1_smem_bytes: ring thresholds + count / min / max tables"""
    return 8 * ((R + 2) & ~1) + 4 * ((R * S + 1) + 2 * R * S)


@pytest.fixture(scope="module")
def capi():
    from erasor_b200 import capi as C
    return C


def _refused(capi, fn):
    """True when fn() raises ERASOR_E_UNSUPPORTED, False when it runs; any other error fails the test"""
    try:
        fn()
        return False
    except capi.ErasorError as e:
        assert e.code == capi.E_UNSUPPORTED, str(e)
        return True


def _tiny_map():
    rng = np.random.default_rng(2)
    n = 3000
    r, t = 50 * np.sqrt(rng.random(n)), rng.uniform(-np.pi, np.pi, n)
    return np.stack([r * np.cos(t), r * np.sin(t), rng.uniform(-1.0, 2.0, n), np.ones(n)], 1).astype(F32)


I7 = np.array([[0, 0, 0, 0, 0, 0, 1.0]])


@pytest.fixture(scope="module")
def limits(capi):
    """(S_node, S_create): at LIMIT_R rings the most sectors node mode runs, and the most erasor_create accepts"""
    m = _tiny_map()
    gm = capi.Map(m)
    qo = np.array([0, 500], np.uint64)

    def node_runs(S):
        try:
            h = capi.Handle(BASE.replace(num_rings=LIMIT_R, num_sectors=S))
        except capi.ErasorError as e:
            assert e.code == capi.E_UNSUPPORTED, str(e)
            return False
        h.attach_map(gm)
        ok = not _refused(capi, lambda: h.process_nodes(I7, m[:500], qo))
        h.close()
        return ok

    def creates(S):
        return not _refused(capi, lambda: capi.Handle(BASE.replace(num_rings=LIMIT_R, num_sectors=S)).close())

    def last_true(f, lo, hi):          # f(lo) true, f(hi) false
        assert f(lo) and not f(hi)
        while hi - lo > 1:
            mid = (lo + hi) // 2
            lo, hi = (mid, hi) if f(mid) else (lo, mid)
        return lo

    s_create = last_true(creates, 100, 300)
    s_node = last_true(node_runs, 100, s_create + 1)
    gm.close()
    import torch
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    # create's limit: the opt-in less a few bytes at most; node mode's: less the 32 KB VoI ring (and the node's pose)
    assert k1_table_bytes(LIMIT_R, s_create) <= optin < k1_table_bytes(LIMIT_R, s_create + 1) + 1024
    assert k1_table_bytes(LIMIT_R, s_node) <= optin - 32768 < k1_table_bytes(LIMIT_R, s_node + 1) + 1024
    print(f"H100 opt-in {optin} B: at {LIMIT_R} rings erasor_create takes {s_create} sectors, node mode {s_node}")
    return s_node, s_create


@pytest.fixture(scope="module", params=GEOMETRIES, ids=IDS)
def geo(request, limits):
    tag, kw = request.param
    if kw is None:
        kw = dict(num_rings=LIMIT_R, num_sectors=limits[0])
    return tag, BASE.replace(**kw)


# ---- scenes ----------------------------------------------------------------------------------------------------------------------
def _pad(xyz, i):
    return np.concatenate([np.asarray(xyz, np.float64), np.full((len(xyz), 1), i)], 1).astype(F32)


def _zg(p):
    return BASE.min_h + 0.4          # seq_05's heights: a geometry whose window holds no float32 bins none of the scene


def _column(p, ring, sector, n, z0, z1, rng):
    x, y = xy_in_bin(p, ring, sector, n, rng)
    z = rng.uniform(z0, z1, n)
    z[0], z[-1] = z0, z1
    return np.stack([x, y, z], 1)


def _rgpf(p, ring, sector, n, rng):
    """one bin the Scan Ratio Test hands to R-GPF: ground within +-3 cm, objects 0.65 m and more above it, a flat low query"""
    zg = _zg(p)
    n_obj = max(2, n // 8)
    g = _column(p, ring, sector, n - n_obj, zg - 0.03, zg + 0.03, rng)
    o = _column(p, ring, sector, n_obj, zg + 0.65, zg + 2.0, rng)
    q = _column(p, ring, sector, max(40, p.minimum_num_pts), zg - 0.02, zg + 0.02, rng)
    return _pad(np.concatenate([g, o]), 40.0), _pad(q, 7.0)


def scene_frames(p, seed=7):
    """[(map, query)] of the geometry: R-GPF bins of every size class (as many per frame as there are bins), then a frame with a
    MERGE bin in sector 0 next to CURR_HIGH bins in sector S - 1 (its true neighbour, which the reference only reaches through
    its wrap by num_rings when S = R) and in sector R - 1 (the bin the wrap reaches when R - 1 < S)"""
    rng = np.random.default_rng(seed)
    R, S, B = p.num_rings, p.num_sectors, p.num_bins
    frames = []
    per = min(B, len(RGPF_SIZES))
    for f0 in range(0, len(RGPF_SIZES), per):
        sizes = RGPF_SIZES[f0:f0 + per]
        bins = [(k * B) // len(sizes) for k in range(len(sizes))]
        parts = [_rgpf(p, b % R, b // R, n, rng) for b, n in zip(bins, sizes)]
        frames.append((rng.permutation(np.concatenate([a for a, _ in parts])), rng.permutation(np.concatenate([b for _, b in parts]))))
    if B >= 2:
        zg, r = _zg(p), R // 2
        ms = [_column(p, r, 0, 60, zg, zg + 1.0, rng)]
        qs = [_column(p, r, 0, 40, zg, zg + 0.9, rng)]
        for sec in sorted({S - 1, R - 1} - {0}):
            if sec < S:
                ms.append(_column(p, r, sec, 30, zg, zg + 0.05, rng))
                qs.append(_column(p, r, sec, 60, zg, zg + 1.5, rng))
        frames.append((rng.permutation(_pad(np.concatenate(ms), 11.0)), rng.permutation(_pad(np.concatenate(qs), 3.0))))
    return frames


def _frames_of(p):
    """the scene frames, then one frame of edge points (every ring radius, sector angle, the gates, the truncated-PI sliver)"""
    e = edge_points(p)
    return scene_frames(p) + [(e, e[::3].copy())]


# ---- oracle comparisons ----------------------------------------------------------------------------------------------------------
def _bits(a):
    return np.ascontiguousarray(a, dtype=F32).view(np.uint32)


def _oracle_keep(o, n):
    _, rej = o.cloud(o.MAP_REJECTED)
    k = np.ones(n, dtype=np.uint8)
    k[rej] = 0
    return k


def cloud_equal(capi, oracle_mod, p, m, q, tag):
    """cloud mode, v3 and v2: bins, tables, status, planes, masks and the four clouds equal the oracle's; bins inside the float64
    reference's candidates"""
    for version in (3, 2):
        pv = p.replace(version=version)
        o = oracle_mod.Oracle(pv)
        o.run(m, q)
        h = capi.Handle(pv)
        h.set_inputs(m, q)
        h.compare(version)
        for which, pts in ((0, m), (1, q)):
            bop, mn, mx, cnt = h.get_bins(which)
            assert np.array_equal(bop, o.bin_of_point(which)), (tag, version, which, int((bop != o.bin_of_point(which)).sum()))
            _assert_bins(bop, polar(p, pts)[1], (tag, which))
            omn, omx, ocnt, _ = o.bins(which)
            occ = ocnt > 0
            assert np.array_equal(cnt, ocnt), (tag, version, which)
            assert np.array_equal(mn[occ].astype(np.float64), omn[occ]) and np.array_equal(mx[occ].astype(np.float64), omx[occ]), (tag, which)
        st, _ = o.status()
        assert np.array_equal(h.get_status(), st.astype(F32)), (tag, version, "status")
        gp, op = h.get_planes(), o.planes()
        assert [g["bin"] for g in gp] == [x["bin"] for x in op], (tag, version, "flagged bins")
        for g, x in zip(gp, op):
            assert (g["n_points"], g["n_seeds"], g["lpr"]) == (x["n_points"], x["n_seeds"], x["lpr"]), (tag, g["bin"])
            assert np.array_equal(g["normal_d"], x["normal_d"]) and np.array_equal(g["n_ground"], x["n_ground"]), (tag, g["bin"])
        keep, gnd = h.get_static_mask()
        assert np.array_equal(keep, _oracle_keep(o, len(m))), (tag, version, "keep")
        arr, cmp_ = h.get_static_estimate()
        mr, cr = h.get_outliers()
        for got, which in ((arr, o.ARRANGED), (cmp_, o.COMPLEMENT), (mr, o.MAP_REJECTED), (cr, o.CURR_REJECTED)):
            ref, _ = o.cloud(which)
            assert got.shape == ref.shape and np.array_equal(_bits(got), _bits(ref)), (tag, version, which)
        h.close()
        o.close()
    return st


def node_reference(oracle_mod, p, map_world, poses, qs):
    out = []
    for pose, q in zip(poses, qs):
        voi, idx = oracle_mod.fetch_voi(map_world, pose, p.max_range)
        o = oracle_mod.Oracle(p)
        o.run(voi, q)
        _, rej = o.cloud(o.MAP_REJECTED)
        k = np.ones(len(map_world), dtype=np.uint8)
        k[idx[rej]] = 0
        out.append(k)
        o.close()
    return np.stack(out)


def _far_pose(p):
    """a rotated pose far from the origin and more than two VoI radii from it"""
    t = 4.0 * p.max_range + 1000.0
    yaw = 0.7315
    return np.array([t, -0.5 * t, 0.0, 0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2)])


def _to_world(oracle_mod, m, pose):
    return oracle_mod.transform(m, oracle_mod.pose_to_matrix(pose))


def _offsets(qs):
    return np.cumsum([0] + [len(q) for q in qs]).astype(np.uint64)


def node_scene(oracle_mod, p):
    """(map_world, poses, queries): the scene frames' maps around the origin and again around a far rotated pose; one node at
    the identity pose and one at the far pose per scene frame"""
    frames = scene_frames(p)
    local = np.concatenate([m for m, _ in frames])
    far = _far_pose(p)
    map_world = np.concatenate([local, _to_world(oracle_mod, local, far)])
    poses, qs = [], []
    for _, q in frames:
        poses += [I7[0], far]
        qs += [q, q]
    return map_world, np.stack(poses), qs


# ---- tests -------------------------------------------------------------------------------------------------------------------------
def test_cloud_mode(capi, oracle_mod, geo):
    tag, p = geo
    sts = [cloud_equal(capi, oracle_mod, p, m, q, (tag, f)) for f, (m, q) in enumerate(_frames_of(p))]
    binned = p.min_h < p.max_h and np.nextafter(F32(p.min_h), F32(np.inf)) < F32(p.max_h)
    if binned:
        # the scene does what it is built for: flagged bins of every size class, and a MERGE bin beside a CURR_HIGH one
        h = capi.Handle(p)
        sizes = []
        for m, q in scene_frames(p):
            h.set_inputs(m, q)
            h.compare(3)
            sizes += [pl["n_points"] for pl in h.get_planes()]
        h.close()
        assert sorted(sizes) == sorted(RGPF_SIZES), (tag, sizes)
        if p.num_sectors >= 2:
            assert (sts[-2] == CURR_HIGH).any() and ((sts[-2] == MERGE) | (sts[-2] == 0.8)).any(), tag


def test_process_frames(capi, oracle_mod, geo):
    tag, p = geo
    frames = _frames_of(p)
    h = capi.Handle(p)
    mo, qo = _offsets([m for m, _ in frames]), _offsets([q for _, q in frames])
    keep = h.process_frames(np.concatenate([m for m, _ in frames]), mo, np.concatenate([q for _, q in frames]), qo)
    for f, (m, q) in enumerate(frames):
        o = oracle_mod.Oracle(p)
        o.run(m, q)
        assert np.array_equal(keep[int(mo[f]):int(mo[f + 1])], _oracle_keep(o, len(m))), (tag, f)
        o.close()
    h.close()


def test_process_nodes(capi, oracle_mod, geo):
    tag, p = geo
    map_world, poses, qs = node_scene(oracle_mod, p)
    ref = node_reference(oracle_mod, p, map_world, poses, qs)
    gm = capi.Map(map_world)
    h = capi.Handle(p)
    h.attach_map(gm)
    keep, fk = h.process_nodes(poses, np.concatenate(qs), _offsets(qs), want_frame_keep=True)
    for f in range(len(qs)):
        assert np.array_equal(fk[f], ref[f]), (tag, f, int((fk[f] != ref[f]).sum()))
    assert np.array_equal(keep, ref.min(axis=0))
    # with inserts: every node's inserted points, bit for bit and in order, against the oracle model
    ins_ref, off_ref, fk_ref = NI.node_inserts(oracle_mod, p, map_world, poses, qs)
    h.set_node_inserts(True)
    gm.reset_keep()
    _, fk2 = h.process_nodes(poses, np.concatenate(qs), _offsets(qs), want_frame_keep=True)
    ins, off = h.node_inserts()
    assert np.array_equal(off, off_ref), (tag, off, off_ref)
    assert np.array_equal(_bits(ins), _bits(ins_ref)), tag
    assert np.array_equal(fk2, fk_ref) and np.array_equal(fk2, ref)
    h.close()
    gm.close()


def test_tune_takes_the_geometry(capi, oracle_mod, geo):
    """the geometry as one tune setting next to the handle's own: each mask equals a plain call with that geometry"""
    import torch
    tag, p = geo
    map_world, poses, qs = node_scene(oracle_mod, p)
    voi = max(p.max_range, BASE.max_range)
    Q, qo = np.concatenate(qs), _offsets(qs)
    n = len(map_world)
    plain = []
    for pp in (BASE, p):
        gm = capi.Map(map_world)
        h = capi.Handle(pp)
        h.attach_map(gm)
        plain.append(h.process_nodes(poses, Q, qo, voi_max_range=voi)[0])
        h.close()
        gm.close()
    own = {f: getattr(BASE, f) for f in capi.GEOMETRY_SWEEP_FIELDS}
    setting = {f: getattr(p, f) for f in capi.GEOMETRY_SWEEP_FIELDS}
    gm = capi.Map(map_world)
    h = capi.Handle(BASE)
    h.attach_map(gm)
    keep = torch.empty(2 * n, dtype=torch.uint8, device="cuda")
    for settings, want in (([own, setting], plain), ([setting, own], plain[::-1])):
        h.reset_keep_mask(keep.data_ptr(), 2 * n)
        h.process_nodes_tune(poses, Q, qo, settings, keep.data_ptr(), voi_max_range=voi)
        got = keep.reshape(2, n).cpu().numpy()
        for v in range(2):
            assert np.array_equal(got[v], want[v]), (tag, settings[v], int((got[v] != want[v]).sum()))
    h.close()
    gm.close()


@pytest.mark.parametrize("which", ["1x1", "3x3", "largest"])
def test_sequential_updater(capi, oracle_mod, limits, which):
    from erasor_b200 import synth
    kw = dict(GEOMETRIES)[which] or dict(num_rings=LIMIT_R, num_sectors=limits[0])
    ep = P.preset("seq_05").replace(**kw)
    up = P.updater_preset("seq_05")
    up.removal_interval = 2
    sc = synth.Scene(seed=31, length=30.0, n_nodes=7, n_dynamic=4)
    scan_kw = dict(n_beams=16, n_az=360)
    nodes = list(range(7))
    initial = sc.build_map(nodes, voxel=0.2, **scan_kw)
    o = oracle_mod.OracleUpdater(up, ep, initial)
    u = capi.Updater(up, ep, initial)
    for k in nodes:
        scan = sc.scan(k, seed_offset=5, **scan_kw)
        a = o.callback_node(k, sc.pose7(k), scan)
        assert a == u.process_node(k, sc.pose7(k), scan)
        if a:
            for c in ("MAP_REJECTED", "MAP_ARRANGED"):
                got, ref = u.cloud(getattr(u, c)), o.cloud(getattr(o, c))[0]
                assert got.shape == ref.shape and np.array_equal(_bits(got), _bits(ref)), (which, k, c)
    got, ref = u.save_static_map(0.2), o.save_static_map(0.2)
    assert got.shape == ref.shape and np.array_equal(_bits(got), _bits(ref)), which
    u.close()
    o.close()


def test_largest_geometry_windows_and_sub_batches(capi, oracle_mod, limits):
    """At the largest grid node mode launches: a frame flagging more bins than one slot window of node mode's SRT + scatter holds,
    and more frames than one submission's records take (kMaxRecords / B), so that the call is split into sub-batches"""
    p = BASE.replace(num_rings=LIMIT_R, num_sectors=limits[0])
    B = p.num_bins
    W = BC.k2_window(B, node=True)
    m, q, pick = BC.fill_flagged(p, W + 5, seed=3)
    assert len(pick) > W
    n_frames = (1 << 21) // B + 2
    assert n_frames > (1 << 21) // B
    rng = np.random.default_rng(8)
    poses, qs = [], []
    for f in range(n_frames):                 # every node a small yaw and shift of the frame, so that frames differ
        yaw = 0.002 * f
        poses.append([0.01 * (f % 7), 0.0, 0.0, 0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2)])
        qs.append(q if f % 4 == 0 else q[rng.permutation(len(q))[:len(q) // 2]])
    poses = np.array(poses)
    ref = node_reference(oracle_mod, p, m, poses, qs)
    gm = capi.Map(m)
    h = capi.Handle(p)
    h.attach_map(gm)
    keep, fk = h.process_nodes(poses, np.concatenate(qs), _offsets(qs), want_frame_keep=True)
    nv, nf, nr = h.node_stats()
    assert nf[0] > W, (int(nf[0]), W)
    for f in range(n_frames):
        assert np.array_equal(fk[f], ref[f]), (f, int((fk[f] != ref[f]).sum()))
    assert np.array_equal(keep, ref.min(axis=0))
    h.close()
    gm.close()


def test_shared_memory_limit(capi, oracle_mod, limits):
    """Between create's limit and node mode's (100 x 180) and past create's: every mode runs the geometry equal to the oracle, or
    refuses it with ERASOR_E_UNSUPPORTED; after a refusal the handle runs a plain call and another handle of the thread runs."""
    import torch
    s_node, s_create = limits
    assert s_node < 180 <= s_create, limits
    m = _tiny_map()
    q = m[::4].copy()
    qo = np.array([0, len(q)], np.uint64)
    n = len(m)
    other = capi.Handle(BASE)
    gm = capi.Map(m)
    other.attach_map(gm)
    other_ref = other.process_nodes(I7, q, qo)[0]

    def others_still_run(h, p):
        if h is not None:                                      # the refusing handle: a plain call
            h.set_inputs(m, q)
            h.compare(3)
            o = oracle_mod.Oracle(p)
            o.run(m, q)
            assert np.array_equal(h.get_static_mask()[0], _oracle_keep(o, n))
            o.close()
        gm.reset_keep()
        assert np.array_equal(other.process_nodes(I7, q, qo)[0], other_ref)

    p = BASE.replace(num_rings=LIMIT_R, num_sectors=180)
    cloud_equal(capi, oracle_mod, p, m, q, "100x180")
    h = capi.Handle(p)
    kf = h.process_frames(m, np.array([0, n], np.uint64), q, qo)
    o = oracle_mod.Oracle(p)
    o.run(m, q)
    assert np.array_equal(kf, _oracle_keep(o, n))
    o.close()
    gm2 = capi.Map(m)
    h.attach_map(gm2)
    keep = torch.empty(2 * n, dtype=torch.uint8, device="cuda")
    geo = {f: getattr(p, f) for f in capi.GEOMETRY_SWEEP_FIELDS}
    calls = [
        ("process_nodes", lambda: h.process_nodes(I7, q, qo)),
        ("process_nodes (again)", lambda: h.process_nodes(I7, q, qo)),
        ("process_nodes_sweep", lambda: h.process_nodes_sweep(I7, q, qo, [dict(), dict(scan_ratio_threshold=0.2)], keep.data_ptr())),
        ("process_nodes_tune", lambda: h.process_nodes_tune(I7, q, qo, [geo, dict(geo, scan_ratio_threshold=0.2)], keep.data_ptr())),
    ]
    for name, call in calls:
        assert _refused(capi, call), name
        others_still_run(h, p)
    # the handle's tune with the 100 x 180 grid as one setting, and the first grid past erasor_create's limit
    t = capi.Handle(BASE)
    t.attach_map(gm2)
    for S in (180, s_create + 1):
        g = dict(geo, num_sectors=S)
        assert _refused(capi, lambda: t.process_nodes_tune(I7, q, qo, [dict(), g], keep.data_ptr(), voi_max_range=BASE.max_range)), S
        others_still_run(t, BASE)
    assert _refused(capi, lambda: capi.Handle(BASE.replace(num_rings=LIMIT_R, num_sectors=s_create + 1)))
    others_still_run(None, None)
    # at node mode's own limit the node call runs and equals the oracle
    p = BASE.replace(num_rings=LIMIT_R, num_sectors=s_node)
    h2 = capi.Handle(p)
    h2.attach_map(gm2)
    gm2.reset_keep()
    assert np.array_equal(h2.process_nodes(I7, q, qo)[0], node_reference(oracle_mod, p, m, I7, [q])[0])
    for x in (h, h2, t, other):
        x.close()
    gm.close()
    gm2.close()


def test_empty_height_window_is_refused(capi):
    """min_h >= max_h: erasor_create and a tune setting refuse it (ERASOR_E_INVALID), and the tuning handle runs on"""
    import torch
    m = _tiny_map()
    q = m[::4].copy()
    qo = np.array([0, len(q)], np.uint64)
    for lo, hi in ((0.5, 0.5), (1.0, -1.0)):
        with pytest.raises(capi.ErasorError) as e:
            capi.Handle(BASE.replace(min_h=lo, max_h=hi))
        assert e.value.code == capi.E_INVALID
    gm = capi.Map(m)
    h = capi.Handle(BASE)
    h.attach_map(gm)
    ref = h.process_nodes(I7, q, qo)[0]
    keep = torch.empty(2 * len(m), dtype=torch.uint8, device="cuda")
    with pytest.raises(capi.ErasorError) as e:
        h.process_nodes_tune(I7, q, qo, [dict(), dict(min_h=0.5, max_h=0.5)], keep.data_ptr(), voi_max_range=BASE.max_range)
    assert e.value.code == capi.E_INVALID
    gm.reset_keep()
    assert np.array_equal(h.process_nodes(I7, q, qo)[0], ref)
    h.close()
    gm.close()
