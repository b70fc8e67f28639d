"""GPU: the pose-driven device paths against the oracle, bit for bit, at poses like a real sequence's and exactly on their cuts.

- node mode (erasor_process_nodes, fetch_VoI fused into K1) on small_workload moved rigidly far from the origin, with a
  full-circle yaw, a tilt and -q; map points crafted so that their body-frame y is exactly 0 (K1's exact path), queries with
  y == -0.0 (the fence);
- node mode on maps made of the boundary shells of tests/pose_cases.py, at lengths that put them at warp-row, unroll-group
  and chunk tails, for several VoI radii;
- node mode's sub-batch split: by the flagged-bin records cap and by the scratch budget (ERASOR_B200_NODE_SCRATCH_GB);
- the sequential updater and mapgen at far, tilted poses, with shells on the submap square and the 2.7 m body cut."""
import numpy as np
import pytest

import pose_cases as pc
from erasor_b200 import params as P
from erasor_b200 import synth

pytestmark = pytest.mark.gpu
D = np.deg2rad
G_FAR = pc.pose7([20000.0, -4000.0, 30.0], pc.quat_rpy(0.0, 0.0, np.pi - 0.01))     # node yaws of +-0.03 cross +-pi
G_TILT = pc.pose7([300.0, 4000.0, -50.0], pc.quat_rpy(D(4), D(-3), -1.9))
G_NEGQ = pc.pose7([-4000.0, 20000.0, 10.0], pc.quat_rpy(0.0, 0.0, np.pi / 2))
TRANSFORMS = {"far": (G_FAR, 1.0), "tilt": (G_TILT, 0.5), "negq": (G_NEGQ, -1.0)}


@pytest.fixture(scope="module")
def capi():
    from erasor_b200 import capi as C
    return C


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _body_y(Tinv, x, y, z):
    """Row 1 of PCL's float affine, the order the device and the oracle evaluate it in (no contraction)."""
    t = Tinv.astype(np.float32)
    return ((t[1, 0] * x + t[1, 1] * y) + t[1, 2] * z) + t[1, 3]


def _y_zero_points(pose, oracle_mod, rng, n=24, reach=40.0, span=64):
    """World points that land exactly on the body frame's x axis (y == 0: sector boundary, K1's exact path)."""
    T = oracle_mod.pose_to_matrix(pose)
    Tinv = oracle_mod.invert4(T)
    ks = np.arange(-span, span + 1)
    out = []
    for _ in range(n):
        body = np.array([rng.uniform(-reach, reach), 0.0, rng.uniform(-1.0, 1.5), 1.0])
        w = (T.astype(np.float64) @ body).astype(np.float32)
        gx = pc.ulp_step(np.full(len(ks), w[0]), ks)
        gy = pc.ulp_step(np.full(len(ks), w[1]), ks)
        X, Y = np.meshgrid(gx, gy, indexing="ij")
        by = _body_y(Tinv, X, Y, np.float32(w[2]))
        hit = np.argwhere(by == 0)
        if len(hit):
            i, j = hit[len(hit) // 2]
            out.append([X[i, j], Y[i, j], w[2], 40.0])
    return np.array(out, dtype=np.float32).reshape(-1, 4)


def _oracle_nodes(oracle_mod, p, map_world, poses, qs, voi_range):
    """fetch_VoI + ERASOR per node: per-frame masks over the map, (|VoI|, flagged bins, rejected) per node, the negzero
    fence count, and the number of VoI points whose body-frame y is exactly 0."""
    n = len(map_world)
    o = oracle_mod.Oracle(p)
    fk, stats, negzero, yzero = [], [], 0, 0
    for pose, q in zip(poses, qs):
        voi, idx = oracle_mod.fetch_voi(map_world, pose, voi_range)
        o.run(voi, q)
        _, rej = o.cloud(o.MAP_REJECTED)
        k = np.ones(n, dtype=np.uint8)
        k[idx[rej]] = 0
        fk.append(k)
        stats.append((len(voi), len(o.planes()), len(rej)))
        negzero += o.negzero_fenced()
        yzero += int((voi[:, 1] == 0).sum())
    o.close()
    return np.stack(fk), np.array(stats, dtype=np.int64), negzero, yzero


def _offsets(qs):
    return np.cumsum([0] + [len(q) for q in qs]).astype(np.uint64)


@pytest.fixture(scope="module")
def far_scenes(small_workload, oracle_mod):
    """small_workload re-placed by each transform, plus exact body-y == 0 points per node; queries with y == -0.0 points."""
    scene = small_workload["scene"]
    poses0 = [scene.pose7(f[2]) for f in small_workload["frames"]]
    negz = np.array([[-7.5, -0.0, 0.3, 40.0], [-12.25, -0.0, -0.9, 40.0]], dtype=np.float32)
    qs = [np.concatenate([f[1], negz]) for f in small_workload["frames"]]
    out = {}
    rng = np.random.default_rng(71)
    for name, (G, qscale) in TRANSFORMS.items():
        moved, poses = pc.replace(small_workload["map_world"], poses0, G, oracle_mod, qscale)
        ties = np.concatenate([_y_zero_points(p, oracle_mod, rng) for p in poses])
        assert len(ties) >= 3 * len(poses)
        out[name] = dict(map=np.concatenate([moved, ties]), poses=poses, qs=qs)
    return out


@pytest.mark.parametrize("G", list(TRANSFORMS))
@pytest.mark.parametrize("name,version", [("seq_05", 3), ("seq_05", 2), ("seq_00", 3), ("synthetic_40x360", 3)])
def test_node_mode_at_far_poses(capi, oracle_mod, far_scenes, name, version, G):
    p = P.preset(name).replace(skip_voxelize=1, version=version)
    sc = far_scenes[G]
    mw, poses, qs = sc["map"], sc["poses"], sc["qs"]
    ofk, ost, negzero, yzero = _oracle_nodes(oracle_mod, p, mw, poses, qs, p.max_range)
    assert (ofk == 0).any(), "the moved workload must reject something"
    assert yzero > 0 and negzero > 0, "the case must reach K1's exact path and the negzero fence"
    m = capi.Map(mw)
    h = capi.Handle(p)
    h.attach_map(m)
    keep, fk = h.process_nodes(poses, np.concatenate(qs), _offsets(qs), want_frame_keep=True)
    bad = np.flatnonzero((fk != ofk).any(axis=1))
    assert len(bad) == 0, f"{name} v{version} {G}: frames {bad.tolist()} differ in {np.count_nonzero(fk != ofk)} points"
    assert np.array_equal(keep, ofk.min(axis=0))
    nv, nf, nr = h.node_stats()
    assert np.array_equal(nv, ost[:, 0]) and np.array_equal(nf, ost[:, 1]) and np.array_equal(nr, ost[:, 2])
    assert h.fence_counts()["negzero_points"] == negzero
    h.close()
    # one-node calls: the per-bin tables of both clouds
    o = oracle_mod.Oracle(p)
    for f in (0, 3):
        h = capi.Handle(p)
        h.attach_map(m)
        h.process_nodes(poses[f:f + 1], qs[f], _offsets(qs[f:f + 1]))
        voi, _ = oracle_mod.fetch_voi(mw, poses[f], p.max_range)
        o.run(voi, qs[f])
        for which in (0, 1):
            _, mn, mx, cnt = h.get_bins(which, per_point=False)
            omn, omx, ocnt, _ = o.bins(which)
            assert np.array_equal(cnt, ocnt), f"node {f} cloud {which}: counts differ in {np.count_nonzero(cnt != ocnt)} bins"
            occ = ocnt > 0
            assert np.array_equal(mn[occ].astype(np.float64), omn[occ]) and np.array_equal(mx[occ].astype(np.float64), omx[occ])
        assert h.fence_counts()["negzero_points"] == o.negzero_fenced()
        h.close()
    o.close()
    m.close()


# ---- node mode on the VoI boundary -------------------------------------------------------------------------------------------
BOUNDARY_PRESET = "seq_05"


def _chunk_size(p):
    """choose_chunk's size for a batch far below one wave of CTAs: max(2048, 5 B) rounded up to 128 points."""
    return (max(2048, 5 * p.num_rings * p.num_sectors) + 127) // 128 * 128


@pytest.fixture(scope="module")
def boundary_nodes(small_workload, oracle_mod):
    """Three nodes: a far one with a near-pi yaw, a tilted one with -q, and one near the origin with qz = 1, qw = 0 (so the
    map's zero padding past its end would sit inside every VoI)."""
    scene = small_workload["scene"]
    f = small_workload["frames"]
    pa = pc.compose(G_FAR, scene.pose7(f[0][2]))
    pb = pc.compose(G_TILT, scene.pose7(f[2][2]))
    pb[3:] *= -1.0
    pcn = pc.pose7([0.5, -0.25, 0.0], [0.0, 0.0, 1.0, 0.0])
    qs = [f[0][1][::2], f[2][1][::2], f[4][1][::2]]
    return np.stack([pa, pb, pcn]), qs


def _boundary_map(poses, r, length, oracle_mod, seed):
    """length points: the shells of every node at radius r (non-finite coordinates included) interleaved with a random fill;
    shell points sit at the warp-row, unroll-group and chunk positions and at the tail."""
    rng = np.random.default_rng(seed)
    shells = []
    for i, pose in enumerate(poses):
        px, py = pc.criterion(pose, oracle_mod)
        xy, _ = pc.shell(px, py, r, seed=seed + i, nonfinite=True)
        shells.append(xy)
    pool = np.concatenate(shells)
    pool = pool[rng.permutation(len(pool))]
    centres = np.array([pc.criterion(p, oracle_mod) for p in poses])
    fill_c = centres[rng.integers(0, len(poses), length)]
    rad = r * np.sqrt(rng.uniform(0.0, 2.0, length))
    th = rng.uniform(-np.pi, np.pi, length)
    fill = np.stack([fill_c[:, 0] + rad * np.cos(th), fill_c[:, 1] + rad * np.sin(th)], 1).astype(np.float32)
    use_shell = (np.arange(length) % 3 != 2)
    special = [i for i in (0, 30, 31, 32, 33, 63, 64, 126, 127, 128, length - 2, length - 1) if 0 <= i < length]
    use_shell[special] = True
    xy = fill.copy()
    xy[use_shell] = np.resize(pool, (int(use_shell.sum()), 2))
    return pc.with_z(xy, rng, -1.2, 2.8, 40.0)


@pytest.mark.parametrize("voi", [0.0, 0.5, 9.5, 1.0e4])
def test_node_mode_on_the_voi_boundary(capi, oracle_mod, boundary_nodes, voi):
    p = P.preset(BOUNDARY_PRESET).replace(skip_voxelize=1)
    poses, qs = boundary_nodes
    r = voi if voi > 0 else p.max_range
    ch = _chunk_size(p)
    n_band = 0
    for length in (1, 31, 32, 33, 127, 128, 129, ch - 1, ch, ch + 1):
        mw = _boundary_map(poses, r, length, oracle_mod, seed=length)
        ofk, ost, _, _ = _oracle_nodes(oracle_mod, p, mw, poses, qs, r)
        for pose in poses:
            px, py = pc.criterion(pose, oracle_mod)
            lo, hi = pc.band(r)
            v = pc.d2f(mw[:, 0], mw[:, 1], px, py)
            n_band += int(((v >= lo) & (v <= hi)).sum())
        m = capi.Map(mw)
        h = capi.Handle(p)
        h.attach_map(m)
        keep, fk = h.process_nodes(poses, np.concatenate(qs), _offsets(qs), voi_max_range=voi, want_frame_keep=True)
        nv, _, _ = h.node_stats()
        assert np.array_equal(nv, ost[:, 0]), f"r={r} n={length}: VoI sizes {nv.tolist()} vs {ost[:, 0].tolist()}"
        assert np.array_equal(fk, ofk), f"r={r} n={length}: masks differ in {np.count_nonzero(fk != ofk)} points"
        assert np.array_equal(keep, ofk.min(axis=0))
        h.close(); m.close()
    assert n_band >= 100


# ---- node mode's sub-batch split -------------------------------------------------------------------------------------------
def _many_nodes(small_workload, oracle_mod, n_nodes, G=G_FAR):
    scene = small_workload["scene"]
    base = [scene.pose7(f[2]) for f in small_workload["frames"]]
    poses = []
    for j in range(n_nodes):
        d = pc.pose7([0.9 * j, -0.35 * j, 0.0], pc.quat_rpy(0.0, 0.0, 0.013 * j))
        poses.append(pc.compose(G, pc.compose(d, base[j % len(base)])))
    qs = [small_workload["frames"][j % len(base)][1] for j in range(n_nodes)]
    return np.stack(poses), qs


def test_node_sub_batch_split_by_records_cap(capi, oracle_mod, small_workload):
    """150 nodes on 40 x 360 bins: the records cap (2^21 / 14400 = 145 frames) splits the call in two.  Every node's mask and
    counters equal the oracle's over the whole call, and keep_out is the AND of all nodes -- host buffers synchronously,
    device buffers asynchronously."""
    import torch
    p = P.preset("synthetic_40x360").replace(skip_voxelize=1)
    assert (1 << 21) // (p.num_rings * p.num_sectors) == 145
    mw = oracle_mod.transform(small_workload["map_world"], oracle_mod.pose_to_matrix(G_FAR))
    poses, qs = _many_nodes(small_workload, oracle_mod, 150)
    ofk, ost, _, _ = _oracle_nodes(oracle_mod, p, mw, poses, qs, p.max_range)
    assert (ofk[:145] == 0).any() and (ofk[145:] == 0).any()
    Q, qo = np.concatenate(qs), _offsets(qs)
    m = capi.Map(mw)
    h = capi.Handle(p)
    h.attach_map(m)
    keep, fk = h.process_nodes(poses, Q, qo, want_frame_keep=True)
    bad = np.flatnonzero((fk != ofk).any(axis=1))
    assert len(bad) == 0, f"nodes {bad.tolist()} differ"
    assert np.array_equal(keep, ofk.min(axis=0))
    nv, nf, nr = h.node_stats()
    for k, (got, col) in enumerate(((nv, 0), (nf, 1), (nr, 2))):
        wrong = np.flatnonzero(got != ost[:, col])
        assert len(wrong) == 0, f"counter {k}: nodes {wrong.tolist()[:10]} differ"
    # device buffers, asynchronous
    m.reset_keep()
    dev = torch.device("cuda", 0)
    dQ = torch.from_numpy(Q).to(dev)
    dfk = torch.zeros((len(qs), len(mw)), dtype=torch.uint8, device=dev)
    dkeep = torch.zeros(len(mw), dtype=torch.uint8, device=dev)
    P7 = np.ascontiguousarray(poses, dtype=np.float64)
    h.process_nodes_ptr(P7, dQ.data_ptr(), qo, 0.0, dfk.data_ptr(), dkeep.data_ptr(), capi.PTR_DEVICE, asynchronous=True)
    h.wait()
    torch.cuda.synchronize()
    assert np.array_equal(dfk.cpu().numpy(), ofk) and np.array_equal(dkeep.cpu().numpy(), ofk.min(axis=0))
    nv2, nf2, nr2 = h.node_stats()
    assert np.array_equal(nv2, ost[:, 0]) and np.array_equal(nf2, ost[:, 1]) and np.array_equal(nr2, ost[:, 2])
    h.close(); m.close()


def test_node_sub_batch_split_by_scratch_budget(capi, oracle_mod, small_workload, monkeypatch):
    """ERASOR_B200_NODE_SCRATCH_GB=1 on an 8 M point map: sub-batches of two frames.  Every output equals the same call with
    the variable unset (one submission)."""
    p = P.preset("seq_05").replace(skip_voxelize=1)
    base = oracle_mod.transform(small_workload["map_world"], oracle_mod.pose_to_matrix(G_TILT))
    tiles = 64
    mw = np.concatenate([base + np.array([500.0 * (t % 8), 400.0 * (t // 8), 0, 0], dtype=np.float32) for t in range(tiles)])
    N = len(mw)
    assert 7_000_000 < N and (1 << 30) // (46 * N) == 2
    scene = small_workload["scene"]
    frames = small_workload["frames"]
    poses, qs = [], []
    for j, t in enumerate((0, 9, 18, 27, 36, 63)):
        off = pc.pose7([500.0 * (t % 8), 400.0 * (t // 8), 0.0], [0, 0, 0, 1.0])
        poses.append(pc.compose(off, pc.compose(G_TILT, scene.pose7(frames[j][2]))))
        qs.append(frames[j][1])
    poses = np.stack(poses)
    Q, qo = np.concatenate(qs), _offsets(qs)
    m = capi.Map(mw)
    outs = {}
    for tag in ("whole", "split"):
        if tag == "split":
            monkeypatch.setenv("ERASOR_B200_NODE_SCRATCH_GB", "1")
        else:
            monkeypatch.delenv("ERASOR_B200_NODE_SCRATCH_GB", raising=False)
        m.reset_keep()
        h = capi.Handle(p)
        h.attach_map(m)
        keep, fk = h.process_nodes(poses, Q, qo, want_frame_keep=True)
        outs[tag] = (keep, fk, h.node_stats())
        h.close()
    monkeypatch.delenv("ERASOR_B200_NODE_SCRATCH_GB", raising=False)
    (k0, f0, s0), (k1, f1, s1) = outs["whole"], outs["split"]
    assert (f0 == 0).any() and (s0[0] > 0).all()
    assert np.array_equal(f1, f0) and np.array_equal(k1, k0)
    for a, b in zip(s0, s1):
        assert np.array_equal(a, b), (a, b)
    m.close()


# ---- the sequential updater at far poses -----------------------------------------------------------------------------------
G_UPD = pc.pose7([4000.0, -20000.0, 35.0], pc.quat_rpy(D(3), D(-4), 2.8))


@pytest.fixture(scope="module")
def far_updater_scene(oracle_mod):
    sc = synth.Scene(seed=31, length=50.0, n_nodes=21, n_dynamic=6)
    kw = dict(n_beams=32, n_az=720)
    nodes = list(range(0, 21))
    initial_map = sc.build_map(nodes, voxel=0.2, **kw)
    scans = [sc.scan(k, seed_offset=5, **kw) for k in nodes]
    moved, poses = pc.replace(initial_map, [sc.pose7(k) for k in nodes], G_UPD, oracle_mod)
    return dict(map=moved, scans=scans, poses=poses)


def _submap_centres(poses, processed, s, oracle_mod):
    """reassign_submap's centres over the processed nodes (OfflineMapUpdater.cpp:332-358)."""
    cs = []
    for k in processed:
        x, y = pc.criterion(poses[k], oracle_mod)
        if not cs or abs(cs[-1][0] - x) > s / 2 or abs(cs[-1][1] - y) > s / 2:
            cs.append((x, y))
    return cs


@pytest.mark.parametrize("name,large", [("seq_05", False), ("large_scale_05", True)])
def test_updater_at_far_poses(capi, oracle_mod, far_updater_scene, name, large):
    ep = P.preset(name)
    up = P.updater_preset(name)
    up.removal_interval = 2
    up.is_large_scale = large
    up.submap_size = 25.0 if large else up.submap_size
    sc = far_updater_scene
    processed = [k for k in range(len(sc["poses"])) if (k + 1) % up.removal_interval == 0]
    rng = np.random.default_rng(13)
    px, py = pc.criterion(sc["poses"][processed[0]], oracle_mod)
    extra = [pc.shell(px, py, up.max_range, seed=3)[0]]
    centres = _submap_centres(sc["poses"], processed, up.submap_size, oracle_mod)
    if large:
        assert len(centres) >= 2
    extra += [pc.square_shell(cx, cy, up.submap_size, seed=i) for i, (cx, cy) in enumerate(centres)]
    extra = np.concatenate(extra)
    mw = np.concatenate([sc["map"], pc.with_z(extra, rng, G_UPD[2] - 1.5, G_UPD[2] + 2.5, 40.0)])
    if large:      # the shells sit exactly on the square's edges, exact ties included
        cx, cy = centres[0]
        on = (np.abs(extra[:, 0].astype(np.float64) - cx) == up.submap_size) & (np.abs(extra[:, 1].astype(np.float64) - cy) < up.submap_size)
        assert on.any()
    o = oracle_mod.OracleUpdater(up, ep, mw)
    u = capi.Updater(up, ep, mw)
    n_proc = 0
    for k, (pose, scan) in enumerate(zip(sc["poses"], sc["scans"])):
        a = o.callback_node(k, pose, scan)
        b = u.process_node(k, pose, scan)
        assert a == b
        if not a:
            continue
        n_proc += 1
        for which in ("QUERY_VOI", "MAP_VOI", "OUTSKIRTS", "MAP_REJECTED", "MAP_ARRANGED"):
            assert _same(u.cloud(getattr(u, which)), o.cloud(getattr(o, which))[0]), f"node {k}: {which}"
    assert n_proc == len(processed)
    assert len(o.cloud(o.TOTAL_MAP_REJECTED)[0]) > 0
    assert _same(u.save_static_map(0.2), o.save_static_map(0.2))
    u.close(); o.close()


# ---- mapgen at far poses -----------------------------------------------------------------------------------------------------
G_MG = pc.pose7([-20000.0, 4000.0, -45.0], pc.quat_rpy(D(-5), D(3), -2.2))


def _far_mapgen_nodes(n_nodes=20, n_pts=300, seed=23):
    rng = np.random.default_rng(seed)
    shell = pc.body_cut_shell(seed=seed)
    out = []
    for k in range(n_nodes):
        r = rng.uniform(0.5, 35.0, n_pts); th = rng.uniform(-np.pi, np.pi, n_pts)
        scan = np.stack([r * np.cos(th), r * np.sin(th), rng.normal(-1.7, 0.2, n_pts), rng.choice([40.0, 48.0, 252.0], n_pts)], axis=1)
        cut = pc.with_z(shell[k % 3::3], rng, -1.9, 0.5, 40.0)
        scan = np.concatenate([scan.astype(np.float32), cut])
        odom = pc.pose7([0.3 * k, 0.02 * k, 0.0], pc.quat_rpy(0.0, 0.0, 0.002 * k))
        pose = pc.compose(G_MG, odom)
        if k % 4 == 3:
            pose[3:] *= -1.0
        out.append((k, pose, np.ascontiguousarray(scan, dtype=np.float32)))
    return out


@pytest.mark.parametrize("large_scale", [False, True])
def test_mapgen_at_far_poses(capi, oracle_mod, large_scale):
    nodes = _far_mapgen_nodes()
    gen = capi.MapGen(0.2, large_scale)
    o = oracle_mod.OracleMapGen(0.2, large_scale)
    for k, pose, scan in nodes:
        gen.accum(pose, scan)
        o.accum(pose, scan)
        assert _same(gen.cloud(gen.CLOUD_CURR), o.cloud(o.CLOUD_CURR)), f"node {k}: cloud_curr"
        assert _same(gen.cloud(gen.CLOUD_MAP), o.cloud(o.CLOUD_MAP)), f"node {k}: cloud_map"
    assert _same(gen.cloud(gen.SAVED_ORIGINAL), o.cloud(o.SAVED_ORIGINAL))
    assert _same(gen.cloud(gen.SAVED_VOXELIZED), o.cloud(o.SAVED_VOXELIZED))
    gen.close(); o.close()
