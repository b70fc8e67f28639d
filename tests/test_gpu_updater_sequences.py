"""The sequential updater (erasor_updater_*) under the call sequences its callers use, against the oracle's caller loop.

- bench.py's offline pass (seq 05 twin, 64 x 1800 scans, removal_interval 8, pinned scans handed to the look-ahead one processed
  node early), run three times on one handle re-armed with reset;
- the look-ahead and the prefetched VoI cut at their capped grids on a dense map, device and pageable scans, mixed in one pass;
- removal intervals, large-scale mode (version 2, reset mid-run), resets that shrink and regrow the buffers, a reset while a
  look-ahead is pending;
- degenerate nodes (empty scan, empty VoI, empty initial map, one point, one voxel) and the fused kernel's size edges;
- the save cache across leaf changes, voxelize calls, resets and large-scale saves.

Every cloud is compared by its bit pattern, order included.  After every processed node the cut is also checked against a float64
restatement of fetch_VoI (and set_submap) that does not go through the oracle.  The CPU tests check the inputs and that
restatement, without a GPU."""
import ctypes
import hashlib

import numpy as np
import pytest

import pose_cases as PC
from erasor_b200 import params as P
from erasor_b200 import synth

FT, PART_CHUNK = 1024, 4096                 # k_node_fused: threads per CTA, points per partition / head chunk
RS_ROWS_MIN, RS_MAX_SEGS = 8, 8192
CLOUDS = ("QUERY_VOI", "MAP_VOI", "OUTSKIRTS", "MAP_REJECTED", "MAP_ARRANGED")
EMPTY = np.zeros((0, 4), dtype=np.float32)
SMALL_SCAN = dict(n_beams=32, n_az=720, seed_offset=5)


def rs_seg_len(n):
    """updater_kernels.cu rs_seg_len: radix-sort segment length of an n-point cloud."""
    rows = (n + 32 * RS_MAX_SEGS - 1) // (32 * RS_MAX_SEGS)
    rows = (rows + RS_ROWS_MIN - 1) // RS_ROWS_MIN * RS_ROWS_MIN
    return 32 * max(rows, RS_ROWS_MIN)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _digest(a):
    return a.shape, hashlib.sha256(np.ascontiguousarray(a).view(np.uint32).tobytes()).hexdigest()


def _matches(got, ref):
    """ref: a cloud, or the _digest of one"""
    return _same(got, ref) if isinstance(ref, np.ndarray) else _digest(got) == ref


def _dev_clouds(u):
    return lambda name: u.cloud(getattr(u, name))


def _ora_clouds(o):
    return lambda name: o.cloud(getattr(o, name))[0]


def _assert_node(u, ref, tag):
    """every per-node cloud of the device caller equals ref[name] (a cloud or a digest)"""
    for name in CLOUDS:
        got = u.cloud(getattr(u, name))
        assert _matches(got, ref[name]), f"{tag}: {name} ({len(got)} points)"


def _oracle_node(o):
    return {name: o.cloud(getattr(o, name))[0] for name in CLOUDS}


class CutModel:
    """fetch_VoI, and in large-scale mode reassign_submap / set_submap, restated in float64 on the map a node starts from
    (pose_cases.criterion / voi_truth / submap_truth).  check() is called after every processed node with a getter of that
    node's clouds; it asserts that the outskirts are the map points outside the radius, in map order, that the VoI has as many
    points as the radius test selects and (large-scale) that the complement is the points outside the window, then takes the
    node's map as the next node's input."""

    def __init__(self, up, initial_map, oracle_mod):
        self.up, self.om = up, oracle_mod
        self.map = np.ascontiguousarray(initial_map, dtype=np.float32).reshape(-1, 4)
        self.complement = EMPTY
        self.center = None

    def expect(self, pose):
        px, py = PC.criterion(pose, self.om)
        window, comp = self.map, self.complement
        if self.up.is_large_scale:
            half = self.up.submap_size / 2.0
            if self.center is None or abs(self.center[0] - px) > half or abs(self.center[1] - py) > half:
                glob = np.concatenate([self.map, self.complement])
                sub = PC.submap_truth(glob[:, 0], glob[:, 1], px, py, self.up.submap_size)
                window, comp = glob[sub], glob[~sub]
                self.center = (px, py)
        pred = PC.voi_truth(window[:, 0], window[:, 1], px, py, self.up.max_range)
        return window, comp, pred

    def check(self, get, pose, tag):
        window, comp, pred = self.expect(pose)
        assert _same(get("OUTSKIRTS"), window[~pred]), f"{tag}: outskirts != map points outside the radius, in map order"
        assert len(get("MAP_VOI")) == int(pred.sum()), f"{tag}: VoI size"
        if self.up.is_large_scale:
            assert _same(get("SUBMAP_COMPLEMENT"), comp), f"{tag}: submap complement"
        self.map, self.complement = get("MAP_ARRANGED"), comp


def _lockstep(u, o, cut, poses, scans, nodes, prefetch=()):
    """Nodes through the oracle's caller loop and the device caller side by side; after every processed node, every cloud and
    the cut.  prefetch: nodes whose scan the device gets through prefetch_scan_ptr just before process_node_ptr."""
    from erasor_b200 import capi
    n = 0
    for k in nodes:
        scan = np.ascontiguousarray(scans[k], dtype=np.float32).reshape(-1, 4)
        a = o.callback_node(k, poses[k], scan)
        if k in prefetch:
            u.prefetch_scan_ptr(scan.ctypes.data, len(scan), capi.PTR_HOST)
            b = u.process_node_ptr(k, poses[k], scan.ctypes.data, len(scan), capi.PTR_HOST)
        else:
            b = u.process_node(k, poses[k], scan)
        assert a == b, f"node {k}: processed"
        if a:
            n += 1
            _assert_node(u, _oracle_node(o), f"node {k}")
            cut.check(_dev_clouds(u), poses[k], f"node {k}")
    return n


def _oracle_trace(oracle_mod, up, ep, initial_map, poses, scans, nodes):
    """One run of the oracle's caller loop: {processed node: {cloud: digest}} and the digest of save_static_map(0.2)."""
    o = oracle_mod.OracleUpdater(up, ep, initial_map)
    trace = {}
    for k in nodes:
        if o.callback_node(k, poses[k], scans.get(k, EMPTY)):
            trace[k] = {name: _digest(c) for name, c in _oracle_node(o).items()}
    save = _digest(o.save_static_map(0.2))
    o.close()
    return trace, save


def _run_pass(u, poses, nodes, src, ahead, on_processed):
    """One pass of bench.py's caller loop.  src[k] = (pointer, points, kind) of processed node k's scan; the scan of a node in
    `ahead` goes to prefetch_scan_ptr while the processed node before it is handed in (the first one before the loop);
    unprocessed nodes get no scan."""
    from erasor_b200 import capi
    proc = sorted(src)
    nxt = dict(zip(proc, proc[1:]))
    if proc and proc[0] in ahead:
        u.prefetch_scan_ptr(*src[proc[0]])
    for k in nodes:
        if k in src:
            if k in nxt and nxt[k] in ahead:
                u.prefetch_scan_ptr(*src[nxt[k]])
            assert u.process_node_ptr(k, poses[k], *src[k]), f"node {k}: not processed"
            on_processed(k)
        else:
            assert not u.process_node_ptr(k, poses[k], 0, 0, capi.PTR_HOST), f"node {k}: processed"


def _presets(name="seq_05", version=None, removal_interval=None, large=None, submap_size=None):
    ep, up = P.preset(name), P.updater_preset(name)
    if version is not None:
        ep = ep.replace(version=version)
        up.version = version
    if removal_interval is not None:
        up.removal_interval = removal_interval
    if large is not None:
        up.is_large_scale = large
    if submap_size is not None:
        up.submap_size = submap_size
    return up, ep


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- inputs -------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small():
    """The 50 m scene of test_gpu_updater.py: 21 nodes, 32 x 720 scans."""
    sc = synth.Scene(seed=31, length=50.0, n_nodes=21, n_dynamic=6)
    nodes = list(range(21))
    m = sc.build_map(nodes, voxel=0.2, n_beams=32, n_az=720)
    return dict(scene=sc, map=m, scans={k: sc.scan(k, **SMALL_SCAN) for k in nodes}, poses={k: sc.pose7(k) for k in nodes}, nodes=nodes)


@pytest.fixture(scope="module")
def bench_pass():
    """bench.py's offline pass: the seq 05 twin (161 nodes), its map, the processed nodes' 64 x 1800 scans."""
    sc = synth.Scene(seed=5, length=160.0, n_nodes=161, n_dynamic=12)
    nodes = list(range(161))
    m = sc.build_map(list(range(0, 161, 2)), voxel=0.2, n_beams=64, n_az=1800)
    ri = P.updater_preset("seq_05").removal_interval
    scans = {k: sc.scan(k, seed_offset=17) for k in nodes if (k + 1) % ri == 0}
    return dict(map=m, scans=scans, poses={k: sc.pose7(k) for k in nodes}, nodes=nodes)


def lattice(n, leaf=0.25, side=128):
    """n points at the centres of distinct leaf-sized cells (exact in float): one voxel per point, far from PCL's overflow."""
    i = np.arange(n)
    c = np.zeros((n, 4), dtype=np.float32)
    c[:, 0], c[:, 1], c[:, 2] = (i % side) * leaf + leaf / 2, (i // side % side) * leaf + leaf / 2, (i // side // side) * leaf + leaf / 2
    c[:, 3] = (i * 7) % 260
    return c


def one_voxel(n, leaf, seed=0, cell=(50, -15, -8)):
    """n points inside one leaf-sized VoxelGrid cell (cells start at multiples of the leaf), 0.1 leaf away from its faces."""
    rng = np.random.default_rng(seed)
    c = np.zeros((n, 4), dtype=np.float32)
    c[:, :3] = (np.asarray(cell) * leaf + rng.uniform(0.1 * leaf, 0.9 * leaf, (n, 3))).astype(np.float32)
    c[:, 3] = rng.integers(0, 260, n)
    return c


def random_cloud(n, seed, span=60.0, zspan=3.0):
    rng = np.random.default_rng(seed)
    c = np.zeros((n, 4), dtype=np.float32)
    c[:, :2] = rng.uniform(-span, span, (n, 2))
    c[:, 2] = rng.uniform(-zspan, zspan, n)
    c[:, 3] = rng.integers(0, 260, n)
    return c


def _voxel_count(c, leaf):
    """distinct VoxelGrid cells of a cloud, floor(p / leaf) in float64 (the clouds above sit far from any cell face)"""
    ijk = np.floor(c[:, :3].astype(np.float64) / leaf).astype(np.int64)
    return len(np.unique(ijk, axis=0))


def dense_world_map(scene, map_world, nodes, n_target, seed=9):
    """map_world cropped to 30 m around the given nodes and replicated with sub-voxel jitter (as test_gpu_capacity_edges.py)."""
    near = np.zeros(len(map_world), dtype=bool)
    for k in nodes:
        t = scene.pose7(k)[:2]
        near |= (map_world[:, 0].astype(np.float64) - t[0]) ** 2 + (map_world[:, 1].astype(np.float64) - t[1]) ** 2 < 30.0 ** 2
    base = map_world[near]
    rng = np.random.default_rng(seed)
    m = np.tile(base, (int(np.ceil(n_target / len(base))), 1))
    m[:, :3] += ((rng.random((len(m), 3)) - 0.5) * np.array([0.19, 0.19, 0.02])).astype(np.float32)
    return m.astype(np.float32)


# ---- CPU: the inputs reach their edges, and the cut restatement agrees with the oracle --------------------------------------
def test_size_edge_inputs():
    assert (rs_seg_len(2_097_152), -(-2_097_152 // rs_seg_len(2_097_152))) == (256, RS_MAX_SEGS)
    assert (rs_seg_len(2_097_153), -(-2_097_153 // rs_seg_len(2_097_153))) == (512, 4097)
    for n in (1023, 1024, 1025, 4095, 4096, 4097, 128 ** 3):
        assert _voxel_count(lattice(n), 0.25) == n
        assert _voxel_count(one_voxel(n, 0.2), 0.2) == 1
    assert -(-1025 // FT) == 2 and -(-4097 // PART_CHUNK) == 2


@pytest.mark.parametrize("large", [False, True])
def test_cut_model_matches_oracle(oracle_mod, small, large):
    """CutModel restates fetch_VoI and the large-scale window split without the oracle; here it is held to the oracle's
    caller loop, so that on the GPU it is an independent second check of the device's cut."""
    up, ep = _presets(removal_interval=2, large=large, submap_size=25.0 if large else None)
    o = oracle_mod.OracleUpdater(up, ep, small["map"])
    cut = CutModel(up, small["map"], oracle_mod)
    splits, n = set(), 0
    for k in small["nodes"]:
        if o.callback_node(k, small["poses"][k], small["scans"][k]):
            cut.check(_ora_clouds(o), small["poses"][k], f"node {k}")
            splits.add(cut.center)
            n += 1
    assert n == 10
    assert len(splits) >= (3 if large else 1)          # the window moves along the 50 m
    o.close()


# ---- 1. bench.py's pass, re-armed ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bench_pass_rearmed(oracle_mod, bench_pass):
    """Three passes of bench.py's offline pass on one handle with reset between them: every processed node and the saved map
    equal the oracle in every pass, and each pass ends with the same map size after the same number of launches."""
    import torch
    from erasor_b200 import capi
    up, ep = _presets()
    assert up.removal_interval == 8 and ep.version == 3
    B = bench_pass
    sm = _sm_count()
    # the look-ahead runs on sm // 4 CTAs: these scans need more, so each CTA loops over several rows and chunks
    assert all(-(-len(s) // FT) > sm // 4 for s in B["scans"].values()), [len(s) for s in B["scans"].values()]
    trace, save = _oracle_trace(oracle_mod, up, ep, B["map"], B["poses"], B["scans"], B["nodes"])
    assert sorted(trace) == sorted(B["scans"]) and len(trace) == 20
    pinned = {k: torch.from_numpy(v).pin_memory() for k, v in B["scans"].items()}
    src = {k: (t.data_ptr(), len(t), capi.PTR_HOST) for k, t in pinned.items()}
    u = capi.Updater(up, ep, B["map"])
    per_pass = []
    for rep in range(3):
        if rep:
            u.reset(B["map"])
        cut = CutModel(up, B["map"], oracle_mod)

        def check(k):
            _assert_node(u, trace[k], f"pass {rep} node {k}")
            cut.check(_dev_clouds(u), B["poses"][k], f"pass {rep} node {k}")
        l0 = u.kernel_launch_count()
        _run_pass(u, B["poses"], B["nodes"], src, set(src), check)
        per_pass.append((u.map_size(), u.kernel_launch_count() - l0))
        assert _digest(u.save_static_map(0.2)) == save, f"pass {rep}: save_static_map"
    assert len(set(per_pass)) == 1, per_pass
    u.close()


# ---- 2. the look-ahead and the prefetched cut at their capped grids -------------------------------------------------------
@pytest.mark.gpu
def test_capped_grids_dense_map(oracle_mod, small_workload):
    """The look-ahead's voxelisation on sm // 4 CTAs and the prefetched VoI cut on the rest, both looping over many rows /
    chunks per CTA (a VoI of more than (sm - sm // 4) x 4096 points): the same clouds as a second handle without look-ahead,
    and as the oracle."""
    from erasor_b200 import capi
    up, ep = _presets(removal_interval=1)
    sm = _sm_count()
    la_ctas = max(1, sm // 4)
    cut_ctas = sm - la_ctas
    sc = small_workload["scene"]
    k0 = small_workload["frames"][2][2]
    nodes = [k0, k0 + 1, k0 + 2, k0 + 3]
    mw = dense_world_map(sc, small_workload["map_world"], nodes, n_target=1_200_000)
    poses = {k: sc.pose7(k) for k in nodes}
    scans = {k: sc.scan(k, seed_offset=17) for k in nodes}
    assert all(-(-len(s) // FT) > la_ctas for s in scans.values())
    trace, save = _oracle_trace(oracle_mod, up, ep, mw, poses, scans, nodes)
    src = {k: (s.ctypes.data, len(s), capi.PTR_HOST) for k, s in scans.items()}
    for ahead in (set(nodes[1:]), set()):
        u = capi.Updater(up, ep, mw)
        cut = CutModel(up, mw, oracle_mod)

        def check(k):
            _assert_node(u, trace[k], f"look-ahead {bool(ahead)} node {k}")
            cut.check(_dev_clouds(u), poses[k], f"node {k}")
            assert len(u.cloud(u.MAP_VOI)) > cut_ctas * PART_CHUNK
        _run_pass(u, poses, nodes, src, ahead, check)
        assert _digest(u.save_static_map(0.2)) == save
        u.close()


# ---- 3. device and pageable scans -------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_and_pageable_scans(oracle_mod, small):
    """process_node_ptr / prefetch_scan_ptr on torch CUDA tensors (PTR_DEVICE) and on pageable numpy arrays, and both mixed in
    one pass (a device scan prefetched, a host one prefetched, then nodes without look-ahead): the pinned-host run's clouds."""
    import torch
    from erasor_b200 import capi
    up, ep = _presets(removal_interval=2)
    nodes, poses = small["nodes"], small["poses"]
    proc = [k for k in nodes if (k + 1) % up.removal_interval == 0]
    scans = {k: np.ascontiguousarray(small["scans"][k]) for k in proc}
    trace, save = _oracle_trace(oracle_mod, up, ep, small["map"], poses, scans, nodes)
    pinned = {k: torch.from_numpy(s).pin_memory() for k, s in scans.items()}
    dev = {k: torch.from_numpy(s).cuda() for k, s in scans.items()}
    torch.cuda.synchronize()
    host_src = {k: (s.ctypes.data, len(s), capi.PTR_HOST) for k, s in scans.items()}
    dev_src = {k: (t.data_ptr(), len(t), capi.PTR_DEVICE) for k, t in dev.items()}
    kinds = ("device, prefetched", "host, prefetched", "device", "host")
    mixed = {k: (dev_src if kinds[i % 4].startswith("device") else host_src)[k] for i, k in enumerate(proc)}
    mixed_ahead = {k for i, k in enumerate(proc) if kinds[i % 4].endswith("prefetched")}
    runs = (("pinned", {k: (t.data_ptr(), len(t), capi.PTR_HOST) for k, t in pinned.items()}, set(proc)),
            ("device", dev_src, set(proc)), ("device, no look-ahead", dev_src, set()),
            ("pageable", host_src, set(proc)), ("mixed", mixed, mixed_ahead))
    pinned_clouds = {}
    for name, src, ahead in runs:
        u = capi.Updater(up, ep, small["map"])
        cut = CutModel(up, small["map"], oracle_mod)

        def check(k):
            got = {c: u.cloud(getattr(u, c)) for c in CLOUDS}
            if name == "pinned":
                _assert_node(u, trace[k], f"{name} node {k}")
                pinned_clouds[k] = got
            else:
                _assert_node(u, pinned_clouds[k], f"{name} node {k}")
            cut.check(lambda c: got[c] if c in got else u.cloud(getattr(u, c)), poses[k], f"{name} node {k}")
        _run_pass(u, poses, nodes, src, ahead, check)
        assert _digest(u.save_static_map(0.2)) == save, name
        u.close()


# ---- 4. sequence variants -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("removal_interval", [1, 3, 8])
def test_removal_interval(oracle_mod, small, removal_interval):
    from erasor_b200 import capi
    up, ep = _presets(removal_interval=removal_interval)
    o = oracle_mod.OracleUpdater(up, ep, small["map"])
    u = capi.Updater(up, ep, small["map"])
    n = _lockstep(u, o, CutModel(up, small["map"], oracle_mod), small["poses"], small["scans"], small["nodes"])
    assert n == len(small["nodes"]) // removal_interval
    assert _same(u.save_static_map(0.2), o.save_static_map(0.2))
    u.close()
    o.close()


@pytest.mark.gpu
def test_large_scale_version2_save_between_nodes(oracle_mod, small):
    """Large-scale mode with version 2 and a 25 m window that moves along the scene; a save in the middle of the run (it merges
    the window and its complement in the double buffer) is followed by more processed nodes."""
    from erasor_b200 import capi
    up, ep = _presets("large_scale_05", version=2, removal_interval=2, submap_size=25.0)
    assert up.is_large_scale
    o = oracle_mod.OracleUpdater(up, ep, small["map"])
    u = capi.Updater(up, ep, small["map"])
    cut = CutModel(up, small["map"], oracle_mod)
    nodes = small["nodes"]
    assert _lockstep(u, o, cut, small["poses"], small["scans"], nodes[:11]) == 5
    assert _same(u.save_static_map(0.2), o.save_static_map(0.2))
    assert _lockstep(u, o, cut, small["poses"], small["scans"], nodes[11:]) == 5
    assert _same(u.save_static_map(0.2), o.save_static_map(0.2))
    assert len(o.cloud(o.TOTAL_MAP_REJECTED)[0]) > 0
    u.close()
    o.close()


@pytest.mark.gpu
def test_large_scale_reset_midrun(oracle_mod, small):
    """reset in large-scale mode re-arms the window: the first processed node after it splits the whole map again around its
    own pose.  Until then the map is the whole initial map (load_global_map), which is what a save right after the reset
    writes."""
    from erasor_b200 import capi
    up, ep = _presets("large_scale_05", removal_interval=2, submap_size=25.0)
    assert up.is_large_scale
    nodes, poses, scans, m = small["nodes"], small["poses"], small["scans"], small["map"]
    o = oracle_mod.OracleUpdater(up, ep, m)
    u = capi.Updater(up, ep, m)
    assert _same(u.save_static_map(0.2), o.save_static_map(0.2))          # before the first node
    assert u.map_size() == len(m) and _same(u.cloud(u.MAP_ARRANGED), o.cloud(o.MAP_ARRANGED)[0])
    _lockstep(u, o, CutModel(up, m, oracle_mod), poses, scans, nodes[:11])
    o.close()
    for reset_map in (m, m[::2]):
        u.reset(reset_map)
        o = oracle_mod.OracleUpdater(up, ep, reset_map)
        assert u.map_size() == len(reset_map)
        assert _same(u.save_static_map(0.2), o.save_static_map(0.2)), "save right after reset"
        cut = CutModel(up, reset_map, oracle_mod)
        assert _lockstep(u, o, cut, poses, scans, nodes[11:]) == 5
        assert _same(u.save_static_map(0.2), o.save_static_map(0.2))
        o.close()
    u.close()


@pytest.mark.gpu
def test_reset_shrinks_then_regrows(oracle_mod, small):
    """reset to a third of the map, then to a map twice the size of the first: the device buffers are kept and regrow."""
    from erasor_b200 import capi
    up, ep = _presets(removal_interval=2)
    m = small["map"]
    rng = np.random.default_rng(4)
    big = np.concatenate([m, m + np.array([0.07, -0.05, 0.01, 0.0], dtype=np.float32) * rng.random((len(m), 1)).astype(np.float32)])
    u = capi.Updater(up, ep, m)
    for mp in (m, m[::3], big):
        if mp is not m:
            u.reset(mp)
        o = oracle_mod.OracleUpdater(up, ep, mp)
        assert u.map_size() == len(mp)
        assert _lockstep(u, o, CutModel(up, mp, oracle_mod), small["poses"], small["scans"], small["nodes"][:12]) == 6
        assert _same(u.save_static_map(0.2), o.save_static_map(0.2))
        o.close()
    u.close()


@pytest.mark.gpu
def test_reset_drops_pending_lookahead(oracle_mod, small):
    """A look-ahead still pending at reset is dropped: the same pinned buffer, refilled with another scan of the same length and
    handed to process_node_ptr without a new prefetch, is voxelised afresh."""
    import torch
    from erasor_b200 import capi
    up, ep = _presets(removal_interval=1)
    nodes, poses, m = small["nodes"], small["poses"], small["map"]
    u = capi.Updater(up, ep, m)
    o = oracle_mod.OracleUpdater(up, ep, m)
    _lockstep(u, o, CutModel(up, m, oracle_mod), poses, small["scans"], nodes[:3], prefetch=set(nodes[:3]))
    o.close()
    a, b = small["scans"][3], small["scans"][9]
    n = min(len(a), len(b))
    a, b = np.ascontiguousarray(a[:n]), np.ascontiguousarray(b[:n])
    buf = torch.from_numpy(a.copy()).pin_memory()
    u.prefetch_scan_ptr(buf.data_ptr(), n, capi.PTR_HOST)
    u.reset(m)
    buf.copy_(torch.from_numpy(b))
    o = oracle_mod.OracleUpdater(up, ep, m)
    cut = CutModel(up, m, oracle_mod)
    assert o.callback_node(3, poses[3], b)
    assert u.process_node_ptr(3, poses[3], buf.data_ptr(), n, capi.PTR_HOST)
    _assert_node(u, _oracle_node(o), "node after reset")
    cut.check(_dev_clouds(u), poses[3], "node after reset")
    _lockstep(u, o, cut, poses, small["scans"], nodes[4:8], prefetch=set(nodes[4:8]))
    assert _same(u.save_static_map(0.2), o.save_static_map(0.2))
    u.close()
    o.close()


# ---- 5. degenerate nodes --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_degenerate_nodes(oracle_mod, small):
    """An empty scan (with and without look-ahead), a node placed 10 km from the map (empty VoI), a one-point scan and a scan
    whose points all fall in one query voxel, each followed by an ordinary node on the same handle."""
    from erasor_b200 import capi
    up, ep = _presets(removal_interval=1)
    m = small["map"]
    poses = dict(small["poses"])
    scans = dict(small["scans"])
    scans[1] = scans[3] = EMPTY
    poses[5] = poses[5].copy()
    poses[5][:2] += 10_000.0
    scans[7] = scans[7][:1]
    scans[9] = one_voxel(3000, up.query_voxel_size, seed=9)
    o = oracle_mod.OracleUpdater(up, ep, m)
    u = capi.Updater(up, ep, m)
    cut = CutModel(up, m, oracle_mod)
    degenerate = {1: ("QUERY_VOI", 0), 3: ("QUERY_VOI", 0), 5: ("MAP_VOI", 0), 7: ("QUERY_VOI", 1), 9: ("QUERY_VOI", 1)}
    for k in range(11):
        assert _lockstep(u, o, cut, poses, scans, [k], prefetch={3, 4}) == 1
        if k in degenerate:
            name, n_want = degenerate[k]
            assert len(u.cloud(getattr(u, name))) == n_want, (k, name)
        else:
            assert len(u.cloud(u.MAP_VOI)) > 0 and len(u.cloud(u.QUERY_VOI)) > 1
    assert _same(u.save_static_map(0.2), o.save_static_map(0.2))
    u.close()
    o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("large", [False, True])
def test_empty_initial_map(oracle_mod, small, large):
    from erasor_b200 import capi
    up, ep = _presets("large_scale_05" if large else "seq_05", removal_interval=2, submap_size=25.0 if large else None)
    o = oracle_mod.OracleUpdater(up, ep, EMPTY)
    u = capi.Updater(up, ep, EMPTY)
    assert u.map_size() == 0 and len(u.save_static_map(0.2)) == 0
    assert _lockstep(u, o, CutModel(up, EMPTY, oracle_mod), small["poses"], small["scans"], small["nodes"][:8]) == 4
    assert u.map_size() == 0
    assert _same(u.save_static_map(0.2), o.save_static_map(0.2))
    u.reset(small["map"])                                   # and usable with a real map afterwards
    o.close()
    o = oracle_mod.OracleUpdater(up, ep, small["map"])
    assert _lockstep(u, o, CutModel(up, small["map"], oracle_mod), small["poses"], small["scans"], small["nodes"][:4]) == 2
    u.close()
    o.close()


# ---- 6. size edges of the fused kernel -----------------------------------------------------------------------------------
EDGES = (1023, 1024, 1025, 4095, 4096, 4097)


@pytest.mark.gpu
def test_voxelize_size_edges(oracle_mod, small):
    """Updater.voxelize (one fused launch, vn = n) at the row / chunk edges, with one voxel per point and with one voxel in all,
    and at the radix segment length's step: 2,097,152 points sort in 8192 segments of 256, one more in 4097 of 512."""
    from erasor_b200 import capi
    up, ep = _presets()
    u = capi.Updater(up, ep, small["map"][:10])
    scan = small["scans"][6]
    assert len(scan) > 4097
    for n in EDGES:
        for c, leaf, n_vox in ((scan[:n], 0.2, None), (lattice(n), 0.25, n), (one_voxel(n, 0.2, seed=n), 0.2, 1)):
            got, ref = u.voxelize(c, leaf), oracle_mod.voxelize(c, leaf)
            assert _same(got, ref), f"n={n} leaf={leaf}"
            assert n_vox is None or len(got) == n_vox
    big = random_cloud(2_097_153, seed=21)
    lat = np.concatenate([lattice(128 ** 3), lattice(1)])               # the extra point repeats the first cell
    for n in (2_097_152, 2_097_153):
        assert rs_seg_len(n) == (256 if n == 2_097_152 else 512)
        for c, leaf in ((big[:n], 0.2), (lat[:n], 0.25)):
            got, ref = u.voxelize(c, leaf), oracle_mod.voxelize(c, leaf)
            assert _same(got, ref), f"n={n} leaf={leaf}"
        assert len(u.voxelize(lat[:n], 0.25)) == 128 ** 3
    u.close()


@pytest.mark.gpu
@pytest.mark.parametrize("grid_from", ["scan", "map"])
def test_process_node_size_edges(oracle_mod, small, grid_from):
    """Nodes whose raw scan has 1023 .. 4097 points.  grid_from = the job that sizes the fused launch: "scan" runs them on a
    map of a few hundred points (vn > pn), "map" on the full map (pn > vn)."""
    from erasor_b200 import capi
    up, ep = _presets(removal_interval=1)
    m = small["map"]
    if grid_from == "scan":
        m = m[np.sort(np.random.default_rng(1).choice(len(m), 900, replace=False))]
    nodes = list(range(len(EDGES)))
    scans = {k: small["scans"][k + 4][:n] for k, n in zip(nodes, EDGES)}
    u = o = None
    for k in nodes:
        if u is None or grid_from == "scan":           # the map grows by the query points a node puts back: one handle per node
            if u is not None:
                u.close(); o.close()
            o = oracle_mod.OracleUpdater(up, ep, m)
            u = capi.Updater(up, ep, m)
            cut = CutModel(up, m, oracle_mod)
        vn, pn = len(scans[k]), u.map_size()
        assert vn == EDGES[k] and ((vn > pn) if grid_from == "scan" else (pn > vn)), (vn, pn)
        assert _lockstep(u, o, cut, small["poses"], scans, [k]) == 1
        assert _same(u.save_static_map(0.2), o.save_static_map(0.2))
    u.close()
    o.close()


# ---- 8. the save cache ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_save_cache(oracle_mod, small):
    """save_static_map keeps its last result for the size query + fetch pattern; a different leaf, a voxelize call (which
    writes the same buffer), a processed node and a reset must each make it voxelise again."""
    from erasor_b200 import capi
    up, ep = _presets(removal_interval=2)
    nodes, poses, scans, m = small["nodes"], small["poses"], small["scans"], small["map"]
    o = oracle_mod.OracleUpdater(up, ep, m)
    u = capi.Updater(up, ep, m)
    cut = CutModel(up, m, oracle_mod)
    _lockstep(u, o, cut, poses, scans, nodes[:10])
    ref = {leaf: o.save_static_map(leaf) for leaf in (0.2, 0.4)}
    assert len(ref[0.2]) != len(ref[0.4])
    for leaf in (0.2, 0.4, 0.2, 0.4):
        assert _same(u.save_static_map(leaf), ref[leaf]), leaf
    # a size query, a voxelize call, then the fetch
    n = ctypes.c_size_t(0)
    u._ck(u.L.erasor_updater_save_static_map(u.h, 0.2, None, 0, ctypes.byref(n)))
    assert n.value == len(ref[0.2])
    assert _same(u.voxelize(scans[3], 0.2), oracle_mod.voxelize(scans[3], 0.2))
    out = np.empty((n.value, 4), dtype=np.float32)
    u._ck(u.L.erasor_updater_save_static_map(u.h, 0.2, out.ctypes.data, n.value, ctypes.byref(n)))
    assert _same(out[:n.value], ref[0.2]), "fetch after voxelize"
    # a processed node changes the map
    _lockstep(u, o, cut, poses, scans, nodes[10:12])
    assert _same(u.save_static_map(0.2), o.save_static_map(0.2))
    # a reset changes it back
    u.reset(m)
    assert _same(u.save_static_map(0.2), oracle_mod.voxelize(m, 0.2)), "save after reset"
    u.close()
    o.close()
