"""GPU parity past the shared-memory limits: R-GPF's class C in global scratch and every sort switch exactly at its boundary, the
in-bin voxeliser (K4b) across its cap and its radix pass counts, the mask-mode SRT + scatter over several slot windows, and a dense
map end to end.  Every case is compared bit for bit with the oracle on the same inputs; tests/test_bin_cases_model.py shows without a
GPU that each crafted case sits on the intended side of its switch."""
import numpy as np
import pytest

import bin_cases as C
from erasor_b200 import params as P

pytestmark = pytest.mark.gpu

IDENTITY = np.array([0, 0, 0, 0, 0, 0, 1], dtype=np.float64)


@pytest.fixture(scope="module")
def capi():
    from erasor_b200 import capi as Cap
    return Cap


def _u32_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _okeep(o, n):
    _, rej = o.cloud(o.MAP_REJECTED)
    k = np.ones(n, dtype=np.uint8)
    k[rej] = 0
    return k


def _cloud_mode(capi, oracle_mod, p, m, q, tag):
    """set_inputs / compare against the oracle: planes, keep and ground masks, the four clouds (bit for bit)."""
    o = oracle_mod.Oracle(p)
    o.run(m, q)
    h = capi.Handle(p)
    h.set_inputs(m, q)
    h.compare(p.version)
    gp, op = h.get_planes(), o.planes()
    assert len(op) > 0 and [g["bin"] for g in gp] == [x["bin"] for x in op], tag
    for g, x in zip(gp, op):
        assert (g["n_points"], g["n_seeds"], g["lpr"]) == (x["n_points"], x["n_seeds"], x["lpr"]), (tag, x["bin"], x["n_points"])
        assert np.array_equal(g["normal_d"], x["normal_d"]) and np.array_equal(g["n_ground"], x["n_ground"]), (tag, x["bin"], x["n_points"])
    keep, gnd = h.get_static_mask()
    assert np.array_equal(keep, _okeep(o, len(m))), tag
    _, gsrc = o.cloud(o.GROUND_VIZ)
    ognd = np.zeros(len(m), dtype=np.uint8)
    ognd[gsrc] = 1
    assert np.array_equal(gnd, ognd), tag
    arr, cmp_ = h.get_static_estimate()
    mr, cr = h.get_outliers()
    for name, dev, which in (("arranged", arr, o.ARRANGED), ("complement", cmp_, o.COMPLEMENT), ("map_rejected", mr, o.MAP_REJECTED),
                             ("curr_rejected", cr, o.CURR_REJECTED)):
        assert _u32_equal(dev, o.cloud(which)[0]), (tag, name)
    h.close()
    return o


# ---- R-GPF: every sort switch at its boundary, class C's cap, bins far beyond it ------------------------------------------------
@pytest.mark.parametrize("version", [3, 2])
@pytest.mark.parametrize("z", C.RGPF_Z_KINDS)
def test_rgpf_sizes_cloud_mode(capi, oracle_mod, z, version):
    p = P.preset("seq_05").replace(skip_voxelize=1, version=version)
    m, q = C.flagged_bins(p, C.rgpf_specs(z), seed=7)
    _cloud_mode(capi, oracle_mod, p, m, q, (z, version))


@pytest.mark.parametrize("version", [3, 2])
def test_rgpf_sizes_frames_and_nodes(capi, oracle_mod, version):
    """The same frames through process_frames (one batch) and process_nodes (each frame as a resident map at the identity pose)."""
    p = P.preset("seq_05").replace(skip_voxelize=1, version=version)
    frames = [C.flagged_bins(p, C.rgpf_specs(z), seed=7) for z in C.RGPF_Z_KINDS]
    mo = np.cumsum([0] + [len(m) for m, _ in frames]).astype(np.uint64)
    qo = np.cumsum([0] + [len(q) for _, q in frames]).astype(np.uint64)
    h = capi.Handle(p)
    keep = h.process_frames(np.concatenate([m for m, _ in frames]), mo, np.concatenate([q for _, q in frames]), qo)
    nf, nr = h.frame_stats()
    for f, (m, q) in enumerate(frames):
        o = oracle_mod.Oracle(p)
        o.run(m, q)
        ok = _okeep(o, len(m))
        assert np.array_equal(keep[int(mo[f]):int(mo[f + 1])], ok), ("frames", C.RGPF_Z_KINDS[f])
        assert nf[f] == len(o.planes()) and nr[f] == int((ok == 0).sum())
    for f, (m, q) in enumerate(frames):
        gm = capi.Map(m)
        h.attach_map(gm)
        kg, fk = h.process_nodes(IDENTITY[None], q, np.array([0, len(q)], dtype=np.uint64), want_frame_keep=True)
        voi, idx = oracle_mod.fetch_voi(m, IDENTITY, p.max_range)
        o = oracle_mod.Oracle(p)
        o.run(voi, q)
        ok = np.ones(len(m), dtype=np.uint8)
        ok[idx[_okeep(o, len(voi)) == 0]] = 0
        assert np.array_equal(fk[0], ok) and np.array_equal(kg, ok), ("nodes", C.RGPF_Z_KINDS[f])
        nv, nfl, nrj = h.node_stats()
        assert nv[0] == len(voi) and nfl[0] == len(o.planes()) and nrj[0] == int((ok == 0).sum())
        h.attach_map(None)
        gm.close()
    h.close()


def test_class_c_global_scratch_turning_up_late(capi, oracle_mod):
    """A 20 000-point bin in a submission launched without class C: erasor_wait's fix-up runs class C in global scratch."""
    p = P.preset("seq_05").replace(skip_voxelize=1)
    small = C.flagged_bins(p, [C.Bin(5, 2, 200)], seed=5)
    big = C.flagged_bins(p, [C.Bin(5, 2, 20000), C.Bin(6, 9, 300)], seed=6)
    h = capi.Handle(p)
    o = oracle_mod.Oracle(p)
    for tag, (m, q) in (("small", small), ("small again (class C now off)", small), ("big (fix-up)", big), ("big (class C launched)", big), ("small", small)):
        keep = h.process_frames(m, np.array([0, len(m)], dtype=np.uint64), q, np.array([0, len(q)], dtype=np.uint64))
        o.run(m, q)
        ok = _okeep(o, len(m))
        assert (ok == 0).any() and np.array_equal(keep, ok), tag
    h.close()


# ---- K4b: both sides of the cap, one to four radix passes, pass-through, adjacent all-ground bins -------------------------------
@pytest.mark.parametrize("leaf", sorted(C.K4B_FRAMES))
def test_k4b_capacity_edges(capi, oracle_mod, leaf):
    p = P.preset("seq_05").replace(skip_voxelize=0, version=3, map_voxel_size=leaf)
    m, q = C.flagged_bins(p, C.K4B_FRAMES[leaf], seed=11)
    _cloud_mode(capi, oracle_mod, p, m, q, leaf)


# ---- K2: the fused SRT + scatter over one, two and all slot windows in mask and node mode -----------------------------------
def test_k2_windows_frames_and_nodes(capi, oracle_mod):
    p = P.preset(C.K2_PRESET)
    B = p.num_bins
    W = C.k2_window(B)
    counts = C.k2_flag_counts(B)
    order = [3, 0, 4, 1, 2]                      # mixed, so that each frame's windows start again from the first
    frames = [C.fill_flagged(p, counts[k], seed=100 + k)[:2] for k in order]
    want = [counts[k] for k in order]
    assert min(want) < W <= sorted(want)[1] and max(want) > 2 * W
    mo = np.cumsum([0] + [len(m) for m, _ in frames]).astype(np.uint64)
    qo = np.cumsum([0] + [len(q) for _, q in frames]).astype(np.uint64)
    h = capi.Handle(p)
    keep = h.process_frames(np.concatenate([m for m, _ in frames]), mo, np.concatenate([q for _, q in frames]), qo)
    nf, nr = h.frame_stats()
    for f, (m, q) in enumerate(frames):
        o = oracle_mod.Oracle(p)
        o.run(m, q)
        assert len(o.planes()) == want[f]
        ok = _okeep(o, len(m))
        assert np.array_equal(keep[int(mo[f]):int(mo[f + 1])], ok), ("frames", want[f])
        assert nf[f] == want[f] and nr[f] == int((ok == 0).sum())
    # node mode: the frames side by side in one resident map, 300 m apart, one node at each
    shift = [np.array([300.0 * f, 0.0, 0.0]) for f in range(len(frames))]
    mw = np.concatenate([m + np.array([*s, 0.0], dtype=np.float32) for (m, _), s in zip(frames, shift)]).astype(np.float32)
    poses = np.stack([np.concatenate([s, [0, 0, 0, 1]]) for s in shift]).astype(np.float64)
    gm = capi.Map(mw)
    h.attach_map(gm)
    kg, fk = h.process_nodes(poses, np.concatenate([q for _, q in frames]), qo, want_frame_keep=True)
    nv, nfl, nrj = h.node_stats()
    for f, (_, q) in enumerate(frames):
        voi, idx = oracle_mod.fetch_voi(mw, poses[f], p.max_range)
        o = oracle_mod.Oracle(p)
        o.run(voi, q)
        assert len(o.planes()) == want[f]
        ok = np.ones(len(mw), dtype=np.uint8)
        ok[idx[_okeep(o, len(voi)) == 0]] = 0
        assert np.array_equal(fk[f], ok), ("nodes", want[f])
        assert nv[f] == len(voi) and nfl[f] == want[f] and nrj[f] == int((ok == 0).sum())
    assert np.array_equal(kg, fk.min(axis=0))
    h.close()
    gm.close()


def test_k2_windows_frames_and_nodes_unfused(capi, oracle_mod, monkeypatch):
    """The same windows through the unfused mask-mode path: k3_srt, then k2_scatter_win over K3's flagged slots."""
    monkeypatch.setenv("ERASOR_B200_UNFUSED_SRT", "1")          # read when the handle is created
    test_k2_windows_frames_and_nodes(capi, oracle_mod)


# ---- a dense map end to end ------------------------------------------------------------------------------------------------------
def dense_frame(small_workload, n_target: int = 6_000_000, seed: int = 5):
    """large_scale_05's geometry on a dense VoI: a frame of the small workload cropped to 30 m, replicated with jitter (the way
    test_full_size_dense_voi_properties builds its 50 M points, at a size the oracle handles)."""
    base, q, _, _ = small_workload["frames"][2]
    r2 = base[:, 0].astype(np.float64) ** 2 + base[:, 1].astype(np.float64) ** 2
    base = base[r2 < 30.0 ** 2]
    reps = int(np.ceil(n_target / len(base)))
    rng = np.random.default_rng(seed)
    m = np.tile(base, (reps, 1))
    m[:, :3] += ((rng.random((len(m), 3)) - 0.5) * np.array([0.19, 0.19, 0.02])).astype(np.float32)
    return m.astype(np.float32), q


@pytest.mark.parametrize("version,skip_voxelize", [(3, 1), (2, 1), (3, 0)])
def test_dense_map_cloud_mode(capi, oracle_mod, small_workload, version, skip_voxelize):
    p = P.preset("large_scale_05").replace(skip_voxelize=skip_voxelize, version=version)
    m, q = dense_frame(small_workload)
    o = _cloud_mode(capi, oracle_mod, p, m, q, ("dense", version, skip_voxelize))
    assert max(x["n_points"] for x in o.planes()) > C.K4_C_CAP, "some flagged bin must take class C's global scratch"
    if version == 3 and not skip_voxelize:
        _, _, cq, _ = o.bins(1)
        assert max(cq[x["bin"]] + x["n_ground"][-1] for x in o.planes()) > C.K4B_CAP, "some flagged bin must take K4b's global scratch"


def dense_world_map(small_workload, nodes, n_target: int = 6_000_000, seed: int = 9):
    """The small workload's world map cropped to 30 m around the given scene nodes and replicated with jitter, as dense_frame."""
    sc, mw = small_workload["scene"], small_workload["map_world"]
    near = np.zeros(len(mw), dtype=bool)
    for k in nodes:
        t = sc.pose7(k)[:2]
        near |= (mw[:, 0].astype(np.float64) - t[0]) ** 2 + (mw[:, 1].astype(np.float64) - t[1]) ** 2 < 30.0 ** 2
    base = mw[near]
    reps = int(np.ceil(n_target / len(base)))
    rng = np.random.default_rng(seed)
    m = np.tile(base, (reps, 1))
    m[:, :3] += ((rng.random((len(m), 3)) - 0.5) * np.array([0.19, 0.19, 0.02])).astype(np.float32)
    return m.astype(np.float32)


def test_dense_map_sequential_updater(capi, oracle_mod, small_workload):
    """Three nodes of the device-resident caller on a dense map against the oracle's caller loop (version 3, in-bin voxelisation):
    the path runs on device-pointer inputs from the fused fetch_VoI and scan voxeliser, and one handle's scratch buffers and
    class-C state carry over from node to node.  The oracle run on each node's VoI shows that class C and K4b both take their
    global-scratch paths."""
    ep = P.preset("large_scale_05").replace(version=3, skip_voxelize=0)
    up = P.updater_preset("large_scale_05")
    up.removal_interval = 1
    sc = small_workload["scene"]
    k0 = small_workload["frames"][2][2]
    nodes = [k0, k0 + 1, k0 + 2]
    mw = dense_world_map(small_workload, nodes)
    o = oracle_mod.OracleUpdater(up, ep, mw)
    u = capi.Updater(up, ep, mw)
    over_c = over_b = 0
    for k in nodes:
        pose, scan = sc.pose7(k), sc.scan(k, n_beams=32, n_az=900, seed_offset=17)
        assert o.callback_node(k, pose, scan) and u.process_node(k, pose, scan)
        for name in ("QUERY_VOI", "MAP_VOI", "OUTSKIRTS", "MAP_REJECTED", "MAP_ARRANGED"):
            assert _u32_equal(u.cloud(getattr(u, name)), o.cloud(getattr(o, name))[0]), f"node {k}: {name}"
        e = oracle_mod.Oracle(ep)
        e.run(o.cloud(o.MAP_VOI)[0], o.cloud(o.QUERY_VOI)[0])
        _, _, cq, _ = e.bins(1)
        over_c += sum(x["n_points"] > C.K4_C_CAP for x in e.planes())
        over_b += sum(cq[x["bin"]] + x["n_ground"][-1] > C.K4B_CAP for x in e.planes())
    assert over_c > 0 and over_b > 0, (over_c, over_b)
    assert len(o.cloud(o.TOTAL_MAP_REJECTED)[0]) > 0
    u.close()
    o.close()
