"""GPU: the captured step graphs of the mask modes (erasor_capi.cu submit()).  A handle that replays cached CUDA graphs must return,
byte for byte, what a handle that launches every step plainly (ERASOR_B200_NO_GRAPH=1) returns -- masks, node, frame and sweep
counters, inserts and kernel launch counts -- over one interleaved sequence that replays graphs across changed sweep settings, fold
on and off, geometry sweeps (the handle's geometry alone, two geometries, one geometry changed), frame_keep null and non-null,
inserts toggled, and host and device pointers.  And erasor_profile_k1 after a replayed step rebins that step's query, not the query
of the step captured last."""
import numpy as np
import pytest

from erasor_b200 import params as P

pytestmark = pytest.mark.gpu
S1 = [dict(scan_ratio_threshold=0.10), dict(scan_ratio_threshold=0.20)]
S2 = [dict(scan_ratio_threshold=0.15), dict(scan_ratio_threshold=0.25, minimum_num_pts=3)]
G1 = [dict(gf_dist_thr=0.10), dict(gf_dist_thr=0.20)]
G2 = [dict(gf_dist_thr=0.10), dict(gf_dist_thr=0.30)]
T0 = [dict(scan_ratio_threshold=0.10), dict(scan_ratio_threshold=0.20, gf_dist_thr=0.30)]     # the handle's geometry only
T1 = [dict(scan_ratio_threshold=0.20), dict(num_rings=20, num_sectors=108)]
T2 = [dict(scan_ratio_threshold=0.20), dict(num_rings=20, num_sectors=90)]                      # T1 with one geometry changed


@pytest.fixture(scope="module")
def capi():
    from erasor_b200 import capi as C
    return C


def _pose(scene, frame):
    return np.ascontiguousarray(scene.pose7(frame[2]), dtype=np.float64).reshape(1, 7)


def _tables(capi, h):
    """K1's count / min / max tables of both clouds of a one-node batch, as bytes (empty bins are NaN)"""
    return [np.concatenate([np.asarray(a).view(np.uint32) for a in h.get_bins(c, per_point=False)[1:]]) for c in (capi.CLOUD_MAP, capi.CLOUD_QUERY)]


def test_graph_replay_equals_plain_launches(capi, small_workload, monkeypatch):
    import torch
    p = P.preset("seq_05")
    mw, frames, scene = small_workload["map_world"], small_workload["frames"], small_workload["scene"]
    n = len(mw)
    picks, others = [0, 2], [3, 5]
    # node batches A and B: the same geometry (B's queries resized to A's), so both stay in the graph cache
    qa = [frames[i][1] for i in picks]
    qb = [np.resize(frames[j][1], q.shape) for j, q in zip(others, qa)]
    qo = np.cumsum([0] + [len(q) for q in qa]).astype(np.uint64)
    poses = {k: np.ascontiguousarray(np.concatenate([_pose(scene, frames[i]) for i in ids])) for k, ids in (("A", picks), ("B", others))}
    QA, QB = np.ascontiguousarray(np.concatenate(qa)), np.ascontiguousarray(np.concatenate(qb))
    dev = {"A": torch.from_numpy(QA).cuda(), "B": torch.from_numpy(QB).cuda(), "Axyz": torch.from_numpy(np.ascontiguousarray(QA[:, :3])).cuda()}
    pin = {"A": torch.from_numpy(QA).pin_memory(), "B": torch.from_numpy(QB).pin_memory()}
    # one batch of (map_voi, query_voi) pairs with its fold index
    MV = np.ascontiguousarray(np.concatenate([frames[i][0] for i in picks]))
    mo = np.cumsum([0] + [len(frames[i][0]) for i in picks]).astype(np.uint64)
    VI = np.concatenate([frames[i][3] for i in picks]).astype(np.uint32)
    fdev = dict(M=torch.from_numpy(MV).cuda(), Q=dev["A"], I=torch.from_numpy(VI.view(np.int32)).cuda())
    fpin = dict(M=torch.from_numpy(MV).pin_memory(), Q=pin["A"])

    def lane():
        h, m = capi.Handle(p), capi.Map(mw)
        h.attach_map(m)
        L = dict(h=h, m=m, fk=torch.empty(2 * n, dtype=torch.uint8, device="cuda"), out=torch.empty(n, dtype=torch.uint8, device="cuda"),
                 hfk=torch.empty(2 * n, dtype=torch.uint8).pin_memory(), hout=torch.empty(n, dtype=torch.uint8).pin_memory(),
                 vk=torch.empty(3 * n, dtype=torch.uint8, device="cuda"), gk=torch.empty(n, dtype=torch.uint8, device="cuda"),
                 keep=torch.empty(int(mo[-1]), dtype=torch.uint8, device="cuda"), hkeep=torch.empty(int(mo[-1]), dtype=torch.uint8).pin_memory())
        h.reset_keep_mask(L["gk"].data_ptr(), n)
        return L

    graphed = lane()
    monkeypatch.setenv("ERASOR_B200_NO_GRAPH", "1")
    plain = lane()
    monkeypatch.delenv("ERASOR_B200_NO_GRAPH")

    def node(L, q, kind="device", fk=True, out=True):
        h = L["h"]
        host = kind == "host"
        qptr = (pin[q] if host else dev[q + ("xyz" if kind == "packed" else "")]).data_ptr()
        fkb, outb = (L["hfk"], L["hout"]) if host else (L["fk"], L["out"])
        ptr_kind = (capi.PTR_HOST if host else capi.PTR_DEVICE) | (capi.PTR_QUERY_XYZ if kind == "packed" else 0)
        h.process_nodes_ptr(poses[q], qptr, qo, 0.0, fkb.data_ptr() if fk else 0, outb.data_ptr() if out else 0, ptr_kind)
        r = dict(map=L["m"].get_keep(), stats=np.stack(h.node_stats()))
        if fk:
            r["fk"] = fkb.cpu().numpy()
        if out:
            r["out"] = outb.cpu().numpy()
        if L.get("inserts"):
            r["ins"], r["ins_off"] = h.node_inserts()
        return r

    def sweep(L, q, settings, ex=False, tune=False):
        h = L["h"]
        V = len(settings)
        h.reset_keep_mask(L["vk"].data_ptr(), V * n)
        fn = h.process_nodes_tune if tune else h.process_nodes_sweep_ex if ex else h.process_nodes_sweep
        fn(poses[q], dev[q].data_ptr(), qo, settings, L["vk"].data_ptr())
        return dict(vk=L["vk"][:V * n].cpu().numpy(), sweep=np.stack(h.sweep_stats()), stats=np.stack(h.node_stats()))

    def batch(L, kind="device", fold=True):
        h = L["h"]
        src, keep = (fpin, L["hkeep"]) if kind == "host" else (fdev, L["keep"])
        h.process_frames_ptr(src["M"].data_ptr(), mo, src["Q"].data_ptr(), qo, keep.data_ptr(), capi.PTR_HOST if kind == "host" else capi.PTR_DEVICE,
                             fold=(fdev["I"].data_ptr(), L["gk"].data_ptr(), n) if fold else None)
        return dict(keep=keep.cpu().numpy(), gk=L["gk"].cpu().numpy(), stats=np.stack(h.frame_stats()))

    def inserts(L, on):
        L["h"].set_node_inserts(on)
        L["inserts"] = on
        return {}

    seq = [
        (node, ("A",), {}), (node, ("B",), {}), (node, ("A",), {}), (node, ("A",), dict(fk=False)), (node, ("B",), dict(fk=False, out=False)),
        (node, ("A",), dict(kind="host")), (node, ("B",), dict(kind="host", fk=False)), (node, ("A",), dict(kind="host")),
        (node, ("A",), dict(kind="packed")), (node, ("A",), {}), (node, ("B",), dict(fk=False)),
        (sweep, ("A", S1), {}), (sweep, ("B", S1), {}), (sweep, ("A", S2), {}), (sweep, ("A", S1), {}), (sweep, ("B", S2), {}),
        (sweep, ("A", G1), dict(ex=True)), (sweep, ("A", G2), dict(ex=True)), (sweep, ("A", G1), dict(ex=True)),
        (sweep, ("A", T0), dict(tune=True)), (sweep, ("A", T1), dict(tune=True)), (sweep, ("A", T1), dict(tune=True)),
        (sweep, ("A", T2), dict(tune=True)), (sweep, ("A", T2), dict(tune=True)), (sweep, ("B", T1), dict(tune=True)),
        (node, ("A",), {}), (inserts, (True,), {}), (node, ("A",), {}), (inserts, (False,), {}), (node, ("A",), {}),
        (inserts, (True,), {}), (node, ("A",), {}), (node, ("B",), dict(fk=False)), (inserts, (False,), {}), (node, ("B",), dict(fk=False)),
        (inserts, (True,), {}), (node, ("B",), dict(fk=False)), (node, ("A",), dict(kind="host")), (inserts, (False,), {}),
        (node, ("A",), dict(kind="host")), (node, ("A",), {}),
        (batch, (), {}), (batch, (), dict(fold=False)), (batch, (), dict(kind="host")), (batch, (), {}), (batch, (), dict(kind="host", fold=False)),
        (batch, (), dict(fold=False)), (batch, (), dict(kind="host")),
    ]
    for i, (fn, args, kw) in enumerate(seq):
        a, b = fn(graphed, *args, **kw), fn(plain, *args, **kw)
        what = f"step {i}: {fn.__name__}{args} {kw}"
        assert a.keys() == b.keys(), what
        for k in a:
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), f"{what}: {k} differs"
        assert graphed["h"].kernel_launch_count() == plain["h"].kernel_launch_count(), f"{what}: kernel launch counts differ"


def test_profile_k1_rebins_the_step_that_ran(capi, small_workload):
    """One-node batches on device query buffers A and B (same size: one set of chunk descriptors, so both graphs stay cached), then
    A and B again as replays: K1's profiling build must rebuild the tables of the step that ran."""
    import torch
    p = P.preset("seq_05")
    mw, frames, scene = small_workload["map_world"], small_workload["frames"], small_workload["scene"]
    qa = np.ascontiguousarray(frames[0][1])
    qb = np.ascontiguousarray(np.resize(frames[3][1], qa.shape))
    qo = np.array([0, len(qa)], dtype=np.uint64)
    bufs = dict(A=(torch.from_numpy(qa).cuda(), _pose(scene, frames[0])), B=(torch.from_numpy(qb).cuda(), _pose(scene, frames[3])))
    h, m = capi.Handle(p), capi.Map(mw)
    h.attach_map(m)
    seen = {}
    for name in "ABABA":
        q, pose = bufs[name]
        h.process_nodes_ptr(pose, q.data_ptr(), qo, 0.0, 0, 0, capi.PTR_DEVICE)
        before = _tables(capi, h)
        h.k1_profile()
        after = _tables(capi, h)
        for c, (x, y) in enumerate(zip(before, after)):
            assert np.array_equal(x, y), f"{name}: erasor_profile_k1 changed the {('map', 'query')[c]} tables"
        seen.setdefault(name, before[1])
        assert np.array_equal(seen[name], before[1])
    assert not np.array_equal(seen["A"], seen["B"]), "A and B must bin differently for this test to see a stale query"
