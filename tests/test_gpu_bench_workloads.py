"""GPU: bench.py's workloads (bench.CONFIGS: seq05, dense, synthetic40x360; 20 frames each, from bench.load_workload) against the
oracle, frame by frame, in every submission form bench.py times, and K1's tables and the Scan Ratio Test's flagged counts on the
same frames against the float64 reference of tests/test_erasor_float64_reference.py.

1. The oracle (oracle_py.fetch_voi + Oracle.run) gives every frame's keep mask on global map indices, its counters
   (len(voi), len(planes), len(map_rejected)) -- what node_stats() returns -- and the folded mask, the AND over the frames.
   It runs once per config in a process pool, one frame per task, on every usable core.
2. The device, in each form bench.py times, against those results:
   - the final step: one synchronous process_nodes_ptr with a device frame_keep [F][N];
   - `value`: four handles on one resident map, asynchronous submissions round-robin (lanes[i % L].wait() first), CUDA graphs
     replayed over 2 L + 1 device query buffers.  The buffers hold different content at identical offsets (copy k: the frames
     rolled by k, each query np.resize'd to its slot's length), so a graph replayed with another buffer's pointer gives a wrong
     mask or wrong counters;
   - `e2e` and `e2e_xyzi`: the same loop with pinned host queries (packed x y z, then x y z i) and a pinned keep output per lane;
   - the per-kernel timing mode (reset_kernel_times(True): no graphs, CUDA events) on one lane;
   - the `configs` block: the seq_00 / 01 / 02 / 07 presets on the seq-05 twin's map, as sweep_presets runs them;
   - ranks on one GPU: seq05 sharded over 2 and 4 ranks, the ranks' masks AND-ed by and_keep_masks.
3. Each frame as a one-node process_nodes call: the map's and the query's count / min / max tables against the float64 polar
   binning, and the flagged-bin count against the float64 Scan Ratio Test, with the reference's EPS_POS band for the float32
   transform of the map to the body frame (the poses are yaw-only at z = 0, so heights cross unchanged).  Counts, minima and
   maxima are exact in every bin no point within a band can reach; a reachable bin's count lies between its certain and its
   possible points.  The flagged count equals the reference's in every frame where no band outcome can change a bin's verdict,
   and lies between the least and the most favourable outcomes elsewhere.

Oracle time per config, on the 8-core host of an H100 80GB HBM3 machine (700 W power limit), one spawned process per core,
starting the workers and reading the cached workload included: seq05 9.2 s (140 frames: 3 rolled copies and the 4 presets of
the configs block), dense 9.3 s (60 frames), synthetic40x360 9.2 s (20 frames: its queries are all one length, so its rolled
copy holds the same frames).  The whole file took 187 s there, generating the workloads into bench.py's cache included.
"""
import dataclasses
import math
import multiprocessing as mp
import time

import numpy as np
import pytest

import bench
from erasor_b200 import params as P
from test_erasor_float64_reference import EPS32, bin_stats, polar, srt_status

pytestmark = pytest.mark.gpu

FRAMES = bench.FRAMES_PER_PASS
LANES = 4
N_BUFS = 2 * LANES + 1                 # coprime with LANES: every lane meets every buffer, and so every content variant
VARIANTS = {"seq05": 3, "dense": 3, "synthetic40x360": 2}
SWEEP_PRESETS = ("seq_00", "seq_01", "seq_02", "seq_07")


# ================================================================================================================================
# the oracle, one frame per task in a process pool (bench.py --impl reference's pattern)
# ================================================================================================================================
_W = {}


def _oracle_task(task):
    """task = (config, frames in the workload, preset or None for the config's own, source frame j, query length): the oracle's
    rejected global indices and node_stats() triple for frame j, its query np.resize'd to the length.  A worker reads the
    workload from bench.py's cache, which the parent process has filled."""
    from oracle import oracle_py
    config, total, preset, j, n_q = task
    if (config, total) not in _W:
        _W[(config, total)] = bench.load_workload(config, 0, 1, total)
    p, map_world, poses, qs = _W[(config, total)]
    if preset is not None:
        p = P.preset(preset).replace(skip_voxelize=1)
    voi, idx = oracle_py.fetch_voi(map_world, poses[j], p.max_range)
    o = oracle_py.Oracle(p)
    o.run(voi, np.resize(qs[j], (n_q, 4)))
    _, rej = o.cloud(o.MAP_REJECTED)
    out = (idx[rej].astype(np.uint32), (len(voi), len(o.planes()), len(rej)))
    o.close()
    return out


def run_oracle(config, total, jobs):
    """jobs: {preset or None: [(j, n_q), ...]} -> {preset or None: {(j, n_q): (rejected indices, stats)}}.  Spawned workers, not
    forked ones: the parent holds CUDA and pytest threads."""
    tasks = [(config, total, preset, j, n_q) for preset, pairs in jobs.items() for j, n_q in pairs]
    cores, _ = bench.usable_cores()
    with mp.get_context("spawn").Pool(max(1, min(cores, len(tasks)))) as pool:
        res = pool.map(_oracle_task, tasks, chunksize=1)
    out = {preset: {} for preset in jobs}
    for (_, _, preset, j, n_q), r in zip(tasks, res):
        out[preset][(j, n_q)] = r
    return out


def keep_of(n, rej):
    k = np.ones(n, dtype=np.uint8)
    k[rej] = 0
    return k


def offsets(qs):
    return np.cumsum([0] + [len(q) for q in qs]).astype(np.uint64)


@dataclasses.dataclass
class Variant:
    """Copy k of a workload: frame i is source frame (i + k) % F, its query resized to slot i's length."""
    poses: np.ndarray
    Q: np.ndarray                      # [sum of slot lengths, 4] float32
    fk: np.ndarray                     # oracle per-frame keep masks [F, N] uint8
    stats: np.ndarray                  # oracle (voi, flagged, rejected) [F, 3]
    fold: np.ndarray                   # AND over the frames


def make_variants(map_world, poses, qs, n_var, results):
    n, F = len(map_world), len(qs)
    out = []
    for k in range(n_var):
        src = [(i + k) % F for i in range(F)]
        res = [results[(j, len(qs[i]))] for i, j in enumerate(src)]
        fk = np.stack([keep_of(n, r[0]) for r in res])
        out.append(Variant(poses=np.ascontiguousarray(poses[src], dtype=np.float64),
                           Q=np.ascontiguousarray(np.concatenate([np.resize(qs[j], qs[i].shape) for i, j in enumerate(src)]), dtype=np.float32),
                           fk=fk, stats=np.array([r[1] for r in res], dtype=np.int64), fold=fk.min(axis=0)))
    return out


def variant_pairs(qs, n_var):
    F = len(qs)
    return sorted({((i + k) % F, len(qs[i])) for k in range(n_var) for i in range(F)})


@pytest.fixture(scope="module", params=list(bench.CONFIGS))
def workload(request, oracle_mod):
    config = request.param
    p, map_world, poses, qs = bench.load_workload(config, 0, 1, FRAMES)
    n_var = VARIANTS[config]
    jobs = {None: variant_pairs(qs, n_var)}
    if config == "seq05":              # the configs block's presets on the same twin
        jobs.update({name: [(j, len(q)) for j, q in enumerate(qs)] for name in SWEEP_PRESETS})
    t0 = time.perf_counter()
    res = run_oracle(config, FRAMES, jobs)
    print(f"\n{config}: oracle over {sum(len(v) for v in jobs.values())} frames in {time.perf_counter() - t0:.1f} s")
    w = dict(config=config, p=p, map_world=map_world, poses=np.ascontiguousarray(poses), qs=qs, qo=offsets(qs),
             variants=make_variants(map_world, poses, qs, n_var, res[None]))
    w["presets"] = {name: make_variants(map_world, poses, qs, 1, res[name])[0] for name in SWEEP_PRESETS if name in res}
    v0 = w["variants"][0]
    assert (v0.fk == 0).any(), "the workload must reject something"
    for a in w["variants"][1:]:          # the copies differ: in their counters always, and in content unless every slot is one size
        assert not np.array_equal(a.stats, v0.stats)
    yield w


# ================================================================================================================================
# the device in bench.py's forms
# ================================================================================================================================
def _check_stats(h, want, tag):
    nv, nf, nr = h.node_stats()
    got = np.stack([nv, nf, nr], 1).astype(np.int64)
    bad = np.nonzero((got != want).any(1))[0]
    assert not len(bad), (tag, "node_stats differ in frames", bad.tolist(), got[bad].tolist(), want[bad].tolist())


def _check_keep(got, want, tag):
    assert got.shape == want.shape
    d = np.count_nonzero(got != want)
    assert d == 0, (tag, f"{d} points differ", int((got == 0).sum()), int((want == 0).sum()))


@pytest.fixture
def lanes(workload):
    from erasor_b200 import capi
    gm = capi.Map(workload["map_world"], device=0)
    hs = [capi.Handle(workload["p"], device=0) for _ in range(LANES)]
    for h in hs:
        h.attach_map(gm)
    yield gm, hs
    for h in hs:
        h.wait()
        h.close()
    gm.close()


def test_final_step(workload, lanes):
    """What bench.py runs after its timed blocks: one synchronous call with a device frame_keep [F][N]."""
    import torch
    from erasor_b200 import capi
    gm, hs = lanes
    v0, n = workload["variants"][0], len(workload["map_world"])
    dQ = torch.from_numpy(v0.Q).cuda()
    dFK = torch.empty((FRAMES, n), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for rep in range(2):               # the second call replays the captured graph
        gm.reset_keep()
        dFK.fill_(7)
        torch.cuda.synchronize()
        hs[0].process_nodes_ptr(v0.poses, dQ.data_ptr(), workload["qo"], 0.0, dFK.data_ptr(), 0, capi.PTR_DEVICE)
        fk = dFK.cpu().numpy()
        for f in range(FRAMES):
            _check_keep(fk[f], v0.fk[f], (workload["config"], rep, "frame", f))
        _check_stats(hs[0], v0.stats, (workload["config"], rep))
        _check_keep(gm.get_keep(), v0.fold, (workload["config"], rep, "fold"))


def _round_robin(workload, gm, hs, submit, n_lanes, label, on_round=None):
    """bench.py's timed() loop: a warm-up that meets every (lane, buffer) pair, reset_keep, then rounds of submissions, each
    checked after wait_all: the map's keep is the AND over the copies submitted since the reset, and every lane's counters are
    those of the copy it ran last."""
    V = workload["variants"]
    var_of = lambda i: (i % N_BUFS) % len(V)
    warmup = N_BUFS * n_lanes
    for i in range(warmup):
        hs[i % n_lanes].wait()
        submit(i, i % n_lanes)
    for h in hs[:n_lanes]:
        h.wait()
    i = warmup
    for r, (reset, count) in enumerate([(True, 1), (False, n_lanes), (False, N_BUFS), (True, n_lanes + 1), (False, 2 * N_BUFS + 3)]):
        if reset:
            gm.reset_keep()
            seen, last = set(), {}
        for _ in range(count):
            lane = i % n_lanes
            hs[lane].wait()
            submit(i, lane)
            seen.add(var_of(i))
            last[lane] = var_of(i)
            i += 1
        for h in hs[:n_lanes]:
            h.wait()
        tag = (workload["config"], label, "round", r, sorted(seen))
        _check_keep(gm.get_keep(), np.min([V[v].fold for v in sorted(seen)], axis=0), tag)
        for lane, v in last.items():
            _check_stats(hs[lane], V[v].stats, tag + ("lane", lane, "copy", v))
        if on_round is not None:
            on_round(last, tag)
    assert len(seen) == len(V)


def _device_buffers(workload):
    import torch
    V = workload["variants"]
    bufs = [torch.from_numpy(V[b % len(V)].Q).cuda() for b in range(N_BUFS)]
    torch.cuda.synchronize()
    return bufs


def test_value_lanes(workload, lanes):
    """bench.py's `value` form: four lanes, device queries, CUDA graphs replayed over 2 L + 1 buffers of different content."""
    from erasor_b200 import capi
    gm, hs = lanes
    V, qo = workload["variants"], workload["qo"]
    dQ = _device_buffers(workload)

    def submit(i, lane):
        b = i % N_BUFS
        hs[lane].process_nodes_ptr(V[b % len(V)].poses, dQ[b].data_ptr(), qo, 0.0, 0, 0, capi.PTR_DEVICE, asynchronous=True)

    _round_robin(workload, gm, hs, submit, LANES, "value")


@pytest.mark.parametrize("form", ["e2e", "e2e_xyzi"])
def test_e2e_lanes(workload, lanes, form):
    """bench.py's `e2e` forms: pinned host queries (packed x y z, or x y z i) and a pinned host keep output per lane."""
    import torch
    from erasor_b200 import capi
    gm, hs = lanes
    V, qo, n = workload["variants"], workload["qo"], len(workload["map_world"])
    packed = form == "e2e"
    hQ = [torch.from_numpy(np.ascontiguousarray(V[b % len(V)].Q[:, :3]) if packed else V[b % len(V)].Q).pin_memory() for b in range(N_BUFS)]
    hK = [torch.empty(n, dtype=torch.uint8).pin_memory() for _ in range(LANES)]
    kind = capi.PTR_HOST | (capi.PTR_QUERY_XYZ if packed else 0)

    def submit(i, lane):
        b = i % N_BUFS
        hs[lane].process_nodes_ptr(V[b % len(V)].poses, hQ[b].data_ptr(), qo, 0.0, 0, hK[lane].data_ptr(), kind, asynchronous=True)

    def own_zeros(last, tag):
        for lane, v in last.items():   # a lane's copy of the map's keep holds at least the zeros of the frames it ran
            k = hK[lane].numpy()
            assert np.all(k[V[v].fold == 0] == 0), tag + ("lane", lane)

    _round_robin(workload, gm, hs, submit, LANES, form, own_zeros)


def test_kernel_timing_mode(workload, lanes):
    """bench.py's per-kernel CUDA-event block: one lane, graphs off, events recorded around every kernel."""
    from erasor_b200 import capi
    gm, hs = lanes
    V, qo = workload["variants"], workload["qo"]
    dQ = _device_buffers(workload)
    hs[0].reset_kernel_times(True)

    def submit(i, lane):
        b = i % N_BUFS
        hs[lane].process_nodes_ptr(V[b % len(V)].poses, dQ[b].data_ptr(), qo, 0.0, 0, 0, capi.PTR_DEVICE, asynchronous=True)

    _round_robin(workload, gm, hs, submit, 1, "kernel times")
    for k in (1, 2, 4):                # K1, K2 and R-GPF; the Scan Ratio Test (3) runs inside K2
        ms, count = hs[0].kernel_time_ms(k)
        assert count > 0 and ms > 0.0, (k, ms, count)
    hs[0].reset_kernel_times(False)


@pytest.mark.parametrize("workload", ["seq05"], indirect=True)
def test_configs_block(workload):
    """bench.py's `configs` block (sweep_presets): the seq 00 / 01 / 02 / 07 presets on the seq-05 twin's map, three synchronous
    steps, then asynchronous ones."""
    import torch
    from erasor_b200 import capi
    v0 = workload["variants"][0]
    dQ = torch.from_numpy(v0.Q).cuda()
    gm = capi.Map(workload["map_world"], device=0)
    folds = []
    for name in SWEEP_PRESETS:
        want = workload["presets"][name]
        folds.append(want.fold)
        h = capi.Handle(P.preset(name).replace(skip_voxelize=1), device=0)
        h.attach_map(gm)
        gm.reset_keep()
        torch.cuda.synchronize()
        for step in range(3):
            h.process_nodes_ptr(workload["poses"], dQ.data_ptr(), workload["qo"], 0.0, 0, 0, capi.PTR_DEVICE)
            _check_stats(h, want.stats, (name, "sync", step))
            _check_keep(gm.get_keep(), want.fold, (name, "sync", step))
        gm.reset_keep()
        for step in range(4):
            h.process_nodes_ptr(workload["poses"], dQ.data_ptr(), workload["qo"], 0.0, 0, 0, capi.PTR_DEVICE, asynchronous=True)
        h.wait()
        _check_stats(h, want.stats, (name, "async"))
        _check_keep(gm.get_keep(), want.fold, (name, "async"))
        h.close()
    assert len({f.tobytes() for f in folds}) == len(folds), "the presets must reject different points"
    gm.close()


@pytest.mark.parametrize("workload", ["seq05"], indirect=True)
@pytest.mark.parametrize("world", [2, 4])
def test_ranks_on_one_gpu(workload, world, oracle_mod):
    """seq05 sharded over `world` ranks as bench.py --gpus shards it, every rank on its own map and lane of one GPU; the ranks'
    masks AND-ed by and_keep_masks (the local half of erasor_allgather_and_keep) equal the oracle over all world x 20 frames."""
    import torch
    from erasor_b200 import capi
    p, mw_all, poses_all, qs_all = bench.load_workload("seq05", 0, 1, world * FRAMES)
    res = run_oracle("seq05", world * FRAMES, {None: [(j, len(q)) for j, q in enumerate(qs_all)]})[None]
    want = np.min([keep_of(len(mw_all), res[(j, len(q))][0]) for j, q in enumerate(qs_all)], axis=0)
    n = len(mw_all)
    masks = torch.empty((world, n), dtype=torch.uint8, device="cuda")
    shards = []
    for r in range(world):
        pr, mw, poses, qs = bench.load_workload("seq05", r, world, FRAMES)
        assert pr == p and np.array_equal(mw, mw_all)
        mine = [int(np.nonzero((poses_all == pose).all(1))[0][0]) for pose in poses]    # which frames of the trajectory rank r got
        assert all(np.array_equal(q, qs_all[j]) for j, q in zip(mine, qs)), ("rank", r, world)
        shards.append(mine)
        gm = capi.Map(mw, device=0)
        h = capi.Handle(p, device=0)
        h.attach_map(gm)
        dQ = torch.from_numpy(np.ascontiguousarray(np.concatenate(qs))).cuda()
        torch.cuda.synchronize()
        P7 = np.ascontiguousarray(poses, dtype=np.float64)
        for step in range(2):
            h.process_nodes_ptr(P7, dQ.data_ptr(), offsets(qs), 0.0, 0, 0, capi.PTR_DEVICE, asynchronous=True)
            h.wait()
        _check_stats(h, np.array([res[(j, len(q))][1] for j, q in zip(shards[-1], qs)]), ("rank", r, world))
        got = gm.get_keep()
        _check_keep(got, np.min([keep_of(n, res[(j, len(qs_all[j]))][0]) for j in shards[-1]], axis=0), ("rank", r, world))
        masks[r] = torch.from_numpy(got).cuda()
        h.close()
        gm.close()
    assert sorted(sum(shards, [])) == list(range(world * FRAMES)), "the shards partition the frames"
    h = capi.Handle(p, device=0)
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    h.and_keep_masks(masks.data_ptr(), world, n, out.data_ptr())
    h.synchronize()
    _check_keep(out.cpu().numpy(), want, ("and_keep_masks", world))
    h.close()


# ================================================================================================================================
# float64: K1's tables and the Scan Ratio Test's flagged count on the bench frames
# ================================================================================================================================
def _possible_stats(p, exact, cand, z):
    """Per bin: the stats of the points certainly in it, and of every point that may be in it (a point within a band counts
    for each of its candidate bins).  Returns (certain cnt, mn, mx), (possible cnt, mn, mx), touched-bin mask."""
    band = ~(cand == cand[:, :1]).all(1)
    certain = bin_stats(p, np.where(band, -1, exact), z)
    c = np.sort(cand[band], axis=1)
    first = np.ones(c.shape, dtype=bool)
    first[:, 1:] = c[:, 1:] != c[:, :-1]
    pb = c[first]
    pz = np.repeat(np.asarray(z, np.float64)[band], first.sum(1))
    possible = bin_stats(p, pb, pz)
    return certain, possible, possible[0] > 0


def _bounds(certain, possible, most):
    """Bin stats that make a bin most (most=True) or least likely to be handed to R-GPF, from the map's or the query's
    certain and possible points: every test of the Scan Ratio Test is monotone in the count and the height spread."""
    (cc, cmn, cmx), (pc, pmn, pmx) = certain, possible
    if most:                           # all possible points in; the spread is the union's
        return cc + pc, np.minimum(cmn, pmn), np.maximum(cmx, pmx)
    return cc, cmn, cmx


def _query_bounds(certain, possible, most):
    (cc, cmn, cmx), (pc, pmn, pmx) = certain, possible
    if most:                           # as many points as may be there, the smallest spread (0 if no point is certain)
        mn = np.where(cc > 0, cmn, 0.0)
        return cc + pc, mn, np.where(cc > 0, cmx, 0.0)
    return cc, np.minimum(cmn, pmn), np.maximum(cmx, pmx)


def body_frame(map_world, idx, pose):
    """The VoI in the body frame, in float64 from the float32 world points (yaw-only poses at z = 0: z stays the world z)."""
    yaw = 2.0 * math.atan2(pose[5], pose[6])
    c, s = math.cos(yaw), math.sin(yaw)
    w = map_world[idx]
    dx, dy = w[:, 0].astype(np.float64) - pose[0], w[:, 1].astype(np.float64) - pose[1]
    return np.stack([c * dx + s * dy, -s * dx + c * dy, w[:, 2].astype(np.float64)], 1)


def check_frame(p, body, q, eps_pos, tables, n_flagged, tag):
    """One frame's K1 tables ((min, max, count) of the map and of the query, as get_bins(per_point=False) returns them) and
    flagged-bin count against the float64 reference.  Returns (bins, bins decided, ambiguous Scan Ratio Test bins)."""
    stats = {}
    for name, pts, eps in (("map", body, eps_pos), ("query", q, 0.0)):
        exact, cand = polar(p, pts, eps_pos=eps)
        stats[name] = _possible_stats(p, exact, cand, pts[:, 2])
    # tables: exact in every bin no band point can reach; elsewhere the count lies between the certain and the possible
    n_bins = n_decided = 0
    for (name, (certain, possible, touched)), (mn, mx, cnt) in zip(stats.items(), tables):
        cc, cmn, cmx = certain
        occ = cnt > 0
        ok = ~touched
        bad = np.nonzero(ok & ((cnt != cc) | (occ & ((mn.astype(np.float64) != cmn) | (mx.astype(np.float64) != cmx)))))[0]
        assert not len(bad), (tag, name, "tables", len(bad), bad[:5].tolist(), cnt[bad[:5]].tolist(), cc[bad[:5]].tolist())
        inside = (cnt >= cc) & (cnt <= cc + possible[0])
        assert inside.all(), (tag, name, "counts outside the band", np.nonzero(~inside)[0][:5].tolist())
        n_bins += int((occ | touched).sum())
        n_decided += int((occ & ok).sum())
    # the Scan Ratio Test: the flagged set under the exact binning, and under the most and least favourable band outcomes
    mstat = bin_stats(p, polar(p, body)[0], body[:, 2])
    qstat = bin_stats(p, polar(p, q)[0], q[:, 2])
    _, flagged, _ = srt_status(p, mstat, qstat)
    _, hi, _ = srt_status(p, _bounds(*stats["map"][:2], True), _query_bounds(*stats["query"][:2], True))
    _, lo, _ = srt_status(p, _bounds(*stats["map"][:2], False), _query_bounds(*stats["query"][:2], False))
    assert not (lo & ~flagged).any() and not (flagged & ~hi).any(), tag
    amb = int((hi & ~lo).sum())
    if amb == 0:
        assert n_flagged == int(flagged.sum()), (tag, "flagged bins", n_flagged, int(flagged.sum()))
    else:
        assert int(lo.sum()) <= n_flagged <= int(hi.sum()), (tag, "flagged bins", n_flagged, int(lo.sum()), int(hi.sum()))
    return n_bins, n_decided, amb


def test_tables_and_flagged_counts_against_float64(workload, oracle_mod):
    from erasor_b200 import capi
    p, mw, poses, qs = workload["p"], workload["map_world"], workload["poses"], workload["qs"]
    assert (poses[:, 2] == 0).all() and (poses[:, 3:5] == 0).all(), "yaw-only poses at z = 0: the body-frame z is the world z"
    gm = capi.Map(mw, device=0)
    h = capi.Handle(p, device=0)
    h.attach_map(gm)
    n_bins = n_bins_decided = n_frames_decided = n_flagged = 0
    report = []
    for f in range(len(qs)):
        q = qs[f]
        h.process_nodes(poses[f:f + 1], q, np.array([0, len(q)], np.uint64))
        nv, nf, _ = (int(x[0]) for x in h.node_stats())
        tables = [h.get_bins(c, per_point=False)[1:] for c in (capi.CLOUD_MAP, capi.CLOUD_QUERY)]
        _, idx = oracle_mod.fetch_voi(mw, poses[f], p.max_range)
        assert nv == len(idx), (f, nv, len(idx))
        eps_pos = 16 * EPS32 * (math.hypot(poses[f, 0], poses[f, 1]) + p.max_range)
        b, d, amb = check_frame(p, body_frame(mw, idx, poses[f]), q, eps_pos, tables, nf, (workload["config"], f))
        n_bins += b
        n_bins_decided += d
        n_frames_decided += amb == 0
        n_flagged += nf
        report.append(amb)
    h.close()
    gm.close()
    print(f"\n{workload['config']}: {n_bins_decided} of {n_bins} bins decided, {n_frames_decided} of {len(qs)} frames without an "
          f"ambiguous Scan Ratio Test bin (ambiguous bins per frame: {report})")
    assert n_bins_decided >= 0.9 * n_bins
    assert n_frames_decided >= 0.5 * len(qs) and sum(report) <= 0.001 * n_flagged
