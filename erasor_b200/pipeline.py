"""The reference's three-stage workflow in one call, ROS stripped (README "How to run": mapgen -> offline_map_updater ->
scripts/analysis_runner.py):

    nodes (erasor_b200.kitti.iter_nodes, a reference bag through read_bag_nodes, or any iterable of (seq, odom7, cloud))
      -> naive map            erasor_b200.mapgen           (src/mapgen)
      -> static map           capi.Updater, one erasor_updater_process_node per node + save_static_map
                              (OfflineMapUpdater::callback_node / save_static_map, OfflineMapUpdater.cpp:174-330)
      -> PR / RR              capi.Evaluator (device), or erasor_b200.evaluate when the updater is injected
                              (scripts/analysis_runner.py)
      -> <name>_naive_map.pcd, <name>_result.pcd (out_dir): capi.PcdCodec (device; ascii, binary or binary_compressed), or
                              write_pcd_ascii when the updater is injected

Everything heavy runs on the device behind the C ABI; this module only sequences the calls.  The updater and the voxeliser are
injectable so that tests/test_pipeline.py can drive the same code with the oracle's objects on a machine without a GPU; with an
injected updater the evaluation stays on the host as well.
"""
from __future__ import annotations

import os
from typing import Callable, Iterable, Optional, Tuple

import numpy as np

from . import evaluate, kitti, mapgen, params

Node = Tuple[int, np.ndarray, np.ndarray]


def run_offline(nodes: Iterable[Node], initial_map: np.ndarray, up, ep, make_updater: Optional[Callable] = None,
                save_voxel_size: Optional[float] = None) -> dict:
    """Feed every node to the map updater, then save_static_map.  make_updater(up, ep, initial_map) must return an object with
    process_node(seq, odom7, cloud) -> bool, save_static_map(voxel) -> cloud (capi.Updater by default: needs a CUDA device)."""
    if make_updater is None:
        from . import capi
        make_updater = lambda u, e, m: capi.Updater(u, e, m)
    upd = make_updater(up, ep, np.ascontiguousarray(initial_map, dtype=np.float32))
    seen = processed = 0
    for seq, odom, cloud in nodes:
        seen += 1
        processed += 1 if upd.process_node(int(seq), odom, cloud) else 0
    static_map = upd.save_static_map(up.map_voxel_size if save_voxel_size is None else save_voxel_size)
    if hasattr(upd, "close"):
        upd.close()
    return {"static_map": static_map, "nodes": seen, "processed_scans": processed}


def processed_nodes(nodes: Iterable[Node], removal_interval: int) -> list:
    """The nodes callback_node processes: the k-th call (1-based) unless k % removal_interval != 0 ("PASS!", :328)."""
    return [nd for k, nd in enumerate(nodes, 1) if k % int(removal_interval) == 0]


def run_frame_independent(nodes: Iterable[Node], initial_map: np.ndarray, up, ep, batch: int = 20, save_voxel_size: Optional[float] = None,
                          prepare: Optional[Callable] = None, inserts: bool = False, retest: bool = False) -> dict:
    """The frame-independent twin of run_offline: every node callback_node would process is tested against the same initial map
    (node mode, erasor_process_nodes), in batches of `batch` nodes, each batch's raw scans voxelised at query_voxel_size and moved
    to the body frame on the device in one submission (erasor_voxelize_batch); then save_static_map of the kept map.  prepare
    (optional) replaces the device query preparation: prepare(raw_xyzi, raw_offsets) -> (queries, query_offsets).  inserts: also
    put back the query points each node's static estimate holds (node-mode inserts), saved with the kept map in node order.
    retest (needs inserts): a second pass over the same batches against the re-test map M2 = kept map ++ every node's inserts
    (DESIGN.md section 8.4.1), node j seeing the kept map and the inserts of the nodes before it; the saved map is then M2 under
    the second pass's mask.  Returns run_offline's dict plus "keep", the map's keep mask after the first pass, and with retest
    "retest_keep" (M2's mask) and "retest_size" (M2's points).  Needs a CUDA device."""
    from . import capi
    if up.is_large_scale:
        raise ValueError("node mode has no large-scale windowing: use run_offline")
    if retest and not inserts:
        raise ValueError("the re-test pass tests the first pass's inserts: retest needs inserts=True")
    nodes = list(nodes)
    sel = processed_nodes(nodes, up.removal_interval)
    m = capi.Map(np.ascontiguousarray(initial_map, dtype=np.float32))
    h = capi.Handle(ep.replace(version=up.version))       # /erasor/version as the updater reads it (OfflineMapUpdater.cpp:81)
    r = None
    l2b = np.asarray(up.lidar2body, dtype=np.float64)
    leaf = up.map_voxel_size if save_voxel_size is None else save_voxel_size

    def batches():
        for b0 in range(0, len(sel), int(batch)):
            chunk = sel[b0:b0 + int(batch)]
            poses = np.stack([np.asarray(o, dtype=np.float64).reshape(7) for _, o, _ in chunk])
            scans = [np.ascontiguousarray(c, dtype=np.float32).reshape(-1, 4) for _, _, c in chunk]
            yield b0, poses, np.concatenate(scans), np.cumsum([0] + [len(s) for s in scans]).astype(np.uint64)

    try:
        h.attach_map(m)
        h.set_node_inserts(inserts)
        for _, poses, raw, off in batches():
            if prepare is None:
                h.process_scans(poses, raw, off, up.query_voxel_size, l2b, voi_max_range=up.max_range)
            else:
                q, qo = prepare(raw, off)
                h.process_nodes(poses, q, qo, voi_max_range=up.max_range)
            if inserts:
                m.append_inserts(h)
        keep = m.get_keep()
        res = {"nodes": len(nodes), "processed_scans": len(sel), "keep": keep}
        if retest:
            r = m.create_retest()
            h.set_node_inserts(False)
            h.attach_map(r)
            for b0, poses, raw, off in batches():
                if prepare is None:
                    h.process_scans_retest(poses, raw, off, up.query_voxel_size, l2b, b0, voi_max_range=up.max_range)
                else:
                    q, qo = prepare(raw, off)
                    h.process_nodes_retest(poses, q, qo, b0, voi_max_range=up.max_range)
            res["retest_keep"] = r.get_keep()
            res["retest_size"] = r.size
            res["static_map"] = h.save_static_map(r, leaf)
        else:
            res["static_map"] = h.save_static_map(m, leaf)
    finally:
        h.close()
        if r is not None:
            r.close()
        m.close()
    return res


def sweep_frame_independent(nodes: Iterable[Node], initial_map: np.ndarray, up, ep, variants, gt: Optional[np.ndarray] = None, batch: int = 20,
                            save_voxel_size: Optional[float] = None) -> list:
    """run_frame_independent under every Scan Ratio Test setting of `variants` (1..32 dicts of scan_ratio_threshold, th_bin_max_h,
    minimum_num_pts; a missing field comes from ep) in one node-mode pass (erasor_process_nodes_sweep, DESIGN.md section 8.5): the
    binning and R-GPF run once per batch, each setting's verdicts go to its own mask.  One row per setting: its three fields, PR /
    RR / F1 of its saved map against gt (default: the initial map, as run_sequence scores) at voxelsize 0.2, the kept map points,
    the saved map's size and the flagged-bin / rejected-point totals.  Row v equals run_frame_independent(nodes, initial_map, up,
    ep.replace(**variants[v])) scored with capi.Evaluator.  Needs a CUDA device."""
    from . import capi
    return _sweep_rows(nodes, initial_map, up, ep, variants, capi.SRT_SWEEP_FIELDS, gt, batch, save_voxel_size)


def tune_frame_independent(nodes: Iterable[Node], initial_map: np.ndarray, up, ep, settings, gt: Optional[np.ndarray] = None, batch: int = 20,
                           save_voxel_size: Optional[float] = None) -> list:
    """sweep_frame_independent over settings that may also vary R-GPF's fields (1..32 dicts of capi.SRT_SWEEP_FIELDS +
    capi.GF_SWEEP_FIELDS; a missing field comes from ep) in one node-mode pass (erasor_process_nodes_sweep_ex, DESIGN.md section
    8.6): each flagged bin is sorted by z once and fitted once per distinct ground-filter tuple.  Rows as sweep_frame_independent's,
    with all eight fields.  When a setting also carries one of capi.GEOMETRY_SWEEP_FIELDS, the pass is erasor_process_nodes_tune
    (section 8.7): each batch's queries are prepared once, the map is cut to every node's VoI once and binned under every
    geometry, and the rows carry all thirteen fields.  Needs a CUDA device."""
    from . import capi
    fields = capi.SRT_SWEEP_FIELDS + capi.GF_SWEEP_FIELDS
    if any(set(dict(s)) & set(capi.GEOMETRY_SWEEP_FIELDS) for s in settings):
        fields += capi.GEOMETRY_SWEEP_FIELDS
    return _sweep_rows(nodes, initial_map, up, ep, settings, fields, gt, batch, save_voxel_size)


def _sweep_rows(nodes, initial_map, up, ep, variants, fields, gt, batch, save_voxel_size) -> list:
    """The rows of sweep_frame_independent (fields: the Scan Ratio Test's) and tune_frame_independent (all eight, or all thirteen
    with the geometry's)."""
    import torch

    from . import capi
    if up.is_large_scale:
        raise ValueError("node mode has no large-scale windowing: use run_offline")
    variants = [dict(v) for v in variants]
    if not 1 <= len(variants) <= capi.MAX_SWEEP_VARIANTS:
        raise ValueError(f"a sweep takes 1 to {capi.MAX_SWEEP_VARIANTS} settings")
    for v in variants:
        if set(v) - set(fields):
            raise ValueError(f"a sweep varies only {fields}, not {sorted(set(v) - set(fields))}")
    ex = len(fields) > len(capi.SRT_SWEEP_FIELDS)
    geo = len(fields) > len(capi.SRT_SWEEP_FIELDS + capi.GF_SWEEP_FIELDS)
    nodes = list(nodes)
    sel = processed_nodes(nodes, up.removal_interval)
    initial_map = np.ascontiguousarray(initial_map, dtype=np.float32)
    m = capi.Map(initial_map)
    h = capi.Handle(ep.replace(version=up.version))       # /erasor/version as the updater reads it (OfflineMapUpdater.cpp:81)
    run, settings_of = ((h.process_nodes_tune, h.tune_settings) if geo else (h.process_nodes_sweep_ex, h.sweep_settings) if ex
                        else (h.process_nodes_sweep, h.sweep_variants))
    V, n = len(variants), m.size
    leaf = up.map_voxel_size if save_voxel_size is None else save_voxel_size
    rows = []
    try:
        h.attach_map(m)
        keep = torch.empty(max(V * n, 1), dtype=torch.uint8, device=f"cuda:{h._device}")
        h.reset_keep_mask(keep.data_ptr(), V * n)
        flagged, rejected = np.zeros(V, dtype=np.int64), np.zeros(V, dtype=np.int64)
        l2b = np.asarray(up.lidar2body, dtype=np.float64)
        for b0 in range(0, len(sel), int(batch)):
            chunk = sel[b0:b0 + int(batch)]
            poses = np.stack([np.asarray(o, dtype=np.float64).reshape(7) for _, o, _ in chunk])
            scans = [np.ascontiguousarray(c, dtype=np.float32).reshape(-1, 4) for _, _, c in chunk]
            off = np.cumsum([0] + [len(s) for s in scans]).astype(np.uint64)
            raw = np.concatenate(scans)
            d, qo = h.voxelize_batch_ptr(raw.ctypes.data if len(raw) else 0, off, up.query_voxel_size, 0, l2b, capi.PTR_HOST)
            run(poses, d, qo, variants, keep.data_ptr(), voi_max_range=up.max_range)
            nf, nr = h.sweep_stats()
            flagged += nf.sum(axis=1, dtype=np.int64)
            rejected += nr.sum(axis=1, dtype=np.int64)
        masks = keep[:V * n].reshape(V, n).cpu().numpy()
        ref = initial_map if gt is None else gt
        with capi.Evaluator() as ev:
            for v in range(V):
                d, oo = h.voxelize_batch_ptr(m.points_ptr, [0, n], leaf, keep.data_ptr() + v * n, None, capi.PTR_DEVICE)
                static_map = np.empty((int(oo[-1]), 4), dtype=np.float32)
                capi._memcpy_from_device(static_map, d)
                q = ev.evaluate(ref, static_map, voxelsize=0.2)
                arr, _ = settings_of([variants[v]])
                parts = (arr[0].geometry, arr[0].s) if geo else (arr[0],)
                value = {f: getattr(part, f) for part in parts for f, _ in type(part)._fields_}
                rows.append(dict(**{f: value[f] for f in fields}, PR=q["PR"], RR=q["RR"], F1=q["F1"],
                                 kept=int(np.count_nonzero(masks[v])), saved=len(static_map), flagged=int(flagged[v]), rejected=int(rejected[v])))
    finally:
        h.close()
        m.close()
    return rows


def run_sequence(nodes, up, ep, voxelize: Optional[mapgen.Voxelizer] = None, make_updater: Optional[Callable] = None,
                 map_leafsize: Optional[float] = None, out_dir: Optional[str] = None, frame_independent: bool = False,
                 inserts: bool = False, pcd_mode: str = "ascii", retest: bool = False) -> dict:
    """mapgen -> updater -> evaluation on one node list.  GT for PR/RR = the naive map itself (it carries the labels), which is
    how the reference scores a run (analysis_runner.py compares <seq>_..._original / voxelised map with the result).
    frame_independent runs node mode (run_frame_independent) on the naive map instead of the sequential updater; inserts (node
    mode only) puts each node's inserted query points back into its static map, and retest (with inserts) tests them again in a
    second node-mode pass (run_frame_independent).  pcd_mode: the DATA mode of the two files written
    to out_dir ("ascii", as the reference writes them, "binary" or "binary_compressed"; the binary modes need the device writer,
    so an injected updater takes only "ascii")."""
    from . import capi
    if pcd_mode not in capi.PCD_MODES:
        raise ValueError(f"pcd_mode must be one of {sorted(capi.PCD_MODES)}")
    if pcd_mode != "ascii" and make_updater is not None:
        raise ValueError("binary PCD files are written on the device: an injected updater writes ascii only")
    nodes = list(nodes)
    leaf = float(up.map_voxel_size if map_leafsize is None else map_leafsize)
    original, naive = mapgen.build_map(nodes, leafsize=leaf, is_large_scale=bool(up.is_large_scale), voxelize=voxelize)
    if frame_independent:
        if make_updater is not None:
            raise ValueError("node mode runs on the device: make_updater does not apply")
        res = run_frame_independent(nodes, naive, up, ep, inserts=inserts, retest=retest)
    else:
        if inserts or retest:
            raise ValueError("inserts and retest are node-mode options: the sequential updater always inserts and re-tests")
        res = run_offline(nodes, naive, up, ep, make_updater=make_updater)
    res["naive_map"] = naive
    if make_updater is None:            # the device updater ran: score on the device too (same counts, same dict)
        from . import capi
        with capi.Evaluator() as ev:
            res["quality"] = ev.evaluate(naive, res["static_map"], voxelsize=0.2)
    else:
        res["quality"] = evaluate.evaluate(naive, res["static_map"], voxelsize=0.2)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        name = getattr(up, "data_name", "seq")
        paths = (os.path.join(out_dir, f"{name}_naive_map.pcd"), os.path.join(out_dir, f"{name}_result.pcd"))   # save_static_map's name (:193)
        if make_updater is None:        # the device updater ran: format the files on the device too (the same bytes)
            from . import capi
            with capi.PcdCodec() as codec:
                codec.write(paths[0], naive, mode=pcd_mode)
                codec.write(paths[1], res["static_map"], mode=pcd_mode)
        else:
            evaluate.write_pcd_ascii(paths[0], naive)
            evaluate.write_pcd_ascii(paths[1], res["static_map"])
    return res


def run_semantickitti(dataset_root: str, sequence: str, init_stamp: int, end_stamp: int, interval: int, config_yaml: str,
                      out_dir: Optional[str] = None, **kw) -> dict:
    """SemanticKITTI files + a reference config/*.yaml -> static map and PR/RR."""
    ep, up = params.load_yaml(config_yaml)
    return run_sequence(kitti.iter_nodes(dataset_root, sequence, init_stamp, end_stamp, interval), up, ep, out_dir=out_dir, **kw)


def read_bag_nodes(bag_path: str, topic: str = "/node/combined/optimized", keep_first: bool = False, device: int = 0) -> list:
    """The (seq, odom7, cloud) list of a ROS bag of erasor/node messages (the reference's <seq>_..._node.bag), as the reference's
    subscribers receive it: the first message dropped unless keep_first.  Indexed on the host, decoded on the device
    (capi.PcdCodec.bag_index / bag_nodes)."""
    from . import capi
    with open(bag_path, "rb") as f:
        data = f.read()
    with capi.PcdCodec(device) as codec:
        codec.bag_index(data, topic, keep_first)
        return list(codec.bag_nodes())


def run_bag(bag: str, config_yaml: str, out_dir: Optional[str] = None, frame_independent: bool = False, **kw) -> dict:
    """A reference bag + a reference config/*.yaml -> naive map, static map and PR/RR: run_sequence on the bag's nodes, with the
    sequential updater or, with frame_independent, node mode (inserts=True in kw: with node-mode inserts; retest=True as well:
    with their re-test pass)."""
    ep, up = params.load_yaml(config_yaml)
    return run_sequence(read_bag_nodes(bag), up, ep, out_dir=out_dir, frame_independent=frame_independent, **kw)
