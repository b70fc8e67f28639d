"""The reference's three-stage workflow in one call, ROS stripped (README "How to run": mapgen -> offline_map_updater ->
scripts/analysis_runner.py):

    nodes (erasor_b200.kitti.iter_nodes, or any iterable of (seq, odom7, cloud))
      -> naive map            erasor_b200.mapgen           (src/mapgen)
      -> static map           capi.Updater, one erasor_updater_process_node per node + save_static_map
                              (OfflineMapUpdater::callback_node / save_static_map, OfflineMapUpdater.cpp:174-330)
      -> PR / RR              capi.Evaluator (device), or erasor_b200.evaluate when the updater is injected
                              (scripts/analysis_runner.py)
      -> <name>_naive_map.pcd, <name>_result.pcd (out_dir): capi.PcdCodec (device), or write_pcd_ascii when the updater is injected

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


def run_sequence(nodes, up, ep, voxelize: Optional[mapgen.Voxelizer] = None, make_updater: Optional[Callable] = None,
                 map_leafsize: Optional[float] = None, out_dir: Optional[str] = None) -> dict:
    """mapgen -> updater -> evaluation on one node list.  GT for PR/RR = the naive map itself (it carries the labels), which is
    how the reference scores a run (analysis_runner.py compares <seq>_..._original / voxelised map with the result)."""
    nodes = list(nodes)
    leaf = float(up.map_voxel_size if map_leafsize is None else map_leafsize)
    original, naive = mapgen.build_map(nodes, leafsize=leaf, is_large_scale=bool(up.is_large_scale), voxelize=voxelize)
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
                codec.write(paths[0], naive)
                codec.write(paths[1], res["static_map"])
        else:
            evaluate.write_pcd_ascii(paths[0], naive)
            evaluate.write_pcd_ascii(paths[1], res["static_map"])
    return res


def run_semantickitti(dataset_root: str, sequence: str, init_stamp: int, end_stamp: int, interval: int, config_yaml: str,
                      out_dir: Optional[str] = None, **kw) -> dict:
    """SemanticKITTI files + a reference config/*.yaml -> static map and PR/RR."""
    ep, up = params.load_yaml(config_yaml)
    return run_sequence(kitti.iter_nodes(dataset_root, sequence, init_stamp, end_stamp, interval), up, ep, out_dir=out_dir, **kw)
