"""ctypes binding of the C ABI in ``include/erasor_b200.h`` (``erasor_b200/_lib/liberasor_b200.so``).

The library is CUDA-only: importing this module without the built ``.so`` raises, and
``Handle(...)`` raises when there is no CUDA device.  There is no CPU fallback anywhere in the
package (the CPU oracle lives under ``oracle/`` and is test infrastructure).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_size_t, c_uint8, c_uint32, c_uint64, c_void_p

import numpy as np

from .params import ErasorParams, ErasorParamsC

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_lib", "liberasor_b200.so")

PTR_HOST, PTR_DEVICE = 0, 1
PTR_QUERY_XYZ = 16          # OR-able (mask modes): the query cloud is packed x y z, three floats per point
CLOUD_MAP, CLOUD_QUERY = 0, 1
OK, E_INVALID, E_CUDA, E_STATE, E_CAPACITY, E_UNSUPPORTED = 0, -1, -2, -3, -4, -5

EXPORTS = [
    "erasor_create", "erasor_destroy", "erasor_last_error", "erasor_abi_version", "erasor_stream", "erasor_synchronize",
    "erasor_set_inputs", "erasor_compare", "erasor_get_output_sizes", "erasor_get_static_estimate", "erasor_get_outliers",
    "erasor_get_max_range", "erasor_device_outputs", "erasor_get_ground_viz", "erasor_get_bins", "erasor_get_status", "erasor_get_planes", "erasor_get_static_mask",
    "erasor_get_fence_counts", "erasor_process_frames", "erasor_process_frames_async", "erasor_wait", "erasor_process_frames_fold",
    "erasor_process_frames_fold_async", "erasor_fold_keep_masks", "erasor_reset_keep_mask", "erasor_get_frame_stats", "erasor_kernel_launch_count",
    "erasor_map_create", "erasor_map_destroy", "erasor_map_size", "erasor_map_reset_keep", "erasor_map_get_keep", "erasor_map_keep_device",
    "erasor_map_points_device", "erasor_attach_map", "erasor_process_nodes", "erasor_process_nodes_async", "erasor_get_node_stats",
    "erasor_process_nodes_sweep", "erasor_process_nodes_sweep_async", "erasor_get_sweep_stats",
    "erasor_process_nodes_sweep_ex", "erasor_process_nodes_sweep_ex_async", "erasor_process_nodes_tune", "erasor_process_nodes_tune_async",
    "erasor_voxelize_batch",
    "erasor_set_node_inserts", "erasor_get_node_inserts", "erasor_map_append_inserts", "erasor_map_inserts", "erasor_map_clear_inserts",
    "erasor_save_node_map",
    "erasor_map_create_retest", "erasor_map_retest_extents", "erasor_process_nodes_retest", "erasor_process_nodes_retest_async",
    "erasor_comm_unique_id", "erasor_comm_init", "erasor_comm_destroy", "erasor_allgather_and_keep", "erasor_and_keep_masks",
    "erasor_get_kernel_time_ms", "erasor_reset_kernel_times", "erasor_forget_run_history", "erasor_get_rgpf_profile", "erasor_get_srt_profile", "erasor_profile_k1",
    "erasor_updater_create", "erasor_updater_destroy", "erasor_updater_reset", "erasor_updater_last_error", "erasor_updater_process_node", "erasor_updater_prefetch_scan",
    "erasor_updater_map_size", "erasor_updater_get_cloud", "erasor_updater_save_static_map", "erasor_updater_voxelize", "erasor_updater_mapgen_node",
    "erasor_updater_erasor", "erasor_updater_kernel_launch_count", "erasor_updater_get_fused_profile",
    "erasor_eval_create", "erasor_eval_destroy", "erasor_eval_last_error", "erasor_evaluate", "erasor_eval_overlap",
    "erasor_eval_count_selected",
    "erasor_pcd_create", "erasor_pcd_destroy", "erasor_pcd_last_error", "erasor_pcd_parse_ascii", "erasor_pcd_format_ascii",
    "erasor_pcd_format", "erasor_pcd_load", "erasor_bag_index", "erasor_bag_nodes", "erasor_bag_load", "erasor_bag_load_list", "erasor_bag_lz4_stats", "erasor_bag_bz2_stats",
    "erasor_mapgen_create", "erasor_mapgen_destroy", "erasor_mapgen_last_error", "erasor_mapgen_accum", "erasor_mapgen_get_cloud",
    "erasor_mapgen_device_cloud", "erasor_mapgen_synchronize", "erasor_mapgen_get_counters",
]
NO_MATCH = 0xFFFFFFFF        # erasor_evaluate's match entry of a GT point without an inlier


class EvalCountsC(ctypes.Structure):
    """erasor_eval_counts_t"""
    _fields_ = [(name, c_uint64) for name in ("gt_static", "gt_dynamic", "preserved_static", "preserved_dynamic", "inliers", "ambiguous_ties")]


class EvalOverlapC(ctypes.Structure):
    """erasor_eval_overlap_t"""
    _fields_ = [(name, c_uint64) for name in ("n", "est_static", "est_dynamic", "below_half", "below_one", "below_two", "far_points")] + [("max", c_double)]


class SrtVariantC(ctypes.Structure):
    """erasor_srt_variant_t"""
    _fields_ = [("scan_ratio_threshold", c_double), ("th_bin_max_h", c_double), ("minimum_num_pts", c_int), ("reserved", c_int)]


SRT_SWEEP_FIELDS = ("scan_ratio_threshold", "th_bin_max_h", "minimum_num_pts")     # what a Scan Ratio Test sweep varies
GF_SWEEP_FIELDS = ("gf_dist_thr", "gf_th_seeds_height", "gf_num_lpr", "num_lowest_pts", "gf_iter")   # R-GPF's, added by sweep_ex
MAX_SWEEP_VARIANTS = 32


class SweepSettingC(ctypes.Structure):
    """erasor_sweep_setting_t"""
    _fields_ = [(name, c_double) for name in ("scan_ratio_threshold", "th_bin_max_h", "gf_dist_thr", "gf_th_seeds_height")] + \
               [(name, c_int) for name in ("minimum_num_pts", "num_lowest_pts", "gf_num_lpr", "gf_iter")]


GEOMETRY_SWEEP_FIELDS = ("max_range", "num_rings", "num_sectors", "min_h", "max_h")    # ERASOR's polar geometry and z window, added by tune


class GeometryC(ctypes.Structure):
    """erasor_geometry_t"""
    _fields_ = [(name, c_double) for name in ("max_range", "min_h", "max_h")] + [(name, c_int) for name in ("num_rings", "num_sectors")]


class TuneSettingC(ctypes.Structure):
    """erasor_tune_setting_t"""
    _fields_ = [("geometry", GeometryC), ("s", SweepSettingC)]


class PcdInfoC(ctypes.Structure):
    """erasor_pcd_info_t"""
    _fields_ = [(name, c_uint64) for name in ("points", "rows", "slow_tokens", "error_line", "header_lines")] + [("fields", c_uint32),
                                                                                                              ("has_intensity", c_uint32)]


class PcdLoadInfoC(ctypes.Structure):
    """erasor_pcd_load_info_t"""
    _fields_ = [(name, c_uint32) for name in ("data_mode", "fields", "intensity_zero_filled", "point_step")] + \
               [(name, c_uint64) for name in ("width", "height", "points", "data_offset", "compressed_size", "uncompressed_size", "lzf_tokens")] + \
               [("ascii", PcdInfoC)]


class PcdFormatInfoC(ctypes.Structure):
    """erasor_pcd_format_info_t"""
    _fields_ = [("data_mode", c_uint32), ("segments", c_uint32)] + \
               [(name, c_uint64) for name in ("header_bytes", "uncompressed_size", "compressed_size", "lzf_tokens")]


PCD_MODES = {"ascii": 0, "binary": 1, "binary_compressed": 2}     # ERASOR_PCD_ASCII / _BINARY / _BINARY_COMPRESSED


class BagInfoC(ctypes.Structure):
    """erasor_bag_info_t"""
    _fields_ = [("version", c_uint32), ("pad_", c_uint32)] + \
               [(name, c_uint64) for name in ("chunks", "connections", "messages", "selected", "unknown_records", "nodes", "total_points",
                                               "intensity_zero_filled", "big_endian")] + [("md5sum", ctypes.c_char * 40)]


class BagCloudC(ctypes.Structure):
    """erasor_bag_cloud_t"""
    _fields_ = [("data_offset", c_uint64), ("data_len", c_uint64)] + \
               [(name, c_uint32) for name in ("width", "height", "point_step", "row_step", "fields", "big_endian")] + [("offset", c_uint32 * 4)]


class BagLz4StatsC(ctypes.Structure):
    """erasor_bag_lz4_stats_t"""
    _fields_ = [(name, c_uint64) for name in ("chunks", "decoded_chunks", "compressed_bytes", "decoded_bytes", "blocks", "stored_blocks",
                                               "block_checksums", "content_checksums")] + [("decode_ms", c_double), ("checksum_ms", c_double)]


class BagBz2StatsC(ctypes.Structure):
    """erasor_bag_bz2_stats_t"""
    _fields_ = [(name, c_uint64) for name in ("chunks", "decoded_chunks", "compressed_bytes", "decoded_bytes", "blocks", "candidates")] + \
               [("streams_by_level", c_uint64 * 9), ("scratch_bytes", c_uint64)] + \
               [(name, c_double) for name in ("scan_ms", "decode_ms", "bwt_ms", "rle_ms")]


class MapGenParamsC(ctypes.Structure):
    """erasor_mapgen_params_t"""
    _fields_ = [("leafsize", c_float), ("is_large_scale", c_int)]


class UpdaterParamsC(ctypes.Structure):
    """erasor_updater_params_t"""
    _fields_ = [
        ("query_voxel_size", c_double), ("map_voxel_size", c_double), ("removal_interval", c_int), ("is_large_scale", c_int),
        ("submap_size", c_double), ("max_range", c_double), ("version", c_int), ("pad_", c_int), ("lidar2body", c_double * 7),
    ]


class ErasorError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"erasor_b200 error {code}: {msg}")
        self.code = code


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with erasor_b200/csrc/build.sh (or __graft_entry__.build()). "
            "erasor_b200 has no CPU fallback.")
    L = ctypes.CDLL(LIB_PATH)
    fp = POINTER(c_float)
    L.erasor_create.restype = c_int
    L.erasor_create.argtypes = [POINTER(ErasorParamsC), c_int, POINTER(c_void_p)]
    L.erasor_destroy.restype = None
    L.erasor_destroy.argtypes = [c_void_p]
    L.erasor_last_error.restype = c_char_p
    L.erasor_last_error.argtypes = [c_void_p]
    L.erasor_abi_version.restype = c_int
    L.erasor_stream.restype = c_void_p
    L.erasor_stream.argtypes = [c_void_p]
    L.erasor_synchronize.argtypes = [c_void_p]
    L.erasor_set_inputs.argtypes = [c_void_p, c_void_p, c_size_t, c_void_p, c_size_t, c_int]
    L.erasor_compare.argtypes = [c_void_p, c_int, c_int]
    L.erasor_get_output_sizes.argtypes = [c_void_p, POINTER(c_size_t), POINTER(c_size_t), POINTER(c_size_t), POINTER(c_size_t)]
    L.erasor_get_static_estimate.argtypes = [c_void_p, c_void_p, c_size_t, POINTER(c_size_t), c_void_p, c_size_t, POINTER(c_size_t), c_int]
    L.erasor_get_outliers.argtypes = [c_void_p, c_void_p, c_size_t, POINTER(c_size_t), c_void_p, c_size_t, POINTER(c_size_t), c_int]
    L.erasor_get_ground_viz.argtypes = [c_void_p, c_void_p, c_size_t, POINTER(c_size_t), c_int]
    L.erasor_get_max_range.restype = c_double
    L.erasor_get_max_range.argtypes = [c_void_p]
    L.erasor_get_bins.argtypes = [c_void_p, c_int, POINTER(c_int32), fp, fp, POINTER(c_uint32)]
    L.erasor_get_status.argtypes = [c_void_p, fp]
    L.erasor_get_planes.argtypes = [c_void_p, POINTER(c_int32), POINTER(c_int32), POINTER(c_int32), POINTER(c_double),
                                    POINTER(c_double), POINTER(c_int32), POINTER(c_size_t)]
    L.erasor_get_static_mask.argtypes = [c_void_p, POINTER(c_uint8), POINTER(c_uint8)]
    L.erasor_get_fence_counts.argtypes = [c_void_p, POINTER(c_uint64), POINTER(c_uint64), POINTER(c_uint64)]
    L.erasor_process_frames.argtypes = [c_void_p, c_void_p, POINTER(c_uint64), c_void_p, POINTER(c_uint64), c_int, c_void_p, c_int]
    L.erasor_process_frames_fold.argtypes = [c_void_p, c_void_p, POINTER(c_uint64), c_void_p, POINTER(c_uint64), c_int, c_void_p, c_int,
                                             c_void_p, c_void_p, c_size_t]
    L.erasor_fold_keep_masks.argtypes = [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_size_t]
    L.erasor_process_frames_async.argtypes = L.erasor_process_frames.argtypes
    L.erasor_process_frames_fold_async.argtypes = L.erasor_process_frames_fold.argtypes
    L.erasor_wait.argtypes = [c_void_p]
    L.erasor_reset_keep_mask.argtypes = [c_void_p, c_void_p, c_size_t]
    L.erasor_map_create.argtypes = [c_void_p, c_size_t, c_int, c_int, POINTER(c_void_p)]
    L.erasor_map_destroy.restype = None
    L.erasor_map_destroy.argtypes = [c_void_p]
    L.erasor_map_size.restype = c_size_t
    L.erasor_map_size.argtypes = [c_void_p]
    L.erasor_map_reset_keep.argtypes = [c_void_p]
    L.erasor_map_get_keep.argtypes = [c_void_p, c_void_p, c_int]
    L.erasor_map_keep_device.restype = c_void_p
    L.erasor_map_keep_device.argtypes = [c_void_p]
    L.erasor_map_points_device.restype = c_void_p
    L.erasor_map_points_device.argtypes = [c_void_p]
    L.erasor_attach_map.argtypes = [c_void_p, c_void_p]
    L.erasor_process_nodes.argtypes = [c_void_p, POINTER(c_double), c_void_p, POINTER(c_uint64), c_int, c_double, c_void_p, c_void_p, c_int]
    L.erasor_process_nodes_async.argtypes = L.erasor_process_nodes.argtypes
    L.erasor_get_node_stats.argtypes = [c_void_p, POINTER(c_uint32), POINTER(c_uint32), POINTER(c_uint32)]
    L.erasor_process_nodes_sweep.argtypes = [c_void_p, POINTER(c_double), c_void_p, POINTER(c_uint64), c_int, c_double, POINTER(SrtVariantC), c_int,
                                             c_void_p, c_int]
    L.erasor_process_nodes_sweep_async.argtypes = L.erasor_process_nodes_sweep.argtypes
    L.erasor_process_nodes_sweep_ex.argtypes = L.erasor_process_nodes_sweep.argtypes[:6] + [POINTER(SweepSettingC)] + L.erasor_process_nodes_sweep.argtypes[7:]
    L.erasor_process_nodes_sweep_ex_async.argtypes = L.erasor_process_nodes_sweep_ex.argtypes
    L.erasor_process_nodes_tune.argtypes = L.erasor_process_nodes_sweep.argtypes[:6] + [POINTER(TuneSettingC)] + L.erasor_process_nodes_sweep.argtypes[7:]
    L.erasor_process_nodes_tune_async.argtypes = L.erasor_process_nodes_tune.argtypes
    L.erasor_get_sweep_stats.argtypes = [c_void_p, POINTER(c_uint32), POINTER(c_uint32)]
    L.erasor_voxelize_batch.argtypes = [c_void_p, c_void_p, POINTER(c_uint64), c_int, c_void_p, c_float, POINTER(c_double), c_int,
                                        POINTER(c_void_p), POINTER(c_uint64)]
    L.erasor_set_node_inserts.argtypes = [c_void_p, c_int]
    L.erasor_get_node_inserts.argtypes = [c_void_p, POINTER(c_void_p), POINTER(c_uint64)]
    L.erasor_map_append_inserts.argtypes = [c_void_p, c_void_p]
    L.erasor_map_inserts.argtypes = [c_void_p, POINTER(c_void_p), POINTER(c_size_t)]
    L.erasor_map_clear_inserts.argtypes = [c_void_p]
    L.erasor_save_node_map.argtypes = [c_void_p, c_void_p, c_float, POINTER(c_void_p), POINTER(c_size_t)]
    L.erasor_map_create_retest.argtypes = [c_void_p, POINTER(c_void_p)]
    L.erasor_map_retest_extents.argtypes = [c_void_p, POINTER(c_size_t), POINTER(c_uint64)]
    L.erasor_process_nodes_retest.argtypes = [c_void_p, POINTER(c_double), c_void_p, POINTER(c_uint64), c_int, c_int, c_double, c_void_p, c_int]
    L.erasor_process_nodes_retest_async.argtypes = L.erasor_process_nodes_retest.argtypes
    L.erasor_comm_unique_id.argtypes = [c_void_p]
    L.erasor_comm_init.argtypes = [c_void_p, c_void_p, c_int, c_int]
    L.erasor_comm_destroy.argtypes = [c_void_p]
    L.erasor_allgather_and_keep.argtypes = [c_void_p, c_void_p, c_size_t]
    L.erasor_and_keep_masks.argtypes = [c_void_p, c_void_p, c_int, c_size_t, c_void_p]
    L.erasor_get_frame_stats.argtypes = [c_void_p, POINTER(c_uint32), POINTER(c_uint32)]
    L.erasor_kernel_launch_count.restype = c_uint64
    L.erasor_kernel_launch_count.argtypes = [c_void_p]
    L.erasor_get_kernel_time_ms.argtypes = [c_void_p, c_int, POINTER(c_double), POINTER(c_uint64)]
    L.erasor_reset_kernel_times.argtypes = [c_void_p, c_int]
    L.erasor_forget_run_history.argtypes = [c_void_p]
    L.erasor_get_rgpf_profile.argtypes = [c_void_p, POINTER(c_uint32), POINTER(c_uint32), POINTER(c_size_t)]
    L.erasor_get_srt_profile.argtypes = [c_void_p, POINTER(c_uint32)]
    L.erasor_profile_k1.argtypes = [c_void_p, POINTER(c_uint32), POINTER(c_size_t), POINTER(c_int)]
    L.erasor_updater_create.argtypes = [POINTER(UpdaterParamsC), POINTER(ErasorParamsC), c_void_p, c_size_t, c_int, POINTER(c_void_p)]
    L.erasor_updater_destroy.restype = None
    L.erasor_updater_destroy.argtypes = [c_void_p]
    L.erasor_updater_reset.argtypes = [c_void_p, c_void_p, c_size_t]
    L.erasor_updater_last_error.restype = c_char_p
    L.erasor_updater_last_error.argtypes = [c_void_p]
    L.erasor_updater_process_node.argtypes = [c_void_p, c_int, POINTER(c_double), c_void_p, c_size_t, c_int, POINTER(c_int)]
    L.erasor_updater_prefetch_scan.argtypes = [c_void_p, c_void_p, c_size_t, c_int]
    L.erasor_updater_map_size.argtypes = [c_void_p, POINTER(c_size_t)]
    L.erasor_updater_get_cloud.argtypes = [c_void_p, c_int, c_void_p, c_size_t, POINTER(c_size_t), c_int]
    L.erasor_updater_save_static_map.argtypes = [c_void_p, c_float, c_void_p, c_size_t, POINTER(c_size_t)]
    L.erasor_updater_voxelize.argtypes = [c_void_p, c_void_p, c_size_t, c_float, c_void_p, c_size_t, POINTER(c_size_t)]
    L.erasor_updater_mapgen_node.argtypes = [c_void_p, POINTER(c_double), c_void_p, c_size_t, c_int, c_void_p, c_size_t, POINTER(c_size_t)]
    L.erasor_updater_erasor.restype = c_void_p
    L.erasor_updater_erasor.argtypes = [c_void_p]
    L.erasor_updater_kernel_launch_count.restype = c_uint64
    L.erasor_updater_kernel_launch_count.argtypes = [c_void_p]
    L.erasor_updater_get_fused_profile.argtypes = [c_void_p, c_void_p]
    L.erasor_eval_create.argtypes = [c_int, POINTER(c_void_p)]
    L.erasor_eval_destroy.restype = None
    L.erasor_eval_destroy.argtypes = [c_void_p]
    L.erasor_eval_last_error.restype = c_char_p
    L.erasor_eval_last_error.argtypes = [c_void_p]
    L.erasor_evaluate.argtypes = [c_void_p, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_double, c_int, c_void_p, POINTER(EvalCountsC)]
    L.erasor_eval_overlap.argtypes = [c_void_p, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p, c_double, c_int, c_void_p, c_size_t, c_void_p,
                                      c_void_p, POINTER(EvalOverlapC)]
    L.erasor_eval_count_selected.argtypes = [c_void_p, c_void_p, c_size_t, c_int, POINTER(c_uint64)]
    L.erasor_pcd_create.argtypes = [c_int, POINTER(c_void_p)]
    L.erasor_pcd_destroy.restype = None
    L.erasor_pcd_destroy.argtypes = [c_void_p]
    L.erasor_pcd_last_error.restype = c_char_p
    L.erasor_pcd_last_error.argtypes = [c_void_p]
    L.erasor_pcd_parse_ascii.argtypes = [c_void_p, c_void_p, c_size_t, c_int, c_void_p, c_size_t, c_int, POINTER(c_size_t), POINTER(PcdInfoC)]
    L.erasor_pcd_format_ascii.argtypes = [c_void_p, c_void_p, c_size_t, c_int, c_void_p, c_size_t, c_int, POINTER(c_size_t)]
    L.erasor_pcd_format.argtypes = [c_void_p, c_void_p, c_size_t, c_int, c_int, c_void_p, c_size_t, c_int, POINTER(c_size_t), POINTER(PcdFormatInfoC)]
    L.erasor_pcd_load.argtypes = [c_void_p, c_void_p, c_size_t, c_int, c_void_p, c_size_t, c_int, POINTER(c_size_t), POINTER(PcdLoadInfoC)]
    L.erasor_bag_index.argtypes = [c_void_p, c_void_p, c_size_t, c_char_p, c_int, POINTER(c_size_t), POINTER(BagInfoC)]
    L.erasor_bag_nodes.argtypes = [c_void_p, c_size_t, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p]
    L.erasor_bag_load.argtypes = [c_void_p, c_size_t, c_size_t, c_void_p, c_size_t, c_int, POINTER(c_uint64)]
    L.erasor_bag_load_list.argtypes = [c_void_p, POINTER(c_uint64), c_size_t, c_void_p, c_size_t, c_int, POINTER(c_uint64)]
    L.erasor_bag_lz4_stats.argtypes = [c_void_p, POINTER(BagLz4StatsC)]
    L.erasor_bag_bz2_stats.argtypes = [c_void_p, POINTER(BagBz2StatsC)]
    L.erasor_mapgen_create.argtypes = [POINTER(MapGenParamsC), c_int, POINTER(c_void_p)]
    L.erasor_mapgen_destroy.restype = None
    L.erasor_mapgen_destroy.argtypes = [c_void_p]
    L.erasor_mapgen_last_error.restype = c_char_p
    L.erasor_mapgen_last_error.argtypes = [c_void_p]
    L.erasor_mapgen_accum.argtypes = [c_void_p, POINTER(c_double), c_void_p, c_size_t, c_int]
    L.erasor_mapgen_get_cloud.argtypes = [c_void_p, c_int, c_void_p, c_size_t, c_int, POINTER(c_size_t)]
    L.erasor_mapgen_device_cloud.argtypes = [c_void_p, c_int, POINTER(c_void_p), POINTER(c_size_t)]
    L.erasor_mapgen_synchronize.argtypes = [c_void_p]
    L.erasor_mapgen_get_counters.argtypes = [c_void_p, POINTER(c_uint64), POINTER(c_uint64), POINTER(c_uint64)]
    return L


_L = None
_CUDART = None


def lib():
    global _L
    if _L is None:
        _L = _load()
    return _L


def _memcpy_from_device(dst: np.ndarray, src_ptr: int):
    """dst <- the dst.nbytes bytes at device address src_ptr (cudaMemcpy of the runtime the library loaded)."""
    global _CUDART
    if _CUDART is None:
        lib()
        _CUDART = ctypes.CDLL("libcudart.so.12")
        _CUDART.cudaMemcpy.restype = c_int
        _CUDART.cudaMemcpy.argtypes = [c_void_p, c_void_p, c_size_t, c_int]
    if dst.nbytes:
        rc = _CUDART.cudaMemcpy(dst.ctypes.data, c_void_p(src_ptr), dst.nbytes, 2)      # cudaMemcpyDeviceToHost
        if rc != 0:
            raise ErasorError(E_CUDA, f"cudaMemcpy: error {rc}")


def _cloud(a) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.size == 0:
        return a.reshape(0, 4)
    if a.ndim != 2 or a.shape[1] != 4:
        raise ValueError("clouds are float32 [n,4] = x,y,z,intensity")
    return a


class _Native:
    """One handle ``h`` of a family of the C ABI, released by ``close`` (or ``with``, or garbage collection).  A subclass names
    the family's ``*_destroy`` and ``*_last_error``; ``_create`` and ``_ck`` raise ``ErasorError`` with the family's message."""
    _DESTROY = _LAST_ERROR = ""
    h = None

    def _create(self, create: str, *args):
        """self.h = the handle L.<create>(*args, &h) makes"""
        self.L = lib()
        h = c_void_p()
        rc = getattr(self.L, create)(*args, ctypes.byref(h))
        if rc != OK:
            raise ErasorError(rc, self._message(None))
        self.h = h

    def _message(self, h) -> str:
        return (getattr(self.L, self._LAST_ERROR)(h) or b"").decode()

    def _ck(self, rc: int):
        if rc != OK:
            raise ErasorError(rc, self._message(self.h))

    def _read_cloud(self, call) -> np.ndarray:
        """A float32 [n,4] cloud from a getter call(out, cap, &n) -> rc: asked for n without a buffer, then filled."""
        n = c_size_t(0)
        self._ck(call(None, 0, ctypes.byref(n)))
        out = np.empty((n.value, 4), dtype=np.float32)
        if n.value:
            self._ck(call(out.ctypes.data, n.value, ctypes.byref(n)))
        return out

    def close(self):
        if self.h:
            getattr(self.L, self._DESTROY)(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class Handle(_Native):
    """One ``erasor_handle_t``: one CUDA device, one stream, fixed parameters."""
    _DESTROY, _LAST_ERROR = "erasor_destroy", "erasor_last_error"

    def __init__(self, params: ErasorParams, device: int = 0):
        self.params = params
        self._pc = params.to_c()
        self._create("erasor_create", ctypes.byref(self._pc), device)
        self._device = device
        self.n_map = 0
        self.n_query = 0
        self._keep = []   # keeps host arrays alive while the library may still read them

    # -- plumbing ---------------------------------------------------------------------------
    @property
    def stream(self) -> int:
        return self.L.erasor_stream(self.h) or 0

    def synchronize(self):
        self._ck(self.L.erasor_synchronize(self.h))

    # -- the per-frame path ---------------------------------------------------------------
    def set_inputs(self, map_voi, query_voi):
        m, q = _cloud(map_voi), _cloud(query_voi)
        self._keep = [m, q]
        self.n_map, self.n_query = len(m), len(q)
        self._ck(self.L.erasor_set_inputs(self.h, m.ctypes.data, len(m), q.ctypes.data, len(q), PTR_HOST))

    def set_inputs_device(self, map_ptr: int, n_map: int, query_ptr: int, n_query: int):
        self.n_map, self.n_query = n_map, n_query
        self._ck(self.L.erasor_set_inputs(self.h, c_void_p(map_ptr), n_map, c_void_p(query_ptr), n_query, PTR_DEVICE))

    def compare(self, version: int | None = None, frame: int = 0):
        self._ck(self.L.erasor_compare(self.h, self.params.version if version is None else version, frame))

    def output_sizes(self):
        a, c, m, q = c_size_t(), c_size_t(), c_size_t(), c_size_t()
        self._ck(self.L.erasor_get_output_sizes(self.h, ctypes.byref(a), ctypes.byref(c), ctypes.byref(m), ctypes.byref(q)))
        return a.value, c.value, m.value, q.value

    def get_static_estimate(self):
        na, nc, _, _ = self.output_sizes()
        arr = np.empty((na, 4), dtype=np.float32)
        cmp_ = np.empty((nc, 4), dtype=np.float32)
        a, c = c_size_t(), c_size_t()
        self._ck(self.L.erasor_get_static_estimate(self.h, arr.ctypes.data, na, ctypes.byref(a), cmp_.ctypes.data, nc, ctypes.byref(c), PTR_HOST))
        return arr, cmp_

    def get_outliers(self):
        _, _, nm, nq = self.output_sizes()
        mr = np.empty((nm, 4), dtype=np.float32)
        cr = np.empty((nq, 4), dtype=np.float32)
        a, c = c_size_t(), c_size_t()
        self._ck(self.L.erasor_get_outliers(self.h, mr.ctypes.data, nm, ctypes.byref(a), cr.ctypes.data, nq, ctypes.byref(c), PTR_HOST))
        return mr, cr

    def get_ground_viz(self) -> np.ndarray:
        return self._read_cloud(lambda out, cap, n: self.L.erasor_get_ground_viz(self.h, out, cap, n, PTR_HOST))

    def get_max_range(self) -> float:
        return self.L.erasor_get_max_range(self.h)

    # -- parity taps ---------------------------------------------------------------------------
    def get_bins(self, which: int, per_point: bool = True):
        """per_point=False: tables only (the form a one-node process_nodes supports); bin_of_point comes back as None."""
        B = self.params.num_bins
        n = self.n_map if which == CLOUD_MAP else self.n_query
        bop = np.empty(n, dtype=np.int32) if per_point else None
        mn, mx = np.empty(B, dtype=np.float32), np.empty(B, dtype=np.float32)
        cnt = np.empty(B, dtype=np.uint32)
        self._ck(self.L.erasor_get_bins(self.h, which, bop.ctypes.data_as(POINTER(c_int32)) if per_point else None,
                                        mn.ctypes.data_as(POINTER(c_float)), mx.ctypes.data_as(POINTER(c_float)),
                                        cnt.ctypes.data_as(POINTER(c_uint32))))
        return bop, mn, mx, cnt

    def get_status(self) -> np.ndarray:
        st = np.empty(self.params.num_bins, dtype=np.float32)
        self._ck(self.L.erasor_get_status(self.h, st.ctypes.data_as(POINTER(c_float))))
        return st

    def get_planes(self):
        n = c_size_t(0)
        self._ck(self.L.erasor_get_planes(self.h, None, None, None, None, None, None, ctypes.byref(n)))
        k, it = n.value, self.params.gf_iter
        bins, npts, nseeds = (np.zeros(k, dtype=np.int32) for _ in range(3))
        lpr = np.zeros(k)
        nd = np.zeros((k, it, 4))
        ng = np.zeros((k, it), dtype=np.int32)
        cap = c_size_t(k)
        if k:
            self._ck(self.L.erasor_get_planes(self.h, bins.ctypes.data_as(POINTER(c_int32)), npts.ctypes.data_as(POINTER(c_int32)),
                                              nseeds.ctypes.data_as(POINTER(c_int32)), lpr.ctypes.data_as(POINTER(c_double)),
                                              nd.ctypes.data_as(POINTER(c_double)), ng.ctypes.data_as(POINTER(c_int32)), ctypes.byref(cap)))
        return [dict(bin=int(bins[i]), n_points=int(npts[i]), n_seeds=int(nseeds[i]), lpr=float(lpr[i]), normal_d=nd[i], n_ground=ng[i])
                for i in range(k)]

    def get_static_mask(self):
        keep = np.empty(self.n_map, dtype=np.uint8)
        gnd = np.empty(self.n_map, dtype=np.uint8)
        self._ck(self.L.erasor_get_static_mask(self.h, keep.ctypes.data_as(POINTER(c_uint8)), gnd.ctypes.data_as(POINTER(c_uint8))))
        return keep, gnd

    def fence_counts(self):
        a, b, c = c_uint64(), c_uint64(), c_uint64()
        self._ck(self.L.erasor_get_fence_counts(self.h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)))
        return dict(negzero_points=a.value, empty_plane_fits=b.value, ambiguous_sector=c.value)

    # -- batch mode ---------------------------------------------------------------------------
    def process_frames(self, map_xyzi, map_offsets, query_xyzi, query_offsets) -> np.ndarray:
        """Host-buffer batch call: returns keep mask (uint8) over all map points of all frames."""
        m, q = _cloud(map_xyzi), _cloud(query_xyzi)
        mo = np.ascontiguousarray(map_offsets, dtype=np.uint64)
        qo = np.ascontiguousarray(query_offsets, dtype=np.uint64)
        F = len(mo) - 1
        keep = np.empty(int(mo[-1]), dtype=np.uint8)
        self._ck(self.L.erasor_process_frames(self.h, m.ctypes.data, mo.ctypes.data_as(POINTER(c_uint64)), q.ctypes.data,
                                              qo.ctypes.data_as(POINTER(c_uint64)), F, keep.ctypes.data, PTR_HOST))
        self.n_frames = F
        return keep

    def process_frames_ptr(self, map_ptr: int, map_offsets: np.ndarray, query_ptr: int, query_offsets: np.ndarray, keep_ptr: int, ptr_kind: int,
                           fold=None, asynchronous: bool = False):
        """Raw-pointer batch call (device tensors or pinned host memory); offsets are host uint64 arrays.
        The ctypes views of the offset arrays are cached per array object so that a caller streaming equally-shaped
        batches pays one foreign call per step and nothing else."""
        key = (id(map_offsets), id(query_offsets))
        c = getattr(self, "_off_cache", None)
        if c is None or c[0] != key:
            mo = np.ascontiguousarray(map_offsets, dtype=np.uint64)
            qo = np.ascontiguousarray(query_offsets, dtype=np.uint64)
            c = (key, mo, qo, mo.ctypes.data_as(POINTER(c_uint64)), qo.ctypes.data_as(POINTER(c_uint64)), len(mo) - 1)
            self._off_cache = c
        if fold is None:
            fn = self.L.erasor_process_frames_async if asynchronous else self.L.erasor_process_frames
            rc = fn(self.h, map_ptr, c[3], query_ptr, c[4], c[5], keep_ptr, ptr_kind)
        else:       # fold = (voi_index device ptr, global_keep device ptr, n_global): the fold runs in R-GPF's epilogue
            fn = self.L.erasor_process_frames_fold_async if asynchronous else self.L.erasor_process_frames_fold
            rc = fn(self.h, map_ptr, c[3], query_ptr, c[4], c[5], keep_ptr, ptr_kind, fold[0], fold[1], fold[2])
        if rc != OK:
            self._ck(rc)
        self.n_frames = c[5]

    def fold_keep_masks(self, keep_ptr: int, voi_index_ptr: int, n: int, global_keep_ptr: int, n_global: int):
        """device pointers; asynchronous on the handle's stream; accumulates (reset_keep_mask starts a job)"""
        self._ck(self.L.erasor_fold_keep_masks(self.h, c_void_p(keep_ptr), c_void_p(voi_index_ptr), n, c_void_p(global_keep_ptr), n_global))

    def reset_keep_mask(self, global_keep_ptr: int, n_global: int):
        self._ck(self.L.erasor_reset_keep_mask(self.h, c_void_p(global_keep_ptr), n_global))

    def wait(self):
        """Complete the handle's asynchronous submission (``*_async``)."""
        rc = self.L.erasor_wait(self.h)
        if rc != OK:
            self._ck(rc)

    # -- map-resident node mode -----------------------------------------------------------------
    def attach_map(self, m: "Map"):
        self._ck(self.L.erasor_attach_map(self.h, m.h if m is not None else None))
        self._map = m

    def process_nodes(self, poses7, query_xyzi, query_offsets, voi_max_range: float = 0.0, want_frame_keep: bool = False, packed_xyz: bool = False):
        """Host-buffer node batch: returns (folded keep mask of the map after this batch, per-frame masks or None).
        packed_xyz: ship the queries as packed x y z (ERASOR_PTR_QUERY_XYZ) -- the masks do not depend on the intensity."""
        P = np.ascontiguousarray(poses7, dtype=np.float64).reshape(-1, 7)
        q = _cloud(query_xyzi)
        if packed_xyz:
            q = np.ascontiguousarray(q[:, :3])
        qo = np.ascontiguousarray(query_offsets, dtype=np.uint64)
        F = len(qo) - 1
        assert len(P) == F
        n = self._map.size
        keep = np.empty(n, dtype=np.uint8)
        fk = np.empty((F, n), dtype=np.uint8) if want_frame_keep else None
        self._ck(self.L.erasor_process_nodes(self.h, P.ctypes.data_as(POINTER(c_double)), q.ctypes.data, qo.ctypes.data_as(POINTER(c_uint64)), F,
                                             float(voi_max_range), fk.ctypes.data if fk is not None else None, keep.ctypes.data,
                                             PTR_HOST | (PTR_QUERY_XYZ if packed_xyz else 0)))
        self.n_frames = F
        return keep, fk

    def process_nodes_ptr(self, poses7: np.ndarray, query_ptr: int, query_offsets: np.ndarray, voi_max_range: float, frame_keep_ptr: int,
                          keep_out_ptr: int, ptr_kind: int, asynchronous: bool = False):
        """Raw-pointer node batch (device tensors or pinned host memory).  poses7: contiguous float64 [F,7]; offsets uint64 [F+1]."""
        key = (id(poses7), id(query_offsets))
        c = getattr(self, "_node_cache", None)
        if c is None or c[0] != key:
            assert poses7.dtype == np.float64 and poses7.flags["C_CONTIGUOUS"] and query_offsets.dtype == np.uint64
            c = (key, poses7, query_offsets, poses7.ctypes.data_as(POINTER(c_double)), query_offsets.ctypes.data_as(POINTER(c_uint64)), len(query_offsets) - 1)
            self._node_cache = c
        fn = self.L.erasor_process_nodes_async if asynchronous else self.L.erasor_process_nodes
        rc = fn(self.h, c[3], query_ptr, c[4], c[5], voi_max_range, frame_keep_ptr or None, keep_out_ptr or None, ptr_kind)
        if rc != OK:
            self._ck(rc)
        self.n_frames = c[5]

    def node_stats(self):
        F = self.n_frames
        nv, nf, nr = (np.zeros(F, dtype=np.uint32) for _ in range(3))
        self._ck(self.L.erasor_get_node_stats(self.h, nv.ctypes.data_as(POINTER(c_uint32)), nf.ctypes.data_as(POINTER(c_uint32)),
                                              nr.ctypes.data_as(POINTER(c_uint32))))
        return nv, nf, nr

    # -- sweeps of the Scan Ratio Test and ground-filter fields (DESIGN.md sections 8.5 and 8.6) -----------------------------------
    def sweep_variants(self, variants):
        """variants (dicts or objects with any of SRT_SWEEP_FIELDS; a missing field takes the handle's value) -> SrtVariantC array"""
        vs = list(variants)
        arr = (SrtVariantC * max(len(vs), 1))()
        for i, v in enumerate(vs):
            get = v.get if isinstance(v, dict) else (lambda k, d, v=v: getattr(v, k, d))
            arr[i].scan_ratio_threshold = float(get("scan_ratio_threshold", self.params.scan_ratio_threshold))
            arr[i].th_bin_max_h = float(get("th_bin_max_h", self.params.th_bin_max_h))
            arr[i].minimum_num_pts = int(get("minimum_num_pts", self.params.minimum_num_pts))
        return arr, len(vs)

    def sweep_settings(self, settings):
        """settings (dicts or objects with any of SRT_SWEEP_FIELDS + GF_SWEEP_FIELDS; a missing field takes the handle's value)
        -> SweepSettingC array"""
        ss = list(settings)
        arr = (SweepSettingC * max(len(ss), 1))()
        for i, v in enumerate(ss):
            get = v.get if isinstance(v, dict) else (lambda k, d, v=v: getattr(v, k, d))
            for name, typ in SweepSettingC._fields_:
                setattr(arr[i], name, (float if typ is c_double else int)(get(name, getattr(self.params, name))))
        return arr, len(ss)

    def process_nodes_sweep(self, poses7, query_xyzi, query_offsets, variants, keep_ptr: int, voi_max_range: float = 0.0,
                            packed_xyz: bool = False, asynchronous: bool = False):
        """erasor_process_nodes_sweep: the node batch against the attached map under every Scan Ratio Test setting of `variants`
        (1..32), mask v folded into the device bytes [keep_ptr + v n_map, keep_ptr + (v + 1) n_map) (they accumulate: start with
        reset_keep_mask(keep_ptr, V n_map)).  query_xyzi: a host float32 [n,4] array (shipped as packed x y z with packed_xyz) or a
        device pointer (int; packed x y z with packed_xyz).  The map's own keep mask is left as it is."""
        arr, V = self.sweep_variants(variants)
        fn = self.L.erasor_process_nodes_sweep_async if asynchronous else self.L.erasor_process_nodes_sweep
        self._sweep(fn, poses7, query_xyzi, query_offsets, arr, V, keep_ptr, voi_max_range, packed_xyz)

    def process_nodes_sweep_ex(self, poses7, query_xyzi, query_offsets, settings, keep_ptr: int, voi_max_range: float = 0.0,
                               packed_xyz: bool = False, asynchronous: bool = False):
        """erasor_process_nodes_sweep_ex: process_nodes_sweep over settings that may also vary GF_SWEEP_FIELDS (DESIGN.md
        section 8.6); arguments as process_nodes_sweep, settings as sweep_settings takes them."""
        arr, V = self.sweep_settings(settings)
        fn = self.L.erasor_process_nodes_sweep_ex_async if asynchronous else self.L.erasor_process_nodes_sweep_ex
        self._sweep(fn, poses7, query_xyzi, query_offsets, arr, V, keep_ptr, voi_max_range, packed_xyz)

    def tune_settings(self, settings):
        """settings (dicts or objects with any of SRT_SWEEP_FIELDS + GF_SWEEP_FIELDS + GEOMETRY_SWEEP_FIELDS; a missing field takes
        the handle's value) -> TuneSettingC array"""
        ss = list(settings)
        arr = (TuneSettingC * max(len(ss), 1))()
        for i, v in enumerate(ss):
            get = v.get if isinstance(v, dict) else (lambda k, d, v=v: getattr(v, k, d))
            for part, ctype in ((arr[i].geometry, GeometryC), (arr[i].s, SweepSettingC)):
                for name, typ in ctype._fields_:
                    setattr(part, name, (float if typ is c_double else int)(get(name, getattr(self.params, name))))
        return arr, len(ss)

    def process_nodes_tune(self, poses7, query_xyzi, query_offsets, settings, keep_ptr: int, voi_max_range: float = 0.0,
                           packed_xyz: bool = False, asynchronous: bool = False):
        """erasor_process_nodes_tune: process_nodes_sweep_ex over settings that may also vary GEOMETRY_SWEEP_FIELDS (DESIGN.md
        section 8.7); arguments as process_nodes_sweep, settings as tune_settings takes them.  voi_max_range <= 0 takes the
        settings' common max_range (refused when they differ)."""
        arr, V = self.tune_settings(settings)
        fn = self.L.erasor_process_nodes_tune_async if asynchronous else self.L.erasor_process_nodes_tune
        self._sweep(fn, poses7, query_xyzi, query_offsets, arr, V, keep_ptr, voi_max_range, packed_xyz)

    def _sweep(self, fn, poses7, query_xyzi, query_offsets, arr, V, keep_ptr, voi_max_range, packed_xyz):
        P = np.ascontiguousarray(poses7, dtype=np.float64).reshape(-1, 7)
        qo = np.ascontiguousarray(query_offsets, dtype=np.uint64)
        F = len(qo) - 1
        assert len(P) == F
        if isinstance(query_xyzi, (int, np.integer)):
            qptr, kind = c_void_p(int(query_xyzi)) if int(query_xyzi) else None, PTR_DEVICE
        else:
            q = _cloud(query_xyzi)
            if packed_xyz:
                q = np.ascontiguousarray(q[:, :3])
            self._keep = [q]
            qptr, kind = q.ctypes.data, PTR_HOST
        self._sweep_args = (P, qo, arr)      # alive until the asynchronous submission has been waited for
        self._ck(fn(self.h, P.ctypes.data_as(POINTER(c_double)), qptr, qo.ctypes.data_as(POINTER(c_uint64)), F, float(voi_max_range),
                    arr, V, c_void_p(keep_ptr) if keep_ptr else None, kind | (PTR_QUERY_XYZ if packed_xyz else 0)))
        self.n_frames = F
        self.n_variants = V

    def sweep_stats(self):
        """(flagged bins, rejected points) of the last sweep, uint32 [V, F] each"""
        V, F = self.n_variants, self.n_frames
        nf, nr = np.zeros((V, F), dtype=np.uint32), np.zeros((V, F), dtype=np.uint32)
        self._ck(self.L.erasor_get_sweep_stats(self.h, nf.ctypes.data_as(POINTER(c_uint32)), nr.ctypes.data_as(POINTER(c_uint32))))
        return nf, nr

    # -- batched voxelize_preserving_labels (query preparation, saving node mode's map) -----------------------------------------
    def voxelize_batch_ptr(self, xyzi_ptr: int, offsets, leaf: float, keep_ptr: int = 0, pose7=None, ptr_kind: int = PTR_HOST):
        """erasor_voxelize_batch on raw pointers -> (device pointer of the voxels, uint64 output offsets [F+1]).  The voxels stay in
        the handle's device memory until its next voxelize_batch call."""
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        F = len(off) - 1
        oo = np.zeros(max(F + 1, 1), dtype=np.uint64)
        P = None if pose7 is None else np.ascontiguousarray(pose7, dtype=np.float64).reshape(7)
        d = c_void_p()
        self._ck(self.L.erasor_voxelize_batch(self.h, c_void_p(xyzi_ptr) if xyzi_ptr else None, off.ctypes.data_as(POINTER(c_uint64)), F,
                                              c_void_p(keep_ptr) if keep_ptr else None, float(leaf),
                                              P.ctypes.data_as(POINTER(c_double)) if P is not None else None, ptr_kind, ctypes.byref(d),
                                              oo.ctypes.data_as(POINTER(c_uint64))))
        return int(d.value or 0), oo

    def voxelize_batch(self, xyzi, offsets, leaf: float, keep=None, pose7=None):
        """Host clouds (float32 [n,4], cloud c = xyzi[offsets[c]:offsets[c+1]]) -> (voxels float32 [m,4], output offsets [F+1]):
        voxelize_preserving_labels of every cloud (keep: optional uint8 [n]), then pose7 (lidar -> body) when given."""
        x = _cloud(xyzi)
        k = None if keep is None else np.ascontiguousarray(keep, dtype=np.uint8)
        d, oo = self.voxelize_batch_ptr(x.ctypes.data if len(x) else 0, offsets, leaf, k.ctypes.data if k is not None and len(k) else 0,
                                        pose7, PTR_HOST)
        out = np.empty((int(oo[-1]), 4), dtype=np.float32)
        _memcpy_from_device(out, d)
        return out, oo

    def process_scans(self, poses7, raw_xyzi, raw_offsets, query_voxel_size: float, lidar2body7, voi_max_range: float = 0.0,
                      want_frame_keep: bool = False, ptr_kind: int = PTR_HOST):
        """Node mode from raw lidar scans (callback_node's query preparation, OfflineMapUpdater.cpp:237-241, then
        erasor_process_nodes): every scan voxelised at query_voxel_size and moved to the body frame in one submission, then the batch
        against the attached map, on the device throughout.  raw_xyzi: float32 [n,4] host array, or a device pointer with
        ptr_kind = PTR_DEVICE.  Returns (the map's keep mask after this batch, per-frame masks or None)."""
        if ptr_kind == PTR_DEVICE:
            d, qo = self.voxelize_batch_ptr(int(raw_xyzi), raw_offsets, query_voxel_size, 0, lidar2body7, PTR_DEVICE)
        else:
            x = _cloud(raw_xyzi)
            d, qo = self.voxelize_batch_ptr(x.ctypes.data if len(x) else 0, raw_offsets, query_voxel_size, 0, lidar2body7, PTR_HOST)
        P = np.ascontiguousarray(poses7, dtype=np.float64).reshape(-1, 7)
        F = len(qo) - 1
        assert len(P) == F
        fk_dev = None
        if want_frame_keep:
            import torch
            fk_dev = torch.empty((F, self._map.size), dtype=torch.uint8, device=f"cuda:{self._device}")
        self._ck(self.L.erasor_process_nodes(self.h, P.ctypes.data_as(POINTER(c_double)), c_void_p(d) if d else None,
                                             qo.ctypes.data_as(POINTER(c_uint64)), F, float(voi_max_range),
                                             c_void_p(fk_dev.data_ptr()) if fk_dev is not None else None, None, PTR_DEVICE))
        self.n_frames = F
        keep = self._map.get_keep()
        return keep, (fk_dev.cpu().numpy() if fk_dev is not None else None)

    # -- node-mode re-test, pass 2 (DESIGN.md section 8.4.1) -----------------------------------------------------------------------
    def process_nodes_retest(self, poses7, query_xyzi, query_offsets, first_node: int, voi_max_range: float = 0.0, packed_xyz: bool = False):
        """erasor_process_nodes_retest with host buffers: node f of the batch is store node first_node + f of the attached re-test
        map (Map.create_retest) and sees only its extent.  Returns the map's keep mask after this batch."""
        P = np.ascontiguousarray(poses7, dtype=np.float64).reshape(-1, 7)
        q = _cloud(query_xyzi)
        if packed_xyz:
            q = np.ascontiguousarray(q[:, :3])
        qo = np.ascontiguousarray(query_offsets, dtype=np.uint64)
        F = len(qo) - 1
        assert len(P) == F
        keep = np.empty(max(self._map.size, 1), dtype=np.uint8)
        self._ck(self.L.erasor_process_nodes_retest(self.h, P.ctypes.data_as(POINTER(c_double)), q.ctypes.data if len(q) else None,
                                                    qo.ctypes.data_as(POINTER(c_uint64)), F, int(first_node), float(voi_max_range),
                                                    keep.ctypes.data, PTR_HOST | (PTR_QUERY_XYZ if packed_xyz else 0)))
        self.n_frames = F
        return keep[:self._map.size]

    def process_nodes_retest_ptr(self, poses7: np.ndarray, query_ptr: int, query_offsets: np.ndarray, first_node: int, voi_max_range: float,
                                 keep_out_ptr: int, ptr_kind: int, asynchronous: bool = False):
        """Raw-pointer form of process_nodes_retest (device tensors or pinned host memory); poses7 and query_offsets must stay alive
        until an asynchronous submission has been waited for."""
        assert poses7.dtype == np.float64 and poses7.flags["C_CONTIGUOUS"] and query_offsets.dtype == np.uint64
        fn = self.L.erasor_process_nodes_retest_async if asynchronous else self.L.erasor_process_nodes_retest
        F = len(query_offsets) - 1
        self._ck(fn(self.h, poses7.ctypes.data_as(POINTER(c_double)), c_void_p(query_ptr) if query_ptr else None,
                    query_offsets.ctypes.data_as(POINTER(c_uint64)), F, int(first_node), float(voi_max_range),
                    c_void_p(keep_out_ptr) if keep_out_ptr else None, ptr_kind))
        self.n_frames = F

    def process_scans_retest(self, poses7, raw_xyzi, raw_offsets, query_voxel_size: float, lidar2body7, first_node: int,
                             voi_max_range: float = 0.0, ptr_kind: int = PTR_HOST):
        """process_scans for the re-test pass: the raw scans voxelised and moved to the body frame again (erasor_voxelize_batch is
        deterministic, so these are the queries pass 1 saw), then erasor_process_nodes_retest from store node first_node.  Returns
        the attached re-test map's keep mask after this batch."""
        if ptr_kind == PTR_DEVICE:
            d, qo = self.voxelize_batch_ptr(int(raw_xyzi), raw_offsets, query_voxel_size, 0, lidar2body7, PTR_DEVICE)
        else:
            x = _cloud(raw_xyzi)
            d, qo = self.voxelize_batch_ptr(x.ctypes.data if len(x) else 0, raw_offsets, query_voxel_size, 0, lidar2body7, PTR_HOST)
        P = np.ascontiguousarray(poses7, dtype=np.float64).reshape(-1, 7)
        F = len(qo) - 1
        assert len(P) == F
        self._ck(self.L.erasor_process_nodes_retest(self.h, P.ctypes.data_as(POINTER(c_double)), c_void_p(d) if d else None,
                                                    qo.ctypes.data_as(POINTER(c_uint64)), F, int(first_node), float(voi_max_range), None,
                                                    PTR_DEVICE))
        self.n_frames = F
        return self._map.get_keep()

    def save_static_map(self, m: "Map", voxel: float) -> np.ndarray:
        """save_static_map of node mode (OfflineMapUpdater.cpp:174-196 without the file): the resident map's points under its keep
        mask, followed by the map's insert store (empty unless inserts were appended), voxelised at `voxel`, in the map frame."""
        d, n = c_void_p(), c_size_t()
        self._ck(self.L.erasor_save_node_map(self.h, m.h, float(voxel), ctypes.byref(d), ctypes.byref(n)))
        out = np.empty((n.value, 4), dtype=np.float32)
        _memcpy_from_device(out, d.value or 0)
        return out

    # -- node-mode inserts (DESIGN.md section 8.4) -------------------------------------------------------------------------------
    def set_node_inserts(self, enable: bool):
        """Opt in (or out) of building each node's inserted points in process_nodes / process_scans."""
        self._ck(self.L.erasor_set_node_inserts(self.h, 1 if enable else 0))

    def node_inserts_ptr(self):
        """The last node call's inserts: (device pointer of float4 points, uint64 offsets [F+1]), valid until the next submission."""
        off = np.zeros(self.n_frames + 1, dtype=np.uint64)
        d = c_void_p()
        self._ck(self.L.erasor_get_node_inserts(self.h, ctypes.byref(d), off.ctypes.data_as(POINTER(c_uint64))))
        return int(d.value or 0), off

    def node_inserts(self):
        """The last node call's inserts in the map frame: (float32 [n,4], uint64 offsets [F+1]; node f = [off[f], off[f+1]))."""
        d, off = self.node_inserts_ptr()
        out = np.empty((int(off[-1]), 4), dtype=np.float32)
        _memcpy_from_device(out, d)
        return out, off

    # -- the exchange step ------------------------------------------------------------------------
    def comm_init(self, id128: bytes, n_ranks: int, rank: int):
        buf = (ctypes.c_uint8 * 128).from_buffer_copy(id128)
        self._ck(self.L.erasor_comm_init(self.h, buf, n_ranks, rank))

    def comm_destroy(self):
        self._ck(self.L.erasor_comm_destroy(self.h))

    def and_keep_masks(self, masks_ptr: int, n_masks: int, n: int, out_ptr: int):
        self._ck(self.L.erasor_and_keep_masks(self.h, c_void_p(masks_ptr), n_masks, n, c_void_p(out_ptr)))

    def allgather_and_keep(self, global_keep_ptr: int, n_global: int):
        """device pointer; asynchronous on the handle's stream; no-op without a communicator"""
        self._ck(self.L.erasor_allgather_and_keep(self.h, c_void_p(global_keep_ptr), n_global))

    def frame_stats(self):
        F = self.n_frames
        nf, nr = np.zeros(F, dtype=np.uint32), np.zeros(F, dtype=np.uint32)
        self._ck(self.L.erasor_get_frame_stats(self.h, nf.ctypes.data_as(POINTER(c_uint32)), nr.ctypes.data_as(POINTER(c_uint32))))
        return nf, nr

    # -- instrumentation ------------------------------------------------------------------------
    def kernel_launch_count(self) -> int:
        return int(self.L.erasor_kernel_launch_count(self.h))

    def reset_kernel_times(self, enable: bool):
        self._ck(self.L.erasor_reset_kernel_times(self.h, 1 if enable else 0))

    def srt_profile(self):
        out = np.zeros(8, dtype=np.uint32)
        self._ck(self.L.erasor_get_srt_profile(self.h, out.ctypes.data_as(POINTER(c_uint32))))
        return out

    def rgpf_profile(self):
        n = c_size_t(0)
        self._ck(self.L.erasor_get_rgpf_profile(self.h, None, None, ctypes.byref(n)))
        k = n.value
        npts = np.zeros(k, dtype=np.uint32)
        prof = np.zeros((k, 8), dtype=np.uint32)
        cap = c_size_t(k)
        if k:
            self._ck(self.L.erasor_get_rgpf_profile(self.h, npts.ctypes.data_as(POINTER(c_uint32)), prof.ctypes.data_as(POINTER(c_uint32)), ctypes.byref(cap)))
        return npts, prof

    def k1_profile(self):
        """K1 of the last node-mode batch as its profiling build: uint32 [chunk, warp, 8] -- SM cycles of scan, compaction,
        transform + bin, table update, list stores, barrier + flush, then the warp's total and dense rows (all ones: query chunk)."""
        n, nw = c_size_t(0), c_int(0)
        self._ck(self.L.erasor_profile_k1(self.h, None, ctypes.byref(n), ctypes.byref(nw)))
        out = np.zeros(n.value, dtype=np.uint32)
        self._ck(self.L.erasor_profile_k1(self.h, out.ctypes.data_as(POINTER(c_uint32)), ctypes.byref(n), ctypes.byref(nw)))
        return out.reshape(-1, nw.value, 8)

    def kernel_time_ms(self, kernel_id: int):
        t, n = c_double(), c_uint64()
        self._ck(self.L.erasor_get_kernel_time_ms(self.h, kernel_id, ctypes.byref(t), ctypes.byref(n)))
        return t.value, n.value


def comm_unique_id() -> bytes:
    """NCCL unique id for erasor_comm_init (call on rank 0, ship the bytes to the other ranks)."""
    buf = (ctypes.c_uint8 * 128)()
    rc = lib().erasor_comm_unique_id(buf)
    if rc != OK:
        raise ErasorError(rc, (lib().erasor_last_error(None) or b"").decode())
    return bytes(buf)


class Map(_Native):
    """One ``erasor_map_t``: the global map resident in HBM plus its global keep mask.  A map keeps no error message of its own:
    erasor_last_error(NULL) reports a failed create, and the other calls' errors name the call."""
    _DESTROY, _LAST_ERROR = "erasor_map_destroy", "erasor_last_error"

    def __init__(self, map_xyzi=None, device: int = 0, device_ptr: int = 0, n: int = 0):
        if device_ptr:
            self._create("erasor_map_create", c_void_p(device_ptr), n, PTR_DEVICE, device)
        else:
            m = _cloud(map_xyzi)
            self._create("erasor_map_create", m.ctypes.data, len(m), PTR_HOST, device)

    @property
    def size(self) -> int:
        return int(self.L.erasor_map_size(self.h))

    @property
    def keep_ptr(self) -> int:
        return self.L.erasor_map_keep_device(self.h) or 0

    @property
    def points_ptr(self) -> int:
        return self.L.erasor_map_points_device(self.h) or 0

    def reset_keep(self):
        rc = self.L.erasor_map_reset_keep(self.h)
        if rc != OK:
            raise ErasorError(rc, "erasor_map_reset_keep")

    def get_keep(self) -> np.ndarray:
        out = np.empty(self.size, dtype=np.uint8)
        rc = self.L.erasor_map_get_keep(self.h, out.ctypes.data, PTR_HOST)
        if rc != OK:
            raise ErasorError(rc, "erasor_map_get_keep")
        return out

    def append_inserts(self, h: "Handle"):
        """Append h's last node call's inserts to the map's store (callers append in node order)."""
        rc = self.L.erasor_map_append_inserts(self.h, h.h)
        if rc != OK:
            raise ErasorError(rc, h._message(h.h))

    def inserts(self) -> np.ndarray:
        d, n = c_void_p(), c_size_t()
        rc = self.L.erasor_map_inserts(self.h, ctypes.byref(d), ctypes.byref(n))
        if rc != OK:
            raise ErasorError(rc, "erasor_map_inserts")
        out = np.empty((n.value, 4), dtype=np.float32)
        _memcpy_from_device(out, d.value or 0)
        return out

    def clear_inserts(self):
        rc = self.L.erasor_map_clear_inserts(self.h)
        if rc != OK:
            raise ErasorError(rc, "erasor_map_clear_inserts")

    # -- node-mode re-test (DESIGN.md section 8.4.1) -------------------------------------------------------------------------------
    def create_retest(self) -> "Map":
        """The re-test map of this map (erasor_map_create_retest): the kept points in map order, then the insert store in node
        order; keep all ones, empty store.  This map is not changed."""
        r = Map.__new__(Map)
        r._create("erasor_map_create_retest", self.h)
        return r

    def retest_extents(self) -> np.ndarray:
        """uint64 [n_nodes]: store node k sees the prefix [0, extents[k]) of this re-test map"""
        n = c_size_t(0)
        rc = self.L.erasor_map_retest_extents(self.h, ctypes.byref(n), None)
        if rc != OK:
            raise ErasorError(rc, "erasor_map_retest_extents: not a re-test map")
        out = np.zeros(n.value, dtype=np.uint64)
        if n.value:
            rc = self.L.erasor_map_retest_extents(self.h, ctypes.byref(n), out.ctypes.data_as(POINTER(c_uint64)))
            if rc != OK:
                raise ErasorError(rc, "erasor_map_retest_extents")
        return out


class Updater(_Native):
    """Device-resident mirror of ``erasor::OfflineMapUpdater`` (one ``erasor_updater_t``)."""
    _DESTROY, _LAST_ERROR = "erasor_updater_destroy", "erasor_updater_last_error"
    MAP_ARRANGED, MAP_VOI, QUERY_VOI, MAP_REJECTED, OUTSKIRTS, SUBMAP_COMPLEMENT = 0, 1, 2, 5, 7, 8

    def __init__(self, up, ep: ErasorParams, initial_map, device: int = 0):
        self.ep, self.up = ep, up
        upc = UpdaterParamsC()
        upc.query_voxel_size, upc.map_voxel_size = up.query_voxel_size, up.map_voxel_size
        upc.removal_interval, upc.is_large_scale = up.removal_interval, 1 if up.is_large_scale else 0
        upc.submap_size, upc.max_range, upc.version = up.submap_size, up.max_range, up.version
        for i in range(7):
            upc.lidar2body[i] = up.lidar2body[i]
        self._upc, self._epc = upc, ep.to_c()
        m = _cloud(initial_map)
        self._create("erasor_updater_create", ctypes.byref(upc), ctypes.byref(self._epc), m.ctypes.data, len(m), device)

    def reset(self, initial_map):
        m = _cloud(initial_map)
        self._ck(self.L.erasor_updater_reset(self.h, m.ctypes.data, len(m)))

    def process_node(self, seq: int, odom7, lidar) -> bool:
        o = np.ascontiguousarray(odom7, dtype=np.float64)
        l = _cloud(lidar)
        done = c_int(0)
        self._ck(self.L.erasor_updater_process_node(self.h, seq, o.ctypes.data_as(POINTER(c_double)), l.ctypes.data, len(l), PTR_HOST, ctypes.byref(done)))
        return bool(done.value)

    def prefetch_scan_ptr(self, lidar_ptr: int, n: int, ptr_kind: int):
        """Look-ahead: start the upload + voxelisation of the NEXT processed node's scan (consumed by the process_node_ptr call
        that is given the same pointer and size)."""
        self._ck(self.L.erasor_updater_prefetch_scan(self.h, c_void_p(lidar_ptr), n, ptr_kind))

    def process_node_ptr(self, seq: int, odom7, lidar_ptr: int, n: int, ptr_kind: int) -> bool:
        o = np.ascontiguousarray(odom7, dtype=np.float64)
        done = c_int(0)
        self._ck(self.L.erasor_updater_process_node(self.h, seq, o.ctypes.data_as(POINTER(c_double)), c_void_p(lidar_ptr), n, ptr_kind, ctypes.byref(done)))
        return bool(done.value)

    def cloud(self, which: int) -> np.ndarray:
        return self._read_cloud(lambda out, cap, n: self.L.erasor_updater_get_cloud(self.h, which, out, cap, n, PTR_HOST))

    def map_size(self) -> int:
        n = c_size_t(0)
        self._ck(self.L.erasor_updater_map_size(self.h, ctypes.byref(n)))
        return n.value

    def save_static_map(self, voxel_size: float) -> np.ndarray:
        return self._read_cloud(lambda out, cap, n: self.L.erasor_updater_save_static_map(self.h, voxel_size, out, cap, n))

    def voxelize(self, cloud, leaf: float) -> np.ndarray:
        c = _cloud(cloud)
        out = np.empty((max(len(c), 1), 4), dtype=np.float32)
        n = c_size_t(0)
        self._ck(self.L.erasor_updater_voxelize(self.h, c.ctypes.data, len(c), leaf, out.ctypes.data, len(out), ctypes.byref(n)))
        return out[:n.value].copy()

    def mapgen_node(self, odom7, lidar) -> np.ndarray:
        """mapgen's accumPointCloud up to cloud_curr, on the device (body cut, lift, pose, 0.2 m voxelisation)."""
        o = np.ascontiguousarray(odom7, dtype=np.float64)
        c = _cloud(lidar)
        out = np.empty((max(len(c), 1), 4), dtype=np.float32)
        n = c_size_t(0)
        self._ck(self.L.erasor_updater_mapgen_node(self.h, o.ctypes.data_as(POINTER(c_double)), c.ctypes.data, len(c), PTR_HOST, out.ctypes.data, len(out),
                                                   ctypes.byref(n)))
        return out[:n.value].copy()

    def kernel_launch_count(self) -> int:
        return int(self.L.erasor_updater_kernel_launch_count(self.h))

    def fused_profile(self):
        """Phase boundaries (ns) of the last fused prologue launch, relative to its start (include/erasor_b200.h)."""
        t = np.zeros(16, dtype=np.uint64)
        self._ck(self.L.erasor_updater_get_fused_profile(self.h, t.ctypes.data))
        return [int(x) - int(t[0]) if x else None for x in t]


class Evaluator(_Native):
    """One ``erasor_eval_t``: PR / RR on the device, the counts of ``evaluate.evaluate`` by an exact grid-indexed 1-NN
    (DESIGN.md section 11).  ``evaluate`` and ``evaluate_map`` return exactly ``evaluate.evaluate``'s dict; ``last_counts()``
    adds ``inliers``, ``ambiguous_ties`` (inliers whose equally-nearest estimate points hold both classes -- the counts equal
    sklearn's whenever it is 0) and, when asked for, ``match``.  Unlike sklearn, an empty estimate is no error: no GT point
    is an inlier."""
    _DESTROY, _LAST_ERROR = "erasor_eval_destroy", "erasor_eval_last_error"

    def __init__(self, device: int = 0):
        self._create("erasor_eval_create", device)
        self._last = None

    def _finish(self, c: EvalCountsC, match) -> dict:
        from . import evaluate
        self._last = {name: int(getattr(c, name)) for name, _ in EvalCountsC._fields_}
        if match is not None:
            self._last["match"] = match
        return evaluate.rates(c.gt_static, c.gt_dynamic, c.preserved_static, c.preserved_dynamic)

    def evaluate(self, gt, est, keep=None, voxelsize: float = 0.2, want_match: bool = False) -> dict:
        """Host clouds (float32 [n,4] x y z intensity); keep: optional uint8 mask over est (nonzero = part of the estimate)."""
        g, e = _cloud(gt), _cloud(est)
        k = None
        if keep is not None:
            k = np.ascontiguousarray(keep, dtype=np.uint8).reshape(-1)
            if len(k) != len(e):
                raise ValueError("keep must have one entry per estimate point")
        match = np.empty(len(g), dtype=np.uint32) if want_match else None
        c = EvalCountsC()
        self._ck(self.L.erasor_evaluate(self.h, g.ctypes.data, len(g), e.ctypes.data, len(e), k.ctypes.data if k is not None else None,
                                        float(voxelsize), PTR_HOST, match.ctypes.data if match is not None else None, ctypes.byref(c)))
        return self._finish(c, match)

    def evaluate_ptr(self, gt_ptr: int, n_gt: int, est_ptr: int, n_est: int, keep_ptr: int = 0, voxelsize: float = 0.2,
                     ptr_kind: int = PTR_DEVICE, match_ptr: int = 0) -> dict:
        """Raw pointers (device memory with PTR_DEVICE, float4-aligned clouds); match_ptr: optional uint32 [n_gt] output."""
        c = EvalCountsC()
        self._ck(self.L.erasor_evaluate(self.h, c_void_p(gt_ptr), n_gt, c_void_p(est_ptr), n_est, c_void_p(keep_ptr) if keep_ptr else None,
                                        float(voxelsize), ptr_kind, c_void_p(match_ptr) if match_ptr else None, ctypes.byref(c)))
        return self._finish(c, None)

    def evaluate_map(self, m: "Map", voxelsize: float = 0.2) -> dict:
        """Score a resident map in place: GT = the initial map, estimate = its points with keep != 0 (what bench.py's
        final_map_quality builds on the host).  The handles that write the mask must have finished."""
        n = m.size
        return self.evaluate_ptr(m.points_ptr, n, m.points_ptr, n, m.keep_ptr, voxelsize, PTR_DEVICE)

    def last_counts(self) -> dict:
        """All six counts of the last call, plus ``match`` (uint32 per GT point, NO_MATCH without an inlier) when requested."""
        return dict(self._last) if self._last is not None else None

    # -- the overlap report (erasor_eval_overlap) ------------------------------------------------------------------------------
    def _overlap(self, gt_ptr, n_gt, est_ptr, n_est, keep_ptr, voxelsize, ptr_kind, dist_ptr, n_sel) -> dict:
        from . import evaluate
        ranks = np.asarray(evaluate.overlap_ranks(n_sel) if n_sel else [], dtype=np.uint64)
        vals = np.empty(len(ranks), dtype=np.float64)
        o = EvalOverlapC()
        self._ck(self.L.erasor_eval_overlap(self.h, gt_ptr, n_gt, est_ptr, n_est, keep_ptr, float(voxelsize), ptr_kind,
                                            ranks.ctypes.data if len(ranks) else None, len(ranks), vals.ctypes.data if len(ranks) else None,
                                            dist_ptr, ctypes.byref(o)))
        self._last_overlap = {name: (float(getattr(o, name)) if name == "max" else int(getattr(o, name))) for name, _ in EvalOverlapC._fields_}
        if o.n != n_sel:
            raise ErasorError(E_STATE, f"the keep mask selects {o.n} points, not the {n_sel} the ranks were computed for")
        if not n_sel:
            return None
        return evaluate.overlap_from_ranks(n_sel, vals, o.max, (o.below_half, o.below_one, o.below_two), voxelsize)

    def overlap(self, gt, est, keep=None, voxelsize: float = 0.2, want_dist: bool = False):
        """evaluate.overlap's dict, bit for bit, for host clouds (keep: optional uint8 mask over est).  With want_dist, returns
        (dict, float64 distance per estimate point, NaN where keep drops it).  The dict is None when nothing is selected; an empty
        GT gives +inf distances.  last_overlap() has the counts, including est_static / est_dynamic and far_points."""
        g, e = _cloud(gt), _cloud(est)
        k = None
        if keep is not None:
            k = np.ascontiguousarray(keep, dtype=np.uint8).reshape(-1)
            if len(k) != len(e):
                raise ValueError("keep must have one entry per estimate point")
        n_sel = len(e) if k is None else int(np.count_nonzero(k))
        dist = np.empty(len(e), dtype=np.float64) if want_dist else None
        r = self._overlap(g.ctypes.data, len(g), e.ctypes.data, len(e), k.ctypes.data if k is not None else None, voxelsize, PTR_HOST,
                          dist.ctypes.data if dist is not None and len(dist) else None, n_sel)
        return (r, dist) if want_dist else r

    def overlap_ptr(self, gt_ptr: int, n_gt: int, est_ptr: int, n_est: int, keep_ptr: int = 0, voxelsize: float = 0.2,
                    ptr_kind: int = PTR_DEVICE, dist_ptr: int = 0, n_sel: int | None = None):
        """Raw pointers (device memory with PTR_DEVICE); dist_ptr: optional float64 [n_est] output.  n_sel: how many points keep
        selects -- without it and with a keep mask, erasor_eval_count_selected counts them first (one pass over the mask)."""
        if n_sel is None:
            n_sel = self.count_selected(keep_ptr, n_est, ptr_kind) if keep_ptr else n_est
        return self._overlap(c_void_p(gt_ptr), n_gt, c_void_p(est_ptr), n_est, c_void_p(keep_ptr) if keep_ptr else None, voxelsize, ptr_kind,
                             c_void_p(dist_ptr) if dist_ptr else None, n_sel)

    def count_selected(self, keep_ptr: int, n: int, ptr_kind: int = PTR_DEVICE) -> int:
        """how many of the n keep bytes at keep_ptr are nonzero"""
        c = c_uint64()
        self._ck(self.L.erasor_eval_count_selected(self.h, c_void_p(keep_ptr), n, ptr_kind, ctypes.byref(c)))
        return int(c.value)

    def overlap_map(self, m: "Map", voxelsize: float = 0.2, dist_ptr: int = 0):
        """The overlap report of a resident map scored in place (GT = the initial map, estimate = its points with keep != 0)."""
        n = m.size
        return self.overlap_ptr(m.points_ptr, n, m.points_ptr, n, m.keep_ptr, voxelsize, PTR_DEVICE, dist_ptr)

    def last_overlap(self) -> dict:
        """The counts of the last overlap call: n, est_static, est_dynamic, below_half / one / two, far_points, max."""
        return dict(self._last_overlap) if getattr(self, "_last_overlap", None) is not None else None

    def _report(self, d: dict, ov) -> dict:
        c = self._last_overlap
        d = dict(d)
        d["est_static"], d["est_dynamic"] = c["est_static"], c["est_dynamic"]
        d["overlap"] = ov
        return d

    def report(self, gt, est, keep=None, voxelsize: float = 0.2) -> dict:
        """evaluate.report's dict: every column of the runner's table and its overlap dict, from both device calls."""
        d = self.evaluate(gt, est, keep, voxelsize)
        return self._report(d, self.overlap(gt, est, keep, voxelsize))

    def report_map(self, m: "Map", voxelsize: float = 0.2) -> dict:
        d = self.evaluate_map(m, voxelsize)
        return self._report(d, self.overlap_map(m, voxelsize))


class PcdCodec(_Native):
    """One ``erasor_pcd_t``: PCD files read and written on the device (DESIGN.md section 12).  ``parse`` / ``read`` give what
    ``evaluate.read_pcd_ascii`` gives, bit for bit (including its KeyError for a file without x, y, z or intensity); ``load`` /
    ``load_bytes`` read any DATA mode (ascii, binary, binary_compressed) as PCL does (section 12.1); ``format`` / ``write`` give the
    bytes ``evaluate.write_pcd_ascii`` writes, except that NaN is written "nan" whatever its sign, or with ``mode`` a binary or
    binary_compressed file (section 12.3).  Files are read and written as raw bytes."""
    _DESTROY, _LAST_ERROR = "erasor_pcd_destroy", "erasor_pcd_last_error"

    def __init__(self, device: int = 0):
        self.device = device
        self._create("erasor_pcd_create", device)
        self._info = None

    def _call_parse(self, ptr, n_bytes, kind, out_ptr, cap, out_kind, require_intensity):
        n, info = c_size_t(0), PcdInfoC()
        rc = self.L.erasor_pcd_parse_ascii(self.h, ptr, n_bytes, kind, out_ptr, cap, out_kind, ctypes.byref(n), ctypes.byref(info))
        self._info = {name: int(getattr(info, name)) for name, _ in PcdInfoC._fields_}
        for bit, name in enumerate(("x", "y", "z", "intensity")):
            if info.header_lines and not (info.fields >> bit) & 1 and (bit < 3 or require_intensity):
                raise KeyError(name)                  # read_pcd_ascii's error for a missing column of a header it could read
        self._ck(rc)
        return n.value

    def parse(self, data, device_out: bool = False, require_intensity: bool = True):
        """data: the whole file -- bytes-like (host) or a CUDA uint8 tensor.  Returns float32 [rows, 4] x y z intensity: a numpy
        array, or a CUDA tensor with device_out.  require_intensity=False reads a file without intensity as the C++ reader does
        (intensity 0) instead of raising KeyError."""
        if hasattr(data, "is_cuda") and data.is_cuda:
            ptr, nb, kind, keep = c_void_p(data.data_ptr()), data.numel() * data.element_size(), PTR_DEVICE, data
        else:
            keep = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data).view(np.uint8)
            ptr, nb, kind = c_void_p(keep.ctypes.data if keep.size else 0), keep.size, PTR_HOST
        pts = self._call_parse(ptr, nb, kind, None, 0, PTR_HOST, require_intensity)
        if device_out:
            import torch
            out = torch.empty((max(pts, 1), 4), dtype=torch.float32, device=f"cuda:{self.device}")
            rows = self._call_parse(ptr, nb, kind, c_void_p(out.data_ptr()), pts, PTR_DEVICE, require_intensity)
        else:
            out = np.empty((max(pts, 1), 4), dtype=np.float32)
            rows = self._call_parse(ptr, nb, kind, c_void_p(out.ctypes.data), pts, PTR_HOST, require_intensity)
        del keep
        return out[:rows]

    def read(self, path: str, device_out: bool = False, require_intensity: bool = True):
        with open(path, "rb") as f:
            data = f.read()
        return self.parse(data, device_out, require_intensity)

    def last_info(self) -> dict:
        """points, rows, slow_tokens, error_line, header_lines, fields and has_intensity of the last parse"""
        return dict(self._info) if self._info is not None else None

    def _call_load(self, ptr, n_bytes, kind, out_ptr, cap, out_kind):
        n, info = c_size_t(0), PcdLoadInfoC()
        rc = self.L.erasor_pcd_load(self.h, ptr, n_bytes, kind, out_ptr, cap, out_kind, ctypes.byref(n), ctypes.byref(info))
        d = {name: int(getattr(info, name)) for name, _ in PcdLoadInfoC._fields_ if name != "ascii"}
        d["ascii"] = {name: int(getattr(info.ascii, name)) for name, _ in PcdInfoC._fields_}
        self._load_info = d
        self._ck(rc)
        return n.value

    def load_bytes(self, data, device_out: bool = False):
        """A PCD file in any DATA mode (ascii, binary, binary_compressed) with PCL's field rules (erasor_pcd_load): data is the
        whole file -- bytes-like (host) or a CUDA uint8 tensor.  A missing intensity, or one that is not F 4 COUNT 1, reads as 0.
        Returns float32 [n, 4] x y z intensity: a numpy array, or a CUDA tensor with device_out."""
        if hasattr(data, "is_cuda") and data.is_cuda:
            ptr, nb, kind, keep = c_void_p(data.data_ptr()), data.numel() * data.element_size(), PTR_DEVICE, data
        else:
            keep = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data).view(np.uint8)
            ptr, nb, kind = c_void_p(keep.ctypes.data if keep.size else 0), keep.size, PTR_HOST
        pts = self._call_load(ptr, nb, kind, None, 0, PTR_HOST)
        if device_out:
            import torch
            out = torch.empty((max(pts, 1), 4), dtype=torch.float32, device=f"cuda:{self.device}")
            rows = self._call_load(ptr, nb, kind, c_void_p(out.data_ptr()), pts, PTR_DEVICE)
        else:
            out = np.empty((max(pts, 1), 4), dtype=np.float32)
            rows = self._call_load(ptr, nb, kind, c_void_p(out.ctypes.data), pts, PTR_HOST)
        del keep
        return out[:rows]

    def load(self, path: str, device_out: bool = False):
        """load_bytes of the file at path"""
        with open(path, "rb") as f:
            data = f.read()
        return self.load_bytes(data, device_out)

    def last_load_info(self) -> dict:
        """erasor_pcd_load_info_t of the last load: data_mode, fields, intensity_zero_filled, point_step, width, height, points,
        data_offset, compressed_size, uncompressed_size, lzf_tokens, and the ascii branch's info as a dict under "ascii" """
        info = getattr(self, "_load_info", None)
        return dict(info) if info is not None else None

    # ---- erasor/node bags (DESIGN.md section 12.2) ----
    BAG_TOPIC = "/node/combined/optimized"

    def bag_index(self, data, topic: str = BAG_TOPIC, keep_first: bool = False) -> dict:
        """Indexes a ROS bag 2.0 file of erasor/node messages (erasor_bag_index): data is the whole file, bytes-like or a CPU uint8
        tensor (pinned memory is read by the device directly, pageable memory through pinned staging).  The codec keeps a reference
        to it until the next bag_index.  The first message on the topic is dropped unless keep_first, as the reference's subscribers
        drop it.  Returns erasor_bag_info_t as a dict."""
        if hasattr(data, "data_ptr"):
            if data.is_cuda:
                raise ValueError("bags are indexed from host memory")
            keep, ptr, nb = data, data.data_ptr(), data.numel() * data.element_size()
        else:
            keep = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data).view(np.uint8)
            ptr, nb = (keep.ctypes.data if keep.size else 0), keep.size
        n, info = c_size_t(0), BagInfoC()
        self._bag = None
        self._ck(self.L.erasor_bag_index(self.h, c_void_p(ptr) if ptr else None, nb, topic.encode(), int(bool(keep_first)), ctypes.byref(n),
                                         ctypes.byref(info)))
        self._bag, self._bag_n = keep, n.value
        d = {name: int(getattr(info, name)) for name, _ in BagInfoC._fields_ if name not in ("md5sum", "pad_")}
        d["md5sum"] = info.md5sum.decode()
        return d

    def _bag_range(self, first: int, count):
        if getattr(self, "_bag", None) is None:
            raise ErasorError(E_STATE, "no bag indexed: call bag_index first")
        return int(first), (self._bag_n - int(first) if count is None else int(count))

    def bag_meta(self, first: int = 0, count=None):
        """(seq uint32 [k], stamp_ns uint64 [k], odom7 float64 [k, 7], clouds) of nodes [first, first + k); clouds: one dict per node
        with erasor_bag_cloud_t's fields"""
        first, count = self._bag_range(first, count)
        seq, stamp, odom = np.zeros(max(count, 0), np.uint32), np.zeros(max(count, 0), np.uint64), np.zeros((max(count, 0), 7))
        cl = (BagCloudC * max(count, 1))()
        self._ck(self.L.erasor_bag_nodes(self.h, first, count, c_void_p(seq.ctypes.data), c_void_p(stamp.ctypes.data), c_void_p(odom.ctypes.data),
                                         ctypes.addressof(cl)))
        clouds = [dict({name: int(getattr(c, name)) for name, _ in BagCloudC._fields_ if name != "offset"}, offset=[int(v) for v in c.offset])
                  for c in cl[:count]]
        return seq, stamp, odom, clouds

    def bag_load(self, first: int = 0, count=None, device_out: bool = False, nodes=None):
        """(xyzi, offsets) of nodes [first, first + count), or of the listed nodes: their clouds back to back as float32 [n, 4] --
        a numpy array, or a CUDA tensor with device_out -- and uint64 offsets [count + 1], from one erasor_bag_load (one gather
        launch)"""
        if nodes is None:
            first, count = self._bag_range(first, count)
            call = lambda out, cap, kind, op: self.L.erasor_bag_load(self.h, first, count, out, cap, kind, op)
        else:
            self._bag_range(0, None)
            lst = np.ascontiguousarray(nodes, dtype=np.uint64)
            count = len(lst)
            lp = lst.ctypes.data_as(POINTER(c_uint64))
            call = lambda out, cap, kind, op: self.L.erasor_bag_load_list(self.h, lp, count, out, cap, kind, op)
        off = np.zeros(max(count, 0) + 1, dtype=np.uint64)
        op = off.ctypes.data_as(POINTER(c_uint64))
        self._ck(call(None, 0, PTR_HOST, op))
        total = int(off[-1])
        if device_out:
            import torch
            out = torch.empty((max(total, 1), 4), dtype=torch.float32, device=f"cuda:{self.device}")
            self._ck(call(c_void_p(out.data_ptr()), total, PTR_DEVICE, op))
        else:
            out = np.empty((max(total, 1), 4), dtype=np.float32)
            self._ck(call(c_void_p(out.ctypes.data), total, PTR_HOST, op))
        return out[:total], off

    def bag_lz4_stats(self) -> dict:
        """erasor_bag_lz4_stats_t of the last bag_index as a dict: lz4 chunks in the file and decoded, compressed bytes uploaded,
        decoded bytes held on the device, blocks and stored blocks, checksums verified, and the decode and checksum kernels' device
        times in ms"""
        st = BagLz4StatsC()
        self._ck(self.L.erasor_bag_lz4_stats(self.h, ctypes.byref(st)))
        return {name: (float if name.endswith("_ms") else int)(getattr(st, name)) for name, _ in BagLz4StatsC._fields_}

    def bag_bz2_stats(self) -> dict:
        """erasor_bag_bz2_stats_t of the last bag_index as a dict: bz2 chunks in the file and decoded, compressed bytes uploaded,
        decoded bytes held on the device, true blocks and block-magic candidates, streams by level (a list of 9), the decode's peak
        scratch, and the device ms of its stage groups (scan + walk + chain, decode, inverse BWT, RLE1 + CRC)"""
        st = BagBz2StatsC()
        self._ck(self.L.erasor_bag_bz2_stats(self.h, ctypes.byref(st)))
        out = {name: (float if name.endswith("_ms") else int)(getattr(st, name)) for name, _ in BagBz2StatsC._fields_ if name != "streams_by_level"}
        out["streams_by_level"] = [int(v) for v in st.streams_by_level]
        return out

    def bag_nodes(self, batch: int = 64, device_out: bool = False):
        """Yields (seq, odom7, cloud) per node of the indexed bag, as erasor_b200.kitti.iter_nodes yields them: clouds decoded
        `batch` nodes per erasor_bag_load; with device_out each cloud is a view of a CUDA tensor holding its batch."""
        _, count = self._bag_range(0, None)
        for b0 in range(0, count, int(batch)):
            nb = min(int(batch), count - b0)
            seq, _, odom, _ = self.bag_meta(b0, nb)
            xyzi, off = self.bag_load(b0, nb, device_out)
            for k in range(nb):
                yield int(seq[k]), odom[k].copy(), xyzi[int(off[k]):int(off[k + 1])]

    def _format(self, xyzi, mode: str) -> np.ndarray:
        if mode not in PCD_MODES:
            raise ValueError(f"mode must be one of {sorted(PCD_MODES)}")
        if hasattr(xyzi, "is_cuda") and xyzi.is_cuda:
            if str(xyzi.dtype) != "torch.float32" or xyzi.dim() != 2 or xyzi.shape[1] != 4 or not xyzi.is_contiguous():
                raise ValueError("device clouds are contiguous float32 [n,4] tensors")
            ptr, n, kind, keep = c_void_p(xyzi.data_ptr()), xyzi.shape[0], PTR_DEVICE, xyzi
        else:
            keep = _cloud(xyzi)
            ptr, n, kind = c_void_p(keep.ctypes.data if len(keep) else 0), len(keep), PTR_HOST
        size, info = c_size_t(0), PcdFormatInfoC()
        m = PCD_MODES[mode]
        self._ck(self.L.erasor_pcd_format(self.h, ptr, n, kind, m, None, 0, PTR_HOST, ctypes.byref(size), ctypes.byref(info)))
        out = np.empty(size.value, dtype=np.uint8)
        self._ck(self.L.erasor_pcd_format(self.h, ptr, n, kind, m, c_void_p(out.ctypes.data), size.value, PTR_HOST, ctypes.byref(size),
                                          ctypes.byref(info)))
        self._format_info = {name: int(getattr(info, name)) for name, _ in PcdFormatInfoC._fields_}
        del keep
        return out

    def format(self, xyzi, mode: str = "ascii") -> bytes:
        """the whole file for a float32 [n, 4] cloud (numpy, or a CUDA tensor) in DATA mode "ascii", "binary" or
        "binary_compressed" (erasor_pcd_format, DESIGN.md section 12.3)"""
        return self._format(xyzi, mode).tobytes()

    def write(self, path: str, xyzi, mode: str = "ascii"):
        out = self._format(xyzi, mode)
        with open(path, "wb") as f:
            f.write(memoryview(out))

    def last_format_info(self) -> dict:
        """erasor_pcd_format_info_t of the last format / write: data_mode, segments, header_bytes, uncompressed_size,
        compressed_size, lzf_tokens"""
        info = getattr(self, "_format_info", None)
        return dict(info) if info is not None else None


class MapGen(_Native):
    """One ``erasor_mapgen_t``: the reference's mapgen (src/mapgen/mapgen.hpp:198-305) with its map resident on the device
    (DESIGN.md section 8.2).  ``accum`` is accumPointCloud -- one launch, no host synchronisation unless a buffer grows; ``cloud``
    gives the four clouds of ``OracleMapGen`` by the same ids; ``save_naive_map`` is saveNaiveMap without the files."""
    _DESTROY, _LAST_ERROR = "erasor_mapgen_destroy", "erasor_mapgen_last_error"
    CLOUD_MAP, CLOUD_CURR, SAVED_ORIGINAL, SAVED_VOXELIZED = 0, 1, 2, 3

    def __init__(self, leafsize: float = 0.05, is_large_scale: bool = False, device: int = 0):
        self.device = device
        self._p = MapGenParamsC(float(leafsize), 1 if is_large_scale else 0)
        self._create("erasor_mapgen_create", ctypes.byref(self._p), device)

    def accum(self, odom7, lidar):
        """accumPointCloud with a host scan (float32 [n, 4] in the lidar frame; odom7 = x y z qx qy qz qw)."""
        o = np.ascontiguousarray(odom7, dtype=np.float64)
        c = _cloud(lidar)
        self._ck(self.L.erasor_mapgen_accum(self.h, o.ctypes.data_as(POINTER(c_double)), c.ctypes.data if len(c) else None, len(c), PTR_HOST))

    def accum_ptr(self, odom7, lidar_ptr: int, n: int, ptr_kind: int = PTR_DEVICE):
        """accumPointCloud with a raw pointer.  A device scan is read asynchronously: keep it unchanged until the next call that
        returns data, or until synchronize()."""
        o = np.ascontiguousarray(odom7, dtype=np.float64)
        self._ck(self.L.erasor_mapgen_accum(self.h, o.ctypes.data_as(POINTER(c_double)), c_void_p(lidar_ptr) if lidar_ptr else None, n, ptr_kind))

    def cloud(self, which: int) -> np.ndarray:
        return self._read_cloud(lambda out, cap, n: self.L.erasor_mapgen_get_cloud(self.h, which, out, cap, PTR_HOST, n))

    def device_cloud(self, which: int):
        """(device pointer, n) of a cloud in the handle's memory, valid until the next accum."""
        p, n = c_void_p(), c_size_t(0)
        self._ck(self.L.erasor_mapgen_device_cloud(self.h, which, ctypes.byref(p), ctypes.byref(n)))
        return int(p.value or 0), n.value

    def save_naive_map(self):
        """-> (original, voxelized): the clouds saveNaiveMap writes"""
        return self.cloud(self.SAVED_ORIGINAL), self.cloud(self.SAVED_VOXELIZED)

    def synchronize(self):
        self._ck(self.L.erasor_mapgen_synchronize(self.h))

    def counters(self) -> dict:
        """kernel launches, host synchronisations and buffer regrowths since creation"""
        a, b, c = c_uint64(), c_uint64(), c_uint64()
        self._ck(self.L.erasor_mapgen_get_counters(self.h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)))
        return {"launches": int(a.value), "host_syncs": int(b.value), "regrowths": int(c.value)}
