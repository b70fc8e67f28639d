"""Naive map builder -- the producer of the path's input map (SURVEY 8f-4; reference src/mapgen/mapgen.hpp:198-309 and its
driver src/mapgen/main.cpp:40-49), ROS stripped.

Per node (`accumPointCloud`):  drop the points within CAR_BODY_SIZE = 2.7 m of the sensor (:218-229), lift by 1.73 m (:209-232),
move to the map frame with the node's pose (:234-237), `voxelize_preserving_labels` at 0.2 m (:239), append to the map (:241-246;
large-scale mode voxelises and parks the accumulated map every 500 nodes, :247-258).  `saveNaiveMap` (:271-307) concatenates and
voxelises once more at the map's leaf size.

The arithmetic that matters for parity is here in float32 exactly as PCL's transformPointCloud does it
(((m0*x + m1*y) + m2*z) + m3, no FMA) and tf's quaternion -> matrix in double; the voxeliser is injected: on a GPU box it is the
device kernel behind `erasor_updater_voxelize` (`device_voxelizer()`), the same one the updater uses for the query scans and
`save_static_map` and that tests/test_gpu_updater.py checks bit for bit.  tests/test_mapgen.py runs this module against the
oracle's C++ restatement of mapgen with the oracle's voxeliser injected.
With `device_producer()` the whole per-node step (cut, lift, transform, voxelise) runs on the device through
`erasor_updater_mapgen_node`; tests/test_gpu_mapgen.py holds both device compositions bit-identical to the oracle's mapgen.
`device_generator()` (the default of `build_map`) keeps the map itself on the device too, behind `erasor_mapgen_*`
(capi.MapGen): one launch per node, parking included; tests/test_gpu_mapgen_resident.py holds it to the oracle.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np

CAR_BODY_SIZE = 2.7            # mapgen.hpp:8
LIDAR_HEIGHT = np.float32(1.73)   # tf_lidar2origin, mapgen.hpp:209-214
NODE_VOXEL = 0.2               # mapgen.hpp:239
SUBMAP_EVERY = 500             # mapgen.hpp:248

Voxelizer = Callable[[np.ndarray, float], np.ndarray]


def pose_to_matrix(odom7) -> np.ndarray:
    """erasor_utils::geoPose2eigen (erasor_utils.cpp:35-55): tf::Matrix3x3(q) in double, then a float 4x4."""
    x, y, z, qx, qy, qz, qw = (float(v) for v in odom7)
    d = qx * qx + qy * qy + qz * qz + qw * qw
    s = 2.0 / d
    xs, ys, zs = qx * s, qy * s, qz * s
    wx, wy, wz = qw * xs, qw * ys, qw * zs
    xx, xy, xz = qx * xs, qx * ys, qx * zs
    yy, yz, zz = qy * ys, qy * zs, qz * zs
    T = np.zeros((4, 4), dtype=np.float32)
    T[:3, :3] = np.array([[1.0 - (yy + zz), xy - wz, xz + wy],
                          [xy + wz, 1.0 - (xx + zz), yz - wx],
                          [xz - wy, yz + wx, 1.0 - (xx + yy)]], dtype=np.float64).astype(np.float32)
    T[0, 3], T[1, 3], T[2, 3], T[3, 3] = np.float32(x), np.float32(y), np.float32(z), np.float32(1.0)
    return T


def transform_point_cloud(cloud: np.ndarray, T: np.ndarray) -> np.ndarray:
    """pcl::transformPointCloud(in, out, Matrix4f) on xyz, intensity untouched: float32, left-to-right sums, no FMA."""
    c = np.ascontiguousarray(cloud, dtype=np.float32)
    T = np.asarray(T, dtype=np.float32)
    x, y, z = c[:, 0], c[:, 1], c[:, 2]
    out = c.copy()
    for r in range(3):
        out[:, r] = ((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3]
    return out


class NaiveMapGenerator:
    """mapgen's accumulate / save cycle.  `voxelize(cloud[n,4] float32, leaf) -> cloud` is voxelize_preserving_labels."""

    def __init__(self, voxelize: Voxelizer, leafsize: float = 0.05, is_large_scale: bool = False, node_producer=None):
        self.voxelize = voxelize
        self.node_producer = node_producer              # optional (odom7, lidar) -> cloud_curr: erasor_updater_mapgen_node
        self.leafsize = float(leafsize)                  # /map/voxelsize, main.cpp:83
        self.is_large_scale = bool(is_large_scale)       # /large_scale/is_large_scale, main.cpp:91
        self.cloud_map = np.zeros((0, 4), dtype=np.float32)
        self.cloud_curr = np.zeros((0, 4), dtype=np.float32)
        self.cloud_maps: List[np.ndarray] = []
        self._is_initial = True
        self._cnt_voxel = 0

    def accum_point_cloud(self, odom7, lidar: np.ndarray) -> None:
        c = np.ascontiguousarray(lidar, dtype=np.float32).reshape(-1, 4)
        if self.node_producer is not None:                  # the whole per-node step on the device
            self.cloud_curr = self.node_producer(odom7, c)
            self._append_curr()
            return
        max_dist_square = np.float64(np.float32(CAR_BODY_SIZE ** 2))                           # float threshold (:219)
        dist_square = c[:, 0].astype(np.float64) ** 2 + c[:, 1].astype(np.float64) ** 2        # double distance (:221)
        c = c[~(dist_square < max_dist_square)]
        lift = np.eye(4, dtype=np.float32)
        lift[2, 3] = LIDAR_HEIGHT
        world = transform_point_cloud(transform_point_cloud(c, lift), pose_to_matrix(odom7))
        self.cloud_curr = self.voxelize(world, NODE_VOXEL)
        self._append_curr()

    def _append_curr(self) -> None:
        if self._is_initial:
            self.cloud_map = self.cloud_curr.copy()
            self._is_initial = False
            return
        self.cloud_map = np.concatenate([self.cloud_map, self.cloud_curr])
        if self.is_large_scale:
            fire = self._cnt_voxel % SUBMAP_EVERY == 0
            self._cnt_voxel += 1
            if fire:
                self.cloud_maps.append(self.voxelize(self.cloud_map, self.leafsize))
                self.cloud_map = np.zeros((0, 4), dtype=np.float32)

    def save_naive_map(self):
        """-> (original, voxelized): what saveNaiveMap writes as <seq>_..._original.pcd and the voxelised map."""
        original = np.concatenate(self.cloud_maps + [self.cloud_map]) if self.is_large_scale else self.cloud_map
        return original, self.voxelize(original, self.leafsize)


def device_voxelizer(device: int = 0) -> Voxelizer:
    """voxelize_preserving_labels on the GPU (erasor_updater_voxelize).  Needs a CUDA device: there is no CPU path."""
    from . import capi, params
    seed_map = np.zeros((1, 4), dtype=np.float32)          # the updater object only lends its stream and buffers here
    upd = capi.Updater(params.updater_preset("seq_05"), params.preset("seq_05"), seed_map, device=device)
    return lambda cloud, leaf: upd.voxelize(cloud, leaf)


def device_producer(device: int = 0):
    """(voxelize, node_producer) backed by one device updater object: the per-node step and the final voxelisation on the GPU."""
    from . import capi, params
    upd = capi.Updater(params.updater_preset("seq_05"), params.preset("seq_05"), np.zeros((1, 4), dtype=np.float32), device=device)
    return (lambda cloud, leaf: upd.voxelize(cloud, leaf)), (lambda odom7, lidar: upd.mapgen_node(odom7, lidar))


class DeviceMapGenerator:
    """NaiveMapGenerator's interface over the resident generator (capi.MapGen, DESIGN.md section 8.2): the map stays on the device,
    one launch per node, no per-node copy back.  cloud_map / cloud_curr are read back on access."""

    def __init__(self, leafsize: float = 0.05, is_large_scale: bool = False, device: int = 0):
        from . import capi
        self.leafsize, self.is_large_scale = float(leafsize), bool(is_large_scale)
        self.gen = capi.MapGen(leafsize, is_large_scale, device=device)

    def accum_point_cloud(self, odom7, lidar: np.ndarray) -> None:
        self.gen.accum(odom7, lidar)

    @property
    def cloud_map(self) -> np.ndarray:
        return self.gen.cloud(self.gen.CLOUD_MAP)

    @property
    def cloud_curr(self) -> np.ndarray:
        return self.gen.cloud(self.gen.CLOUD_CURR)

    def save_naive_map(self):
        return self.gen.save_naive_map()

    def close(self):
        self.gen.close()


def device_generator(leafsize: float = 0.05, is_large_scale: bool = False, device: int = 0) -> DeviceMapGenerator:
    """The whole of mapgen on the device (needs a CUDA device: there is no CPU path)."""
    return DeviceMapGenerator(leafsize, is_large_scale, device)


def build_map(nodes, leafsize: float = 0.05, is_large_scale: bool = False, voxelize: Optional[Voxelizer] = None, node_producer=None):
    """nodes: iterable of (seq, odom7, cloud) (e.g. erasor_b200.kitti.iter_nodes) -> (original, voxelized) map clouds.
    Without an injected voxeliser everything runs on the device, map included (device_generator; needs a CUDA device)."""
    if voxelize is None:
        gen = device_generator(leafsize, is_large_scale)
        try:
            for _, odom, cloud in nodes:
                gen.accum_point_cloud(odom, cloud)
            return gen.save_naive_map()
        finally:
            gen.close()
    gen = NaiveMapGenerator(voxelize, leafsize, is_large_scale, node_producer)
    for _, odom, cloud in nodes:
        gen.accum_point_cloud(odom, cloud)
    return gen.save_naive_map()
