"""The resident map generator's bookkeeping (erasor_b200/csrc/mapgen_capi.cu, DESIGN.md section 8.2) as a numpy model, held to
NaiveMapGenerator -- the reference's mapgen restated -- cloud for cloud, with the oracle's voxeliser injected into both.

The model keeps what the device keeps: one buffer [parked, voxelised submaps | current chunk, raw] with a tail and a chunk start;
each node's voxels written at the tail; parking voxelising [chunk start, tail) and moving the result to the chunk start; and the
host's upper bounds on the map and chunk sizes, which only a read-back tightens and which decide when a buffer has to grow.
Plus: the new C ABI symbols exist in the library and capi gives each of them a ctypes signature."""
import ctypes
import os
import re

import numpy as np
import pytest

from erasor_b200 import mapgen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class ResidentModel:
    def __init__(self, voxelize, leafsize, is_large_scale, min_cap=64, period=500):
        self.voxelize, self.leafsize, self.is_large_scale, self.period = voxelize, leafsize, is_large_scale, period
        self.buf = np.zeros((0, 4), dtype=np.float32)
        self.min_cap = min_cap
        self.tail = self.chunk = 0                  # device words
        self.ub_tail = self.ub_chunk = 0            # host bounds
        self.initial, self.cnt_voxel = True, 0
        self.curr = np.zeros((0, 4), dtype=np.float32)
        self.launches = self.syncs = self.regrowths = 0

    def _read_back(self):
        self.syncs += 1
        self.ub_tail, self.ub_chunk = self.tail, self.tail - self.chunk

    def _node_voxels(self, odom, lidar):
        c = lidar
        d2 = c[:, 0].astype(np.float64) ** 2 + c[:, 1].astype(np.float64) ** 2
        c = c[~(d2 < np.float64(np.float32(2.7 ** 2)))]
        lift = np.eye(4, dtype=np.float32)
        lift[2, 3] = np.float32(1.73)
        world = mapgen.transform_point_cloud(mapgen.transform_point_cloud(c, lift), mapgen.pose_to_matrix(odom))
        return self.voxelize(world, 0.2)

    def accum(self, odom, lidar):
        n = len(lidar)
        if self.ub_tail + n > len(self.buf):
            self._read_back()
            new = np.zeros((max(self.tail + n, 2 * len(self.buf), self.min_cap), 4), dtype=np.float32)
            new[:self.tail] = self.buf[:self.tail]
            self.buf = new
            self.regrowths += 1
        v = self._node_voxels(odom, lidar)
        assert len(v) <= n
        self.buf[self.tail:self.tail + len(v)] = v
        self.tail += len(v)
        self.curr = v
        self.launches += 1
        self.ub_tail += n
        self.ub_chunk += n
        assert self.tail <= self.ub_tail and self.tail - self.chunk <= self.ub_chunk
        if self.initial:
            self.initial = False
            return False
        if self.is_large_scale:
            fire = self.cnt_voxel % self.period == 0
            self.cnt_voxel += 1
            if fire:
                src = self.buf[self.chunk:self.tail].copy()        # the 1-NN reads the chunk to the end: the move comes after
                vox = self.voxelize(src, self.leafsize)
                assert len(vox) <= len(src) <= self.ub_chunk
                self.buf[self.chunk:self.chunk + len(vox)] = vox
                self.tail = self.chunk = self.chunk + len(vox)
                self.ub_chunk = 0
                self.launches += 1
                return True
        return False

    @property
    def cloud_map(self):
        return self.buf[self.chunk:self.tail]

    def save_naive_map(self):
        original = self.buf[:self.tail].copy()
        return original, self.voxelize(original, self.leafsize)


def _small_nodes(n_nodes, seed=5):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_nodes):
        if k % 97 == 3:
            scan = np.zeros((0, 4), dtype=np.float32)                                  # empty scan
        else:
            m = int(rng.integers(10, 60))
            r = rng.uniform(0.5, 2.6, m) if k % 89 == 5 else rng.uniform(0.5, 30.0, m)  # k % 89 == 5: all inside the 2.7 m cut
            th = rng.uniform(-np.pi, np.pi, m)
            scan = np.stack([r * np.cos(th), r * np.sin(th), rng.normal(-1.7, 0.3, m), rng.choice([40.0, 48.0, 252.0], m)], axis=1)
        yaw = 0.01 * k
        odom = np.array([0.5 * k, 0.05 * k, 0.0, 0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2)])
        out.append((k, odom, np.ascontiguousarray(scan, dtype=np.float32)))
    return out


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("large_scale", [True, False])
def test_resident_bookkeeping_equals_naive_map_generator(oracle_mod, large_scale):
    vox = lambda c, leaf: oracle_mod.voxelize(c, leaf)
    nodes = _small_nodes(1100)
    ref = mapgen.NaiveMapGenerator(vox, leafsize=0.2, is_large_scale=large_scale)
    model = ResidentModel(vox, 0.2, large_scale)
    parked_at = []
    for k, odom, scan in nodes:
        ref.accum_point_cloud(odom, scan)
        if model.accum(odom, scan):
            parked_at.append(k)
        assert _same(model.curr, ref.cloud_curr), f"node {k}: cloud_curr"
        assert _same(model.cloud_map, ref.cloud_map), f"node {k}: cloud_map"
    o_ref, v_ref = ref.save_naive_map()
    o_mod, v_mod = model.save_naive_map()
    assert _same(o_mod, o_ref) and _same(v_mod, v_ref)
    if large_scale:
        assert parked_at == [1, 501, 1001]                       # the 2nd, 502nd and 1002nd node
        assert model.launches == len(nodes) + 3
        assert len(ref.cloud_maps) == 3
    else:
        assert parked_at == [] and model.launches == len(nodes)
    # geometric growth: a handful of read-backs for 1100 nodes, each one a regrowth
    assert 3 <= model.regrowths == model.syncs <= 20


def test_new_abi_symbols_and_signatures():
    from erasor_b200 import capi
    hdr = open(os.path.join(ROOT, "include", "erasor_b200.h")).read()
    names = set(re.findall(r"\b(erasor_mapgen_[a-z_]+)\s*\(", hdr))
    assert names == {"erasor_mapgen_create", "erasor_mapgen_destroy", "erasor_mapgen_last_error", "erasor_mapgen_accum",
                     "erasor_mapgen_get_cloud", "erasor_mapgen_device_cloud", "erasor_mapgen_synchronize", "erasor_mapgen_get_counters"}
    assert names <= set(capi.EXPORTS)
    raw = ctypes.CDLL(capi.LIB_PATH)                # loads without a GPU
    L = capi.lib()
    for s in sorted(names):
        assert hasattr(raw, s), s
        f = getattr(L, s)
        assert f.argtypes is not None, s
    assert len(L.erasor_mapgen_accum.argtypes) == 5 and len(L.erasor_mapgen_get_cloud.argtypes) == 6
    assert [n for n, _ in capi.MapGenParamsC._fields_] == ["leafsize", "is_large_scale"]
    assert ctypes.sizeof(capi.MapGenParamsC) == 8
    assert (capi.MapGen.CLOUD_MAP, capi.MapGen.CLOUD_CURR, capi.MapGen.SAVED_ORIGINAL, capi.MapGen.SAVED_VOXELIZED) == (0, 1, 2, 3)
