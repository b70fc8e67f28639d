"""erasor_voxelize_batch (voxelize_batch.cu) restated in numpy: per-cloud bounds, grid set-up and overflow decision, voxel keys, the
two-stage stable sort (voxel key, then cloud index), run heads of (cloud, key), per-cloud output offsets and the output order; then
centroids summed in cloud order and the exact 1-NN label restore among each cloud's selected points (brute force).  Held cloud by
cloud to the oracle's voxelize_preserving_labels on batches that mix empty and 1-point clouds, an overflowing cloud, duplicates with
different labels and clouds of different key widths.  Also checks the C ABI symbol and its ctypes signature.  No GPU needed."""
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

F32 = np.float32
NO_KEY = 0xFFFFFFFF


def segment_model(xyzi, offsets, leaf, keep=None):
    """The device's segmentation of a batch: dict of per-cloud grids, keys, sorted order, voxel starts / clouds and output offsets."""
    x = np.ascontiguousarray(xyzi, dtype=F32).reshape(-1, 4)
    off = np.asarray(offsets, dtype=np.int64)
    F, n = len(off) - 1, int(off[-1])
    sel = np.ones(n, dtype=bool) if keep is None else (np.asarray(keep) != 0)
    cloud = np.repeat(np.arange(F), np.diff(off))
    inv = F32(1.0) / F32(leaf)
    key = np.full(n, NO_KEY, dtype=np.uint32)
    grids = []
    for c in range(F):                                     # k_vb_bounds + k_vb_setup + k_vb_keys, one cloud at a time
        idx = np.nonzero(sel[off[c]:off[c + 1]])[0] + off[c]
        if not len(idx):
            grids.append(None)
            continue
        p = x[idx, :3]
        mn, mx = p.min(axis=0), p.max(axis=0)
        d = ((mx - mn) * inv).astype(np.int64) + 1
        ovf = int(d[0]) * int(d[1]) * int(d[2]) > 2147483647
        min_b = np.floor(mn * inv).astype(np.int64)
        div = np.floor(mx * inv).astype(np.int64) - min_b + 1
        grids.append(dict(overflow=ovf, min_b=min_b, div=div, cells=int(div[0] * div[1] * div[2])))
        if ovf:
            key[idx] = (idx - off[c]).astype(np.uint32)     # one voxel per point, in cloud order
        else:
            ijk = (np.floor(p * inv) - min_b.astype(F32)).astype(np.int32).astype(np.int64)
            k = ijk[:, 0] + ijk[:, 1] * int(div[0]) + ijk[:, 2] * ((int(div[0]) * int(div[1])) & 0xFFFFFFFF)
            key[idx] = (k & 0xFFFFFFFF).astype(np.uint32)  # PCL's int32 arithmetic, unsigned order
    o1 = np.argsort(key, kind="stable")                    # 4 passes over the voxel key
    ck = np.where(sel, cloud, F)[o1]                       # deselected points: cloud F, behind every cloud
    order = o1[np.argsort(ck, kind="stable")]              # then the passes over the cloud index
    ns = int(sel.sum())
    order = order[:ns]
    scl, skey = cloud[order], key[order]
    head = np.ones(ns, dtype=bool)
    head[1:] = (skey[1:] != skey[:-1]) | (scl[1:] != scl[:-1])
    vstart = np.nonzero(head)[0]
    vcloud = scl[vstart]
    out_off = np.concatenate([[0], np.cumsum(np.bincount(vcloud, minlength=F))]).astype(np.uint64)
    return dict(grids=grids, key=key, order=order, vstart=vstart, vcloud=vcloud, out_off=out_off, n_sel=ns)


def voxelize_model(xyzi, offsets, leaf, keep=None):
    """-> (voxels float32 [m, 4], output offsets [F + 1]) as erasor_voxelize_batch returns them (no pose)."""
    x = np.ascontiguousarray(xyzi, dtype=F32).reshape(-1, 4)
    s = segment_model(x, offsets, leaf, keep)
    order, vstart, ns = s["order"], s["vstart"], s["n_sel"]
    nv = len(vstart)
    cnt = np.diff(np.append(vstart, ns))
    sums = np.zeros((nv, 4), dtype=F32)
    for r in range(int(cnt.max()) if nv else 0):           # members in cloud order: sequential float32 sums
        m = cnt > r
        sums[m] += x[order[vstart[m] + r]]
    cen = sums / cnt.astype(F32)[:, None]
    off = np.asarray(offsets, dtype=np.int64)
    sel = np.ones(len(x), dtype=bool) if keep is None else (np.asarray(keep) != 0)
    for c in range(len(off) - 1):                          # exact 1-NN among the cloud's selected points, ties to the lowest index
        idx = np.nonzero(sel[off[c]:off[c + 1]])[0] + off[c]
        a, b = int(s["out_off"][c]), int(s["out_off"][c + 1])
        for v0 in range(a, b, 256):
            v1 = min(b, v0 + 256)
            q = cen[v0:v1, None, :3]
            dxyz = q - x[None, idx, :3]
            d2 = (dxyz[..., 0] * dxyz[..., 0] + dxyz[..., 1] * dxyz[..., 1]) + dxyz[..., 2] * dxyz[..., 2]
            cen[v0:v1, 3] = x[idx[np.argmin(d2, axis=1)], 3]
    return cen, s["out_off"]


def batch_of(clouds):
    off = np.cumsum([0] + [len(c) for c in clouds]).astype(np.uint64)
    xyzi = np.concatenate([np.asarray(c, dtype=F32).reshape(-1, 4) for c in clouds]) if int(off[-1]) else np.zeros((0, 4), F32)
    return xyzi, off


def mixed_clouds(seed=3):
    """Empty and 1-point clouds, an overflowing cloud (10 km wide), a small scan, a cloud held in one voxel,
    duplicates with different labels, coordinates on voxel faces and 1 ulp either side, and a 1 m cloud (narrow keys)."""
    from erasor_b200 import synth
    rng = np.random.default_rng(seed)
    sc = synth.Scene(seed=seed, n_nodes=11)
    scan = sc.scan(3, n_beams=8, n_az=120, seed_offset=1)
    one_voxel = np.column_stack([rng.uniform(0.21, 0.39, (40, 3)), rng.integers(0, 260, 40)]).astype(F32)
    dup = np.repeat(rng.uniform(-5, 5, (30, 3)), 3, axis=0)
    dup = np.column_stack([dup, np.tile([40.0, 252.0, 9.0], 30)]).astype(F32)
    faces = np.arange(-6, 7, dtype=F32) * F32(0.2)
    face_pts = []
    for f in faces:
        for u in (-1, 0, 1):
            v = f
            for _ in range(abs(u)):
                v = np.nextafter(v, F32(np.inf) if u > 0 else F32(-np.inf), dtype=F32)
            face_pts.append([v, -v, v * F32(0.5), float(len(face_pts) % 7)])
    far = np.column_stack([rng.uniform(-5000, 5000, (150, 3)), rng.integers(0, 260, 150)]).astype(F32)
    far[10] = far[3]
    far[10, 3] = 77.0                                      # a duplicate inside the overflowing cloud, other label
    tiny = np.column_stack([rng.uniform(0, 1, (60, 3)), rng.integers(0, 260, 60)]).astype(F32)
    return [np.zeros((0, 4), F32), scan, np.array([[1.0, 2.0, 3.0, 5.0]], F32), one_voxel, far, dup, np.zeros((0, 4), F32),
            np.array(face_pts, F32), tiny]


def test_segmentation_grids_and_order():
    clouds = mixed_clouds()
    xyzi, off = batch_of(clouds)
    s = segment_model(xyzi, off, 0.2)
    g = s["grids"]
    assert g[0] is None and g[6] is None and not g[2]["overflow"] and g[2]["cells"] == 1
    assert g[4]["overflow"] and not g[1]["overflow"]
    assert g[8]["cells"] < g[1]["cells"] < 2 ** 31                    # key widths differ between clouds
    # output order: clouds in order, ascending key within a cloud, members in cloud order within a voxel
    order, vstart, vcloud = s["order"], s["vstart"], s["vcloud"]
    cl = np.repeat(np.arange(len(off) - 1), np.diff(off.astype(np.int64)))
    assert np.all(np.diff(cl[order]) >= 0)
    for c in range(len(off) - 1):
        seg = order[cl[order] == c]
        k = s["key"][seg]
        assert np.all(np.diff(k.astype(np.int64)) >= 0)
        same = np.diff(k.astype(np.int64)) == 0
        assert np.all(np.diff(seg)[same] > 0)
    assert np.all(np.diff(s["out_off"].astype(np.int64)) >= 0) and int(s["out_off"][-1]) == len(vstart)
    assert np.array_equal(np.bincount(vcloud, minlength=len(off) - 1), np.diff(s["out_off"].astype(np.int64)))
    assert int(np.diff(s["out_off"].astype(np.int64))[4]) == len(clouds[4])          # overflow: one voxel per point


@pytest.mark.parametrize("leaf", [0.01, 0.2, 1.0])
def test_model_equals_oracle_cloud_by_cloud(oracle_mod, leaf):
    clouds = mixed_clouds()
    xyzi, off = batch_of(clouds)
    vox, oo = voxelize_model(xyzi, off, leaf)
    for c, cloud in enumerate(clouds):
        want = oracle_mod.voxelize(cloud, leaf)
        got = vox[int(oo[c]):int(oo[c + 1])]
        assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"cloud {c} at leaf {leaf}"


def test_model_keep_mask_equals_oracle_on_selection(oracle_mod):
    clouds = mixed_clouds(seed=8)
    xyzi, off = batch_of(clouds)
    rng = np.random.default_rng(1)
    keep = (rng.random(len(xyzi)) < 0.6).astype(np.uint8)
    vox, oo = voxelize_model(xyzi, off, 0.2, keep)
    o = off.astype(np.int64)
    for c in range(len(clouds)):
        want = oracle_mod.voxelize(xyzi[o[c]:o[c + 1]][keep[o[c]:o[c + 1]] != 0], 0.2)
        got = vox[int(oo[c]):int(oo[c + 1])]
        assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"cloud {c}"


def test_capi_declares_voxelize_batch():
    from erasor_b200 import capi
    assert "erasor_voxelize_batch" in capi.EXPORTS
    hdr = open(os.path.join(ROOT, "include", "erasor_b200.h")).read()
    assert "int erasor_voxelize_batch(erasor_handle_t h, const float* xyzi, const uint64_t* offsets, int n_clouds, const uint8_t* keep, float leaf," in hdr
    L = capi.lib()
    f = L.erasor_voxelize_batch
    assert [t for t in f.argtypes] == [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64), ctypes.c_int, ctypes.c_void_p,
                                       ctypes.c_float, ctypes.POINTER(ctypes.c_double), ctypes.c_int, ctypes.POINTER(ctypes.c_void_p),
                                       ctypes.POINTER(ctypes.c_uint64)]
