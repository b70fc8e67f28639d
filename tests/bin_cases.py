"""Test-side generators of crafted flagged bins (numpy only), for the size switches of R-GPF, the in-bin voxeliser and the
mask-mode scatter.

- ``flagged_bins(p, specs, seed)``: one frame (map, query) in the body frame holding the bins of ``specs``.  Every bin is "tall
  object over ground, low query" -- or, for ``ramp``, a plane tilted enough to span more than 0.5 m, every point of which R-GPF
  keeps as ground -- so that the Scan Ratio Test flags it (MAP_IS_HIGHER) in both versions.  Points sit strictly inside their
  bin: 10 % of the ring and sector widths clear of the thresholds, and well inside the z window.
- ``K4_C_CAP`` / ``K4B_CAP`` / ``k2_window``: the size switches of the device path, restated from the launch code.
- ``fill_flagged(p, n_flagged, seed)``: one frame that flags exactly ``n_flagged`` bins, a few points each.
- ``voxel_cells`` / ``voxel_ids``: pcl::VoxelGrid's cell count and per-point cells for one bin's input (device_common.cuh).
"""
from collections import namedtuple

import numpy as np

F32 = np.float32

# kernels.cu launch_k4 / launch_k4_class: class C runs in a 180 KB slice of 21 bytes per point (+ 32); beyond it, global scratch
K4_C_CAP = (180 * 1024 - 32) // 21                 # 8775
# kernels.cu launch_k4b: 160 KB of shared memory at 36 bytes per point (+ 64); beyond it, global scratch
K4B_CAP = (160 * 1024 - 64) // 36                  # 4549
# kernels.cu k4_rgpf / k4_process_bin: the sort paths of R-GPF (class A networks, class B networks then radix, class C)
RGPF_SWITCHES = (128, 256, 512, 1024, 2048, 2560)


def k2_window(B: int, with_complement: bool = False, node: bool = False) -> int:
    """kernels.cu k2_smem_plan: slots per window of the SRT + scatter kernel (W = 8 warps, two CTAs per SM in 111 KB; node mode
    also stages kK2Stage = 512 VoI entries of 2 bytes per warp)."""
    W = 8
    fixed = ((2 * (B + 2) + 15) & ~15) + (2 * W * 512 if node else 0)
    n_slots_max = B + 1 if with_complement else B
    full = 4 * (W + 1) * n_slots_max + fixed
    budget = min(full, 111 * 1024)
    return min(max(n_slots_max, 1), max(1, (budget - fixed) // (4 * (W + 1))))


# ring, sector: the bin; n: map points; z: rough | dup | equal | ulp | ramp; nq: query points;
# extent: None (the bin's inner 80 %) or the side in metres of a square cluster at the bin's centre; span: ramp height (m);
# distinct_leaf: if set, no two points of the bin (map and query) share a voxel of this leaf
Bin = namedtuple("Bin", "ring sector n z nq extent span distinct_leaf", defaults=("rough", 40, None, 1.2, None))


def geometry(p):
    ring_size = p.max_range / p.num_rings
    sector_size = 2.0 * np.pi / p.num_sectors
    zg = p.min_h + 0.4                              # ground height: 0.4 m above the z window's floor
    top = min(zg + 2.9, p.max_h - 0.1)              # object top
    return ring_size, sector_size, zg, top


def bin_id(p, ring: int, sector: int) -> int:
    return sector * p.num_rings + ring


def _xy(p, s: Bin, rng, n):
    """n (x, y) strictly inside bin s (or its central cluster), plus the bin's radial axis angle and radial range."""
    rs, ss, _, _ = geometry(p)
    r0, r1 = (s.ring + 0.1) * rs, (s.ring + 0.9) * rs
    t0, t1 = (s.sector + 0.1) * ss, (s.sector + 0.9) * ss
    thc = (s.sector + 0.5) * ss
    if s.extent is None:
        r = rng.uniform(r0, r1, n)
        th = rng.uniform(t0, t1, n)
        u0, u1 = r0 * np.cos(max(abs(t0 - thc), abs(t1 - thc))), r1
    else:
        rc = (s.ring + 0.5) * rs
        h = s.extent / 2
        u0, u1 = rc - h, rc + h
        u = rng.uniform(u0, u1, n)
        t = rng.uniform(-h, h, n)
        r = np.hypot(u, t)
        th = thc + np.arctan2(t, u)
        assert r0 < r.min() and r.max() < r1 and t0 < th.min() and th.max() < t1, "cluster does not fit in the bin"
    return r * np.cos(th), r * np.sin(th), thc, u0, u1


def _bin_points(p, s: Bin, rng):
    rs, ss, zg, top = geometry(p)
    n, nq = s.n, s.nq
    if s.z == "ramp":
        x, y, thc, u0, u1 = _xy(p, s, rng, n)
        u = x * np.cos(thc) + y * np.sin(thc)
        z = zg + s.span * (u - u0) / (u1 - u0)
        m = np.stack([x, y, z, np.full(n, 40.0)], 1)
    else:
        n_obj = min(60, max(2, n // 8))
        ng = n - n_obj
        x, y, *_ = _xy(p, s, rng, ng)
        if s.z == "dup":            # a handful of distinct heights, many exact duplicates (and both zeros)
            z = rng.choice(np.array([zg - 0.1, zg - 0.05, zg, np.nextafter(F32(zg), F32(-1)), -0.0, 0.0], dtype=F32), ng)
        elif s.z == "equal":        # every ground point at the same height
            z = np.full(ng, zg, dtype=F32)
        elif s.z == "ulp":          # clusters a few ulps wide
            z = F32(zg) + rng.integers(0, 7, ng).astype(F32) * F32(6e-8)
        elif s.z == "rough":
            z = rng.normal(zg, 0.04, ng)
        else:
            raise ValueError(s.z)
        g = np.stack([x, y, z, np.full(ng, 40.0)], 1)
        ox, oy, *_ = _xy(p, s, rng, n_obj)
        oz = rng.uniform(zg + 0.3, top, n_obj)
        oz[0] = top
        m = np.concatenate([g, np.stack([ox, oy, oz, np.full(n_obj, 252.0)], 1)])
    qx, qy, *_ = _xy(p, s, rng, nq)
    q = np.stack([qx, qy, rng.uniform(zg - 0.02, zg + 0.02, nq), np.full(nq, 40.0)], 1)
    m, q = m.astype(F32), q.astype(F32)
    if s.distinct_leaf is not None:
        m, q = _distinct(p, s, rng, m, q)
    return m, q


def _distinct(p, s: Bin, rng, m, q):
    """Redraw map and query points of the bin until no two share a voxel (ramp bins only: their z follows from x, y)."""
    assert s.z == "ramp"
    for _ in range(50):
        pts = np.concatenate([q, m])
        ids = voxel_ids(pts, s.distinct_leaf)
        _, first = np.unique(ids, axis=0, return_index=True)
        dup = np.ones(len(pts), dtype=bool)
        dup[first] = False
        if not dup.any():
            return m, q
        fresh_m, fresh_q = _bin_points(p, s._replace(distinct_leaf=None, n=len(m), nq=len(q)), rng)
        pts = np.where(dup[:, None], np.concatenate([fresh_q, fresh_m]), pts)
        q, m = pts[:len(q)], pts[len(q):]
    raise RuntimeError("could not place the points in distinct voxels")


def flagged_bins(p, specs, seed: int = 0):
    """(map, query) float32 [n, 4] of one frame holding the bins of specs (each map and each query cloud shuffled as a whole)."""
    rng = np.random.default_rng(seed)
    keys = [(s.ring, s.sector) for s in specs]
    assert len(set(keys)) == len(keys), "one spec per bin"
    ms, qs = zip(*[_bin_points(p, s, rng) for s in specs]) if specs else ([], [])
    m = np.concatenate(ms) if ms else np.zeros((0, 4), F32)
    q = np.concatenate(qs) if qs else np.zeros((0, 4), F32)
    return rng.permutation(m), rng.permutation(q)


def fill_flagged(p, n_flagged: int, seed: int = 0):
    """One frame that flags exactly n_flagged bins of p's grid (8 map points and max(8, minimum_num_pts) query points each);
    returns (map, query, bin ids)."""
    rng = np.random.default_rng(seed)
    B = p.num_bins
    pick = np.sort(rng.choice(B, n_flagged, replace=False))
    specs = [Bin(int(b % p.num_rings), int(b // p.num_rings), 8, "rough", max(8, p.minimum_num_pts)) for b in pick]
    m, q = flagged_bins(p, specs, seed=seed + 1)
    return m, q, pick


def voxel_ids(pts, leaf: float) -> np.ndarray:
    """Per point (floor(x / leaf), floor(y / leaf), floor(z / leaf)) as pcl::VoxelGrid computes it (float product with 1 / leaf)."""
    inv = F32(1.0) / F32(leaf)
    return np.floor(np.asarray(pts, dtype=F32)[:, :3] * inv).astype(np.int64)


def voxel_cells(pts, leaf: float):
    """(cells of the bin's voxel grid, PCL's overflow flag) for one bin's K4b input (device_common.cuh voxel_grid_setup)."""
    a = np.asarray(pts, dtype=F32)[:, :3]
    inv = F32(1.0) / F32(leaf)
    mn, mx = a.min(0), a.max(0)
    d = np.prod([int((mx[k] - mn[k]) * inv) + 1 for k in range(3)])
    div = np.floor(mx * inv).astype(np.int64) - np.floor(mn * inv).astype(np.int64) + 1
    return int(np.prod(div)), d > 2147483647


def radix_passes(cells: int) -> int:
    """kernels.cu k4b_voxelize: 8-bit passes of the voxel-key sort."""
    bits = 1
    while bits < 31 and (1 << bits) < cells:
        bits += 1
    return (bits + 7) // 8


# ---- the cases the capacity-edge tests run (seq_05 geometry: 15 rings x 60 sectors) ----------------------------------------------
# R-GPF: both sides of every sort switch and of class C's shared-memory cap, and two bins far beyond it
RGPF_SIZES = (128, 129, 256, 257, 512, 513, 1024, 1025, 2048, 2049, 2560, 2561, K4_C_CAP, K4_C_CAP + 1, K4_C_CAP + 2, 20000, 150000)
RGPF_Z_KINDS = ("rough", "dup", "equal", "ulp")     # equal / ulp only from class C's cap upwards
# Not every bin of these frames rejects points: in the equal and ulp frames the oracle keeps the whole 20 000-point bin as ground
# (its 60 object points included), so that bin checks the plane fields only; their other bins and every bin of the rough / dup frames do reject.


def rgpf_specs(z: str):
    sizes = [n for n in RGPF_SIZES if z in ("rough", "dup") or n >= K4_C_CAP]
    return [Bin(2 + i % 10, 3 * i + 1, n, z) for i, n in enumerate(sizes)]


# K4b (version 3, in-bin voxelisation): ramp bins, so that n = qc + n_ground_final = n_map + nq exactly.  Per leaf: bins on both
# sides of the shared-memory cap and far beyond it, whole bins and central clusters, so that the voxel-key sort takes each of its
# pass counts; at leaf 0.01 also two adjacent bins (consecutive bin ids) over the cap with one point per voxel -- the geometry
# in which each bin's scratch footprint reaches the next bin's region unless the regions are padded; at leaf 0.001 the grid
# overflows PCL's INT_MAX check and the bin passes through.
def _k4b(ring, sector, n_total, nq, **kw):
    return Bin(ring, sector, n_total - nq, "ramp", nq, **kw)


K4B_FRAMES = {
    0.2:   [_k4b(5, 0, K4B_CAP, 549, span=0.8), _k4b(5, 30, K4B_CAP + 1, 550, span=0.8),
            _k4b(5, 15, 12000, 2000, extent=0.8, span=0.8), _k4b(7, 45, 40000, 10000, extent=0.8, span=0.8)],
    0.05:  [_k4b(5, 0, K4B_CAP, 549, span=0.8), _k4b(5, 30, K4B_CAP + 1, 550, span=0.8),
            _k4b(8, 15, 12000, 2000, span=0.8), _k4b(9, 45, 40000, 10000, span=0.8)],
    0.01:  [_k4b(5, 0, K4B_CAP, 549, extent=1.0, span=0.8), _k4b(5, 30, K4B_CAP + 1, 550, extent=1.0, span=0.8),
            _k4b(13, 45, 12000, 1000, span=1.6), _k4b(12, 15, 40000, 10000, extent=1.0, span=0.8),
            _k4b(3, 20, 4600, 100, span=0.8, distinct_leaf=0.01), _k4b(4, 20, 4600, 100, span=0.8, distinct_leaf=0.01)],
    0.001: [_k4b(5, 0, 5000, 100, span=0.8)],
}
K4B_ADJACENT = ((3, 20), (4, 20))        # (ring, sector) of the adjacent pair at leaf 0.01

# K2 windows (synthetic_40x360): flagged bins per frame on both sides of one and two windows, and every bin
K2_PRESET = "synthetic_40x360"


def k2_flag_counts(B: int):
    W = k2_window(B)
    return (W - 1, W, W + 1, 2 * W + 1, B)
