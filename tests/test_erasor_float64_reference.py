"""R-POD binning, the Scan Ratio Test and R-GPF against an independent float64 reference, at the inputs where a float32 port
can be wrong without the oracle noticing: points on ring radii, sector angles, azimuth +-pi, the range and height gates; bins of
0 to 3 points, collinear points, equal heights and a wall without ground; SRT quantities exactly on their thresholds; the same
scene at +-1000 m and +-10 000 m; sizes around the shared-memory and launch limits; empty and one-point inputs.

The reference below is written from the algorithm (DESIGN.md, include/erasor_b200.h, params.py), in NumPy float64:

- binning: r = sqrt(x^2 + y^2), azimuth in [0, 2*PI) with PI = 3.1415926535 (the constant the sector size is defined with,
  binning.h), ring = min(floor(r / ring_size), R - 1), sector = min(floor(theta / sector_size), S - 1); binned iff
  min_h < z < max_h and r <= max_range.  The sign of a zero y is ignored (-0.0 is +0.0), so azimuth is 0 or pi there, never -pi.
- bin statistics: count, min z, max z per bin.
- SRT (version 3): LITTLE if the map bin is empty, the query bin has fewer than minimum_num_pts points (the reference compares
  a size_t with the int, so a negative minimum_num_pts is a huge bound: every bin is LITTLE) or the query bin is empty; else
  ratio = min(dh_map / dh_query, dh_query / dh_map) (C++ std::min: a NaN first argument wins); ratio < threshold gives MAP_HIGH
  (dh_map >= dh_query) or CURR_HIGH, otherwise MERGE.  Second pass: MAP_HIGH with dh_map > 0.5 is handed to R-GPF, else the bin
  is left alone (status 0); MERGE next to a CURR_HIGH bin (ring +-1, sector +-1; a sector index below 0 or past S - 1 is wrapped by
  num_rings, as the reference does) is BLOCKED.  Version 2: the same first pass on the bins occupied in both clouds, no second
  pass, and MAP_HIGH is handed to R-GPF when the map bin's top is above th_bin_max_h (in double).
- R-GPF on a handed-over bin: z sorted stably; lpr = mean of sorted z[num_lowest_pts : num_lowest_pts + gf_num_lpr] (0 if
  empty); seeds = points with z < lpr + gf_th_seeds_height; gf_iter times: plane through the current ground set (mean, two-pass
  mean-centred covariance, np.linalg.eigh, normal = eigenvector of the smallest eigenvalue; an empty set gives normal (0, 0, 1) and
  d = 0, the fallback the device documents), ground = points with normal . (p - mean) < gf_dist_thr.  The test is one-sided, so
  the sign of the normal decides which side is ground: the reference takes the device's sign (every other property is compared
  up to sign).  Map points of a handed-over bin that end up non-ground are removed (with gf_iter 0: every point that is not a
  seed, since only the seeds return to the map); every other map point is kept.

Tolerances (every one of them is stated next to its use):
- EPS32 = 2^-23 (float32 machine epsilon).
- Bins: exact, except within EPS_R = 1e-12 * max_range of a ring radius or the range gate and within EPS_THETA = 1e-9 rad of a
  sector angle; there either neighbour is accepted (the device decides such points exactly on the double expression; the band
  only absorbs libm differences, which are below 1e-15).  Points on an axis (x or y zero) have an exactly known r and azimuth
  and get no band.  Poses add EPS_POS = 16 * EPS32 * (|t| + max_range) metres: the transform to the body frame runs in float32.
- SRT: exact.  Both sides take the same double operations on the same float32 extrema, so a tie is decided identically.
- Plane normals (up to sign): the first-order eigenvector perturbation of a float32 covariance,
      tol_k = (16 * EPS32 * sqrt(m) * a_0 * a_k + 8 * sqrt(EPS32) * lambda_max) / (lambda_k - lambda_0),   tol = max(tol_1, tol_2),
  with lambda_0 <= lambda_1 <= lambda_2 the float64 eigenvalues, v_k their eigenvectors and a_k = sum_i |v_k,i| * max |p_i - c_i|
  the largest product size along v_k that the accumulation adds up.  sqrt(m) is the random-walk size of m float32 roundings and
  16 the margin.  The second term is the float32 Jacobi SVD's (Eigen 3.3's, which the device reproduces bit for bit): on these
  inputs its normal is off by up to 1.3 * sqrt(EPS32) * lambda_max / gap, measured with the oracle (bit-identical to the device)
  on the frames below, so 8 * sqrt(EPS32) leaves a margin of 6.  c is the point the device's accumulation is centred on: the first
  point of the ground list for cov_mode 1 (PCL >= 1.11's shifted formula), the body-frame origin for the default cov_mode 0
  (PCL <= 1.10's one-pass formula, which the oracle shares).  So cov_mode 1 is held to the centred spread of the bin, and cov_mode
  0 only as tightly as its coordinates, at most max_range, allow: R-GPF always fits in the body frame, so a world offset never
  enters it.  A fit with tol >= 0.05 rad is degenerate (fewer than three points, collinear points): the device's normal must be
  finite, of unit length, and orthogonal to every eigenvector k whose own tol_k is below 0.05 rad.
- Ground labels: the reference classifies with its own normal where tol < 0.05 rad, else with the device's.  Exact for points
  further than tol * |p - mean| + 8 * EPS32 * (sqrt(m) * max |g| + |p| + |mean|) from the threshold (the float32 dot products and
  mean of the device); a bin with a point inside that band is reported, and its later iterations and labels are not compared.
"""
import math

import numpy as np
import pytest

import bin_cases as BC
from erasor_b200 import params as P

F32 = np.float32
EPS32 = float(np.finfo(np.float32).eps)
PI_CFG = 3.1415926535
EPS_THETA = 1e-9
LITTLE, MERGE, MAP_HIGH, BLOCKED, CURR_HIGH = 0.0, 0.25, 0.5, 0.8, 1.0


def _has_cuda() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


needs_gpu = pytest.mark.skipif(not _has_cuda(), reason="needs a CUDA device")


# ================================================================================================================================
# float64 reference
# ================================================================================================================================
def polar(p, xyz, eps_pos: float = 0.0, eps_z: float = 0.0):
    """(bin or -1, candidate bins [n, k]) of every point.  The candidates are the bins of the point moved by the band widths
    (EPS_R / EPS_THETA, plus eps_pos metres and eps_z in z); a point whose candidates differ lies on a boundary."""
    x, y, z = (np.asarray(xyz[:, k], dtype=np.float64) for k in range(3))
    R, S = p.num_rings, p.num_sectors
    rs, ss = p.max_range / R, 2.0 * PI_CFG / S
    y0 = np.where(y == 0.0, 0.0, y)
    r = np.sqrt(x * x + y0 * y0)
    th = np.arctan2(y0, x)
    th = np.where(th < 0.0, th + 2.0 * PI_CFG, th)
    axis = (x == 0.0) | (y == 0.0)
    er = np.where(axis, 0.0, 1e-12 * p.max_range) + eps_pos
    et = np.where(axis, 0.0, EPS_THETA) + np.where(r > 0.0, eps_pos / np.maximum(r, 1e-300), np.where(eps_pos > 0, np.pi, 0.0))
    et = np.minimum(et, np.pi)

    def one(rr, tt, zz):
        tt = np.where(tt < 0.0, tt + 2.0 * PI_CFG, tt)          # a band across azimuth 0 reaches the last sector
        ring = np.minimum(np.floor(rr / rs), R - 1).astype(np.int64)
        sec = np.minimum(np.floor(tt / ss), S - 1).astype(np.int64)
        ok = (zz > p.min_h) & (zz < p.max_h) & (rr <= p.max_range)
        return np.where(ok, sec * R + np.maximum(ring, 0), -1)

    exact = one(r, th, z)
    cand = [one(np.maximum(r + dr * er, 0.0), th + dt * et, z + dz * eps_z)
            for dr in (-1, 0, 1) for dt in (-1, 0, 1) for dz in (-1, 0, 1)]
    return exact, np.stack(cand, 1)


def bin_stats(p, bins, z):
    B = p.num_bins
    sel = bins >= 0
    cnt = np.bincount(bins[sel], minlength=B)
    mn, mx = np.full(B, np.inf), np.full(B, -np.inf)
    np.minimum.at(mn, bins[sel], np.asarray(z, np.float64)[sel])
    np.maximum.at(mx, bins[sel], np.asarray(z, np.float64)[sel])
    return cnt, mn, mx


def _cpp_min(a, b):
    return b if b < a else a


def srt_status(p, mstat, qstat, eps_dh: float = 0.0):
    """Status per bin (version 3, or version 2 when p.version == 2), which bins are handed to R-GPF, and the bins whose decisive
    quantity lies within the band of its threshold (node mode moves every z by up to eps_dh; in cloud mode eps_dh = 0 and nothing
    is ambiguous).  The query count is compared as the reference's size_t against the int minimum_num_pts, which the int is
    converted to: a negative minimum_num_pts is a huge bound and sends every bin to LITTLE.  Only a bin occupied in both clouds
    takes the ratio test (an empty query bin has no heights); version 3 gives the others LITTLE, version 2 leaves them unassigned
    (0, the value of LITTLE)."""
    R, S = p.num_rings, p.num_sectors
    (mc, mmn, mmx), (qc, qmn, qmx) = mstat, qstat
    enough = (qc >= p.minimum_num_pts) if p.minimum_num_pts >= 0 else np.zeros(R * S, dtype=bool)
    if p.version == 2:
        return _srt_status_v2(p, mstat, qstat, enough, eps_dh)
    pass1 = np.zeros(R * S)
    near = np.zeros(R * S, dtype=bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        for b in np.nonzero((mc > 0) & (qc > 0) & enough)[0]:
            mdh, cdh = mmx[b] - mmn[b], qmx[b] - qmn[b]
            ratio = _cpp_min(np.float64(mdh) / np.float64(cdh), np.float64(cdh) / np.float64(mdh))
            if ratio < p.scan_ratio_threshold:
                pass1[b] = MAP_HIGH if mdh >= cdh else CURR_HIGH
            else:
                pass1[b] = MERGE
            if eps_dh > 0.0:
                if mdh > 0 and cdh > 0:
                    near[b] |= abs(ratio - p.scan_ratio_threshold) <= ratio * 2 * eps_dh * (1 / mdh + 1 / cdh)
                near[b] |= abs(mdh - cdh) <= 4 * eps_dh or min(mdh, cdh) <= 2 * eps_dh
    st = pass1.copy()
    flagged = np.zeros(R * S, dtype=bool)
    for b in np.nonzero(pass1 == MAP_HIGH)[0]:
        mdh = mmx[b] - mmn[b]
        near[b] |= eps_dh > 0.0 and abs(mdh - 0.5) <= 2 * eps_dh
        if mdh > 0.5:
            flagged[b] = True
        else:
            st[b] = 0.0
    for b in np.nonzero(pass1 == MERGE)[0]:
        theta, r = divmod(int(b), R)
        close = False
        for j in (theta - 1, theta, theta + 1):
            tj = j + R if j < 0 else (j - R if j >= S else j)
            if not 0 <= tj < S:
                continue
            for rr in range(max(0, r - 1), min(r + 1, R - 1) + 1):
                if (rr, tj) != (r, theta) and pass1[tj * R + rr] == CURR_HIGH:
                    close = True
        st[b] = BLOCKED if close else MERGE
    return st, flagged, near


def _srt_status_v2(p, mstat, qstat, enough, eps_dh):
    """Version 2: one pass, no neighbour test; MAP_HIGH goes to R-GPF when the map bin's top is above th_bin_max_h (in double)."""
    (mc, mmn, mmx), (qc, qmn, qmx) = mstat, qstat
    st = np.zeros(len(mc))
    flagged = np.zeros(len(mc), dtype=bool)
    near = np.zeros(len(mc), dtype=bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        for b in np.nonzero((mc > 0) & (qc > 0) & enough)[0]:
            mdh, cdh = mmx[b] - mmn[b], qmx[b] - qmn[b]
            ratio = _cpp_min(np.float64(mdh) / np.float64(cdh), np.float64(cdh) / np.float64(mdh))
            if ratio < p.scan_ratio_threshold:
                st[b] = MAP_HIGH if mdh >= cdh else CURR_HIGH
                flagged[b] = bool(mdh >= cdh and np.float64(mmx[b]) > np.float64(p.th_bin_max_h))
            else:
                st[b] = MERGE
            if eps_dh > 0.0:
                if mdh > 0 and cdh > 0:
                    near[b] |= abs(ratio - p.scan_ratio_threshold) <= ratio * 2 * eps_dh * (1 / mdh + 1 / cdh)
                near[b] |= abs(mdh - cdh) <= 4 * eps_dh or min(mdh, cdh) <= 2 * eps_dh or abs(mmx[b] - p.th_bin_max_h) <= eps_dh
    return st, flagged, near


def fit_plane(pts):
    """Two-pass float64 plane fit: (unit normal, mean, eigenvalues ascending, eigenvectors).  Empty: (0, 0, 1) through the origin."""
    pts = np.asarray(pts, dtype=np.float64).reshape(-1, 3)
    if len(pts) == 0:
        return np.array([0.0, 0.0, 1.0]), np.zeros(3), np.zeros(3), np.eye(3)
    mean = pts.mean(0)
    c = pts - mean
    lam, vec = np.linalg.eigh(c.T @ c / len(pts))
    return vec[:, 0], mean, lam, vec


def _axis_extent(pts, centre, v):
    """sum_i |v_i| * max |p_i - c_i|: the largest size of the products along v that a float32 accumulation centred on c adds up."""
    A = np.max(np.abs(pts - centre), axis=0)
    return float(np.abs(v) @ A)


def normal_tol(pts, lam, vec, centre, normal=None):
    """Angle tolerances of a float32 fit of pts whose accumulation is centred on `centre` (see the module docstring): of the normal
    as a whole, and of its component along each in-plane eigenvector k = 1, 2 (the normal may be the device's, for a degenerate set)."""
    pts = np.asarray(pts, dtype=np.float64).reshape(-1, 3)
    m = len(pts)
    if m == 0:
        return 0.0, [np.inf, np.inf]
    n = vec[:, 0] if normal is None else normal
    a0 = _axis_extent(pts, centre, n)
    per_k = []
    for k in (1, 2):
        num = 16.0 * EPS32 * math.sqrt(m) * a0 * _axis_extent(pts, centre, vec[:, k]) + 8.0 * math.sqrt(EPS32) * lam[2]
        gap = lam[k] - lam[0]
        per_k.append(num / gap if gap > 0 else np.inf)
    return max(per_k), per_k


def lpr_and_seeds(p, z_sorted):
    take = z_sorted[p.num_lowest_pts:p.num_lowest_pts + p.gf_num_lpr] if p.num_lowest_pts >= 0 else z_sorted[:0]
    lpr = float(np.sum(take) / len(take)) if len(take) else 0.0
    return lpr, lpr + p.gf_th_seeds_height


def rgpf(p, pts, dev_normals=None, cov_mode: int = 0, eps_pos: float = 0.0):
    """R-GPF of one bin's map points (float32 [n, 3], source order).  dev_normals: the device's normal per iteration, for the sign,
    and for classifying where the fit is degenerate.  eps_pos: how far (m) the device's copy of each point may be from this one.
    Returns dict(lpr, n_seeds, and per iteration normals, tols, checks, n_ground; ground = the final labels; ambiguous_from = the
    first iteration with a point inside the label band, or None)."""
    x = np.asarray(pts, dtype=np.float64).reshape(-1, 3)
    order = np.argsort(x[:, 2], kind="stable")
    lpr, thr = lpr_and_seeds(p, x[order, 2])
    gset = order[x[order, 2] < thr]
    out = dict(lpr=lpr, n_seeds=len(gset), normals=[], tols=[], checks=[], n_ground=[], ground=None, ambiguous_from=None)
    label = np.zeros(len(x), dtype=bool)
    for it in range(p.gf_iter):
        g = x[gset]
        nrm, mean, lam, vec = fit_plane(g)
        centre = (g[0] if len(g) else np.zeros(3)) if cov_mode == 1 else np.zeros(3)
        dev = None if dev_normals is None else np.asarray(dev_normals[it], dtype=np.float64)
        if dev is not None and float(nrm @ dev) < 0.0:
            nrm = -nrm
        tol, _ = normal_tol(g, lam, vec, centre)
        # a degenerate fit: the device's normal must still be orthogonal to each well-determined direction of the set
        _, per_k = normal_tol(g, lam, vec, centre, normal=dev if dev is not None else nrm)
        checks = [(vec[:, k], t) for k, t in zip((1, 2), per_k) if len(g) and t < 0.05]
        out["normals"].append(nrm)
        out["tols"].append(tol)
        out["checks"].append(checks)
        # classify with the reference's normal where the plane is determined to 0.05 rad, else with the device's
        if tol < 0.05 or dev is None:
            use, t_ang = nrm, min(tol, 0.05)
        else:
            use, t_ang = dev / np.linalg.norm(dev), 0.0
        dist = (x - mean) @ use
        label = dist < p.gf_dist_thr
        mg = float(np.max(np.linalg.norm(g, axis=1))) if len(g) else 0.0
        band = (t_ang * np.linalg.norm(x - mean, axis=1) +
                8 * EPS32 * (math.sqrt(max(len(g), 1)) * mg + np.linalg.norm(x, axis=1) + np.linalg.norm(mean)) + eps_pos)
        if out["ambiguous_from"] is None and np.any(np.abs(dist - p.gf_dist_thr) <= band):
            out["ambiguous_from"] = it
        out["n_ground"].append(int(label.sum()))
        gset = np.nonzero(label)[0]
    out["ground"] = label if p.gf_iter > 0 else np.isin(np.arange(len(x)), gset)
    return out


# ================================================================================================================================
# generated inputs
# ================================================================================================================================
def _bin_frame(p):
    rs, ss = p.max_range / p.num_rings, 2.0 * np.pi / p.num_sectors
    return rs, ss, p.min_h + 0.4


def xy_in_bin(p, ring, sector, n, rng, extent=None, lo=0.15, hi=0.85):
    """n (x, y) strictly inside bin (ring, sector): lo..hi of its ring and sector widths, or a square of side `extent` at its centre."""
    rs, ss, _ = _bin_frame(p)
    if extent is None:
        r = rng.uniform((ring + lo) * rs, (ring + hi) * rs, n)
        th = rng.uniform((sector + lo) * ss, (sector + hi) * ss, n)
        return r * np.cos(th), r * np.sin(th)
    rc, tc = (ring + 0.5) * rs, (sector + 0.5) * ss
    u = rc + rng.uniform(-extent / 2, extent / 2, n)
    t = rng.uniform(-extent / 2, extent / 2, n)
    x, y = u * np.cos(tc) - t * np.sin(tc), u * np.sin(tc) + t * np.cos(tc)
    r, th = np.hypot(x, y), np.arctan2(y, x) % (2 * np.pi)
    assert ((ring + lo) * rs < r).all() and (r < (ring + hi) * rs).all() and ((sector + lo) * ss < th).all() and (th < (sector + hi) * ss).all()
    return x, y


def rgpf_bin(p, ring, sector, kind, n, rng, extent=None):
    """(map, query) float32 [., 4] of one bin that the SRT hands to R-GPF.  Ground sits within +-3 cm of its plane, objects at
    least 0.65 m above it, so that no ground label lies near gf_dist_thr and no object is a seed; the degenerate kinds are
    stated with their point counts."""
    rs, ss, zg = _bin_frame(p)
    top = min(zg + 2.9, p.max_h - 0.1)
    tc = (sector + 0.5) * ss
    if kind in ("flat", "tight", "equal", "ulp", "dup", "slope"):
        n_obj = max(2, n // 8)
        gx, gy = xy_in_bin(p, ring, sector, n - n_obj, rng, extent)
        ox, oy = xy_in_bin(p, ring, sector, n_obj, rng, extent)
        ng = n - n_obj
        if kind == "flat":
            gz = zg + rng.uniform(-0.03, 0.03, ng)
        elif kind == "tight":      # +-5 mm: with a small extent, a bin whose normal a one-pass covariance cannot resolve
            gz = zg + rng.uniform(-0.005, 0.005, ng)
        elif kind == "equal":
            gz = np.full(ng, zg)
        elif kind == "ulp":
            gz = F32(zg) + rng.integers(0, 7, ng).astype(F32) * F32(6e-8)
        elif kind == "dup":
            gz = rng.choice(np.array([zg - 0.02, zg, np.nextafter(F32(zg), F32(-10)), zg + 0.01], dtype=F32), ng)
        else:   # a 10 degree radial slope
            u0 = (ring + 0.15) * rs
            slope = lambda xx, yy: zg + math.tan(math.radians(10.0)) * (xx * np.cos(tc) + yy * np.sin(tc) - u0)
            gz = slope(gx, gy) + rng.uniform(-0.02, 0.02, ng)
        base = slope(ox, oy) if kind == "slope" else zg
        oz = np.minimum(base + rng.uniform(0.65, 2.0, n_obj), top)
        m = np.concatenate([np.stack([gx, gy, gz], 1), np.stack([ox, oy, oz], 1)])
    elif kind == "wall":           # a vertical wall across the bin at its radial centre, no ground
        u = (ring + 0.5) * rs
        t = rng.uniform(-0.3, 0.3, n) * ss * u
        z = rng.uniform(zg, zg + 2.0, n)
        z[0] = zg
        m = np.stack([u * np.cos(tc) - t * np.sin(tc), u * np.sin(tc) + t * np.cos(tc), z], 1)
    elif kind in ("two", "three", "collinear"):
        k = {"two": 2, "three": 3, "collinear": 6}[kind]
        if kind == "collinear":    # six points on one 3-D segment: a rank-1 covariance
            s = np.linspace(0.0, 1.0, k)
            u, t = (ring + 0.3 + 0.4 * s) * rs, (0.2 * s - 0.1) * ss * (ring + 0.5) * rs
            z = zg + 0.7 * s
        else:
            x, y = xy_in_bin(p, ring, sector, k, rng)
            z = np.array([zg, zg + 0.7]) if k == 2 else np.array([zg, zg + 0.05, zg + 0.7])
            m = np.stack([x, y, z], 1)
        if kind == "collinear":
            m = np.stack([u * np.cos(tc) - t * np.sin(tc), u * np.sin(tc) + t * np.cos(tc), z], 1)
    elif kind == "high":           # three points all above lpr + gf_th_seeds_height: no seed, the empty-fit fallback
        x, y = xy_in_bin(p, ring, sector, 3, rng)
        m = np.stack([x, y, np.array([0.6, 0.9, 1.3])], 1)
    else:
        raise ValueError(kind)
    nq = max(40, p.minimum_num_pts)
    qx, qy = xy_in_bin(p, ring, sector, nq, rng)
    q = np.stack([qx, qy, zg + rng.uniform(-0.02, 0.02, nq)], 1)
    pad = lambda a, i: np.concatenate([a, np.full((len(a), 1), i)], 1).astype(F32)
    return pad(m, 40.0), pad(q, 7.0)


def frame_of(p, specs, seed):
    """(map, query, map bin of each point's spec) of one frame holding the bins of specs = [(ring, sector, kind, n, extent)]."""
    rng = np.random.default_rng(seed)
    ms, qs = [], []
    for ring, sector, kind, n, ext in specs:
        m, q = rgpf_bin(p, ring, sector, kind, n, rng, ext)
        ms.append(m)
        qs.append(q)
    m, q = np.concatenate(ms), np.concatenate(qs)
    pm, pq = rng.permutation(len(m)), rng.permutation(len(q))
    return m[pm], q[pq]


RGPF_PRESET = "seq_00"         # 20 rings of 4 m, 108 sectors, max_range 80 m
RGPF_KINDS = ([("flat", n) for n in (128, 129, 512, 513, 2560, 2561, BC.K4_C_CAP - 1, BC.K4_C_CAP, BC.K4_C_CAP + 1)] +
              [("equal", 300), ("ulp", 300), ("dup", 300), ("slope", 600), ("wall", 200), ("two", 2), ("three", 3), ("collinear", 6),
               ("high", 3)])
FAR_COMPACT = (19, 100, "tight", 400, 0.1)     # a 0.1 m cluster at 78 m: the one-pass covariance's worst case inside max_range


def rgpf_specs():
    return [(2 + i % 16, 5 * i + 2, k, n, None) for i, (k, n) in enumerate(RGPF_KINDS)] + [FAR_COMPACT]


def pi_sliver(steps: int = 400):
    """float32 [n, 2]: the sliver between azimuth pi and the sector boundary at PI_CFG (the truncated pi the sector size is defined
    with): |y| = (pi - PI_CFG) * |x| and up to `steps` float32 steps either side, both signs of y, x = -1, -7.3, -33, -79.9.  They
    lie inside EPS_THETA of the boundary, so the float64 reference takes either neighbour; the device must equal the oracle."""
    pts = []
    for x in (1.0, 7.3, 33.0, 79.9):
        y0 = F32((math.pi - PI_CFG) * x)
        ys = [y0]
        a = b = y0
        for _ in range(steps):
            a, b = np.nextafter(a, F32(np.inf)), np.nextafter(b, F32(0))
            ys += [a, b]
        for y in ys:
            pts += [(-x, y), (-x, -y)]
    return np.array(pts, dtype=np.float64).astype(F32)


def edge_points(p, seed=3, sliver=True):
    """float32 [n, 4]: points on every ring radius and sector angle and one ulp either side, azimuth +-pi and +-0, the truncated-pi
    sliver (pi_sliver; all inside the bands, sliver=False leaves it out), the range gate, the origin, z on the height gates and
    one ulp either side, and a seeded bulk over the whole disc."""
    rng = np.random.default_rng(seed)
    R, S, rmax = p.num_rings, p.num_sectors, p.max_range
    rs, ss = rmax / R, 2.0 * PI_CFG / S
    zmid = F32(0.5 * (p.min_h + p.max_h))
    pts = []
    up = lambda v: np.nextafter(F32(v), F32(np.inf))
    dn = lambda v: np.nextafter(F32(v), F32(-np.inf))
    for k in range(R + 1):                                     # ring radii on the axes (exact) and on two diagonals
        r = F32(k * rs)
        for v in (r, up(r), dn(r)):
            for x, y in ((v, 0.0), (0.0, v), (-v, 0.0), (-v, -0.0), (0.0, -v), (F32(0.6) * v, F32(0.8) * v), (-F32(0.8) * v, -F32(0.6) * v)):
                pts.append((x, y))
    for j in range(S):                                         # sector angles at three radii, and one ulp either side in x and y
        for rr in (0.37, 3.3, 0.93 * rmax):
            x, y = F32(rr * math.cos(j * ss)), F32(rr * math.sin(j * ss))
            for dx in (dn(x), x, up(x)):
                for dy in (dn(y), y, up(y)):
                    pts.append((dx, dy))
    for r in (1.0, 7.3, rmax):                                 # azimuth pi from both sides, both zeros, and the smallest y
        for y in (0.0, -0.0, 1e-45, -1e-45, 1e-30, -1e-30, float(np.spacing(F32(r))), -float(np.spacing(F32(r)))):
            pts.append((-r, y))
            pts.append((r, y))
    for x, y in ((0.0, 0.0), (-0.0, 0.0), (0.0, -0.0), (-0.0, -0.0), (1e-45, 0.0), (-1e-45, 0.0), (0.0, 1e-45), (0.0, -1e-45)):
        pts.append((x, y))                                     # the lower edge of ring 0: the origin
    xy = np.concatenate([np.array(pts, dtype=np.float64).astype(F32)] + ([pi_sliver()] if sliver else []))
    out = [np.stack([xy[:, 0], xy[:, 1], np.full(len(xy), zmid)], 1)]
    # z on the gates: float32 nearest and one ulp either side, at points well inside a bin
    gz = []
    for h in (p.min_h, p.max_h):
        for v in (F32(h), up(h), dn(h), up(up(h)), dn(dn(h))):
            gz.append(v)
    bx, by = xy_in_bin(p, 3, 5, len(gz), rng)
    out.append(np.stack([bx, by, np.array(gz)], 1))
    # bulk: uniform over a disc 5 % wider than max_range, z over the gate window and beyond
    n = 20000
    r = rmax * 1.05 * np.sqrt(rng.random(n))
    th = rng.uniform(-np.pi, np.pi, n)
    out.append(np.stack([r * np.cos(th), r * np.sin(th), rng.uniform(p.min_h - 0.5, p.max_h + 0.5, n)], 1))
    xyz = np.concatenate(out).astype(F32)
    return np.concatenate([xyz, np.full((len(xyz), 1), 1.0, F32)], 1)


def srt_cases(p):
    """(map, query, {bin: expected status}) of bins whose SRT quantities sit exactly on their thresholds (seq_05's 0.3 scan
    ratio).  Every height is a float32 value whose double differences and quotients are exact, asserted below."""
    assert p.scan_ratio_threshold == 0.3 and p.minimum_num_pts == 10
    rng = np.random.default_rng(17)
    nx = lambda v, d: float(np.nextafter(F32(v), F32(d)))
    # (ring, sector, map z range, query z range, query count, expected status)
    cases = [
        (3, 4, (-1.0, 1.5), (-1.0, -0.25), 12, MERGE),                     # ratio = 0.75 / 2.5 == 0.3 exactly: not below
        (3, 8, (-1.0, 1.5), (-1.0, nx(-0.25, -9)), 12, MAP_HIGH),           # one ulp below 0.3: handed to R-GPF
        (3, 12, (-1.0, -0.5), (-1.0, -0.98), 12, 0.0),                      # dh_map == 0.5 exactly: not above, left alone
        (3, 16, (-1.0, nx(-0.5, 9)), (-1.0, -0.98), 12, MAP_HIGH),          # one ulp above 0.5: handed to R-GPF
        (3, 20, (-1.0, 1.5), (-1.0, nx(-0.25, -9)), 9, LITTLE),             # minimum_num_pts - 1 query points
        (3, 24, (-1.0, 1.5), (-1.0, nx(-0.25, -9)), 10, MAP_HIGH),          # exactly minimum_num_pts
        (3, 28, (-1.0, 0.0), (-0.5, 0.5), 12, MERGE),                       # dh_map == dh_query: ratio 1
        (3, 32, (-1.0, 1.5), (-1.0, -1.0), 12, MAP_HIGH),                   # dh_query == 0: ratio min(inf, 0) = 0
        (3, 36, (-1.0, -1.0), (-1.0, -1.0), 12, MERGE),                     # both 0: ratio NaN, not below
        (6, 40, (-1.0, -1.0), (-1.0, -0.5), 12, CURR_HIGH),                 # dh_map == 0: ratio 0, query higher
        (6, 41, (-1.0, 0.0), (-0.5, 0.5), 12, BLOCKED),                     # MERGE beside a CURR_HIGH bin
        (6, 14, (-1.0, -1.0), (-1.0, -0.5), 12, CURR_HIGH),                 # sector 14 = num_rings - 1 ...
        (6, 0, (-1.0, 0.0), (-0.5, 0.5), 12, BLOCKED),                      # ... blocks sector 0 (sector -1 wraps by num_rings)
        (9, 59, (-1.0, -1.0), (-1.0, -0.5), 12, CURR_HIGH),                 # sector S - 1 ...
        (9, 0, (-1.0, 0.0), (-0.5, 0.5), 12, MERGE),                        # ... does not block sector 0
        (11, 50, None, (-1.0, -0.5), 12, LITTLE),                           # empty map bin
    ]
    ms, qs, want = [], [], {}
    for ring, sec, mz, qz, nq, st in cases:
        for z2, cnt, dst in ((mz, 12, ms), (qz, nq, qs)):
            if z2 is None:
                continue
            x, y = xy_in_bin(p, ring, sec, cnt, rng, lo=0.25, hi=0.75)
            # both extrema, the rest within 2 cm of the lower one: ground under a tall object, so that R-GPF's labels are clear
            fill = rng.uniform(z2[0], z2[0] + min(0.02, z2[1] - z2[0]), cnt - 2)
            z = np.concatenate([[z2[0], z2[1]], fill])
            dst.append(np.stack([x, y, z, np.full(cnt, 3.0)], 1))
        want[sec * p.num_rings + ring] = st
    d = np.float64(F32(-0.25)) - np.float64(F32(-1.0))
    assert d / 2.5 == 0.3 and np.float64(F32(nx(-0.25, -9))) - (-1.0) < 0.75           # the two ratio cases straddle 0.3 exactly
    m, q = np.concatenate(ms).astype(F32), np.concatenate(qs).astype(F32)
    return m, q, want


# -- the sweep paths' inputs (tests/test_gpu_sweep_float64.py): every frame below is also held to the oracle on the CPU ----------
SWEEP_THRESHOLDS = (0.10, 0.15, 0.20, 0.25, 0.30)
nx32 = lambda v, d: float(np.nextafter(F32(v), F32(d)))       # the float32 next to v towards d


def _case_cloud(p, ring, sec, zr, cnt, rng, tag):
    """cnt points of bin (ring, sector) holding both extrema of zr = (lo, hi), the rest within 2 cm of lo (ground under a tall
    object, so that R-GPF's labels are clear), intensity tag."""
    x, y = xy_in_bin(p, ring, sec, cnt, rng, lo=0.25, hi=0.75)
    fill = rng.uniform(zr[0], zr[0] + min(0.02, zr[1] - zr[0]), max(cnt - 2, 0))
    z = np.concatenate([[zr[0], zr[1]], fill])[:cnt]
    return np.stack([x, y, z, np.full(cnt, tag)], 1)


def _tie_frame(p, cases, seed):
    """(map, query, [(bin, case)]) of cases = [(map z range or None, map count, query z range or None, query count)], one bin each"""
    rng = np.random.default_rng(seed)
    ms, qs, where = [], [], []
    for k, (mz, mc, qz, qc) in enumerate(cases):
        ring, sec = 2 + k % 12, 1 + 2 * (k // 12)
        assert sec < p.num_sectors
        if mz is not None:
            ms.append(_case_cloud(p, ring, sec, mz, mc, rng, 3.0))
        if qz is not None and qc:
            qs.append(_case_cloud(p, ring, sec, qz, qc, rng, 7.0))
        where.append((sec * p.num_rings + ring, (mz, mc, qz, qc)))
    return np.concatenate(ms).astype(F32), np.concatenate(qs).astype(F32), where


def srt_tie_frame(p):
    """Version 3 on seq_05's geometry: every Scan Ratio Test quantity of the sweep grid exactly on its threshold and one float32
    step off it.  Each bin's lowest point is at z = 0 (inside (-1.3, 3.2)), so dh is exactly the float32 top height and the double
    ratio of two such heights is exact; asserted below."""
    cases = []
    for t in SWEEP_THRESHOLDS:
        top = F32(t * 2.5)
        assert np.float64(top) / 2.5 == t and np.float64(nx32(top, 0)) / 2.5 < t     # on the threshold, one step below
        cases += [((0.0, 2.5), 24, (0.0, float(top)), 45), ((0.0, 2.5), 24, (0.0, nx32(top, 0)), 45)]
    cases += [((0.0, 0.5), 24, (0.0, 0.02), 45), ((0.0, nx32(0.5, 9)), 24, (0.0, 0.02), 45)]        # map_dh 0.5 and one ulp above
    for k in (1, 10, 40):                                              # qc == minimum_num_pts and one below
        cases += [((0.0, 2.5), 24, (0.0, 0.1) if k > 2 else (0.0, 0.0), k), ((0.0, 2.5), 24, (0.0, 0.1) if k > 2 else (0.0, 0.0), k - 1)]
    cases += [((0.0, 2.5), 24, None, 0),                               # an empty query bin beside an occupied map bin
              ((0.0, 2.5), 24, (0.0, 0.0), 45),                        # dh_query 0: ratio min(inf, 0) = 0
              ((0.0, 0.0), 24, (0.0, 0.0), 45),                        # both 0: ratio NaN, not below any threshold
              ((0.0, 0.0), 24, (0.0, 0.5), 45),                        # dh_map 0: CURR_HIGH
              (None, 0, (0.0, 0.5), 45)]                               # an empty map bin
    return _tie_frame(p, cases, seed=31)


TIE_SETTINGS = ([dict(scan_ratio_threshold=t, minimum_num_pts=k) for k in (0, 1, 10, 40, -1, -5) for t in SWEEP_THRESHOLDS] +
                [dict(scan_ratio_threshold=0.3, minimum_num_pts=9), dict(scan_ratio_threshold=0.1, minimum_num_pts=39)])
V2_MAX_H = (-1.0, 0.0, 0.5, 1.5)


def srt_v2_frame(p):
    """Version 2: the map bin's top exactly on each th_bin_max_h and one float32 step above (for 0.0 the smallest denormal), a
    low query so that the ratio is far below every threshold."""
    cases = []
    for h in V2_MAX_H:
        assert np.float64(F32(h)) == h
        lo = max(h - 1.0, -1.25)
        for top in (h, nx32(h, 9)):
            cases.append(((lo, top), 24, (lo, lo + 0.005), 45))
    return _tie_frame(p, cases, seed=37)


V2_SETTINGS = ([dict(th_bin_max_h=h, scan_ratio_threshold=t) for h in V2_MAX_H for t in (0.1, 0.3)] +
               [dict(th_bin_max_h=0.0, minimum_num_pts=k) for k in (0, -1)])

# R-GPF under ground-filter groups: RGPF_KINDS plus the remaining sort switches (256, 1024, 2048) and one point past each
GROUP_KINDS = RGPF_KINDS + [("flat", n) for n in (256, 257, 1024, 1025, 2048, 2049)]


def group_specs():
    return [(2 + i % 16, 4 * i + 2, k, n, None) for i, (k, n) in enumerate(GROUP_KINDS)] + [FAR_COMPACT]


# each list is one sweep_ex call (two or more ground-filter groups); the gf_iter 0 group and a num_lowest_pts >= n group each run
# first in one of them, because a bin's plane record comes from the first group.  num_lowest_pts 2 and 3 are n and n - 1 of the
# 'three' bin and n of the 'two' bin; where num_lowest_pts >= n empties the LPR window (lpr 0), a seeds height of -0.5 keeps the
# objects out of the seeds, so that the fit stays determined
GROUP_CALLS = [
    [dict(gf_iter=0), dict(gf_iter=1), dict(gf_iter=3, scan_ratio_threshold=0.3), dict(gf_iter=8)],
    [dict(num_lowest_pts=600, gf_th_seeds_height=-0.5), dict(num_lowest_pts=0), dict(num_lowest_pts=5), dict(num_lowest_pts=2),
     dict(num_lowest_pts=3), dict(num_lowest_pts=512, gf_th_seeds_height=-0.5)],
    [dict(gf_num_lpr=1), dict(gf_num_lpr=20), dict(gf_num_lpr=10000), dict(gf_num_lpr=10000, num_lowest_pts=2560, gf_th_seeds_height=-0.5, gf_iter=1)],
    [dict(gf_th_seeds_height=s, gf_dist_thr=d) for s in (0.1, 0.3, 0.6) for d in (0.1, 0.3)] + [dict(gf_iter=0, num_lowest_pts=600)],
]


def witness_geometries():
    """(name, geometry fields) of the geometries the bin-edge witnesses run under"""
    return [("kitti_60x15x60", dict(max_range=60.0, num_rings=15, num_sectors=60)),
            ("kitti_60x15x108", dict(max_range=60.0, num_rings=15, num_sectors=108)),
            ("kitti_80x20x108", dict(max_range=80.0, num_rings=20, num_sectors=108)),
            ("exact_gates", dict(max_range=64.0, num_rings=16, num_sectors=64, min_h=-1.25, max_h=3.0)),
            ("40x360", dict(max_range=80.0, num_rings=40, num_sectors=360)),
            ("4x12", dict(max_range=60.0, num_rings=4, num_sectors=12)),
            ("26x181", dict(max_range=60.0, num_rings=26, num_sectors=181)),
            ("26x182", dict(max_range=60.0, num_rings=26, num_sectors=182))]


def witness_frame(p, seed=41):
    """(map, query, witnesses) of one geometry's bin-edge scene.  Each edge lies between a bin X that the Scan Ratio Test always
    hands to R-GPF (a 'flat' bin with a low query) and a bin Y that it never can (Y's query spans 2.5 m, its map at most 1.02 m with
    every witness) or no bin at all.  A map witness is a point 1 m above X's ground: non-ground in X (removed), kept in Y.
    - a ring radius on the -x axis (r exact, azimuth pi) and one ulp either side: X = ring k - 1, Y = ring k;
    - the range gate r = max_range on the -y axis and one ulp either side: X = the outer ring;
    - azimuth 0 (y = +-0, +-denormal, +-1 ulp): X = sector S - 1, Y = sector 0; azimuth pi the same way (for an even S, where pi is
      a sector edge): X = sector S/2 - 1, Y = sector S/2;
    - z on max_h and one and two ulps under it, and one over it, inside X = (the outer ring, sector 1);
    - min_h: three bins Z of ground 4 cm above min_h and one point 0.47 m over it, each with one witness on min_h, one ulp over it
      or one under it; a binned witness widens Z's map dh to 0.51 > 0.5 and hands Z to R-GPF (the query's 0.02 m puts the ratio
      under every threshold), which removes the top point;
    - the minimum_num_pts-th query point of a flat bin X = ring k - 1, on the ring radius k (+y axis: it lands in ring k, and X
      stays below minimum_num_pts) or one ulp inside it (-y axis: X has enough query points and goes to R-GPF).
    witnesses: list of dict(group, cloud ('map' / 'query'), idx (row in its cloud), alt (float32 x, y, z on the other side of the
    edge))."""
    rng = np.random.default_rng(seed)
    R, S, rs, ss = p.num_rings, p.num_sectors, p.max_range / p.num_rings, 2.0 * PI_CFG / p.num_sectors
    zg = p.min_h + 0.4
    zw = float(F32(zg + 1.0))
    ms, qs, wit = [], [], []

    def x_bin(ring, sec, nq=None):
        m, q = rgpf_bin(p, ring, sec, "flat", 48, rng)
        ms.append(m); qs.append(q if nq is None else q[:nq])

    def y_bin(ring, sec):
        x, y = xy_in_bin(p, ring, sec, 6, rng)
        ms.append(np.stack([x, y, zg + rng.uniform(0.0, 0.02, 6), np.full(6, 40.0)], 1).astype(F32))
        x, y = xy_in_bin(p, ring, sec, 45, rng)
        qz = np.concatenate([[zg, zg + 2.5], zg + rng.uniform(0.0, 2.5, 43)])
        qs.append(np.stack([x, y, qz, np.full(45, 7.0)], 1).astype(F32))

    def add(group, pts, alts, cloud="map"):
        dst = ms if cloud == "map" else qs
        base = sum(len(a) for a in dst)
        dst.append(np.array([(x, y, z, 9.0) for x, y, z in pts], dtype=F32))
        for i, a in enumerate(alts):
            wit.append(dict(group=group, cloud=cloud, idx=base + i, alt=np.array(a, dtype=F32)))

    up, dn = (lambda v: nx32(v, np.inf)), (lambda v: nx32(v, -np.inf))
    s_pi, k = S // 2, max(1, R // 2)
    rk = F32(k * rs)
    x_bin(k - 1, s_pi); y_bin(k, s_pi)                                        # a ring radius
    add("ring", [(-rk, 0.0, zw), (-dn(rk), 0.0, zw), (-up(rk), 0.0, zw)],
        [(-dn(rk), 0.0, zw), (-rk, 0.0, zw), (-dn(rk), 0.0, zw)])
    ug = F32(p.max_range)                                                      # the range gate
    sec_ny = int(polar(p, np.array([[0.0, -1.0, zg]]))[0][0]) // R
    x_bin(R - 1, sec_ny)
    add("range", [(0.0, -ug, zw), (0.0, -dn(ug), zw), (0.0, -up(ug), zw)],
        [(0.0, -up(ug), zw), (0.0, -up(ug), zw), (0.0, -ug, zw)])
    ra = F32((R - 0.5) * rs)                                                    # azimuth 0 and pi, in the outer ring
    ul = float(np.spacing(ra))
    x_bin(R - 1, S - 1); y_bin(R - 1, 0)
    ys = (0.0, -0.0, 1e-45, -1e-45, ul, -ul)
    flip = lambda y: -y if y != 0.0 else -1e-45                               # the other side of the edge
    add("azimuth 0", [(ra, y, zw) for y in ys], [(ra, flip(y), zw) for y in ys])
    if S % 2 == 0:
        x_bin(R - 1, s_pi - 1); y_bin(R - 1, s_pi)
        ys = (0.0, 1e-45, -1e-45, ul, -ul)
        add("azimuth pi", [(-ra, y, zw) for y in ys], [(-ra, flip(y), zw) for y in ys])
    # the height gates, in the outer ring, sectors 1 to 4
    at = lambda sec: (F32((R - 0.5) * rs * math.cos((sec + 0.5) * ss)), F32((R - 0.5) * rs * math.sin((sec + 0.5) * ss)))
    x_bin(R - 1, 1)
    hin = float(F32(p.max_h)) if float(F32(p.max_h)) < p.max_h else dn(p.max_h)      # the largest float32 under max_h
    zs = (up(hin), hin, dn(hin), dn(dn(hin)))
    add("max_h", [(*at(1), z) for z in zs], [(*at(1), up(hin) if z < p.max_h else hin) for z in zs])
    lin = float(F32(p.min_h)) if float(F32(p.min_h)) > p.min_h else up(p.min_h)      # the smallest float32 over min_h
    for j, z0 in enumerate((dn(lin), lin, up(lin))):
        sec = 2 + j
        x, y = xy_in_bin(p, R - 1, sec, 31, rng)
        mzs = np.concatenate([[lin + 0.04, lin + 0.51], lin + 0.04 + rng.uniform(0.0, 0.005, 29)])
        ms.append(np.stack([x, y, mzs, np.full(31, 40.0)], 1).astype(F32))
        x, y = xy_in_bin(p, R - 1, sec, 45, rng)
        qs.append(np.stack([x, y, lin + 0.1 + rng.uniform(0.0, 0.02, 45), np.full(45, 7.0)], 1).astype(F32))
        add("min_h", [(*at(sec), z0)], [(*at(sec), dn(lin) if z0 > p.min_h else lin)])
    # the query witnesses: X = ring k - 1 with minimum_num_pts - 1 query points, on the +y axis (witness on the radius: Y) and on
    # the -y axis (witness one ulp inside X)
    need = max(p.minimum_num_pts, 1)
    sec_y = int(polar(p, np.array([[0.0, 1.0, zg]]))[0][0]) // R
    for sec in (sec_y, sec_ny):
        x_bin(k - 1, sec, nq=need - 1); y_bin(k, sec)
    add("query", [(0.0, rk, zg), (0.0, -dn(rk), zg)], [(0.0, dn(rk), zg), (0.0, -rk, zg)], cloud="query")
    m, q = np.concatenate(ms).astype(F32), np.concatenate(qs).astype(F32)
    return m, q, wit


def witness_settings():
    """every witness geometry under two thresholds: 4 x 12 and 26 x 181 first (their K1 tables add up to exactly 56 KB)"""
    geos = dict(witness_geometries())
    order = ["4x12", "26x181"] + [g for g in geos if g not in ("4x12", "26x181")]
    return [dict(geos[g], scan_ratio_threshold=t) for g in order for t in (0.1, 0.3)]


WITNESS_VOI = 160.0                  # the VoI radius of the witness calls: beyond every max_range and the range-gate witnesses
CLASS_C_COARSE = dict(max_range=60.0, num_rings=4, num_sectors=12)     # 15 m x 30 degree bins


def class_c_frame(p):
    """(map, query) of nine flat seq_05 bins (rings 4 to 6 x sectors 11 to 13: 16-28 m, 66-84 degrees) of 1500 to 200 points, all
    inside one bin (ring 1, sector 2) of CLASS_C_COARSE: 3600 points there, a class-C bin, and class-A/B bins in seq_05's geometry."""
    sizes = (1500, 400, 300, 300, 250, 250, 200, 200, 200)
    specs = [(4 + i % 3, 11 + i // 3, "flat", n, None) for i, n in enumerate(sizes)]
    return frame_of(p, specs, seed=43)


CLASS_C_SETTINGS = [dict(scan_ratio_threshold=t) for t in (0.1, 0.3)] + [dict(CLASS_C_COARSE, scan_ratio_threshold=t) for t in (0.1, 0.3)]


def clear_witnesses(p, m, q, wit):
    """The witness frame without the witnesses that lie within the reference's band under p (either neighbour is right for them):
    (map, query, map rows kept, query rows kept, band witnesses)."""
    keep_m, keep_q = np.ones(len(m), bool), np.ones(len(q), bool)
    band = []
    for w in wit:
        cloud = m if w["cloud"] == "map" else q
        _, cand = polar(p, cloud[w["idx"]:w["idx"] + 1])
        if not (cand == cand[:, :1]).all():
            band.append(w)
            (keep_m if w["cloud"] == "map" else keep_q)[w["idx"]] = False
    rows_m, rows_q = np.nonzero(keep_m)[0], np.nonzero(keep_q)[0]
    return m[rows_m], q[rows_q], rows_m, rows_q, band


def moved(m, q, w):
    """(map, query) with witness w moved to its other side"""
    m, q = m.copy(), q.copy()
    (m if w["cloud"] == "map" else q)[w["idx"], :3] = w["alt"]
    return m, q


# ================================================================================================================================
# CPU self-tests of the reference
# ================================================================================================================================
def test_polar_reference_by_hand():
    p = P.preset("seq_05")                 # 15 rings of 4 m, 60 sectors, max_range 60, z window (-1.3, 3.2)
    pts = np.array([
        [0.0, 0.0, 0.0], [4.0, 0.0, 0.0], [np.nextafter(F32(4.0), F32(0)), 0.0, 0.0], [12.0, 16.0, 0.0],      # r = 20: ring 5
        [60.0, 0.0, 0.0], [np.nextafter(F32(60.0), F32(99)), 0.0, 0.0], [0.0, -60.0, 0.0],
        [-5.0, 0.0, 0.0], [-5.0, -0.0, 0.0], [-5.0, -1e-30, 0.0], [5.0, -1e-30, 0.0], [0.0, 5.0, 0.0],
        [5.0, 1.0, float(F32(-1.3))], [5.0, 1.0, float(np.nextafter(F32(-1.3), F32(-9)))],             # -1.3f > -1.3 > the next float
        [5.0, 1.0, float(F32(3.2))], [5.0, 1.0, float(np.nextafter(F32(3.2), F32(0)))],                 # 3.2f > 3.2 > the previous float
    ], dtype=np.float64).astype(F32)
    b, cand = polar(p, pts)
    R = 15
    want = [0, 1, 0, 8 * R + 5,                     # (12, 16): atan2 = 0.9273 rad = 8.85 sectors of 0.10472 rad
            14, -1,                                  # r == max_range is in the last ring; one ulp further is out
            44 * R + 14,                             # (0, -60): 2 * 3.1415926535 - pi / 2 is 44.99999999957 sectors
            30 * R + 1, 30 * R + 1,                  # azimuth pi, with y = +0 and y = -0: pi / (2 * 3.1415926535 / 60) = 30.0000000009
            29 * R + 1,                              # y = -1e-30, x < 0: 2 * 3.1415926535 - pi is 29.999999999 sectors
            59 * R + 1,                              # y = -1e-30, x > 0: azimuth 2 * 3.1415926535, clamped to the last sector
            15 * R + 1,                              # azimuth pi / 2
            1 * R + 1, -1, -1, 1 * R + 1]            # (5, 1): ring 1, sector 1 (0.1974 rad)
    assert b.tolist() == want
    # axis points carry no band: their candidates are all the exact bin
    assert (cand[[0, 1, 4, 7, 8, 11]] == b[[0, 1, 4, 7, 8, 11], None]).all()
    # a sector index never leaves [0, S) and a ring index never leaves [0, R), also for y = -tiny and theta = 2*pi - tiny
    rng = np.random.default_rng(0)
    x = rng.uniform(-60, 60, 50000).astype(F32)
    y = np.where(rng.random(50000) < 0.2, -np.abs(rng.normal(0, 1e-20, 50000)), rng.uniform(-60, 60, 50000)).astype(F32)
    bb, _ = polar(p, np.stack([x, y, np.zeros_like(x)], 1))
    ok = bb >= 0
    assert ok.any() and (bb[ok] // R < 60).all() and (bb[ok] % R < R).all()


def test_polar_reference_matches_the_numpy_restatement():
    """tests/np_restatement.py is a second reading of the same binning (the reference's double expression): away from the bands
    the two must agree point for point."""
    import np_restatement as NR
    for name in ("seq_05", "seq_00", "synthetic_40x360"):
        p = P.preset(name)
        pts = edge_points(p, sliver=False)
        b, cand = polar(p, pts)
        nb, _ = NR.bin_of_points(p, pts)
        clear = (cand == cand[:, :1]).all(1)
        assert clear.mean() > 0.95
        assert np.array_equal(b[clear], nb[clear]), name


def test_plane_fit_on_exact_planes():
    rng = np.random.default_rng(1)
    for offset in (0.0, 80.0, 1e3, 1e4):
        for _ in range(20):
            nrm = rng.normal(size=3)
            nrm /= np.linalg.norm(nrm)
            a = np.cross(nrm, [1.0, 0, 0] if abs(nrm[0]) < 0.9 else [0, 1.0, 0])
            a /= np.linalg.norm(a)
            b = np.cross(nrm, a)
            uv = rng.uniform(-2, 2, (50, 2))
            pts = offset + uv[:, :1] * a + uv[:, 1:] * b
            n, mean, lam, _ = fit_plane(pts)
            assert abs(abs(n @ nrm) - 1.0) < 1e-12, offset           # the two-pass fit does not care where the plane is
            assert lam[0] < 1e-12 * lam[2] + 1e-18
    n, mean, lam, _ = fit_plane(np.zeros((0, 3)))
    assert n.tolist() == [0.0, 0.0, 1.0] and mean.tolist() == [0.0, 0.0, 0.0]
    # degenerate sets: one point, two points, collinear points -- a finite unit normal orthogonal to the set's directions
    for pts in (np.array([[3.0, 1.0, -1.0]]), np.array([[3.0, 1.0, -1.0], [4.0, 1.5, -0.2]]), np.linspace([1, 2, 3], [2, 4, 7], 6)):
        n, mean, lam, vec = fit_plane(pts)
        assert np.isfinite(n).all() and abs(np.linalg.norm(n) - 1) < 1e-12
        if len(pts) > 1:
            d = pts[-1] - pts[0]
            assert abs(n @ d) < 1e-12 * np.linalg.norm(d)


def test_rgpf_reference_on_a_hand_made_bin():
    p = P.preset("seq_00")                  # num_lowest_pts 5, gf_num_lpr 20, th_seeds 0.5, gf_dist_thr 0.15, 3 iterations
    gx, gy = np.meshgrid(np.linspace(10.0, 11.0, 6), np.linspace(2.0, 2.5, 5))
    z_ground = -0.92 + 0.04 * (gx.ravel() - 10.0)          # a plane rising 4 cm per metre in x
    g = np.stack([gx.ravel(), gy.ravel(), z_ground], 1)
    obj = np.array([[10.5, 2.1, 0.5], [10.6, 2.2, 1.0]])
    pts = np.concatenate([obj, g])
    out = rgpf(p, pts, dev_normals=[np.array([0, 0, 1.0])] * 3)
    assert out["lpr"] == pytest.approx(np.mean(np.sort(z_ground)[5:25]), abs=1e-15)
    assert out["n_seeds"] == 30
    assert out["n_ground"] == [30, 30, 30] and out["ground"].tolist() == [False, False] + [True] * 30
    n0 = out["normals"][0]
    assert n0[2] > 0 and abs(n0 @ np.array([1.0, 0, 0.04]) / np.linalg.norm([1, 0, 0.04])) < 1e-12 and abs(n0[1]) < 1e-12
    # the empty-seed fallback: every point above lpr + 0.5 -> normal (0, 0, 1), d = 0, nothing is ground below 0.15
    out = rgpf(p, np.array([[10.0, 2.0, 0.6], [10.2, 2.0, 0.9], [10.4, 2.0, 1.3]]))
    assert out["n_seeds"] == 0 and out["normals"][0].tolist() == [0, 0, 1.0] and out["n_ground"] == [0, 0, 0]


def test_srt_reference_on_its_threshold_cases():
    p = P.preset("seq_05")
    m, q, want = srt_cases(p)
    mb, _ = polar(p, m)
    qb, _ = polar(p, q)
    assert (mb >= 0).all() and (qb >= 0).all()
    st, flagged, near = srt_status(p, bin_stats(p, mb, m[:, 2]), bin_stats(p, qb, q[:, 2]))
    for b, s in want.items():
        assert st[b] == s, (b % p.num_rings, b // p.num_rings, st[b], s)
        assert flagged[b] == (s == MAP_HIGH)
    assert not near.any()
    others = np.setdiff1d(np.arange(p.num_bins), list(want))
    assert (st[others] == 0).all()


def test_generated_bins_stay_inside_their_bins():
    p = P.preset(RGPF_PRESET)
    m, q = frame_of(p, rgpf_specs(), seed=2)
    for cloud in (m, q):
        b, cand = polar(p, cloud)
        assert (b >= 0).all() and (cand == b[:, None]).all()
    mb, _ = polar(p, m)
    qb, _ = polar(p, q)
    st, flagged, _ = srt_status(p, bin_stats(p, mb, m[:, 2]), bin_stats(p, qb, q[:, 2]))
    assert flagged.sum() == len(rgpf_specs()) and set(np.unique(mb)) == set(np.nonzero(flagged)[0])


def test_srt_reference_new_rules_by_hand():
    """Version 2's th_bin_max_h, the both-occupied test and the size_t comparison of the query count, on hand-made bin tables."""
    p = P.preset("seq_05")
    B = p.num_bins
    inf = np.inf

    def tables(rows):      # rows: {bin: (count, min z, max z)}
        c, mn, mx = np.zeros(B, np.int64), np.full(B, inf), np.full(B, -inf)
        for b, (n, lo, hi) in rows.items():
            c[b], mn[b], mx[b] = n, lo, hi
        return c, mn, mx
    # bin 0: map dh 2.5, query dh 0.25 (ratio 0.1); bin 1: the same map, no query; bin 2: the same map, one query point (dh 0)
    mst = tables({0: (20, 0.0, 2.5), 1: (20, 0.0, 2.5), 2: (20, 0.0, 2.5)})
    qst = tables({0: (12, 0.0, 0.25), 2: (1, 0.0, 0.0)})
    for k, want in ((13, [False] * 3), (12, [True, False, False]), (1, [True, False, True]), (0, [True, False, True]), (-1, [False] * 3), (-5, [False] * 3)):
        st, fl, _ = srt_status(p.replace(minimum_num_pts=k, scan_ratio_threshold=0.3), mst, qst)
        assert fl[:3].tolist() == want, k
        assert st[1] == LITTLE and (k >= 0 or (st == LITTLE).all()), k
    # ratio 0.1 is not below 0.1 (MERGE); version 2 has no neighbour test and no dh > 0.5 rule
    st, fl, _ = srt_status(p.replace(minimum_num_pts=1, scan_ratio_threshold=0.1), mst, qst)
    assert st[0] == MERGE and not fl[0] and st[2] == MAP_HIGH and fl[2]
    for top, th, want in ((1.5, 1.5, False), (float(np.nextafter(F32(1.5), F32(9))), 1.5, True), (0.0, 0.0, False), (1e-45, 0.0, True),
                          (-1.0, -1.0, False), (0.4, 0.05, True)):
        pv = p.replace(version=2, th_bin_max_h=th, minimum_num_pts=10)
        m2 = tables({0: (20, top - 0.45, top)})
        q2 = tables({0: (12, top - 0.45, top - 0.44)})
        st, fl, _ = srt_status(pv, m2, q2)
        assert st[0] == MAP_HIGH and fl[0] == want and fl.sum() == want, (top, th)      # map dh 0.45 <= 0.5: flagged all the same
    st, fl, _ = srt_status(p.replace(version=2, th_bin_max_h=0.0), tables({0: (20, 0.0, 0.5)}), tables({0: (12, -1.0, 1.0)}))
    assert st[0] == CURR_HIGH and not fl.any()
    st, fl, _ = srt_status(p.replace(version=2, minimum_num_pts=0), tables({0: (20, 0.0, 2.5)}), tables({}))
    assert not fl.any() and (st == 0).all()
    st, fl, _ = srt_status(p.replace(version=2, minimum_num_pts=-1), mst, qst)
    assert not fl.any() and (st == LITTLE).all()


def test_sweep_frames_hold_their_ties():
    """The tie frames put each case in its own bin, with the intended exact heights and counts, and the reference flags each of
    them as the hand count says under every setting."""
    p = P.preset("seq_05").replace(skip_voxelize=1)
    m, q, where = srt_tie_frame(p)
    mb, cm = polar(p, m)
    qb, cq = polar(p, q)
    assert (mb >= 0).all() and (qb >= 0).all() and (cm == mb[:, None]).all() and (cq == qb[:, None]).all()
    ms, qs = bin_stats(p, mb, m[:, 2]), bin_stats(p, qb, q[:, 2])
    f32 = lambda zr: None if zr is None else tuple(float(F32(v)) for v in zr)
    where = [(b, (f32(mz), mc, f32(qz), qc)) for b, (mz, mc, qz, qc) in where]
    for b, (mz, mc, qz, qc) in where:
        assert ms[0][b] == mc and qs[0][b] == qc
        if mz is not None:
            assert (ms[1][b], ms[2][b]) == mz
        if qc:
            assert (qs[1][b], qs[2][b]) == qz
    assert sorted(set(np.unique(mb))) == sorted(b for b, c in where if c[0] is not None)
    for s in TIE_SETTINGS:
        pv = p.replace(**s)
        _, fl, near = srt_status(pv, ms, qs)
        want = 0
        for b, (mz, mc, qz, qc) in where:
            if mz is None or qc == 0 or pv.minimum_num_pts < 0 or qc < pv.minimum_num_pts:
                continue
            mdh, cdh = mz[1] - mz[0], qz[1] - qz[0]
            ratio = 0.0 if cdh == 0 and mdh > 0 else (np.nan if mdh == 0 and cdh == 0 else min(mdh / cdh, cdh / mdh) if mdh and cdh else 0.0)
            want += bool(ratio < pv.scan_ratio_threshold and mdh >= cdh and mdh > 0.5)
        assert fl.sum() == want and not near.any(), s
    pv2 = p.replace(version=2)
    m, q, where = srt_v2_frame(pv2)
    ms, qs = bin_stats(pv2, polar(pv2, m)[0], m[:, 2]), bin_stats(pv2, polar(pv2, q)[0], q[:, 2])
    for s in V2_SETTINGS:
        pv = pv2.replace(**s)
        _, fl, _ = srt_status(pv, ms, qs)
        want = 0 if pv.minimum_num_pts < 0 else sum(float(F32(c[0][1])) > pv.th_bin_max_h for _, c in where)
        assert fl.sum() == want, s


def _oracle_against_reference(p, m, q, tag):
    """The C++ oracle (bit-identical to the device) against the reference on one frame under p: bin tables, statuses, flagged bins
    and the keep mask outside ambiguous bins.  Returns (reference keep, known, ambiguous bins)."""
    from oracle import oracle_py
    o = oracle_py.Oracle(p)
    try:
        o.run(m, q)
        mb, _ = polar(p, m)
        assert np.array_equal(o.bin_of_point(0), mb), tag
        mn, mx, cnt, _ = o.bins(0)
        rc, rmn, rmx = bin_stats(p, mb, m[:, 2])
        occ = rc > 0
        assert np.array_equal(cnt, rc) and np.array_equal(mn[occ], rmn[occ]) and np.array_equal(mx[occ], rmx[occ]), tag
        report, ambiguous = [], []
        st, keep, known = _reference_keep(p, m, q, {pl["bin"]: pl for pl in o.planes()}, p.cov_mode, tag, report, ambiguous)
        assert np.array_equal(o.status()[0], st), (tag, np.nonzero(o.status()[0] != st)[0][:10])
        # the map points the static map keeps: those of the arranged bins and of the complement (a query point's source index
        # carries the top bit).  Without a plane-fit iteration R-GPF rejects nothing, but only the seeds return to the map.
        okeep = np.zeros(len(m), np.uint8)
        for which in (o.ARRANGED, o.COMPLEMENT):
            _, src = o.cloud(which)
            okeep[src[src < 0x80000000]] = 1
        _, rej = o.cloud(o.MAP_REJECTED)
        assert not okeep[rej].any() and (p.gf_iter == 0 or (okeep == 0).sum() == len(rej)), tag
        assert np.array_equal(okeep[known], keep[known]), tag
        return keep, known, ambiguous
    finally:
        o.close()


def test_sweep_frames_reference_against_the_oracle():
    """Every frame of the sweep tests under every setting they run: the reference and the oracle agree, so the GPU comparisons
    rest on a reference pinned on the CPU."""
    base = P.preset("seq_05").replace(skip_voxelize=1)
    m, q, _ = srt_tie_frame(base)
    for s in TIE_SETTINGS:
        _oracle_against_reference(base.replace(**s), m, q, ("tie", s))
    pv2 = base.replace(version=2)
    m, q, _ = srt_v2_frame(pv2)
    for s in V2_SETTINGS:
        _oracle_against_reference(pv2.replace(**s), m, q, ("v2", s))
    m, q = class_c_frame(base)
    for s in CLASS_C_SETTINGS:
        _, known, _ = _oracle_against_reference(base.replace(**s), m, q, ("class C", s))
        assert known.all()
    for name, g in witness_geometries():
        m, q, wit = witness_frame(base.replace(**g))
        for s in witness_settings():
            pv = base.replace(**s)
            mc, qc, _, _, _ = clear_witnesses(pv, m, q, wit)
            _oracle_against_reference(pv, mc, qc, ("witness", name, s))
    # the oracle's polar binning with the band witnesses in: every point in one of the reference's candidate bins
    from oracle import oracle_py
    for name, g in witness_geometries():
        pv = base.replace(**g)
        m, q, _ = witness_frame(pv)
        o = oracle_py.Oracle(pv)
        o.run(m, q)
        _, cand = polar(pv, m)
        assert (o.bin_of_point(0)[:, None] == cand).any(1).all(), name
        o.close()


@pytest.mark.parametrize("cov_mode", [0, 1])
def test_group_frame_reference_against_the_oracle(cov_mode):
    p = P.preset(RGPF_PRESET).replace(skip_voxelize=1, cov_mode=cov_mode)
    m, q = frame_of(p, group_specs(), seed=47)
    n_amb = []
    for call in GROUP_CALLS:
        for s in call:
            _, _, amb = _oracle_against_reference(p.replace(**s), m, q, ("groups", s))
            n_amb.append(len(amb))
    assert max(n_amb) <= 1, n_amb


def test_witnesses_are_decisive():
    """Moving any witness to the other side of its edge changes the reference's keep mask, and both sides are binned exactly as
    intended (a ring, sector or gate apart): the GPU comparison of the witnesses cannot pass by keeping or removing everything."""
    base = P.preset("seq_05").replace(skip_voxelize=1)
    from oracle import oracle_py
    for name, g in witness_geometries():
        p = base.replace(**g)
        m, q, wit = witness_frame(p)
        groups = {w["group"] for w in wit}
        assert groups >= {"ring", "range", "azimuth 0", "max_h", "min_h", "query"} and (("azimuth pi" in groups) == (p.num_sectors % 2 == 0))

        def keep_of(mm, qq):
            o = oracle_py.Oracle(p)
            o.run(mm, qq)
            planes = {pl["bin"]: pl for pl in o.planes()}
            o.close()
            report, amb = [], []
            _, keep, known = _reference_keep(p, mm, qq, planes, 0, name, report, amb)
            assert known.all() and not amb, name
            return keep
        k0 = keep_of(m, q)
        for w in wit:
            cloud = m if w["cloud"] == "map" else q
            b0 = polar(p, cloud[w["idx"]:w["idx"] + 1])[0][0]
            b1 = polar(p, w["alt"][None, :].astype(np.float64))[0][0]
            assert b0 != b1, (name, w["group"], w["idx"])
            k1 = keep_of(*moved(m, q, w))
            assert not np.array_equal(k0, k1), (name, w["group"], cloud[w["idx"]].tolist(), w["alt"].tolist())


def _cov_f32(pts, shift: bool):
    """The device's covariance arithmetic restated in float32: nine sequential sums of products, / m, minus the mean products,
    about the first point of the list (cov_mode 1) or about the origin (cov_mode 0)."""
    a = np.asarray(pts, dtype=F32)
    k = a[0] if shift else np.zeros(3, F32)
    d = (a - k).astype(F32)
    m = F32(len(a))
    s = lambda v: np.cumsum(v.astype(F32), dtype=F32)[-1] / m
    mx, my, mz = s(d[:, 0]), s(d[:, 1]), s(d[:, 2])
    xx, xy, xz = s(d[:, 0] * d[:, 0]) - mx * mx, s(d[:, 0] * d[:, 1]) - mx * my, s(d[:, 0] * d[:, 2]) - mx * mz
    yy, yz, zz = s(d[:, 1] * d[:, 1]) - my * my, s(d[:, 1] * d[:, 2]) - my * mz, s(d[:, 2] * d[:, 2]) - mz * mz
    return np.array([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]], dtype=np.float64)


def test_normal_tolerance_separates_the_shifted_from_the_one_pass_covariance():
    """At the far compact cluster of the R-GPF frame the centred tolerance admits the shifted float32 covariance with a wide margin
    and rejects the one-pass one: so the GPU test at cov_mode 1 fails if the device drops the shift."""
    p = P.preset(RGPF_PRESET)
    ring, sector, kind, n, ext = FAR_COMPACT
    errs1, errs0, tols = [], [], []
    for seed in range(8):
        m, _ = rgpf_bin(p, ring, sector, kind, n, np.random.default_rng(seed), ext)
        x = m[:, :3].astype(np.float64)
        order = np.argsort(x[:, 2], kind="stable")
        _, thr = lpr_and_seeds(p, x[order, 2])
        seeds = x[order][x[order, 2] < thr]
        nrm, _, lam, vec = fit_plane(seeds)
        tol, _ = normal_tol(seeds, lam, vec, seeds[0])
        ang = lambda c: math.acos(min(1.0, abs(float(np.linalg.eigh(c)[1][:, 0] @ nrm))))
        errs1.append(ang(_cov_f32(seeds, True)))
        errs0.append(ang(_cov_f32(seeds, False)))
        tols.append(tol)
    assert max(e / t for e, t in zip(errs1, tols)) < 0.05          # measured: 4e-5
    assert min(e / t for e, t in zip(errs0, tols)) > 3.0           # measured: 6


# ================================================================================================================================
# GPU comparisons
# ================================================================================================================================
@pytest.fixture(scope="module")
def capi():
    from erasor_b200 import capi as Cap
    return Cap


def _assert_bins(dev, cand, tag):
    ok = (dev[:, None] == cand).any(1)
    bad = np.nonzero(~ok)[0]
    assert not len(bad), (tag, bad[:10].tolist(), dev[bad[:10]].tolist(), cand[bad[:10]].tolist())


def _tables_equal(a, b):
    (_, amn, amx, ac), (_, bmn, bmx, bc) = a, b
    return np.array_equal(ac, bc) and np.array_equal(amn, bmn, equal_nan=True) and np.array_equal(amx, bmx, equal_nan=True)


@pytest.mark.gpu
@needs_gpu
@pytest.mark.parametrize("preset", ["seq_05", "seq_00", "exact_gates"])
def test_binning_edges(capi, oracle_mod, preset):
    if preset == "exact_gates":   # gates and radii that float32 represents exactly, so that z == max_h and r == max_range are hit
        p = P.preset("seq_05").replace(min_h=-1.25, max_h=3.0, max_range=64.0, num_rings=16, num_sectors=64)
    else:
        p = P.preset(preset)
    p = p.replace(skip_voxelize=1)
    pts = edge_points(p)
    exact, cand = polar(p, pts)
    h = capi.Handle(p)
    h.set_inputs(pts, pts)
    h.compare(3)
    bm, *tm = h.get_bins(capi.CLOUD_MAP)
    bq, *_ = h.get_bins(capi.CLOUD_QUERY)
    _assert_bins(bm, cand, preset)
    assert np.array_equal(bm, bq), "the map and the query path bin the same point differently"
    amb = ~(cand == cand[:, :1]).all(1)
    assert np.array_equal(bm[~amb], exact[~amb])
    # inside the bands (the truncated-pi sliver among them) the reference takes either neighbour: the oracle decides
    o = oracle_mod.Oracle(p)
    o.run(pts, pts[:0])
    assert np.array_equal(bm, o.bin_of_point(0)), (preset, int((bm != o.bin_of_point(0)).sum()))
    o.close()
    print(f"{preset}: {len(pts)} points, {int(amb.sum())} within a band, {int((bm[amb] != exact[amb]).sum())} of them in the other neighbour")
    # the node path (fetch_VoI + K1 at the identity pose) builds the same tables, and the mask mode keeps the same points
    keep_cloud, _ = h.get_static_mask()
    k_frames = h.process_frames(pts, np.array([0, len(pts)], np.uint64), pts, np.array([0, len(pts)], np.uint64))
    assert np.array_equal(k_frames, keep_cloud)
    # node mode moves the map to the body frame first, and a float32 transform may turn x = -0.0 (azimuth pi) into +0.0
    # (azimuth 0), as the reference's does: those points are left out of this comparison
    sub = pts[~((pts[:, 0] == 0) & np.signbit(pts[:, 0]))]
    h.set_inputs(sub, sub)
    h.compare(3)
    bs, *ts = h.get_bins(capi.CLOUD_MAP)
    _assert_bins(bs, polar(p, sub)[1], (preset, "subset"))
    gm = capi.Map(sub)
    h.attach_map(gm)
    kg, _ = h.process_nodes(np.array([[0, 0, 0, 0, 0, 0, 1.0]]), sub, np.array([0, len(sub)], np.uint64), voi_max_range=2 * p.max_range)
    tn = h.get_bins(capi.CLOUD_MAP, per_point=False)
    assert (np.hypot(sub[:, 0].astype(np.float64), sub[:, 1].astype(np.float64)) < 2 * p.max_range).all()
    diff = np.nonzero((ts[2] != tn[3]))[0]
    assert _tables_equal((None, *ts), tn), ("node mode bins the map differently from cloud mode", diff[:10].tolist(), ts[2][diff[:10]].tolist(),
                                            tn[3][diff[:10]].tolist())
    assert (kg == 1).all()
    h.close()
    gm.close()


def _planes_by_bin(h):
    return {pl["bin"]: pl for pl in h.get_planes()}


def _check_bin_fit(p, mpts, pl, cov_mode, tag, report, check_planes=True, eps_pos=0.0):
    """Device R-GPF record of one bin against the reference; returns the reference's final ground labels (None if ambiguous).
    check_planes=False: the record is of a copy of the points up to eps_pos metres away; only its normals' signs are used."""
    nd = np.asarray(pl["normal_d"], dtype=np.float64)
    ref = rgpf(p, mpts[:, :3], dev_normals=[nd[i, :3] for i in range(p.gf_iter)], cov_mode=cov_mode, eps_pos=eps_pos)
    assert pl["n_points"] == len(mpts) and pl["n_seeds"] == ref["n_seeds"], tag
    if not check_planes:
        return ref["ground"] if ref["ambiguous_from"] is None else None
    assert pl["lpr"] == pytest.approx(ref["lpr"], rel=1e-12, abs=1e-12), tag
    last = p.gf_iter if ref["ambiguous_from"] is None else ref["ambiguous_from"] + 1
    for it in range(last):
        n_dev = nd[it, :3]
        assert np.isfinite(nd[it]).all() and abs(np.linalg.norm(n_dev) - 1.0) < 1e-5, (tag, it, n_dev)
        tol = ref["tols"][it]
        if tol < 0.05:
            ang = math.acos(min(1.0, abs(float(n_dev @ ref["normals"][it]))))
            assert ang <= tol, (tag, it, ang, tol)
            report.append(ang / tol if tol > 0 else 0.0)
        else:                                             # degenerate: orthogonal to every well-determined direction
            for v, t in ref["checks"][it]:
                assert abs(float(n_dev @ v)) <= t, (tag, it, "degenerate", float(n_dev @ v), t)
        if it < last - 1 or ref["ambiguous_from"] is None:
            assert pl["n_ground"][it] == ref["n_ground"][it], (tag, it)
    return ref["ground"] if ref["ambiguous_from"] is None else None


def _reference_keep(p, m, q, planes, cov_mode, tag, report, ambiguous, check_planes=True, eps_pos=0.0):
    """Reference status and keep mask of one frame (and which points it knows: not those of an ambiguous bin), the device's
    planes giving each normal's sign; every flagged bin's plane record is checked on the way."""
    mb, _ = polar(p, m)
    qb, _ = polar(p, q)
    st, flagged, _ = srt_status(p, bin_stats(p, mb, m[:, 2]), bin_stats(p, qb, q[:, 2]))
    keep = np.ones(len(m), dtype=np.uint8)
    known = np.ones(len(m), dtype=bool)
    assert sorted(planes) == sorted(np.nonzero(flagged)[0].tolist()), tag
    for b in np.nonzero(flagged)[0]:
        idx = np.nonzero(mb == b)[0]
        g = _check_bin_fit(p, m[idx], planes[int(b)], cov_mode, (tag, int(b) % p.num_rings, int(b) // p.num_rings), report,
                           check_planes, eps_pos)
        if g is None:
            ambiguous.append((tag, int(b)))
            known[idx] = False
        else:
            keep[idx[~g]] = 0
    return st, keep, known


@pytest.mark.gpu
@needs_gpu
@pytest.mark.parametrize("cov_mode", [0, 1])
def test_rgpf_against_float64(capi, cov_mode):
    p = P.preset(RGPF_PRESET).replace(skip_voxelize=1, cov_mode=cov_mode)
    m, q = frame_of(p, rgpf_specs(), seed=2)
    h = capi.Handle(p)
    h.set_inputs(m, q)
    h.compare(3)
    report, ambiguous = [], []
    st, keep, known = _reference_keep(p, m, q, _planes_by_bin(h), cov_mode, "rgpf", report, ambiguous)
    assert np.array_equal(h.get_status(), st.astype(np.float32))
    dkeep, _ = h.get_static_mask()
    assert np.array_equal(dkeep[known], keep[known])
    print(f"cov_mode {cov_mode}: {len(report)} fits, worst angle / tolerance {max(report):.3g}, ambiguous bins {ambiguous}")
    assert len(ambiguous) <= 1
    assert h.fence_counts()["empty_plane_fits"] >= p.gf_iter          # the 'high' bin: no seed, gf_iter empty fits
    h.close()


@pytest.mark.gpu
@needs_gpu
def test_srt_thresholds_against_float64(capi):
    p = P.preset("seq_05").replace(skip_voxelize=1)
    m, q, want = srt_cases(p)
    h = capi.Handle(p)
    h.set_inputs(m, q)
    h.compare(3)
    report, ambiguous = [], []
    st, keep, known = _reference_keep(p, m, q, _planes_by_bin(h), 0, "srt", report, ambiguous)
    dst = h.get_status()
    for b, s in want.items():
        assert dst[b] == np.float32(s), (b % p.num_rings, b // p.num_rings, float(dst[b]), s)
    assert np.array_equal(dst, st.astype(np.float32))
    dkeep, _ = h.get_static_mask()
    assert known.all() and np.array_equal(dkeep, keep)
    h.close()


@pytest.mark.gpu
@needs_gpu
def test_k2_windows_against_float64(capi):
    """Frames that hand one fewer, exactly, and one more bin to R-GPF than one slot window of the mask-mode SRT + scatter holds,
    through cloud mode and the batched mask mode, against the reference."""
    p = P.preset(BC.K2_PRESET).replace(skip_voxelize=1)
    W = BC.k2_window(p.num_bins)
    rng = np.random.default_rng(23)
    frames, refs = [], []
    h = capi.Handle(p)
    report, ambiguous = [], []
    for k, n_flag in enumerate((W - 1, W, W + 1)):
        pick = np.sort(rng.choice(p.num_bins, n_flag, replace=False))
        specs = [(int(b % p.num_rings), int(b // p.num_rings), "flat", 24, None) for b in pick]
        m, q = frame_of(p, specs, seed=40 + k)
        h.set_inputs(m, q)
        h.compare(3)
        planes = _planes_by_bin(h)
        assert len(planes) == n_flag
        st, keep, known = _reference_keep(p, m, q, planes, 0, ("k2", n_flag), report, ambiguous)
        dkeep, _ = h.get_static_mask()
        assert np.array_equal(h.get_status(), st.astype(np.float32)) and np.array_equal(dkeep[known], keep[known])
        frames.append((m, q))
        refs.append((keep, known))
    assert len(ambiguous) <= 0.01 * sum(len(f[0]) for f in frames) / 24
    mo = np.cumsum([0] + [len(m) for m, _ in frames]).astype(np.uint64)
    qo = np.cumsum([0] + [len(q) for _, q in frames]).astype(np.uint64)
    kb = h.process_frames(np.concatenate([m for m, _ in frames]), mo, np.concatenate([q for _, q in frames]), qo)
    for f, (keep, known) in enumerate(refs):
        got = kb[int(mo[f]):int(mo[f + 1])]
        assert np.array_equal(got[known], keep[known]), ("process_frames", f)
    h.close()


FAR_POSES = [(tx, ty, yaw) for tx, ty in ((1000.0, -1000.0), (-1000.0, 1000.0), (10000.0, 10000.0), (-10000.0, -10000.0))
             for yaw in (0.0, math.pi / 2, math.pi, 0.7315)]


@pytest.mark.gpu
@needs_gpu
def test_far_from_origin_node_mode(capi):
    """One local scene (flagged bins of every kind plus merged bins), placed in a world map at +-1000 m and +-10 000 m and four
    yaws, run in node mode: the keep mask matches the float64 reference on the body-frame points at every pose."""
    p = P.preset(RGPF_PRESET).replace(skip_voxelize=1)
    # not the degenerate bins, nor the far compact cluster whose normal the default one-pass covariance does not resolve
    # (test_rgpf_against_float64 holds it to the cov_mode 1 tolerance): a degenerate or unresolved normal changes with the
    # last bits of the points, so its sign from the frame at the origin does not carry over to the same frame elsewhere
    specs = [s for s in rgpf_specs() if s[2] not in ("two", "three", "collinear", "high", "tight")]
    m_loc, q = frame_of(p, specs, seed=5)
    rng = np.random.default_rng(6)
    # merged bins: map and query of equal height spread
    mx, my = xy_in_bin(p, 8, 60, 400, rng)
    mz = rng.uniform(-1.0, 1.0, 400)
    extra = np.stack([mx, my, mz, np.full(400, 5.0)], 1).astype(F32)
    m_loc = np.concatenate([m_loc, extra])
    q = np.concatenate([q, extra[::2]])
    h = capi.Handle(p)
    h.set_inputs(m_loc, q)
    h.compare(3)
    planes0 = _planes_by_bin(h)
    keep0, _ = h.get_static_mask()
    for tx, ty, yaw in FAR_POSES:
        c, s = math.cos(yaw), math.sin(yaw)
        xl, yl = m_loc[:, 0].astype(np.float64), m_loc[:, 1].astype(np.float64)
        world = np.stack([c * xl - s * yl + tx, s * xl + c * yl + ty, m_loc[:, 2], m_loc[:, 3]], 1).astype(F32)
        pose = np.array([[tx, ty, 0.0, 0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2)]])
        # the body-frame points the reference sees: the float32 world points moved back exactly
        dx, dy = world[:, 0].astype(np.float64) - tx, world[:, 1].astype(np.float64) - ty
        body = np.stack([c * dx + s * dy, -s * dx + c * dy, world[:, 2]], 1)
        eps_pos = 16 * EPS32 * (math.hypot(tx, ty) + p.max_range)
        b, cand = polar(p, body, eps_pos=eps_pos)
        assert (cand == b[:, None]).all(), "the scene keeps every point clear of the bin boundaries by more than EPS_POS"
        bodyf = body.astype(F32)
        report, ambiguous = [], []
        _, keep, known = _reference_keep(p, bodyf, q, planes0, 0, ("far", tx, ty, yaw), report, ambiguous, check_planes=False,
                                         eps_pos=eps_pos)
        assert known.all() and not ambiguous
        gm = capi.Map(world)
        h.attach_map(gm)
        kg, fk = h.process_nodes(pose, q, np.array([0, len(q)], np.uint64), want_frame_keep=True)
        assert np.array_equal(fk[0], keep), (tx, ty, yaw, int((fk[0] != keep).sum()))
        assert np.array_equal(fk[0], keep0), "the same local scene gives the same mask far from the origin"
        h.attach_map(None)
        gm.close()
    h.close()


@pytest.mark.gpu
@needs_gpu
def test_empty_and_single_point_inputs(capi):
    """Empty and one-point clouds through every entry point: correctly shaped empty or trivial results, no CUDA error, nothing
    left over from the previous, larger call."""
    p = P.preset("seq_05").replace(skip_voxelize=1)
    none = np.zeros((0, 4), F32)
    one = np.array([[5.0, 1.0, -0.5, 7.0]], F32)
    big_m, big_q = frame_of(p, [(4, 7, "flat", 600, None), (6, 20, "flat", 300, None)], seed=9)
    b_one = int(polar(p, one)[0][0])
    h = capi.Handle(p)
    for tag, m, q in (("big", big_m, big_q), ("0/0", none, none), ("1/0", one, none), ("0/1", none, one), ("1/1", one, one),
                      ("big again", big_m, big_q), ("1/1 after big", one, one)):
        h.set_inputs(m, q)
        h.compare(3)
        bm, mn, mx, cnt = h.get_bins(capi.CLOUD_MAP)
        bq, _, _, cq = h.get_bins(capi.CLOUD_QUERY)
        assert bm.shape == (len(m),) and bq.shape == (len(q),), tag
        assert np.array_equal(bm, polar(p, m)[0]) and np.array_equal(bq, polar(p, q)[0]), tag
        assert cnt.sum() == len(m) and cq.sum() == len(q), tag
        keep, gnd = h.get_static_mask()
        assert keep.shape == (len(m),) and gnd.shape == (len(m),), tag
        if len(m) <= 1:
            assert h.get_planes() == [] and (h.get_status() == 0).all() and (keep == 1).all(), tag
            if len(m):
                assert cnt[b_one] == 1 and mn[b_one] == one[0, 2] and mx[b_one] == one[0, 2], tag
            arr, cmp_ = h.get_static_estimate()
            mr, cr = h.get_outliers()
            assert arr.shape[1:] == (4,) and cmp_.shape[1:] == (4,) and mr.shape == (0, 4) and cr.shape == (0, 4), tag
            assert len(arr) + len(cmp_) >= len(m), tag
    # the batched mask mode with empty frames between non-empty ones
    for sizes in (((0, 0),), ((1, 0), (0, 1)), ((0, 0), (1, 1), (0, 0))):
        ms = [one if a else none for a, _ in sizes]
        qs = [one if c else none for _, c in sizes]
        mo = np.cumsum([0] + [len(x) for x in ms]).astype(np.uint64)
        qo = np.cumsum([0] + [len(x) for x in qs]).astype(np.uint64)
        keep = h.process_frames(np.concatenate(ms), mo, np.concatenate(qs), qo)
        nf, nr = h.frame_stats()
        assert keep.shape == (int(mo[-1]),) and (keep == 1).all() and (nf == 0).all() and (nr == 0).all(), sizes
    # node mode: a one-point map, an empty query, an empty node between two others
    gm = capi.Map(one)
    h.attach_map(gm)
    I7 = np.array([0, 0, 0, 0, 0, 0, 1.0])
    for qs in ([none], [one], [one, none, one]):
        kg, fk = h.process_nodes(np.stack([I7] * len(qs)), np.concatenate(qs), np.cumsum([0] + [len(x) for x in qs]).astype(np.uint64),
                                 want_frame_keep=True)
        assert kg.shape == (1,) and fk.shape == (len(qs), 1) and (kg == 1).all() and (fk == 1).all(), len(qs)
    h.attach_map(None)
    gm.close()
    # the batched voxeliser: empty clouds, one-point clouds
    for sizes in ((0,), (1,), (0, 1, 0), (1, 0, 1)):
        xyzi = np.concatenate([one if s else none for s in sizes])
        vox, oo = h.voxelize_batch(xyzi, np.cumsum([0] + list(sizes)).astype(np.uint64), 0.2)
        assert oo.tolist() == np.cumsum([0] + list(sizes)).tolist() and vox.shape == (sum(sizes), 4), sizes
        if len(vox):
            assert (vox == one).all(), sizes
    h.close()

