"""Test-side generators for the pose-driven paths (numpy only).

- ``POSES``: body -> origin poses [x y z qx qy qz qw] like a real sequence's -- yaw over the whole circle (both signs of qz and
  qw at +-pi), a few degrees of roll and pitch plus one 30 degree tilt, z within +-50 m, translations of 0 to 20 000 m along
  each axis and diagonally -- each also as -q, 0.5 q and 2 q (geoPose2eigen divides by |q|^2, so these are the same rotation).
- ``replace``: a scene moved rigidly by a world transform G: the map through the oracle's float transform, the node poses
  composed with G in double; body-frame queries are unchanged.
- Boundary shells around a criterion point: exact ties, ulp walks across the limit, and points whose float pre-test lands in
  the radius cut's guard band (pose_math.h).  ``d2f`` restates the kernel's float pre-test only to show that the band is hit;
  the truth is always the reference's double expression (``voi_truth``).
"""
import numpy as np

F32 = np.float32
RADII = (0.5, 9.5, 80.0, 1.0e4)
BODY_CUT = 2.7                      # mapgen's CAR_BODY_SIZE


# ---- poses ----------------------------------------------------------------------------------------------------------------
def quat_rpy(roll: float, pitch: float, yaw: float) -> np.ndarray:
    """[qx qy qz qw] of R = Rz(yaw) Ry(pitch) Rx(roll)."""
    cr, sr, cp, sp, cy, sy = (np.cos(roll / 2), np.sin(roll / 2), np.cos(pitch / 2), np.sin(pitch / 2), np.cos(yaw / 2), np.sin(yaw / 2))
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


def qmul(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Hamilton product of [x y z w] quaternions."""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def rot(q: np.ndarray) -> np.ndarray:
    """Rotation matrix of a (not necessarily unit) quaternion, in double."""
    x, y, z, w = np.asarray(q, dtype=np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def pose7(t, q) -> np.ndarray:
    return np.concatenate([np.asarray(t, dtype=np.float64), np.asarray(q, dtype=np.float64)])


def _base_poses():
    d = np.deg2rad
    rng = np.random.default_rng(2024)
    out = [
        ("origin", pose7([0, 0, 0], [0, 0, 0, 1])),
        ("yaw+pi/2 x300", pose7([300, 0, 0], quat_rpy(0, 0, np.pi / 2))),
        ("yaw-pi/2 y-4000", pose7([0, -4000, 12.5], quat_rpy(0, 0, -np.pi / 2))),
        ("qz+1 qw+0 x20000", pose7([20000, 0, -50], [0, 0, 1, 0])),
        ("qz-1 qw+0 y20000", pose7([0, 20000, 50], [0, 0, -1, 0])),
        ("qz+1 qw-0 x-300", pose7([-300, 0, 3], [0, 0, 1, -0.0])),
        ("yaw+pi y-20000", pose7([0, -20000, -7], quat_rpy(0, 0, np.pi))),
        ("yaw-pi x-4000", pose7([-4000, 0, 0], quat_rpy(0, 0, -np.pi))),
        ("diag 300", pose7([300, 300, 1], quat_rpy(0, 0, rng.uniform(-np.pi, np.pi)))),
        ("diag 4000", pose7([-4000, 4000, -25], quat_rpy(0, 0, rng.uniform(-np.pi, np.pi)))),
        ("diag 20000", pose7([20000, -20000, 40], quat_rpy(0, 0, rng.uniform(-np.pi, np.pi)))),
        ("diag -20000", pose7([-20000, -20000, -50], quat_rpy(0, 0, rng.uniform(-np.pi, np.pi)))),
        ("tilt 3/-5 deg", pose7([4000, 300, 20], quat_rpy(d(3), d(-5), 1.1))),
        ("tilt -5/4 deg", pose7([-300, 20000, -40], quat_rpy(d(-5), d(4), -2.5))),
        ("tilt 30 deg", pose7([300, -4000, 5], quat_rpy(d(30), d(2), 0.7))),
        ("random far", pose7(rng.uniform(-20000, 20000, 2).tolist() + [rng.uniform(-50, 50)],
                             quat_rpy(*rng.uniform(-d(5), d(5), 2), rng.uniform(-np.pi, np.pi)))),
    ]
    return out


def _variants(base):
    out = []
    for name, p in base:
        for tag, s in (("", 1.0), (" -q", -1.0), (" 0.5q", 0.5), (" 2q", 2.0)):
            v = p.copy()
            v[3:] *= s
            out.append((name + tag, v))
    return out


POSES = _variants(_base_poses())


# ---- rigid re-placement of a scene --------------------------------------------------------------------------------------------
def compose(G7: np.ndarray, P7: np.ndarray) -> np.ndarray:
    """Pose of G o P as a 7-vector, in double (quaternion product, rotated translation)."""
    t = rot(G7[3:]) @ P7[:3] + G7[:3]
    q = qmul(G7[3:] / np.linalg.norm(G7[3:]), P7[3:] / np.linalg.norm(P7[3:]))
    return pose7(t, q)


def replace(map_world: np.ndarray, poses7, G7: np.ndarray, oracle_mod, q_scale: float = 1.0):
    """Move a map by G with the oracle's float transform and compose every node pose with G (the quaternion then scaled by
    q_scale, e.g. -1 for -q).  Returns (moved map, poses [F,7])."""
    moved = oracle_mod.transform(map_world, oracle_mod.pose_to_matrix(G7))
    P = np.stack([compose(G7, p) for p in poses7])
    P[:, 3:] *= q_scale
    return moved, P


# ---- the cut predicates, restated -----------------------------------------------------------------------------------------
def criterion(pose: np.ndarray, oracle_mod):
    """(px, py) of fetch_VoI: the float translation of the oracle's pose matrix, as double."""
    T = oracle_mod.pose_to_matrix(pose)
    return float(T[0, 3]), float(T[1, 3])


def voi_truth(x, y, px: float, py: float, r: float) -> np.ndarray:
    """fetch_VoI: pow(pt.x - x, 2) + pow(pt.y - y, 2) < pow(r, 2), in double on the float coordinates."""
    dx = np.asarray(x, dtype=np.float32).astype(np.float64) - px
    dy = np.asarray(y, dtype=np.float32).astype(np.float64) - py
    with np.errstate(invalid="ignore"):
        return dx * dx + dy * dy < r * r


def submap_truth(x, y, cx: float, cy: float, s: float) -> np.ndarray:
    """set_submap: fabs(x - pt.x) < submap_size && fabs(y - pt.y) < submap_size, in double."""
    dx = np.abs(cx - np.asarray(x, dtype=np.float32).astype(np.float64))
    dy = np.abs(cy - np.asarray(y, dtype=np.float32).astype(np.float64))
    with np.errstate(invalid="ignore"):
        return (dx < s) & (dy < s)


def body_cut_kept(x, y) -> np.ndarray:
    """mapgen's body cut: a point is kept unless pow(x, 2) + pow(y, 2) (double) < (float)pow(2.7, 2)."""
    x64 = np.asarray(x, dtype=np.float32).astype(np.float64)
    y64 = np.asarray(y, dtype=np.float32).astype(np.float64)
    with np.errstate(invalid="ignore"):
        return ~(x64 * x64 + y64 * y64 < float(F32(BODY_CUT ** 2)))


def band(r: float):
    """The radius pre-test's guard band [lim_lo, lim_hi] (pose_math.h node_pose_of)."""
    lim = float(r) ** 2
    return (np.nextafter(F32(lim * (1.0 - 1.0e-6)), F32(-np.inf)), np.nextafter(F32(lim * (1.0 + 1.0e-6)), F32(np.inf)))


def _fma_f32(a: np.ndarray, b: np.ndarray, c: np.ndarray) -> np.ndarray:
    """fmaf(a, b, c) for float32 inputs: a * b is exact in double; the double sum's rounding error (TwoSum) breaks the rare
    double-rounding ties when the sum is rounded to float."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)
    r = s.astype(np.float32)
    lo = np.nextafter(r, F32(-np.inf)).astype(np.float64)
    hi = np.nextafter(r, F32(np.inf)).astype(np.float64)
    r64 = r.astype(np.float64)
    mid_lo, mid_hi = (lo + r64) / 2, (hi + r64) / 2
    r = np.where((s == mid_lo) & (e < 0), lo.astype(np.float32), r)
    r = np.where((s == mid_hi) & (e > 0), hi.astype(np.float32), r)
    return r


def d2f(x, y, pxf, pyf) -> np.ndarray:
    """The kernel's float pre-test: fmaf(dyf, dyf, dxf * dxf) on float differences."""
    with np.errstate(invalid="ignore", over="ignore"):
        dxf = np.asarray(x, dtype=np.float32) - F32(pxf)
        dyf = np.asarray(y, dtype=np.float32) - F32(pyf)
        return _fma_f32(dyf, dyf, dxf * dxf)


# ---- boundary shells ---------------------------------------------------------------------------------------------------------
TIE, WALK, BAND, NONFINITE = range(4)


def ulp_step(a: np.ndarray, k) -> np.ndarray:
    """a moved by k float ulps (k > 0 towards +inf), elementwise."""
    a = np.asarray(a, dtype=np.float32).copy()
    k = np.broadcast_to(np.asarray(k), a.shape)
    for j in range(int(np.abs(k).max()) if k.size else 0):
        a = np.where(np.abs(k) > j, np.nextafter(a, np.where(k > 0, F32(np.inf), F32(-np.inf))), a)
    return a


def _nonfinite(px, py):
    n, i = np.nan, np.inf
    return np.array([[n, py], [px, n], [n, n], [i, py], [-i, py], [px, i], [px, -i], [i, i], [-i, -i], [i, n]], dtype=np.float32)


def shell(px: float, py: float, r: float, seed: int = 0, n_angles: int = 64, walk: int = 8, band_min: int = 100,
          band_max: int = 2000, nonfinite: bool = False):
    """Float x y around (px, py) at radius r in the classes TIE / WALK / BAND (/ NONFINITE): returns (xy [n,2] float32, class [n]).

    TIE: axis-aligned points with px +- r (py +- r) representable, so that the double distance equals r^2 exactly.
    WALK: at n_angles angles, the nearest float point on the circle moved by +-1..+-walk ulps in x, in y and in both.
    BAND: points from the walk's neighbourhoods whose d2f lands in the guard band; where the float grid is too coarse for
    band_min distinct ones (far from the origin, small r), the ones found are repeated (the caller gives them distinct z)."""
    rng = np.random.default_rng(seed)
    pxf, pyf = F32(px), F32(py)
    xs, cls = [], []
    # TIE
    ties = []
    for sx, sy in ((1, 0), (-1, 0), (0, 1), (0, -1)):
        x, y = F32(px + sx * r), F32(py + sy * r)
        if (float(x) - px) ** 2 + (float(y) - py) ** 2 == r * r:
            ties.append((x, y))
    if ties:
        xs.append(np.array(ties, dtype=np.float32)); cls.append(np.full(len(ties), TIE))
    # WALK
    th = np.concatenate([np.arange(8) * (np.pi / 4), rng.uniform(-np.pi, np.pi, max(n_angles - 8, 0))])
    bx, by = (px + r * np.cos(th)).astype(np.float32), (py + r * np.sin(th)).astype(np.float32)
    sgx, sgy = np.where(np.cos(th) >= 0, 1, -1), np.where(np.sin(th) >= 0, 1, -1)
    wk = [np.stack([bx, by], 1)]
    for k in list(range(1, walk + 1)) + list(range(-walk, 0)):
        wk.append(np.stack([ulp_step(bx, sgx * k), by], 1))
        wk.append(np.stack([bx, ulp_step(by, sgy * k)], 1))
        wk.append(np.stack([ulp_step(bx, sgx * k), ulp_step(by, sgy * k)], 1))
    wk = np.concatenate(wk)
    xs.append(wk); cls.append(np.full(len(wk), WALK))
    # BAND: a (2 walk + 1)^2 ulp neighbourhood of every angle's circle point
    ks = np.arange(-walk, walk + 1)
    gx = np.concatenate([ulp_step(bx, k) for k in ks])
    gy = np.concatenate([ulp_step(by, k) for k in ks])
    cx = np.repeat(gx.reshape(len(ks), -1)[:, None, :], len(ks), axis=1).reshape(-1)
    cy = np.repeat(gy.reshape(len(ks), -1)[None, :, :], len(ks), axis=0).reshape(-1)
    cand = np.unique(np.stack([cx, cy], 1), axis=0)
    lo, hi = band(r)
    v = d2f(cand[:, 0], cand[:, 1], pxf, pyf)
    inb = cand[(v >= lo) & (v <= hi)]
    if len(inb) > band_max:
        inb = inb[rng.choice(len(inb), band_max, replace=False)]
    if 0 < len(inb) < band_min:
        inb = np.tile(inb, (-(-band_min // len(inb)), 1))
    xs.append(inb.astype(np.float32)); cls.append(np.full(len(inb), BAND))
    if nonfinite:
        nf = _nonfinite(pxf, pyf)
        xs.append(nf); cls.append(np.full(len(nf), NONFINITE))
    return np.concatenate(xs).astype(np.float32), np.concatenate(cls)


def square_shell(cx: float, cy: float, s: float, seed: int = 0, n_per_edge: int = 48, walk: int = 8, nonfinite: bool = False):
    """Float x y on and next to both edges of set_submap's square on each axis: per edge the edge coordinate itself (an exact
    tie where cx +- s is representable) and +-1..+-walk ulps off it, the other coordinate inside, on or beyond the square."""
    rng = np.random.default_rng(seed)
    out = []
    for axis in (0, 1):
        c0, c1 = (cx, cy) if axis == 0 else (cy, cx)
        for sg in (1, -1):
            e = F32(c0 + sg * s)
            other = np.concatenate([(c1 + rng.uniform(-s, s, n_per_edge)), [c1, c1 + s, c1 - s]]).astype(np.float32)
            for k in range(-walk, walk + 1):
                a = np.full(len(other), ulp_step(np.array([e]), k)[0], dtype=np.float32)
                out.append(np.stack([a, other], 1) if axis == 0 else np.stack([other, a], 1))
    xy = np.concatenate(out).astype(np.float32)
    if nonfinite:
        xy = np.concatenate([xy, _nonfinite(F32(cx), F32(cy))])
    return xy


def body_cut_shell(seed: int = 0, n_angles: int = 96, walk: int = 8):
    """Float x y around the lidar origin at mapgen's 2.7 m body cut: ulp walks across the float limit at many angles,
    the axis points r, r -+ ulps, and the points whose double distance rounds onto the float limit."""
    xy, _ = shell(0.0, 0.0, BODY_CUT, seed=seed, n_angles=n_angles, walk=walk, band_min=0)
    lim = float(F32(BODY_CUT ** 2))
    rt = np.float32(np.sqrt(lim))
    extra = np.array([[rt, 0], [0, rt], [-rt, 0], [0, -rt]], dtype=np.float32)
    extra = np.concatenate([extra] + [np.stack([ulp_step(extra[:, 0], k), ulp_step(extra[:, 1], k)], 1) for k in (-2, -1, 1, 2)])
    return np.concatenate([xy, extra]).astype(np.float32)


def with_z(xy: np.ndarray, rng: np.random.Generator, z_lo: float = -1.5, z_hi: float = 2.5, label: float = 9.0) -> np.ndarray:
    """xyzi cloud from x y: z uniform in [z_lo, z_hi), intensity = label."""
    out = np.empty((len(xy), 4), dtype=np.float32)
    out[:, :2] = xy
    out[:, 2] = rng.uniform(z_lo, z_hi, len(xy))
    out[:, 3] = label
    return out
