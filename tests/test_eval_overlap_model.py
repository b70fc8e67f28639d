"""CPU suite: a numpy model of the device overlap report (erasor_eval_overlap, DESIGN.md section 11.1) -- the GT cell grid, the
shell search with its stopping bound, the coarse far path -- held to an all-pairs brute force on adversarial sets; the percentile
reconstruction from two order statistics held to numpy bit for bit; and evaluate.format_report / `python -m erasor_b200.analysis
--host` held byte for byte to the reference script's stdout on two golden pairs.  tests/test_gpu_eval_overlap.py holds the device
to sklearn and to this model."""
import os
import subprocess
import sys

import numpy as np
import pytest

from erasor_b200 import evaluate as E
from test_eval_grid_model import grid_setup, is_dynamic, seed41_pass, sq_dist, voxel_cell

F = np.float32
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN_STDOUT = {name: os.path.join(HERE, "golden", f"analysis_runner_{name}_stdout.txt") for name in ("seed41", "seed41_jittered")}
SHELL_MAX = 4          # kOvlShellMax: fine shells searched before a point takes the far path
COARSE_DIV = 32        # kOvlCoarseDiv: coarse cells per axis at most


def jittered_estimate(est):
    """the second golden pair's estimate: every point moved by up to 0.3 m (0.17 m per axis), plus 300 of them 1 km away"""
    rng = np.random.default_rng(43)
    j = est.copy()
    j[:, :3] += rng.uniform(-0.17, 0.17, (len(j), 3)).astype(np.float32)
    far = est[rng.choice(len(est), 300, replace=False)].copy()
    far[:, 0] += F(1000.0)
    return np.concatenate([j, far]).astype(np.float32)


# ---- the model -------------------------------------------------------------------------------------------------------------------
def ovl_grids(gt, voxelsize):
    """ovl_setup: the fine grid (eval_grid_setup over the GT), its face margin marg = R 2^-21, and the coarse grid: blocks of
    2^cshift fine cells per axis, cshift the smallest with at most COARSE_DIV blocks per axis"""
    pts = gt[:, :3] + F(0.0)
    mn, mx = pts.min(axis=0), pts.max(axis=0)
    g = grid_setup(mn, mx, voxelsize)
    cmax = max(max(abs(float(g["min_b"][k])), abs(float(g["min_b"][k] + g["div"][k] - 1)) + 1.0) for k in range(3))
    g["marg"] = (cmax + 3.0) * float(g["leaf"]) / 2 ** 21
    sh = 0
    while np.any(((g["div"] - 1) >> sh) + 1 > COARSE_DIV):
        sh += 1
    return g, dict(cshift=sh, cdiv=((g["div"] - 1) >> sh) + 1)


def _cells(pts, grid, shift=0):
    c = np.stack([voxel_cell(pts[:, k], grid["inv"], grid["min_b"][k]) for k in range(3)], axis=1) >> shift
    table = {}
    for i, key in enumerate(map(tuple, c)):
        table.setdefault(key, []).append(i)
    return {k: np.array(v) for k, v in table.items()}


SHRINK, GROW = 1.0 - 2.0 ** -40, 1.0 + 2.0 ** -40


def model_overlap(gt, est, keep=None, voxelsize=0.2):
    """What k_ovl_query computes: (distance per estimate point -- NaN where deselected, +inf for an empty GT --, far-path flag)."""
    gt = np.asarray(gt, np.float32).reshape(-1, 4)
    est = np.asarray(est, np.float32).reshape(-1, 4)
    sel = np.ones(len(est), bool) if keep is None else np.asarray(keep).astype(bool)
    dist = np.full(len(est), np.nan)
    far = np.zeros(len(est), bool)
    if len(gt) == 0:
        dist[sel] = np.inf
        return dist, far
    g, cg = ovl_grids(gt, voxelsize)
    fine, coarse = _cells(gt, g), _cells(gt, g, cg["cshift"])
    cdiv = cg["cdiv"]
    order = sorted(coarse, key=lambda k: k[0] + k[1] * cdiv[0] + k[2] * cdiv[0] * cdiv[1])     # coarse key order
    boxes = [(k, gt[coarse[k], :3].min(axis=0).astype(np.float64), gt[coarse[k], :3].max(axis=0).astype(np.float64)) for k in order]
    leaf, marg, div, mb = float(g["leaf"]), g["marg"], g["div"], g["min_b"]

    def axis_gap(x, c0, c1):
        return max(0.0, c0 * leaf - marg - x, x - ((c1 + 1) * leaf + marg))

    def scan_row(qrow, x0, x1, jj, kk, best):
        for x in range(x0, x1 + 1):
            if (x, jj, kk) in fine:
                best = min(best, sq_dist(qrow[None], gt[fine[(x, jj, kk)]]).min())
        return best

    def centre_out(c, t, lo, hi):
        v = c + (-((t + 1) >> 1) if t & 1 else t >> 1)
        return None if v < lo or v > hi else v

    def clamped_cell(x, a, lo, hi):
        return int(min(max(np.floor(x / leaf) - mb[a], lo), hi))

    def visit_block(key, qrow, qd, ub, best):
        """ovl_visit_block: the block's fine rows, nearest first along y and z, each pruned by its gap and x window"""
        w = 1 << cg["cshift"]
        lo = [key[a] * w for a in range(3)]
        hi = [min(lo[a] + w - 1, div[a] - 1) for a in range(3)]
        jc, kc = clamped_cell(qd[1], 1, lo[1], hi[1]), clamped_cell(qd[2], 2, lo[2], hi[2])
        for tk in range(2 * (hi[2] - lo[2]) + 2):
            kk = centre_out(kc, tk, lo[2], hi[2])
            if kk is None:
                continue
            gz = axis_gap(qd[2], kk + mb[2], kk + mb[2])
            if gz * gz * SHRINK > min(ub, best):
                continue
            for tj in range(2 * (hi[1] - lo[1]) + 2):
                jj = centre_out(jc, tj, lo[1], hi[1])
                if jj is None:
                    continue
                gy = axis_gap(qd[1], jj + mb[1], jj + mb[1])
                gyz, bound = gy * gy + gz * gz, min(ub, best)
                if gyz * SHRINK > bound:
                    continue
                r = np.sqrt(max(bound * GROW - gyz, 0.0)) * GROW
                xl = max(np.floor((qd[0] - r - marg) / leaf) - mb[0] - 1.0, lo[0])
                xh = min(np.floor((qd[0] + r + marg) / leaf) - mb[0] + 1.0, hi[0])
                if not xl <= xh:
                    continue
                x0, x1 = int(xl), int(xh)
                gx = axis_gap(qd[0], x0 + mb[0], x1 + mb[0])
                if (gx * gx + gyz) * SHRINK > bound:
                    continue
                best = scan_row(qrow, x0, x1, jj, kk, best)
        return best

    def face_bound(x, c, s, a):
        lb = np.inf
        if c + s + 1 <= div[a] - 1:
            lb = (c + s + 1 + mb[a]) * leaf - marg - x
        if c - s - 1 >= 0:
            lb = min(lb, x - ((c - s + mb[a]) * leaf + marg))
        return lb

    for i in np.flatnonzero(sel):
        q = est[i]
        qd = q[:3].astype(np.float64)
        best, settled = np.inf, False
        a = q[:3] * g["inv"]
        if np.all((a >= g["lo"]) & (a < g["hi"])):
            c = [int(voxel_cell(q[k:k + 1], g["inv"], mb[k])[0]) for k in range(3)]
            for s in range(SHELL_MAX + 1):
                for b in range(-s, s + 1):
                    jj = c[1] + b
                    if not 0 <= jj < div[1]:
                        continue
                    gy = axis_gap(qd[1], jj + mb[1], jj + mb[1])
                    for cc in range(-s, s + 1):
                        kk = c[2] + cc
                        if not 0 <= kk < div[2]:
                            continue
                        gz = axis_gap(qd[2], kk + mb[2], kk + mb[2])
                        gyz = gy * gy + gz * gz
                        if gyz * SHRINK > best:
                            continue
                        face = abs(b) == s or abs(cc) == s
                        for x0, x1 in ([(c[0] - s, c[0] + s)] if face else [(c[0] - s, c[0] - s), (c[0] + s, c[0] + s)]):
                            x0, x1 = max(x0, 0), min(x1, div[0] - 1)
                            if x0 > x1:
                                continue
                            gx = axis_gap(qd[0], x0 + mb[0], x1 + mb[0])
                            if (gx * gx + gyz) * SHRINK > best:
                                continue
                            best = scan_row(q, x0, x1, jj, kk, best)
                lb = min(face_bound(qd[k], c[k], s, k) for k in range(3))
                if lb == np.inf or (best < np.inf and np.sqrt(best) <= lb * SHRINK):
                    settled = True
                    break
        if not settled:
            far[i] = True
            ub, gmin, vmin = best, np.inf, 0
            for v, (_, lo, hi) in enumerate(boxes):
                f = np.maximum(np.abs(qd - lo), np.abs(qd - hi))
                ub = min(ub, float(f @ f) * GROW)
                gp = np.maximum(0.0, np.maximum(lo - qd, qd - hi))
                if float(gp @ gp) < gmin:
                    gmin, vmin = float(gp @ gp), v
            best = visit_block(boxes[vmin][0], q, qd, ub, best)
            for v, (k, lo, hi) in enumerate(boxes):
                gp = np.maximum(0.0, np.maximum(lo - qd, qd - hi))
                if v == vmin or float(gp @ gp) * SHRINK > min(ub, best):
                    continue
                best = visit_block(k, q, qd, ub, best)
        dist[i] = np.sqrt(best)
    return dist, far


def brute_overlap(gt, est, keep=None):
    gt = np.asarray(gt, np.float32).reshape(-1, 4)
    est = np.asarray(est, np.float32).reshape(-1, 4)
    sel = np.ones(len(est), bool) if keep is None else np.asarray(keep).astype(bool)
    dist = np.full(len(est), np.nan)
    if len(gt) == 0:
        dist[sel] = np.inf
    elif sel.any():
        dist[sel] = np.sqrt(sq_dist(est[sel][:, None, :], gt[None, :, :]).min(axis=1))
    return dist


# ---- adversarial sets ------------------------------------------------------------------------------------------------------------
def _lab(rng, n):
    return rng.choice([40.0, 252.0, 259.0, 50.0], n).astype(np.float32)


def overlap_sets():
    """name -> (gt, est, keep, voxelsize)"""
    rng = np.random.default_rng(29)
    sets = {}
    base = rng.uniform(-6, 6, (400, 3)).astype(np.float32)
    gt = np.c_[base, _lab(rng, 400)].astype(np.float32)
    # estimate a subset of the GT (d = 0), with duplicates on both sides, plus jittered points
    est = np.concatenate([gt[::3], gt[::3], gt[5:9], np.c_[base[:100] + rng.normal(0, 0.3, (100, 3)).astype(np.float32), _lab(rng, 100)]])
    sets["subset_dups"] = (np.concatenate([gt, gt[:20]]), est.astype(np.float32), None, 0.2)
    # pairs at the stopping bound of shell s and one ulp either side, in a sparse GT box (corners at +-10 m)
    box = np.array([[sx, sy, sz, 40.0] for sx in (-10, 10) for sy in (-10, 10) for sz in (-10, 10)], np.float32)
    g, _ = ovl_grids(box, 0.2)
    leaf, marg = float(g["leaf"]), g["marg"]
    q, p = [], []
    for s in range(SHELL_MAX + 1):
        for u in (-1, 0, 1):
            for axis in range(3):
                y0 = F(-8.0 + 3.0 * (3 * s + u + 1) / 2.0)
                qq = np.array([0.03, y0, 1.5 * axis - 3.0], np.float32)           # a query inside its cell
                cell = int(np.floor(F(qq[axis]) * g["inv"])) - int(g["min_b"][axis])
                lb = (cell + s + 1 + g["min_b"][axis]) * leaf - marg - float(qq[axis])
                x = F(float(qq[axis]) + lb)
                for _ in range(abs(u)):
                    x = np.nextafter(x, F(np.sign(u) * 1e9))
                pp = qq.copy()
                pp[axis] = x
                q.append(qq)
                p.append(pp)
    q, p = np.array(q, np.float32), np.array(p, np.float32)
    sets["stop_bound_ulps"] = (np.concatenate([box, np.c_[p, _lab(rng, len(p))]]).astype(np.float32), np.c_[q, _lab(rng, len(q))].astype(np.float32), None, 0.2)
    # points within ulps of cell faces, GT on the far side of the face
    faces = (np.arange(-20, 20) * F(0.2)).astype(np.float32)
    e, t = [], []
    for f in faces:
        for u in (-2, -1, 0, 1, 2):
            x = f
            for _ in range(abs(u)):
                x = np.nextafter(x, F(np.sign(u) * 1e9))
            y, z = rng.uniform(-1, 1, 2).astype(np.float32)
            e.append([x, y, z, 40.0])
            t.append([np.nextafter(x, F(-1e9)) - F(0.35) * rng.random(), y, z, 252.0])
            t.append([x + F(0.45), y + F(0.1), z, 40.0])
    sets["cell_faces"] = (np.array(t, np.float32), np.array(e, np.float32), None, 0.2)
    # a GT over +-10 km (the fine cell doubles: 0.2 m cells would need more than 2^32 keys), queries near its clusters
    corners = np.array([[sx, sy, sz] for sx in (-1e4, 1e4) for sy in (-1e4, 1e4) for sz in (-50.0, 50.0)])
    ce = np.concatenate([c + rng.uniform(-0.5, 0.5, (30, 3)) for c in corners]).astype(np.float32)
    cq = (ce + rng.normal(0, 0.4, ce.shape)).astype(np.float32)
    sets["10km_extent"] = (np.c_[ce, _lab(rng, len(ce))], np.c_[cq, _lab(rng, len(cq))], None, 0.2)
    # estimate points 1 km and 10 km out in every octant of a small GT, with a keep mask
    oct_ = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], np.float64)
    fe = np.concatenate([base[:50] + (r * oct_[k] / np.sqrt(3)).astype(np.float32) for r in (1e3, 1e4) for k in range(8)])
    near = base[:40] + rng.normal(0, 0.5, (40, 3)).astype(np.float32)
    fe = np.concatenate([fe, near]).astype(np.float32)
    sets["far_octants"] = (gt, np.c_[fe, _lab(rng, len(fe))].astype(np.float32), rng.random(len(fe)) < 0.8, 0.2)
    # a single GT point
    sets["single_gt"] = (gt[:1], est, None, 0.2)
    sets["stop_bound_rounding"] = stop_bound_rounding_set()
    sets["far_box_order"] = far_box_order_set()
    return sets


def stop_bound_rounding_set():
    """The stopping bound at its margin.  At |x| ~ 800 m, 0.2 m cells, floats exist that the float cell assignment puts in cell N
    although they lie up to 3.6e-5 m below the face N leaf; only marg (4.9e-4 m here) keeps them inside the bound.  Per case, a query
    q sits near the top of cell N - s - 1 (so after shell s the nearest unseen face is x = N leaf), its nearest GT point p is such a
    float in cell N, and a competitor c inside the searched block lies at a distance between |p - q| and N leaf - q.x (the bound
    without marg): a stop rule without marg, or looser, stops at c; the true answer is p, found in shell s + 1."""
    box = np.array([[-1030, -2, -2, 40], [1030, 2, 2, 40]], np.float32)
    g, _ = ovl_grids(box, 0.2)
    leaf, inv = float(g["leaf"]), g["inv"]
    gt, q = [box], []
    for k, N in enumerate(range(4003, 5100, 40)):
        face = N * leaf
        x = F(face)
        while not (int(np.floor(x * inv)) == N and float(x) < face):
            x = np.nextafter(x, F(-1e9))
            assert int(np.floor(x * inv)) == N, "no float below the face in cell N"
        s = 1 + k % 3
        xq = F((N - s) * leaf - 0.01)
        d_p, d_free = float(x) - float(xq), face - float(xq)
        t = 0.5 * (d_p + d_free)
        yc = F(0.1 + t / np.sqrt(2.0))
        zc = F(0.1 + np.sqrt(t * t - (float(yc) - 0.1) ** 2))
        d_c = np.sqrt((float(yc) - float(F(0.1))) ** 2 + (float(zc) - float(F(0.1))) ** 2)
        assert d_p < d_c < d_free * (1 - 2.0 ** -30), (d_p, d_c, d_free)
        gt.append(np.array([[x, 0.1, 0.1, 40.0], [xq, yc, zc, 252.0]], np.float32))
        q.append([xq, 0.1, 0.1, 40.0])
    return np.concatenate(gt).astype(np.float32), np.array(q, np.float32), None, 0.2


def far_box_order_set():
    """The far path's box pruning at its edge.  In a GT spanning 100 m in x and y (coarse blocks of 3.2 m), a query 1 km out in -x sees box A
    first: its points (0, -1.9) and (1.1, 1.1) span the query's y, so the box's gap is 1000 m, but its nearest point is 1000.0018 m
    away.  Box B, one point in the next block in y, lies 2e-7 m nearer than that (a relative gap of 2e-10): pruning B by any factor
    above that returns A's point instead of B's."""
    a2 = np.sqrt(1000.0 ** 2 + float(F(-1.9)) ** 2)
    bx = F(np.sqrt((a2 - 2e-7) ** 2 - float(F(-2.1)) ** 2) - 1000.0)
    db = np.sqrt((1000.0 + float(bx)) ** 2 + float(F(-2.1)) ** 2)
    assert 1000.0 < db < a2, (db, a2)
    corners = [[sx, sy, sz, 40.0] for sx in (20.0, 100.0) for sy in (-50.0, 50.0) for sz in (-1.0, 1.0)]
    gt = np.array(corners + [[0.0, -1.9, 0.0, 40.0], [1.1, 1.1, 0.0, 40.0], [bx, -2.1, 0.0, 252.0]], np.float32)
    q = np.array([[-1000.0, 0.0, 0.0, 40.0], [-1000.0, -0.5, 0.0, 40.0]], np.float32)
    return gt, q, None, 0.2


OSETS = overlap_sets()


@pytest.mark.parametrize("name", sorted(OSETS))
def test_model_equals_brute_force(name):
    gt, est, keep, vs = OSETS[name]
    d, far = model_overlap(gt, est, keep, vs)
    want = brute_overlap(gt, est, keep)
    assert np.array_equal(d, want, equal_nan=True)
    if name in ("far_octants", "single_gt"):
        assert far.any()
    if name == "subset_dups":
        assert (d == 0).sum() >= len(est) - 100


def test_sets_bite():
    gt, est, keep, vs = OSETS["far_octants"]
    _, far = model_overlap(gt, est, keep, vs)
    assert far[:800][keep[:800]].all()                       # every 1 km / 10 km point takes the far path
    g, _ = ovl_grids(OSETS["10km_extent"][0], 0.2)
    assert float(g["leaf"]) > 0.3
    # the stopping-bound pairs: each query's nearest point is its planted one, at the bound of shell s (to float rounding)
    gt, est, _, vs = OSETS["stop_bound_ulps"]
    d, far = model_overlap(gt, est, None, vs)
    assert np.all(d < 1.0) and not far[:3 * 3 * (SHELL_MAX - 1)].any()


def test_empty_gt_and_selection():
    gt, est, _, _ = OSETS["subset_dups"]
    d, _ = model_overlap(gt[:0], est)
    assert np.all(np.isinf(d))
    d, _ = model_overlap(gt, est, keep=np.zeros(len(est), bool))
    assert np.all(np.isnan(d))


# ---- the percentiles from two order statistics ---------------------------------------------------------------------------------
def _from_sorted(d, voxelsize=0.2):
    s = np.sort(d)
    n = len(d)
    vals = [s[r] for r in E.overlap_ranks(n)]
    below = tuple(int((d < t).sum()) for t in (0.5 * voxelsize, voxelsize, 2 * voxelsize))
    return E.overlap_from_ranks(n, vals, s[-1], below, voxelsize)


def _numpy(d, voxelsize=0.2):
    half, one = 0.5 * voxelsize, voxelsize
    return {"median": float(np.median(d)), "p90": float(np.percentile(d, 90)), "p99": float(np.percentile(d, 99)), "max": float(d.max()),
            "frac_half": float(np.mean(d < half) * 100), "frac_one": float(np.mean(d < one) * 100), "frac_two": float(np.mean(d < 2 * one) * 100)}


# besides 1..50: n where the p99 virtual index (n - 1) * 0.99 is an integer in float64 (no interpolation)
INTEGER_P99 = [n for n in range(51, 1002, 50) if float((n - 1) * np.float64(0.99)).is_integer()]


def test_integer_p99_sizes_exist():
    assert INTEGER_P99[:3] == [101, 201, 301]          # the percentile path without interpolation (gamma = 0) is exercised


@pytest.mark.parametrize("n", list(range(1, 51)) + INTEGER_P99[:4] + [1001, 10001, 100001])
def test_percentiles_from_order_statistics_equal_numpy(n):
    rng = np.random.default_rng(n)
    for d in (rng.exponential(0.1, n), np.round(rng.uniform(0, 0.5, n), 2), rng.uniform(0, 1e3, n) ** 2):
        assert _from_sorted(d) == _numpy(d)


# ---- the runner's stdout, byte for byte ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden_pairs(oracle_mod):
    gt, est = seed41_pass(oracle_mod)
    return {"seed41": (gt, est), "seed41_jittered": (gt, jittered_estimate(est))}


def write_pair(d, gt, est):
    E.write_pcd_ascii(os.path.join(d, "gt.pcd"), gt)
    E.write_pcd_ascii(os.path.join(d, "est.pcd"), est)


@pytest.mark.parametrize("name", sorted(GOLDEN_STDOUT))
def test_format_report_reproduces_the_runner(tmp_path, golden_pairs, name):
    write_pair(tmp_path, *golden_pairs[name])
    gt, est = E.read_pcd_ascii(str(tmp_path / "gt.pcd")), E.read_pcd_ascii(str(tmp_path / "est.pcd"))
    r = E.report(gt, est)
    assert E.format_report(r, 0.2, "gt.pcd", "est.pcd") == open(GOLDEN_STDOUT[name]).read()


@pytest.mark.parametrize("name", sorted(GOLDEN_STDOUT))
def test_host_cli_reproduces_the_runner(tmp_path, golden_pairs, name):
    write_pair(tmp_path, *golden_pairs[name])
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    out = subprocess.run([sys.executable, "-m", "erasor_b200.analysis", "--gt", "gt.pcd", "--est", "est.pcd", "--host"], cwd=tmp_path,
                         env=env, check=True, capture_output=True, text=True).stdout
    assert out == open(GOLDEN_STDOUT[name]).read()
