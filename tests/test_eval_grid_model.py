"""CPU suite: a numpy model of the device PR/RR evaluator (erasor_b200/csrc/eval_kernels.cu, DESIGN.md section 11), step by
step as the kernels do it -- float32 cell assignment, the leaf-doubling rule, the 9 contiguous key ranges per GT point with the
optional conservative gap skip, the no-FMA double distance, lowest-index ties and the tie counter -- held to an all-pairs float64
brute force on adversarial sets, and to erasor_b200.evaluate (sklearn) and through it the reference script's golden table.
tests/test_gpu_evaluate.py holds the device to this model."""
import json

import numpy as np
import pytest

from erasor_b200 import evaluate as E

NO_MATCH = 0xFFFFFFFF
F = np.float32


def thr_of(voxelsize: float) -> float:
    return voxelsize * 1.7320508075688772 / 2          # == voxelsize * np.sqrt(3) / 2, as evaluate.py computes it


def is_dynamic(v) -> np.ndarray:
    """(uint32_t)(int64_t)v & 0xFFFF in 252..259 for finite |v| < 2^63; NaN, +-inf and larger values are class 0."""
    v = np.asarray(v, dtype=np.float32).reshape(-1)
    ok = np.isfinite(v) & (np.abs(v) < F(2.0 ** 63))
    s = np.zeros(len(v), dtype=np.uint32)
    s[ok] = v[ok].astype(np.int64).astype(np.uint32) & 0xFFFF
    return ok & (s >= 252) & (s <= 259)


def grid_setup(mn, mx, voxelsize: float):
    """eval_grid_setup: cell edge voxelsize, doubled until (a) the cell count fits a 32-bit key below 0xFFFFFFFF, (b) every
    converted coordinate scales below 2^22 cells, (c) thr (1 + 1e-12) + R 2^-21 < leaf, R = (max |cell| + 3) leaf.  (c) is the
    rounding margin: fl(x * fl(1 / leaf)) is within |x| / leaf * 2^-22.99 of x / leaf, so two points closer than thr along an
    axis, both within R of the origin, land at most one cell apart."""
    thr = thr_of(voxelsize)
    leaf = F(voxelsize)
    for _ in range(300):
        inv = F(1.0) / leaf
        a, b = np.floor(mn * inv), np.floor(mx * inv)
        ok = bool(np.all(np.abs(a) < F(2 ** 22)) and np.all(np.abs(b) < F(2 ** 22)))
        if ok:
            min_b = a.astype(np.int64)
            div = b.astype(np.int64) - min_b + 1
            cells = int(div[0]) * int(div[1]) * int(div[2])
            cmax = max(max(abs(float(a[k])), abs(float(b[k])) + 1.0) for k in range(3))
            R = (cmax + 3.0) * float(leaf)
            if cells <= 0xFFFFFFFE and thr * (1.0 + 1e-12) + R / 2 ** 21 < float(leaf):
                return dict(leaf=leaf, inv=inv, min_b=min_b, div=div, cells=cells, thr=thr, thr2f=F(thr * thr),
                            lo=(min_b - 2).astype(np.float32), hi=(min_b + div + 2).astype(np.float32))
        leaf = leaf * F(2.0)
    raise AssertionError("no grid")


def voxel_cell(x, inv, min_b):
    """device_common.cuh voxel_cell: (int)(floorf(x * inv) - (float)min_b), all in float32"""
    with np.errstate(invalid="ignore"):            # dropped estimate points may be non-finite; their cells are never used
        return (np.floor(np.asarray(x, dtype=np.float32) * inv) - np.float32(min_b)).astype(np.int64)


def cell_gap(x, cell, off: int, leaf, slack):
    """device_common.cuh cell_gap, float32"""
    if off == 0:
        return np.zeros(len(x), dtype=np.float32)
    c = np.asarray(cell, dtype=np.float32)
    g = c * leaf - x if off > 0 else x - (c + F(1.0)) * leaf
    return np.maximum(g - slack, F(0.0))


def sq_dist(q, p):
    """sklearn's squared distance: (dx*dx + dy*dy) + dz*dz in float64 from float32 coordinates (numpy never contracts)"""
    d = q[..., :3].astype(np.float64) - p[..., :3].astype(np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _counts(gt_dyn, inl, best_dyn, amb):
    return dict(gt_static=int((~gt_dyn).sum()), gt_dynamic=int(gt_dyn.sum()),
                preserved_static=int((inl & ~gt_dyn & ~best_dyn).sum()), preserved_dynamic=int((inl & gt_dyn & best_dyn).sum()),
                inliers=int(inl.sum()), ambiguous_ties=int((inl & amb).sum()))


def model_eval(gt, est, keep=None, voxelsize=0.2, gap_skip=True, return_grid=False):
    """What the kernels compute: (the six counts, match per GT point).  gap_skip: drop a range whose conservative y / z gap is
    at least thr.  The kernel also drops a range whose gap is strictly beyond its best distance so far; such a range holds
    neither the nearest point nor a tie, by the same argument, so the result is the one computed here with or without skips."""
    gt = np.ascontiguousarray(gt, dtype=np.float32).reshape(-1, 4)
    est = np.ascontiguousarray(est, dtype=np.float32).reshape(-1, 4)
    sel = np.ones(len(est), bool) if keep is None else np.asarray(keep).astype(bool)
    if not np.all(np.isfinite(est[sel, :3])) or not np.all(np.isfinite(gt[:, :3])):
        raise ValueError("non-finite coordinate")
    gt_dyn, est_dyn = is_dynamic(gt[:, 3]), is_dynamic(est[:, 3])
    n = len(gt)
    match = np.full(n, NO_MATCH, dtype=np.uint32)
    if n == 0 or not sel.any():
        z = np.zeros(n, bool)
        out = (_counts(gt_dyn, z, z, z), match)
        return out + (None,) if return_grid else out
    pts = est[sel, :3] + F(0.0)
    g = grid_setup(pts.min(axis=0), pts.max(axis=0), voxelsize)
    # keys (uint32 arithmetic; dropped points 0xFFFFFFFF), stable sort, run heads
    cell = np.stack([voxel_cell(est[:, k], g["inv"], g["min_b"][k]) for k in range(3)], axis=1)
    key = np.full(len(est), 0xFFFFFFFF, dtype=np.int64)
    key[sel] = cell[sel, 0] + cell[sel, 1] * g["div"][0] + cell[sel, 2] * (g["div"][0] * g["div"][1])
    assert np.all(cell[sel] >= 0) and np.all(cell[sel] < g["div"])
    order = np.argsort(key, kind="stable")[: int(sel.sum())]
    skey = key[order]
    heads = np.flatnonzero(np.r_[True, skey[1:] != skey[:-1]])
    vox_key, vox_start = skey[heads], np.r_[heads, len(skey)]
    # query: guard window, then the 9 ranges (i-1..i+1, j+b, k+c)
    a = gt[:, :3] * g["inv"]
    inside = np.all((a >= g["lo"]) & (a < g["hi"]), axis=1)
    qi = np.flatnonzero(inside)
    q = gt[qi]
    c = np.stack([voxel_cell(q[:, k], g["inv"], g["min_b"][k]) for k in range(3)], axis=1)
    i0, i1 = np.maximum(c[:, 0] - 1, 0), np.minimum(c[:, 0] + 1, g["div"][0] - 1)
    slack = F(1e-3) * g["leaf"] + F(4e-6) * np.maximum(np.abs(q[:, 1]), np.abs(q[:, 2]))
    owner, lo_pos, hi_pos = [], [], []
    for b in (-1, 0, 1):
        jj = c[:, 1] + b
        gy = cell_gap(q[:, 1], jj + g["min_b"][1], b, g["leaf"], slack)
        for cc in (-1, 0, 1):
            kk = c[:, 2] + cc
            gz = cell_gap(q[:, 2], kk + g["min_b"][2], cc, g["leaf"], slack)
            ok = (i0 <= i1) & (jj >= 0) & (jj < g["div"][1]) & (kk >= 0) & (kk < g["div"][2])
            if gap_skip:
                ok &= ~(F(0.999) * (gy * gy + gz * gz) >= g["thr2f"])
            k_lo = i0 + jj * g["div"][0] + kk * (g["div"][0] * g["div"][1])
            k_hi = k_lo + (i1 - i0)
            v0 = np.searchsorted(vox_key, k_lo, side="left")
            v1 = np.searchsorted(vox_key, k_hi, side="right")
            ok &= v1 > v0
            owner.append(qi[ok]); lo_pos.append(vox_start[v0[ok]]); hi_pos.append(vox_start[v1[ok]])
    owner, lo_pos, hi_pos = np.concatenate(owner), np.concatenate(lo_pos), np.concatenate(hi_pos)
    lens = hi_pos - lo_pos
    pg = np.repeat(owner, lens)
    pos = np.repeat(lo_pos - np.r_[0, np.cumsum(lens)[:-1]], lens) + np.arange(int(lens.sum()))
    pe = order[pos]
    d2 = sq_dist(gt[pg], est[pe])
    best = np.full(n, np.inf)
    np.minimum.at(best, pg, d2)
    eq = d2 == best[pg]
    best_i = np.full(n, np.iinfo(np.int64).max, dtype=np.int64)
    np.minimum.at(best_i, pg[eq], pe[eq])
    tie_d = np.zeros(n, bool); tie_s = np.zeros(n, bool)
    tie_d[pg[eq & est_dyn[pe]]] = True
    tie_s[pg[eq & ~est_dyn[pe]]] = True
    inl = np.isfinite(best) & (np.sqrt(best) < g["thr"])
    best_dyn = np.zeros(n, bool)
    best_dyn[inl] = est_dyn[best_i[inl]]
    match[inl] = best_i[inl]
    out = (_counts(gt_dyn, inl, best_dyn, tie_d & tie_s), match)
    return out + (g,) if return_grid else out


def brute_eval(gt, est, keep=None, voxelsize=0.2):
    """All pairs, the same distance formula, lowest index among the equally nearest."""
    gt = np.asarray(gt, dtype=np.float32).reshape(-1, 4)
    est = np.asarray(est, dtype=np.float32).reshape(-1, 4)
    sel = np.ones(len(est), bool) if keep is None else np.asarray(keep).astype(bool)
    gt_dyn, est_dyn = is_dynamic(gt[:, 3]), is_dynamic(est[:, 3])
    n = len(gt)
    match = np.full(n, NO_MATCH, dtype=np.uint32)
    idx = np.flatnonzero(sel)
    if n == 0 or len(idx) == 0:
        z = np.zeros(n, bool)
        return _counts(gt_dyn, z, z, z), match
    d2 = sq_dist(gt[:, None, :], est[None, idx, :])
    best = d2.min(axis=1)
    eq = d2 == best[:, None]
    first = idx[np.argmax(eq, axis=1)]
    inl = np.sqrt(best) < thr_of(voxelsize)
    amb = (eq & est_dyn[idx][None, :]).any(axis=1) & (eq & ~est_dyn[idx][None, :]).any(axis=1)
    match[inl] = first[inl]
    return _counts(gt_dyn, inl, est_dyn[first] & inl, amb), match


def exact_thr_voxelsize():
    """A voxelsize near 0.2 whose thr = voxelsize * sqrt(3) / 2 is a float32 value, so a pair can sit at exactly thr."""
    for t in np.nextafter(F(0.17320508), F(1.0)) + np.arange(200, dtype=np.float32) * np.spacing(F(0.17)):
        vs = float(t) * 2.0 / 1.7320508075688772
        for k in range(-4, 5):
            v = vs + k * np.spacing(vs)
            if thr_of(v) == float(F(thr_of(v))):
                return v, F(thr_of(v))
    raise AssertionError("no voxelsize with a float32 thr")


def adversarial_sets():
    """name -> (gt, est, keep, voxelsize)"""
    rng = np.random.default_rng(17)
    sets = {}
    # pairs at exactly thr and one / two ulp either side, along each axis and both directions
    vs, t = exact_thr_voxelsize()
    gt, est = [], []
    for axis in range(3):
        for sgn in (1, -1):
            for k, d in enumerate([np.nextafter(np.nextafter(t, F(0)), F(0)), np.nextafter(t, F(0)), t, np.nextafter(t, F(1)),
                                   np.nextafter(np.nextafter(t, F(1)), F(1))]):
                base = np.zeros(3, dtype=np.float32)                # 0 along `axis`, so the offset is exact
                base[(axis + 1) % 3] = 2.0 * k + 12.0 * (sgn > 0)
                base[(axis + 2) % 3] = 30.0 * axis
                gt.append(np.r_[base, F(252.0 if k % 2 else 40.0)])
                p = base.copy(); p[axis] = p[axis] + F(sgn) * d
                assert abs(float(p[axis]) - float(base[axis])) == float(d)
                est.append(np.r_[p, F(252.0 if k < 3 else 50.0)])
    sets["thr_ulps"] = (np.array(gt, np.float32), np.array(est, np.float32), None, vs)
    # points within ulps of cell faces at 0.2 m, GT on the other side of the face
    faces = (np.arange(-40, 40) * F(0.2)).astype(np.float32)
    e, q = [], []
    for f in faces:
        for u in (-2, -1, 0, 1, 2):
            x = f
            for _ in range(abs(u)):
                x = np.nextafter(x, F(np.sign(u) * 1e9))
            y, z = rng.uniform(-1, 1, 2).astype(np.float32)
            e.append([x, y, z, 252.0 if u % 2 else 30.0])
            q.append([np.nextafter(x, F(-1e9)) - F(0.1) * rng.random(), y + F(0.05), np.nextafter(z, F(1e9)), 40.0 if u else 253.0])
            q.append([x + F(0.17), y, z, 258.0])
    sets["cell_faces"] = (np.array(q, np.float32), np.array(e, np.float32), None, 0.2)
    # +-10 km: clusters at the corners of a 20 km box (also forces the leaf to double: the cell count would exceed 2^32)
    corners = np.array([[sx, sy, sz] for sx in (-1e4, 1e4) for sy in (-1e4, 1e4) for sz in (-50.0, 50.0)])
    ce = np.concatenate([c + rng.uniform(-0.5, 0.5, (40, 3)) for c in corners]).astype(np.float32)
    cq = np.concatenate([ce[:, :3] + rng.normal(0, 0.08, ce.shape).astype(np.float32), ce[:, :3] + F(0.15)]).astype(np.float32)
    lab_e = rng.choice([40.0, 252.0, 256.0, 51.0], len(ce)).astype(np.float32)
    lab_q = rng.choice([40.0, 252.0, 259.0], len(cq)).astype(np.float32)
    sets["10km"] = (np.c_[cq, lab_q], np.c_[ce, lab_e], None, 0.2)
    # a far cloud (3e5 m): the rounding margin alone doubles the leaf
    fe = (np.array([3.0e5, -2.0e5, 10.0]) + rng.uniform(-2, 2, (300, 3))).astype(np.float32)
    fq = (fe + rng.normal(0, 0.1, fe.shape)).astype(np.float32)
    sets["far"] = (np.c_[fq, rng.choice([40.0, 252.0], 300)], np.c_[fe, rng.choice([40.0, 252.0], 300)], None, 0.2)
    # duplicates and exact dynamic / static ties: the same point twice with both classes, and mirrored pairs
    base = rng.uniform(-5, 5, (100, 3)).astype(np.float32)
    d = np.array([0.05, 0.0, 0.0], np.float32)
    te = np.concatenate([np.c_[base, np.full(100, 252.0)], np.c_[base, np.full(100, 40.0)],             # duplicates, both classes
                         np.c_[base + d + F(20), np.full(100, 40.0)], np.c_[base - d + F(20), np.full(100, 254.0)],   # mirrored
                         np.c_[base + F(40), np.full(100, 40.0)], np.c_[base + F(40), np.full(100, 41.0)]]).astype(np.float32)
    tq = np.concatenate([np.c_[base, np.full(100, 40.0)], np.c_[base + F(20), np.full(100, 252.0)], np.c_[base + F(40), np.full(100, 40.0)]])
    perm = rng.permutation(len(te))
    sets["ties"] = (tq.astype(np.float32), te[perm], None, 0.2)
    # label edge values, NaN intensities, and a keep mask
    labels = np.array([252, 259, 251, 260, -65284.0, 65788.0, 65536 + 255, -1.0, 2.0 ** 63, -2.0 ** 63, 1e20, np.nan, np.inf, -np.inf,
                       252.7, 259.9, 4294967548.0], np.float32)
    le = rng.uniform(-3, 3, (600, 3)).astype(np.float32)
    lq = (le + rng.normal(0, 0.12, le.shape)).astype(np.float32)
    sets["labels"] = (np.c_[lq, rng.choice(labels, 600)], np.c_[le, rng.choice(labels, 600)], rng.random(600) < 0.6, 0.2)
    return sets


ADV = adversarial_sets()


@pytest.mark.parametrize("name", sorted(ADV))
def test_model_equals_brute_force(name):
    gt, est, keep, vs = ADV[name]
    want, want_m = brute_eval(gt, est, keep, vs)
    for skip in (True, False):
        got, m = model_eval(gt, est, keep, vs, gap_skip=skip)
        assert got == want, (skip, got, want)
        assert np.array_equal(m, want_m)
    assert want["inliers"] > 0


def test_adversarial_sets_bite():
    """the sets exercise what they are named after"""
    gt, est, _, vs = ADV["thr_ulps"]
    c, m = brute_eval(gt, est, None, vs)
    assert c["inliers"] == 12                             # two ulp below and one ulp below thr, 6 directions; exactly thr is out
    assert brute_eval(*ADV["ties"][:2])[0]["ambiguous_ties"] > 100     # every duplicate pair, and the mirrored pairs float32 keeps exact
    *_, g = model_eval(*ADV["10km"][:2], return_grid=True)
    assert float(g["leaf"]) > 0.2 * 1.5                 # cells at 0.2 m would need > 2^32 keys
    *_, g = model_eval(*ADV["far"][:2], return_grid=True)
    assert float(g["leaf"]) > 0.2 * 1.5 and g["cells"] < 10 ** 6   # only the rounding margin forces this one
    *_, g = model_eval(*ADV["cell_faces"][:2], return_grid=True)
    assert float(g["leaf"]) == float(F(0.2))


def test_dynamic_label_edges():
    v = np.array([252, 259, 251, 260, -65284.0, 65788.0, 65536 + 255, -1.0, 252.7, 259.9, 4294967548.0, -2.0 ** 40 + 253], np.float32)
    with np.errstate(invalid="ignore"):
        assert np.array_equal(is_dynamic(v), np.isin(E.semantic(v), E.DYNAMIC_CLASSES))
    assert list(is_dynamic(np.array([-65284.0, 65788.0, np.nan, np.inf, -np.inf, 2.0 ** 63], np.float32))) == [True, True, False, False, False, False]


def test_empty_and_invalid():
    gt, est, _, _ = ADV["ties"]
    c, m = model_eval(gt, est[:0])
    assert c["inliers"] == 0 and c["gt_static"] + c["gt_dynamic"] == len(gt) and np.all(m == NO_MATCH)
    c, _ = model_eval(gt, est, keep=np.zeros(len(est), np.uint8))
    assert c["inliers"] == 0
    c, _ = model_eval(gt[:0], est)
    assert all(v == 0 for v in c.values())
    bad = gt.copy(); bad[3, 1] = np.nan
    with pytest.raises(ValueError):
        model_eval(bad, est)
    bad = est.copy(); bad[5, 2] = np.inf
    with pytest.raises(ValueError):
        model_eval(gt, bad)
    model_eval(gt, bad, keep=np.arange(len(bad)) != 5)     # a dropped point may be non-finite


def _rates_of(c):
    return E.rates(c["gt_static"], c["gt_dynamic"], c["preserved_static"], c["preserved_dynamic"])


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_model_equals_sklearn_on_random_clouds(seed):
    rng = np.random.default_rng(seed)
    n = 20000
    xyz = rng.uniform(-20, 20, (n, 3)) * np.array([1.0, 1.0, 0.1])
    lab = rng.choice([40.0, 50.0, 252.0, 255.0], n)
    gt = np.c_[xyz, lab].astype(np.float32)
    keep = rng.random(n) < 0.7
    est = gt[keep].copy()
    est[:, :3] += rng.normal(0, 0.1, (len(est), 3)).astype(np.float32)
    c, _ = model_eval(gt, est)
    assert c["ambiguous_ties"] == 0
    assert _rates_of(c) == E.evaluate(gt, est)
    # the keep-mask form scores the same estimate
    full = np.concatenate([est, gt[~keep]])
    c2, _ = model_eval(gt, full, keep=np.r_[np.ones(len(est), bool), np.zeros((~keep).sum(), bool)])
    assert c2 == c


def test_model_equals_sklearn_and_golden_table_on_seed41_pass(oracle_mod):
    from test_evaluate import REF_TABLE
    gt, est = seed41_pass(oracle_mod)
    c, _ = model_eval(gt, est)
    assert c["ambiguous_ties"] == 0
    assert _rates_of(c) == E.evaluate(gt, est)
    t = json.load(open(REF_TABLE))["table"]
    assert (c["gt_static"], c["gt_dynamic"], c["preserved_static"], c["preserved_dynamic"]) == (t["gt_S"], t["gt_D"], t["kept_S"], t["kept_D"])


def seed41_pass(oracle_mod):
    """tests/test_evaluate.py's run_pass fixture body: the clouds the golden analysis_runner table was made from"""
    from erasor_b200 import params as P
    from erasor_b200 import synth
    sc = synth.Scene(seed=41, length=40.0, n_nodes=17, n_dynamic=6)
    kw = dict(n_beams=24, n_az=480)
    nodes = list(range(17))
    m = sc.build_map(nodes, voxel=0.2, **kw)
    ep, up = P.preset("seq_05"), P.updater_preset("seq_05")
    up.removal_interval = 2
    o = oracle_mod.OracleUpdater(up, ep, m)
    for k in nodes:
        o.callback_node(k, sc.pose7(k), sc.scan(k, seed_offset=3, **kw))
    est = o.save_static_map(0.2)
    return m, est
