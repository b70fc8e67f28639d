"""CPU model (numpy float32, no FMA -- like the kernels' _rn intrinsics) of the grid-pruned exact 1-NN that labels voxel centroids
(erasor_b200/csrc/device_common.cuh voxel_grid_nn + cell_gap, used by k4b_voxelize and k_node_fused): own cell first, then the 26 around it --
each skipped when 0.999 * (conservative gap)^2 > best -- and further shells while something unseen could still be closer.
The claim is EXACTNESS: the same (distance, lowest index) as comparing against every point.  The pruning is where that could
break (a float cell assignment puts the faces a few ulp off k * leaf), so the model is driven with adversarial layouts: points
and queries within ulps of cell faces, coordinates up to kilometres, leaves down to 5 cm, exact ties across cells."""
import numpy as np
import pytest

f32 = np.float32


def cell_gap(x, cell, off, leaf, slack):
    if off == 0:
        return f32(0.0)
    g = (f32(cell) * leaf - x) if off > 0 else (x - f32(cell + 1) * leaf)
    return max(f32(g - slack), f32(0.0))


def pruned_nn(c, pts, cells, leaf, inv, min_b, div):
    """cells: dict cell -> ascending point indices.  Returns (best_d, best_i, cells_searched)."""
    ci = int(f32(np.floor(f32(c[0] * inv))) - f32(min_b[0]))
    cj = int(f32(np.floor(f32(c[1] * inv))) - f32(min_b[1]))
    ck = int(f32(np.floor(f32(c[2] * inv))) - f32(min_b[2]))
    slack = f32(f32(1.0e-3) * leaf + f32(4.0e-6) * max(abs(c[0]), abs(c[1]), abs(c[2])))
    best_d, best_i, searched = f32(np.inf), -1, 0
    rad = 0
    while True:
        for a in range(-rad, rad + 1):
            ii = ci + a
            if ii < 0 or ii >= div[0]:
                continue
            for b in range(-rad, rad + 1):
                jj = cj + b
                if jj < 0 or jj >= div[1]:
                    continue
                for cc in range(-rad, rad + 1):
                    if max(abs(a), abs(b), abs(cc)) != rad:
                        continue
                    kk = ck + cc
                    if kk < 0 or kk >= div[2]:
                        continue
                    if rad > 0:
                        gx = cell_gap(c[0], ii + min_b[0], a, leaf, slack)
                        gy = cell_gap(c[1], jj + min_b[1], b, leaf, slack)
                        gz = cell_gap(c[2], kk + min_b[2], cc, leaf, slack)
                        if f32(f32(0.999) * f32(f32(gx * gx + gy * gy) + gz * gz)) > best_d:
                            continue
                    members = cells.get((ii, jj, kk))
                    if members is None:
                        continue
                    searched += 1
                    for i in members:
                        dx, dy, dz = f32(c[0] - pts[i, 0]), f32(c[1] - pts[i, 1]), f32(c[2] - pts[i, 2])
                        d = f32(f32(dx * dx + dy * dy) + dz * dz)
                        if d < best_d or (d == best_d and i < best_i):
                            best_d, best_i = d, i
        reach = f32(f32(f32(rad) * leaf) * f32(0.9999))
        if best_i >= 0 and best_d < f32(reach * reach):
            break
        rad += 1
        if rad > 64 and best_i >= 0:
            break
        if rad > 4096:
            break
    return best_d, best_i, searched


def brute_nn(c, pts):
    dx, dy, dz = c[0] - pts[:, 0], c[1] - pts[:, 1], c[2] - pts[:, 2]
    d = (dx * dx + dy * dy) + dz * dz
    i = int(np.argmin(d))                      # the first minimum = the lowest index among ties
    return d[i], i


def build_grid(pts, leaf):
    inv = f32(1.0) / leaf
    mn, mx = pts.min(axis=0), pts.max(axis=0)
    min_b = np.floor(mn * inv).astype(np.int64)
    max_b = np.floor(mx * inv).astype(np.int64)
    div = max_b - min_b + 1
    ijk = (np.floor(pts * inv) - min_b.astype(f32)).astype(np.int64)
    cells = {}
    for i, key in enumerate(map(tuple, ijk)):
        cells.setdefault(key, []).append(i)
    return inv, min_b, div, cells


@pytest.mark.parametrize("seed,leaf,centre,span", [(1, 0.2, 0.0, 3.0), (2, 0.2, 3900.0, 3.0), (3, 0.05, -780.0, 1.0), (4, 0.4, 25.0, 8.0), (5, 0.2, -0.1, 0.6)])
def test_pruned_grid_search_is_exact(seed, leaf, centre, span):
    rng = np.random.default_rng(seed)
    leaf = f32(leaf)
    n = 1500
    pts = (centre + rng.uniform(-span, span, size=(n, 3))).astype(f32)
    # adversarial layers: a third of the points snapped to within a few ulp of cell faces, exact duplicates, and points mirrored
    # across a face at equal distance from it (ties across cells)
    snap = rng.integers(0, n, n // 3)
    ax = rng.integers(0, 3, len(snap))
    face = (np.round(pts[snap, ax] / leaf) * leaf).astype(f32)
    ulps = rng.integers(-3, 4, len(snap))
    for k, a, fv, u in zip(snap, ax, face, ulps):
        v = fv
        for _ in range(abs(int(u))):
            v = np.nextafter(v, f32(np.inf) if u > 0 else f32(-np.inf), dtype=f32)
        pts[k, a] = v
    pts[n - 60:n - 30] = pts[:30]
    m = rng.integers(0, n, 30)
    mirror = pts[m].copy()
    fx = (np.round(mirror[:, 0] / leaf) * leaf).astype(f32)
    mirror[:, 0] = (fx + (fx - mirror[:, 0])).astype(f32)
    pts[n - 30:] = mirror
    inv, min_b, div, cells = build_grid(pts, leaf)
    # queries: voxel centroids (what the kernels label), points themselves, and arbitrary positions near faces
    queries = []
    for key, members in list(cells.items())[:250]:
        acc = np.zeros(3, dtype=f32)
        for i in members:
            acc = (acc + pts[i]).astype(f32)
        queries.append((acc / f32(len(members))).astype(f32))
    queries += [pts[i] for i in rng.integers(0, n, 100)]
    for _ in range(150):
        q = (centre + rng.uniform(-span, span, size=3)).astype(f32)
        a = rng.integers(0, 3)
        q[a] = f32(np.round(q[a] / leaf) * leaf)
        if rng.random() < 0.5:
            q[a] = np.nextafter(q[a], f32(np.inf) if rng.random() < 0.5 else f32(-np.inf), dtype=f32)
        queries.append(q)
    searched_total = 0
    for q in queries:
        if np.any(q < pts.min(axis=0)) or np.any(q > pts.max(axis=0)):
            continue                            # the kernels only ever label centroids, which lie inside the cloud's box
        bd, bi = brute_nn(q, pts)
        pd, pi, searched = pruned_nn(q, pts, cells, leaf, inv, min_b, div)
        searched_total += searched
        assert (pd, pi) == (bd, bi), f"query {q}: pruned ({pd}, {pi}) != brute force ({bd}, {bi})"
    assert searched_total < 12 * len(queries), "the pruning must actually prune (27 cells per query without it)"


def test_pruned_grid_search_is_exact_on_sparse_and_skewed_clouds():
    """Sparse clouds (most cells empty: the search has to go to shells 2, 3, ...), flat and line-like clouds, and queries whose
    nearest point sits in a diagonal neighbour -- 40 random configurations."""
    rng = np.random.default_rng(2024)
    worst_shell = 0
    for trial in range(40):
        leaf = f32(rng.choice([0.05, 0.1, 0.2, 0.25, 0.4]))
        centre = float(rng.choice([0.0, 17.3, -250.0, 1800.0, -3999.0]))
        n = int(rng.integers(5, 400))
        shape = np.array([1.0, 1.0, 1.0]) if trial % 3 == 0 else (np.array([1.0, 1.0, 0.02]) if trial % 3 == 1 else np.array([1.0, 0.03, 0.03]))
        span = float(leaf) * float(rng.choice([2.0, 6.0, 25.0]))
        pts = (centre + rng.uniform(-span, span, size=(n, 3)) * shape).astype(f32)
        inv, min_b, div, cells = build_grid(pts, leaf)
        lo, hi = pts.min(axis=0), pts.max(axis=0)
        for _ in range(60):
            q = (lo + rng.random(3).astype(f32) * (hi - lo)).astype(f32)
            q = np.minimum(np.maximum(q, lo), hi)
            bd, bi = brute_nn(q, pts)
            pd, pi, _ = pruned_nn(q, pts, cells, leaf, inv, min_b, div)
            assert (pd, pi) == (bd, bi), f"trial {trial} leaf {leaf} centre {centre}: query {q}: ({pd}, {pi}) != ({bd}, {bi})"
            worst_shell = max(worst_shell, int(np.ceil(np.sqrt(float(bd)) / float(leaf))))
    assert worst_shell >= 3, "the configurations must reach beyond the first shell"
