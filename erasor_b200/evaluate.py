"""Preservation Rate / Rejection Rate / F1 exactly as the reference's evaluator defines them
(reference scripts/analysis.py:124-155,189-191; identical in scripts/analysis_runner.py:74-105):
1-NN from every ground-truth point into the estimate, inlier if the distance is below voxelsize*sqrt(3)/2;
PR = GT-static inliers whose match is static / GT static; RR = (GT dynamic - GT-dynamic inliers whose match is
dynamic) / GT dynamic; dynamic = SemanticKITTI classes 252..259 carried numerically in `intensity`.
Host-side quality judge, not part of the path.  tests/test_evaluate.py checks it against the reference's own script
when /root/reference is present.  capi.Evaluator computes the same counts on the device (DESIGN.md section 11).
overlap / report / format_report restate the rest of the runner's output: its estimate -> GT distance report and est_S / est_D.
"""
from __future__ import annotations

import numpy as np

DYNAMIC_CLASSES = (252, 253, 254, 255, 256, 257, 258, 259)


def semantic(intensity: np.ndarray) -> np.ndarray:
    return intensity.astype(np.uint32) & 0xFFFF


def evaluate(gt_xyzi: np.ndarray, est_xyzi: np.ndarray, voxelsize: float = 0.2) -> dict:
    from sklearn.neighbors import NearestNeighbors
    gt_xyz, est_xyz = gt_xyzi[:, :3].astype(np.float32), est_xyzi[:, :3].astype(np.float32)
    gt_sem, est_sem = semantic(gt_xyzi[:, 3]), semantic(est_xyzi[:, 3])
    gt_dyn_all = np.isin(gt_sem, DYNAMIC_CLASSES)
    ns_gt, nd_gt = int((~gt_dyn_all).sum()), int(gt_dyn_all.sum())
    nn = NearestNeighbors(n_neighbors=1, algorithm="kd_tree").fit(est_xyz)
    dists, idx = nn.kneighbors(gt_xyz)
    dists, idx = dists.reshape(-1), idx.reshape(-1)
    is_in = dists < voxelsize * np.sqrt(3) / 2
    gt_is_dyn = np.isin(gt_sem[is_in], DYNAMIC_CLASSES)
    est_is_dyn = np.isin(est_sem[idx[is_in]], DYNAMIC_CLASSES)
    preserved_static = int(np.sum((~gt_is_dyn) & (~est_is_dyn)))
    preserved_dynamic = int(np.sum(gt_is_dyn & est_is_dyn))
    return rates(ns_gt, nd_gt, preserved_static, preserved_dynamic)


def rates(ns_gt: int, nd_gt: int, preserved_static: int, preserved_dynamic: int) -> dict:
    """The four counts -> evaluate()'s dict with PR, RR and F1.  The device evaluator (capi.Evaluator) calls this too, so equal
    counts give identical floats."""
    ns_gt, nd_gt, preserved_static, preserved_dynamic = int(ns_gt), int(nd_gt), int(preserved_static), int(preserved_dynamic)
    pr = preserved_static / ns_gt * 100.0 if ns_gt else 0.0
    rr = (nd_gt - preserved_dynamic) / nd_gt * 100.0 if nd_gt else 0.0
    f1 = 2 * (pr / 100) * (rr / 100) / ((pr / 100) + (rr / 100)) if (pr + rr) > 0 else 0.0
    return {"gt_static": ns_gt, "gt_dynamic": nd_gt, "preserved_static": preserved_static,
            "preserved_dynamic": preserved_dynamic, "PR": pr, "RR": rr, "F1": f1}


def est_counts(est_xyzi: np.ndarray) -> tuple:
    """(static, dynamic) points of the estimate: the runner's est_S / est_D (count_dyn_stat)"""
    nd = int(np.isin(semantic(est_xyzi[:, 3]), DYNAMIC_CLASSES).sum())
    return len(est_xyzi) - nd, nd


def overlap_distances(gt_xyzi: np.ndarray, est_xyzi: np.ndarray) -> np.ndarray:
    """The runner's overlap_report distances: sklearn's 1-NN from every estimate point into the GT, unbounded (float64)."""
    from sklearn.neighbors import NearestNeighbors
    nn = NearestNeighbors(n_neighbors=1, algorithm="kd_tree").fit(gt_xyzi[:, :3].astype(np.float32))
    d, _ = nn.kneighbors(est_xyzi[:, :3].astype(np.float32))
    return d.reshape(-1)


def overlap(gt_xyzi: np.ndarray, est_xyzi: np.ndarray, voxelsize: float = 0.2) -> dict:
    """The reference's overlap_report (scripts/analysis_runner.py:55-71) as a dict: median, p90, p99 and max of the estimate ->
    GT distances, and the percentage of them below 0.5, 1 and 2 voxels, each computed as the runner computes it."""
    d = overlap_distances(gt_xyzi, est_xyzi)
    half, one = 0.5 * voxelsize, voxelsize
    return {"median": float(np.median(d)), "p90": float(np.percentile(d, 90)), "p99": float(np.percentile(d, 99)), "max": float(d.max()),
            "frac_half": float(np.mean(d < half) * 100), "frac_one": float(np.mean(d < one) * 100), "frac_two": float(np.mean(d < 2 * one) * 100)}


# ---- the same numbers from order statistics (capi.Evaluator.overlap: the device returns the sorted distances at given ranks) ----
PERCENTILES = (90, 99)


def percentile_ranks(n: int, p) -> tuple:
    """np.percentile(d, p)'s method 'linear' on n values: (lower rank, upper rank, gamma) as numpy derives them -- virtual index
    (n - 1) * (p / 100) in float64, its floor and floor + 1; at or past the last index both ranks are n - 1 and gamma is measured
    from index -1, as numpy does."""
    q = np.true_divide(p, np.float64(100))
    v = np.asanyarray((n - 1) * q)
    prev = np.floor(v)
    if v >= n - 1:
        lo = hi = n - 1
        prev = np.float64(-1)
    else:
        lo = int(prev)
        hi = lo + 1
    gamma = np.asanyarray(v - prev, dtype=v.dtype)[()]
    return lo, hi, gamma


def lerp(a, b, t):
    """numpy's _lerp on float64 scalars"""
    a, b = np.float64(a), np.float64(b)
    with np.errstate(invalid="ignore"):             # inf - inf is NaN, as in numpy's percentile
        diff = b - a
        return b - diff * (1 - t) if t >= 0.5 else a + diff * t


def median_ranks(n: int) -> tuple:
    return ((n - 1) // 2,) if n % 2 else (n // 2 - 1, n // 2)


def overlap_ranks(n: int) -> list:
    """every rank overlap_from_ranks needs, in a fixed order"""
    r = list(median_ranks(n))
    for p in PERCENTILES:
        lo, hi, _ = percentile_ranks(n, p)
        r += [lo, hi]
    return r


def overlap_from_ranks(n: int, values, max_d: float, below: tuple, voxelsize: float = 0.2) -> dict:
    """overlap()'s dict from the sorted distances at overlap_ranks(n) (values, same order), the max and the three counts below
    0.5, 1 and 2 voxels: np.median is the mean of the middle value(s), np.percentile the lerp of its two neighbours, np.mean of
    the comparisons the count over n, each with numpy's float64 operations in numpy's order."""
    v = [np.float64(x) for x in values]
    m = median_ranks(n)
    med = v[0] if len(m) == 1 else (v[0] + v[1]) / np.float64(2)
    out = {"median": float(med)}
    k = len(m)
    for p in PERCENTILES:
        _, _, t = percentile_ranks(n, p)
        out[f"p{p}"] = float(lerp(v[k], v[k + 1], t))
        k += 2
    out["max"] = float(max_d)
    for name, c in zip(("frac_half", "frac_one", "frac_two"), below):
        out[name] = float(np.float64(c) / np.float64(n) * 100)
    return out


def report(gt_xyzi: np.ndarray, est_xyzi: np.ndarray, voxelsize: float = 0.2) -> dict:
    """Everything the runner prints: evaluate()'s dict, est_static / est_dynamic, and overlap()'s dict under "overlap"."""
    r = evaluate(gt_xyzi, est_xyzi, voxelsize)
    r["est_static"], r["est_dynamic"] = est_counts(est_xyzi)
    r["overlap"] = overlap(gt_xyzi, est_xyzi, voxelsize)
    return r


def format_report(r: dict, voxelsize: float = 0.2, gt_path=None, est_path=None) -> str:
    """The runner's stdout for report()'s dict, character for character (with its "GT :" / "Est:" lines when the paths are given)."""
    from tabulate import tabulate
    ov = r["overlap"]
    half, one = 0.5 * voxelsize, voxelsize
    lines = [] if gt_path is None else [f"GT : {gt_path}", f"Est: {est_path}"]
    lines.append(f"est->GT dist: median={ov['median']:.4f}m  p90={ov['p90']:.4f}m  p99={ov['p99']:.4f}m  max={ov['max']:.4f}m")
    lines.append(f"  fraction <0.5*v ({half:.2f}m): {ov['frac_half']:.2f}%  <1*v ({one:.2f}m): {ov['frac_one']:.2f}%  "
                 f"<2*v ({2 * one:.2f}m): {ov['frac_two']:.2f}%")
    lines.append(tabulate(
        [[r["gt_static"], r["gt_dynamic"], r["est_static"], r["est_dynamic"], r["preserved_static"], r["preserved_dynamic"],
          f'{r["PR"]:.3f}', f'{r["RR"]:.3f}', f'{r["F1"]:.4f}']],
        headers=["gt_S", "gt_D", "est_S", "est_D", "kept_S", "kept_D", "PR%", "RR%", "F1"], tablefmt="orgtbl"))
    return "\n".join(lines) + "\n"


def write_pcd_ascii(path: str, xyzi: np.ndarray):
    """ASCII PCD in the layout pcl::io::savePCDFileASCII produces for PointXYZI (what analysis_runner.py reads)."""
    n = len(xyzi)
    with open(path, "w") as f:
        f.write("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\nTYPE F F F F\n"
                f"COUNT 1 1 1 1\nWIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA ascii\n")
        np.savetxt(f, xyzi, fmt="%.8g")


def read_pcd_ascii(path: str) -> np.ndarray:
    with open(path, "r") as f:
        fields, n = None, None
        for line in f:
            line = line.strip()
            if line.startswith("FIELDS"):
                fields = line.split()[1:]
            elif line.startswith("POINTS"):
                n = int(line.split()[1])
            elif line.startswith("DATA"):
                assert line.split()[1] == "ascii"
                break
        arr = np.loadtxt(f, dtype=np.float64, max_rows=n).reshape(-1, len(fields))
    cols = {name: arr[:, i] for i, name in enumerate(fields)}
    return np.stack([cols["x"], cols["y"], cols["z"], cols["intensity"]], axis=1).astype(np.float32)
