"""Tune the Scan Ratio Test and the ground filter on new data in one node-mode pass: every setting of the Cartesian product of the
listed values (at most 32) runs through pipeline.sweep_frame_independent, which bins each node and fits R-GPF once and keeps one map
mask per setting (DESIGN.md section 8.5), or, when a ground-filter or geometry field is listed, through
pipeline.tune_frame_independent, which sorts each flagged bin once and fits it once per distinct ground-filter tuple (section 8.6)
and bins each node under every listed geometry in one scan of the map (section 8.7).  Prints one row per setting (PR / RR / F1
against the GT, kept and saved points, flagged bins and rejected points; a column per listed ground-filter or geometry field) and
marks the F1 maximum with '*'; --save-best writes that setting's saved map.

    python -m erasor_b200.sweep <config.yaml> <file.bag | data_dir> [--scan-ratio 0.10,0.15,0.20,0.25,0.30] [--min-pts 6,10]
                                [--th-bin-max-h 0.05,0.2] [--gf-dist-thr 0.075,0.15] [--gf-seeds-height 0.5] [--gf-num-lpr 10,20]
                                [--num-lowest-pts 1,5] [--gf-iter 3] [--max-range 60,80] [--num-rings 15,20] [--num-sectors 60,108]
                                [--min-h -1.5] [--max-h 3.0] [--gt gt.pcd] [--save-best out.pcd] [--pcd-mode ascii] [--batch 20]

A field left out keeps the yaml's value; --save-best reruns run_frame_independent for the chosen setting.  Inputs are read on
the device: a ROS bag of erasor/node messages (the map is the yaml's initial_map_path, as static_map_nodes_main reads it), or
<data_dir>/dense_global_map.pcd, <data_dir>/poses_lidar2body.csv and <data_dir>/pcds/%06d.pcd.  GT defaults to the initial map,
as run_sequence scores.
"""
from __future__ import annotations

import argparse
import itertools
import os
import sys

import numpy as np

from . import capi, params, pipeline


def _floats(s):
    return [float(x) for x in s.split(",") if x.strip()]


def _ints(s):
    return [int(x) for x in s.split(",") if x.strip()]


# the ground-filter fields: (setting field, command-line flag, column header, column width, value format)
GF_COLUMNS = (("gf_dist_thr", "--gf-dist-thr", "gf_dist_thr", 11, ".4g"), ("gf_th_seeds_height", "--gf-seeds-height", "seeds_height", 12, ".4g"),
              ("gf_num_lpr", "--gf-num-lpr", "num_lpr", 7, "d"), ("num_lowest_pts", "--num-lowest-pts", "lowest_pts", 10, "d"),
              ("gf_iter", "--gf-iter", "gf_iter", 7, "d"))
# the geometry fields, the same way
GEOMETRY_COLUMNS = (("max_range", "--max-range", "max_range", 9, ".4g"), ("num_rings", "--num-rings", "rings", 5, "d"),
                    ("num_sectors", "--num-sectors", "sectors", 7, "d"), ("min_h", "--min-h", "min_h", 7, ".4g"),
                    ("max_h", "--max-h", "max_h", 7, ".4g"))


def variants_of(scan_ratio=None, min_pts=None, th_bin_max_h=None, **gf) -> list:
    """The Cartesian product of the listed values, as sweep settings (a field with no list is left to the yaml).  gf: lists of
    the ground-filter and geometry fields (capi.GF_SWEEP_FIELDS, capi.GEOMETRY_SWEEP_FIELDS), by field name."""
    if set(gf) - set(capi.GF_SWEEP_FIELDS + capi.GEOMETRY_SWEEP_FIELDS):
        raise ValueError(f"unknown fields {sorted(set(gf) - set(capi.GF_SWEEP_FIELDS + capi.GEOMETRY_SWEEP_FIELDS))}")
    axes = [(k, v) for k, v in (("scan_ratio_threshold", scan_ratio), ("minimum_num_pts", min_pts), ("th_bin_max_h", th_bin_max_h)) if v]
    axes += [(k, gf[k]) for k, *_ in GF_COLUMNS + GEOMETRY_COLUMNS if gf.get(k)]
    if not axes:
        return [{}]
    return [dict(zip([k for k, _ in axes], combo)) for combo in itertools.product(*[v for _, v in axes])]


def best_row(rows) -> int:
    """Index of the F1 maximum (the first one on ties)."""
    return int(np.argmax([r["F1"] for r in rows]))


def format_rows(rows, gf_fields=()) -> str:
    """The table: one line per row, the F1 maximum marked; gf_fields adds a column per listed ground-filter or geometry field."""
    best = best_row(rows)
    cols = [(f, hd, w, spec) for f, _, hd, w, spec in GF_COLUMNS + GEOMETRY_COLUMNS if f in gf_fields]
    head = f"{'':1} {'scan_ratio':>10} {'min_pts':>7} {'th_bin_max_h':>12} " + "".join(f"{hd:>{w}} " for _, hd, w, _ in cols) + \
           f"{'PR%':>8} {'RR%':>8} {'F1':>7} {'kept':>10} {'saved':>10} {'flagged':>9} {'rejected':>10}"
    lines = [head]
    for i, r in enumerate(rows):
        lines.append(f"{'*' if i == best else ' '} {r['scan_ratio_threshold']:>10.4g} {r['minimum_num_pts']:>7d} {r['th_bin_max_h']:>12.4g} " +
                     "".join(f"{r[f]:>{w}{spec}} " for f, _, w, spec in cols) +
                     f"{r['PR']:>8.3f} {r['RR']:>8.3f} {r['F1']:>7.4f} {r['kept']:>10d} {r['saved']:>10d} {r['flagged']:>9d} {r['rejected']:>10d}")
    return "\n".join(lines) + "\n"


def read_data_dir(codec, data_dir: str):
    """(nodes, initial map) of the env layout: poses_lidar2body.csv rows idx,time,x,y,z,qx,qy,qz,qw and pcds/%06d.pcd in node order."""
    rows = np.loadtxt(os.path.join(data_dir, "poses_lidar2body.csv"), delimiter=",", skiprows=1, dtype=np.float64, ndmin=2)
    nodes = [(int(r[1]), r[2:9].copy(), codec.load(os.path.join(data_dir, "pcds", f"{i:06d}.pcd"))) for i, r in enumerate(rows)]
    return nodes, codec.load(os.path.join(data_dir, "dense_global_map.pcd"))


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("config")
    ap.add_argument("data", help="a .bag of erasor/node messages, or a data directory")
    ap.add_argument("--scan-ratio", type=_floats)
    ap.add_argument("--min-pts", type=_ints)
    ap.add_argument("--th-bin-max-h", type=_floats)
    for field, flag, _, _, spec in GF_COLUMNS + GEOMETRY_COLUMNS:
        ap.add_argument(flag, dest=field, type=_ints if spec == "d" else _floats)
    ap.add_argument("--gt", help="GT cloud (default: the initial map)")
    ap.add_argument("--save-best", help="write the F1 maximum's saved map here")
    ap.add_argument("--pcd-mode", default="ascii", choices=sorted(capi.PCD_MODES))
    ap.add_argument("--batch", type=int, default=20)
    args = ap.parse_args(argv)
    gf = {f: getattr(args, f) for f, *_ in GF_COLUMNS + GEOMETRY_COLUMNS if getattr(args, f)}
    variants = variants_of(args.scan_ratio, args.min_pts, args.th_bin_max_h, **gf)
    if len(variants) > capi.MAX_SWEEP_VARIANTS:
        ap.error(f"{len(variants)} settings: a sweep takes at most {capi.MAX_SWEEP_VARIANTS}")
    ep, up = params.load_yaml(args.config)
    with capi.PcdCodec() as codec:
        if args.data.endswith(".bag"):
            nodes = pipeline.read_bag_nodes(args.data)
            initial = codec.load(up.initial_map_path)
        else:
            nodes, initial = read_data_dir(codec, args.data)
        gt = codec.load(args.gt) if args.gt else None
    if gf:
        rows = pipeline.tune_frame_independent(nodes, initial, up, ep, variants, gt=gt, batch=args.batch)
    else:
        rows = pipeline.sweep_frame_independent(nodes, initial, up, ep, variants, gt=gt, batch=args.batch)
    sys.stdout.write(format_rows(rows, tuple(gf)))
    if args.save_best:
        best = variants[best_row(rows)]
        res = pipeline.run_frame_independent(nodes, initial, up, ep.replace(**best), batch=args.batch)
        with capi.PcdCodec() as codec:
            codec.write(args.save_best, res["static_map"], mode=args.pcd_mode)
    return 0


if __name__ == "__main__":
    sys.exit(main())
