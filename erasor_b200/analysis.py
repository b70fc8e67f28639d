"""The reference's scripts/analysis_runner.py on the device: prints exactly what it prints for two ASCII PCDs -- the estimate -> GT
distance report, then the PR / RR table -- computed by capi.Evaluator (erasor_evaluate + erasor_eval_overlap) on clouds read by
capi.PcdCodec.load (erasor_pcd_load: ASCII files bit-identical to read_pcd_ascii, and binary and binary_compressed files as PCL
reads them).
--host reads ASCII files only, with read_pcd_ascii and computes with sklearn instead (erasor_b200.evaluate), for machines without a GPU.

    python -m erasor_b200.analysis --gt gt.pcd --est est.pcd [--voxelsize 0.2] [--host] [--device N]
"""
from __future__ import annotations

import argparse
import os
import sys

from . import evaluate as E


def main(argv=None) -> int:
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--gt", required=True)
    p.add_argument("--est", required=True)
    p.add_argument("--voxelsize", type=float, default=0.2)
    p.add_argument("--host", action="store_true", help="sklearn on the host instead of the device evaluator")
    p.add_argument("--device", type=int, default=0)
    args = p.parse_args(argv)
    for path in (args.gt, args.est):
        if not os.path.isfile(path):
            p.error(f"no such file: {path}")
    if args.host:
        gt, est = E.read_pcd_ascii(args.gt), E.read_pcd_ascii(args.est)
        r = E.report(gt, est, args.voxelsize)
    else:
        from . import capi
        with capi.PcdCodec(device=args.device) as codec:
            gt, est = codec.load(args.gt), codec.load(args.est)
        with capi.Evaluator(device=args.device) as ev:
            r = ev.report(gt, est, voxelsize=args.voxelsize)
    sys.stdout.write(E.format_report(r, args.voxelsize, args.gt, args.est))
    return 0


if __name__ == "__main__":
    sys.exit(main())
