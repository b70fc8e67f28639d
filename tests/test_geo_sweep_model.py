"""CPU suite: the geometry sweep's host side and its workload (DESIGN.md section 8.7), on the oracle alone.

  - variants_of takes the geometry fields as axes and format_rows gives each listed one a column after the ground-filter ones;
    without them the table is the one the Scan Ratio Test and ground-filter sweeps print;
  - on the shared node workload (one VoI radius for every setting, as a tune call cuts it), settings that differ only in the polar
    geometry, or only in min_h / max_h, give different oracle masks, so the GPU tests that compare them bit for bit discriminate.
"""
import numpy as np
import pytest

from erasor_b200 import capi
from erasor_b200 import params as P
from erasor_b200 import sweep as cli

VOI = 80.0


def test_variants_of_geometry_axes():
    vs = cli.variants_of([0.1, 0.3], None, None, gf_dist_thr=[0.1], num_rings=[15, 20], max_h=[3.0])
    assert vs == [dict(scan_ratio_threshold=t, gf_dist_thr=0.1, num_rings=r, max_h=3.0) for t in (0.1, 0.3) for r in (15, 20)]
    assert cli.variants_of(None, None, None, max_range=[60.0, 80.0], min_h=[-1.3]) == [dict(max_range=m, min_h=-1.3) for m in (60.0, 80.0)]
    with pytest.raises(ValueError):
        cli.variants_of([0.1], None, None, version=[2])
    assert set(capi.GEOMETRY_SWEEP_FIELDS) == {f for f, *_ in cli.GEOMETRY_COLUMNS}


def test_format_rows_geometry_columns():
    row = dict(scan_ratio_threshold=0.2, minimum_num_pts=6, th_bin_max_h=0.05, gf_dist_thr=0.125, max_range=60.0, num_rings=15,
               num_sectors=108, min_h=-1.3, max_h=3.2, PR=99.5, RR=90.25, F1=0.9453, kept=1000, saved=900, flagged=12, rejected=345)
    rows = [row, dict(row, num_rings=20, F1=0.95)]
    plain = cli.format_rows(rows)
    out = cli.format_rows(rows, ("num_sectors", "gf_dist_thr", "num_rings"))
    head, first, second = out.splitlines()
    assert head.split()[2:6] == ["th_bin_max_h", "gf_dist_thr", "rings", "sectors"]
    assert first.split()[2:6] == ["0.05", "0.125", "15", "108"] and second.startswith("*") and second.split()[5] == "20"
    # the columns slot in between th_bin_max_h and PR%: dropping them gives the plain table back
    widths = 12 + 8 + 6                                   # gf_dist_thr, rings, sectors with their separators
    cut = len(f"{'':1} {'scan_ratio':>10} {'min_pts':>7} {'th_bin_max_h':>12} ")
    assert "\n".join(line[:cut] + line[cut + widths:] for line in out.splitlines()) + "\n" == plain


def test_geometry_and_height_window_change_the_oracle_masks(oracle_mod, small_workload):
    base = P.preset("seq_05").replace(skip_voxelize=1)
    scene = small_workload["scene"]
    settings = [dict(), dict(num_rings=20, num_sectors=108), dict(num_sectors=108), dict(max_range=40.0),
                dict(max_h=1.5), dict(max_h=1.0), dict(min_h=-2.0, max_h=4.0), dict(min_h=-1.6, max_h=2.5)]
    masks = np.zeros((len(settings), 0), dtype=np.uint8)
    for _, q, k, _ in small_workload["frames"][:3]:
        voi, _ = oracle_mod.fetch_voi(small_workload["map_world"], scene.pose7(k), VOI)
        keeps = []
        for s in settings:
            o = oracle_mod.Oracle(base.replace(**s))
            o.run(voi, q)
            keep = np.ones(len(voi), dtype=np.uint8)
            keep[o.cloud(o.MAP_REJECTED)[1]] = 0
            keeps.append(keep)
        masks = np.concatenate([masks, np.stack(keeps)], axis=1)
    assert (masks == 0).any()
    assert len({m.tobytes() for m in masks}) == len(settings), "every geometry and height window must give its own mask"
