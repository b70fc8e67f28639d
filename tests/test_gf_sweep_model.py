"""CPU suite: the facts a ground-filter sweep rests on (DESIGN.md section 8.6), on the oracle alone.

In the mask modes a bin's flag reads only the Scan Ratio Test fields, and R-GPF on a flagged bin reads only that bin's points, their
z order and the five ground-filter fields (gf_dist_thr, gf_th_seeds_height, gf_num_lpr, num_lowest_pts, gf_iter).  So one pass that
flags the union of the settings' bins and fits each union bin once per distinct ground-filter tuple among the settings that flag it,
zeroing each fit's rejected points in the masks of exactly those settings, gives each setting's own mask.  Checked per frame, with
settings that vary the ground-filter fields alongside the thresholds, on the presets and frames of test_srt_sweep_model:
  - a setting's flagged bins are the restated Scan Ratio Test mask, whatever its ground-filter fields;
  - in a bin, settings with equal ground-filter tuples reject the same points, and different tuples differ on some bin;
  - so the grouped union rule rebuilds every setting's keep mask exactly.
"""
import pathlib

import numpy as np
import pytest

from erasor_b200 import params as P
from test_srt_sweep_model import GOLDEN, frames, srt_variant_masks

GF_FIELDS = ("gf_dist_thr", "gf_th_seeds_height", "gf_num_lpr", "num_lowest_pts", "gf_iter")


def gf_settings(version: int) -> list:
    """Thresholds x gf_dist_thr (the bench twin's grid), then each other ground-filter field on its own (num_lowest_pts 600: beyond
    every small bin, whose LPR is then 0), a minimum_num_pts setting and, for version 2, a th_bin_max_h one; two settings repeat a
    ground-filter tuple of the grid under another threshold."""
    vs = [dict(scan_ratio_threshold=t, gf_dist_thr=d) for t in (0.10, 0.20, 0.30) for d in (0.075, 0.15, 0.25)]
    vs += [dict(gf_num_lpr=k) for k in (5, 20)] + [dict(num_lowest_pts=k) for k in (0, 1, 600)]
    vs += [dict(gf_th_seeds_height=h) for h in (0.1, 1.5)] + [dict(gf_iter=k) for k in (0, 1, 8)]
    vs += [dict(minimum_num_pts=25, gf_dist_thr=0.25)]
    if version == 2:
        vs += [dict(th_bin_max_h=0.5, gf_iter=1)]
    return vs


def gf_tuple(p, var) -> tuple:
    return tuple(var.get(f, getattr(p, f)) for f in GF_FIELDS)


@pytest.mark.parametrize("key", sorted(GOLDEN))
def test_grouped_union_rule_reproduces_every_setting(oracle_mod, small_workload, key):
    name, version = key
    p = P.preset(name).replace(skip_voxelize=1, version=version)
    settings = gf_settings(version)
    tuples = [gf_tuple(p, s) for s in settings]
    groups = list(dict.fromkeys(tuples))                      # in order of their lowest setting
    assert 1 < len(groups) < len(settings)
    golden_dir = pathlib.Path(__file__).parent / "golden"
    tuples_differ = 0
    for fi, (m, q) in enumerate(frames(small_workload, oracle_mod, p, golden_dir, key)):
        o = oracle_mod.Oracle(p)
        o.run(m, q)
        bm = o.bin_of_point(0)
        mmn, mmx, mcnt, _ = o.bins(0)
        qmn, qmx, qcnt, _ = o.bins(1)
        masks = srt_variant_masks(version, settings, p, mmn, mmx, mcnt, qmn, qmx, qcnt)
        rej_of = {}                                           # (bin, ground-filter tuple) -> rejected points of that fit
        keeps = []
        for v, s in enumerate(settings):
            ov = oracle_mod.Oracle(p.replace(**s))
            ov.run(m, q)
            flagged = np.array(sorted(pl["bin"] for pl in ov.planes()), dtype=np.int64)
            want = np.nonzero((masks >> np.uint32(v)) & 1)[0]
            assert np.array_equal(flagged, want), f"frame {fi} {s}: flagged bins depend on more than the Scan Ratio Test fields"
            _, rej = ov.cloud(ov.MAP_REJECTED)
            assert np.isin(bm[rej], flagged).all(), "only flagged bins reject"
            for b in flagged:
                r = np.sort(rej[bm[rej] == b])
                k = (int(b), tuples[v])
                if k in rej_of:
                    assert np.array_equal(rej_of[k], r), f"frame {fi} bin {b}: equal ground-filter tuples reject different points"
                else:
                    rej_of[k] = r
            keep = np.ones(len(m), dtype=np.uint8)
            keep[rej] = 0
            keeps.append(keep)
        for b in {b for b, _ in rej_of}:
            fits = [r for (bb, _), r in rej_of.items() if bb == b]
            tuples_differ += int(len({r.tobytes() for r in fits}) > 1)
        # the grouped union rule: per union bin, one fit per group among the settings that flag it, zeroed in those settings' masks
        rebuilt = np.ones((len(settings), len(m)), dtype=np.uint8)
        for b in np.nonzero(masks)[0]:
            for g in groups:
                vm = [v for v in range(len(settings)) if tuples[v] == g and (int(masks[b]) >> v) & 1]
                if vm:
                    rebuilt[np.ix_(vm, rej_of[(int(b), g)])] = 0
        for v in range(len(settings)):
            assert np.array_equal(rebuilt[v], keeps[v]), f"frame {fi} {settings[v]}"
    assert tuples_differ > 0, "different ground-filter tuples must reject different points in some bin"
