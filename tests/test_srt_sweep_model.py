"""CPU suite: the fact a Scan Ratio Test sweep rests on (DESIGN.md section 8.5), on the oracle alone.

In the mask modes a map point's verdict depends on scan_ratio_threshold, minimum_num_pts and th_bin_max_h only through the set of
flagged bins, and R-GPF on a flagged bin reads only that bin's points and the gf_* parameters.  So one pass that flags the union of
the settings' bins, fits each union bin once and zeroes a rejected point in the mask of every setting that flags its bin gives
each setting's own mask.  Checked per frame, for every setting:
  - the oracle's flagged bins equal the per-bin mask restated here from the oracle's bin tables (srt_variant_masks);
  - in every bin two settings flag, the rejected points are the same;
  - so the union rule rebuilds the setting's keep mask exactly.
"""
import numpy as np
import pytest

from erasor_b200 import params as P

GOLDEN = {("seq_05", 3): "seq05_v3.npz", ("seq_00", 3): "seq00_v3.npz", ("seq_05", 2): "seq05_v2.npz"}
THRESHOLDS = (0.10, 0.15, 0.20, 0.25, 0.30)


def sweep_variants(version: int) -> list:
    """The README's threshold sweep, minimum_num_pts settings (App. B-9: a negative one flags nothing) and, for version 2,
    th_bin_max_h settings."""
    vs = [dict(scan_ratio_threshold=t) for t in THRESHOLDS]
    vs += [dict(minimum_num_pts=k) for k in (0, 3, 25, -1)]
    if version == 2:
        vs += [dict(th_bin_max_h=h) for h in (-1.0, 0.0, 0.5, 1.5)]
    return vs


def srt_variant_masks(version, variants, base, mmn, mmx, mcnt, qmn, qmx, qcnt) -> np.ndarray:
    """uint32 per bin, bit v set when setting v flags the bin: srt_is_flagged with the setting's three fields (missing ones from
    base).  mmn .. qcnt: the map / query bin tables (z as float64, counts)."""
    masks = np.zeros(len(mcnt), dtype=np.uint32)
    occ = (mcnt > 0) & (qcnt > 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        mdh = np.where(occ, mmx - mmn, 0.0)
        cdh = np.where(occ, qmx - qmn, 0.0)
        a, c = mdh / cdh, cdh / mdh
    ratio = np.where(c < a, c, a)          # std::min(a, c) returns a unless c < a
    for v, var in enumerate(variants):
        k = int(var.get("minimum_num_pts", base.minimum_num_pts))
        thr = float(var.get("scan_ratio_threshold", base.scan_ratio_threshold))
        hmax = float(var.get("th_bin_max_h", base.th_bin_max_h))
        if k < 0:
            continue
        fl = occ & (qcnt >= k) & (ratio < thr) & (mdh >= cdh)
        fl &= (mdh > 0.5) if version == 3 else (mmx > hmax)
        masks[fl] |= np.uint32(1 << v)
    return masks


def frames(small_workload, oracle_mod, p, golden_dir, key):
    scene = small_workload["scene"]
    out = []
    for voi_map, q, k, _ in small_workload["frames"]:
        voi, _ = oracle_mod.fetch_voi(small_workload["map_world"], scene.pose7(k), p.max_range)
        out.append((voi, q))
    g = np.load(golden_dir / GOLDEN[key])
    out.append((g["map_voi"], g["query_voi"]))
    return out


@pytest.mark.parametrize("key", sorted(GOLDEN))
def test_union_rule_reproduces_every_setting(oracle_mod, small_workload, key):
    import pathlib
    name, version = key
    p = P.preset(name).replace(skip_voxelize=1, version=version)
    variants = sweep_variants(version)
    golden_dir = pathlib.Path(__file__).parent / "golden"
    differ = 0
    for fi, (m, q) in enumerate(frames(small_workload, oracle_mod, p, golden_dir, key)):
        o = oracle_mod.Oracle(p)
        o.run(m, q)
        bm = o.bin_of_point(0)
        mmn, mmx, mcnt, _ = o.bins(0)
        qmn, qmx, qcnt, _ = o.bins(1)
        masks = srt_variant_masks(version, variants, p, mmn, mmx, mcnt, qmn, qmx, qcnt)
        rej_of_bin, keeps = {}, []
        for v, var in enumerate(variants):
            ov = oracle_mod.Oracle(p.replace(**var))
            ov.run(m, q)
            assert np.array_equal(ov.bin_of_point(0), bm), "the binning does not depend on the Scan Ratio Test"
            flagged = np.array(sorted(pl["bin"] for pl in ov.planes()), dtype=np.int64)
            want = np.nonzero((masks >> np.uint32(v)) & 1)[0]
            assert np.array_equal(flagged, want), f"frame {fi} {var}: flagged bins differ from the restated mask"
            _, rej = ov.cloud(ov.MAP_REJECTED)
            assert np.isin(bm[rej], flagged).all(), "only flagged bins reject"
            for b in flagged:
                r = np.sort(rej[bm[rej] == b])
                if b in rej_of_bin:
                    assert np.array_equal(rej_of_bin[b], r), f"frame {fi} bin {b}: R-GPF depends on the setting"
                else:
                    rej_of_bin[b] = r
            keep = np.ones(len(m), dtype=np.uint8)
            keep[rej] = 0
            keeps.append(keep)
        # the union rule: each union bin's rejected points, zeroed in the mask of every setting whose bit the bin carries
        for v in range(len(variants)):
            keep = np.ones(len(m), dtype=np.uint8)
            for b in np.nonzero(masks)[0]:
                if (int(masks[b]) >> v) & 1:
                    keep[rej_of_bin[b]] = 0
            assert np.array_equal(keep, keeps[v]), f"frame {fi} {variants[v]}"
        differ += int(len({k.tobytes() for k in keeps}) > 1)
        assert np.count_nonzero(masks) > 0
    assert differ > 0, "the settings must give different masks on some frame"
