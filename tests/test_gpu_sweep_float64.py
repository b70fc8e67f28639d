"""GPU: the node-mode sweeps (erasor_process_nodes_sweep, _sweep_ex and _tune, DESIGN.md sections 8.5-8.7) against the float64
reference of tests/test_erasor_float64_reference.py, at the inputs where the sweep code does not reuse the plain path: Scan Ratio
Test quantities exactly on their thresholds (srt_variant_mask), R-GPF at every sort switch and size class under several
ground-filter groups (k4_process_bin's group loop), points on ring radii, sector angles and gates under eight geometries packed
into K1 launches (k1_geo_bin), and a class-C bin in one geometry only.

Every call runs in node mode at the identity pose with a VoI that covers the scene, and every setting v is checked three ways:
its mask equals a plain erasor_process_nodes run with p.replace(**setting_v) bit for bit; it equals the reference on every point
the reference knows (not those of an ambiguous R-GPF bin, nor a witness within the reference's band), the normals' signs taken
from a cloud-mode run of the same frame under that setting; and its flagged and rejected counts equal the reference's when the
frame has no ambiguous bin.  The frames hold no point with x = -0.0 (the float32 transform to the body frame makes it +0.0)."""
import numpy as np
import pytest

import test_erasor_float64_reference as F
from erasor_b200 import params as P
from test_erasor_float64_reference import _reference_keep
from test_gpu_geo_sweep import tune
from test_gpu_gf_sweep import sweep_ex
from test_gpu_srt_sweep import capi, offsets, sweep  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
I7 = np.array([[0, 0, 0, 0, 0, 0, 1.0]])


def _no_negative_zero_x(m):
    assert not ((m[:, 0] == 0) & np.signbit(m[:, 0])).any()


def plain_runs(capi, p, m, q, settings, voi):
    """One erasor_process_nodes run per setting on a fresh map: masks [V, n], flagged [V], rejected [V], and each run's
    ambiguous_sector count (points the exact binning path decided)."""
    ks, nf, nr, fence = [], [], [], []
    for s in settings:
        gm = capi.Map(m)
        h = capi.Handle(p.replace(**s))
        h.attach_map(gm)
        keep, _ = h.process_nodes(I7, q, offsets([q]), voi_max_range=voi)
        _, f, r = h.node_stats()
        ks.append(keep); nf.append(int(f[0])); nr.append(int(r[0])); fence.append(h.fence_counts()["ambiguous_sector"])
        h.close(); gm.close()
    return dict(keep=np.stack(ks), nf=np.array(nf), nr=np.array(nr), fence=fence)


def cloud_planes(capi, p, m, q):
    h = capi.Handle(p)
    h.set_inputs(m, q)
    h.compare()
    planes = {pl["bin"]: pl for pl in h.get_planes()}
    h.close()
    return planes


def reference(capi, p, m, q, settings, tag):
    """The reference's keep mask per setting, with the points it knows, its flagged and rejected counts and its ambiguous bins."""
    out = []
    for s in settings:
        pv = p.replace(**s)
        planes = cloud_planes(capi, pv, m, q)
        report, amb = [], []
        _, keep, known = _reference_keep(pv, m, q, planes, pv.cov_mode, (tag, s), report, amb)
        out.append(dict(keep=keep, known=known, n_flag=len(planes), n_rej=int((keep == 0).sum()), amb=amb))
    return out


def check_call(got, stats, plain, refs, settings, tag, rows=None, exact_counts=True):
    """got: the call's masks [V, n]; stats: its sweep_stats; rows: the map rows the reference ran on (all by default)."""
    nf, nr = stats
    for v, s in enumerate(settings):
        assert np.array_equal(got[v], plain["keep"][v]), (tag, s, "plain", int((got[v] != plain["keep"][v]).sum()))
        assert nf[v, 0] == plain["nf"][v] and nr[v, 0] == plain["nr"][v], (tag, s, "plain counts")
        r = refs[v]
        g = got[v] if rows is None else got[v][rows]
        bad = np.nonzero(g[r["known"]] != r["keep"][r["known"]])[0]
        assert not len(bad), (tag, s, "reference", len(bad), bad[:10].tolist())
        if exact_counts and not r["amb"]:
            assert (nf[v, 0], nr[v, 0]) == (r["n_flag"], r["n_rej"]), (tag, s, "reference counts")


def _report(tag, refs, band=0):
    amb = sum(len(r["amb"]) for r in refs)
    unknown = sum(int((~r["known"]).sum()) for r in refs)
    print(f"{tag}: {len(refs)} settings, {band} points within a band, {amb} ambiguous bins ({unknown} points)")
    assert max(len(r["amb"]) for r in refs) <= 1, tag         # test_rgpf_against_float64's bound, per frame and setting


# ================================================================================================================================
# a. Scan Ratio Test ties through sweep, sweep_ex and tune
# ================================================================================================================================
@pytest.mark.parametrize("version", [3, 2])
def test_srt_ties(capi, version):
    p = P.preset("seq_05").replace(skip_voxelize=1, version=version)
    m, q, _ = (F.srt_tie_frame if version == 3 else F.srt_v2_frame)(p)
    settings = F.TIE_SETTINGS if version == 3 else F.V2_SETTINGS
    _no_negative_zero_x(m)
    n, V = len(m), len(settings)
    refs = reference(capi, p, m, q, settings, ("ties", version))
    _report(f"ties v{version}", refs)
    assert all(r["known"].all() and not r["amb"] for r in refs), "the tie frames are exact: no band, no ambiguous bin"
    assert len({r["keep"].tobytes() for r in refs}) >= (12 if version == 3 else 5), "the settings must decide different bins"
    plain = plain_runs(capi, p, m, q, settings, 0.0)
    own = {f: getattr(p, f) for f in capi.GEOMETRY_SWEEP_FIELDS}
    gm = capi.Map(m)
    h = capi.Handle(p)
    h.attach_map(gm)
    for call in ("sweep", "sweep_ex", "tune", "sweep packed"):
        if call == "sweep":
            keep = sweep(capi, h, n, I7, [q], settings)
        elif call == "sweep packed":
            keep = sweep(capi, h, n, I7, [q], settings, "packed")
        elif call == "sweep_ex":
            keep = sweep_ex(h, n, I7, [q], settings)
        else:
            keep = tune(h, n, I7, [q], [dict(s, **own) for s in settings], voi=0.0)
        check_call(keep.reshape(V, n).cpu().numpy(), h.sweep_stats(), plain, refs, settings, (call, version))
    h.close(); gm.close()


# ================================================================================================================================
# b. R-GPF under ground-filter groups
# ================================================================================================================================
@pytest.mark.parametrize("cov_mode", [0, 1])
def test_rgpf_groups(capi, cov_mode):
    """Every sort switch and class boundary (128 to K4_C_CAP + 1 points) and the degenerate bins, through sweep_ex calls of two to
    seven ground-filter groups.  Each call runs three times on one handle: after a frame without class-C bins (class C off: its
    bins turn up late), and twice after the full frame (class C running)."""
    p = P.preset(F.RGPF_PRESET).replace(skip_voxelize=1, cov_mode=cov_mode)
    m, q = F.frame_of(p, F.group_specs(), seed=47)
    m_small, q_small = F.frame_of(p, [s for s in F.group_specs() if s[3] <= 2560], seed=48)
    _no_negative_zero_x(m)
    n = len(m)
    h = capi.Handle(p)
    all_refs = []
    for ci, settings in enumerate(F.GROUP_CALLS):
        refs = reference(capi, p, m, q, settings, ("groups", cov_mode, ci))
        all_refs += refs
        plain = plain_runs(capi, p, m, q, settings, 0.0)
        for stage in ("late", "running", "running again"):
            if stage == "late":
                gs = capi.Map(m_small)
                h.attach_map(gs)
                sweep_ex(h, len(m_small), I7, [q_small], settings)
                h.attach_map(None); gs.close()
            gm = capi.Map(m)
            h.attach_map(gm)
            keep = sweep_ex(h, n, I7, [q], settings)
            check_call(keep.reshape(len(settings), n).cpu().numpy(), h.sweep_stats(), plain, refs, settings, (ci, stage, cov_mode))
            h.attach_map(None); gm.close()
    _report(f"groups cov_mode {cov_mode}", all_refs)
    h.close()


# ================================================================================================================================
# c. bin edges through tune, under eight geometries
# ================================================================================================================================
@pytest.mark.parametrize("scene", [name for name, _ in F.witness_geometries()])
def test_bin_edge_witnesses_through_tune(capi, scene):
    """One tune call with every witness geometry's settings (4 x 12 and 26 x 181 first: one K1 launch of exactly 56 KB; 40 x 360 and
    26 x 182 each a 32-warp launch of their own) on the witness scene built for one of them, with host, device and packed queries.
    The exact binning path must run on the same points as in the plain runs: the ambiguous_sector count of the call equals the sum
    of one plain run per geometry."""
    base = P.preset("seq_05").replace(skip_voxelize=1)
    m, q, wit = F.witness_frame(base.replace(**dict(F.witness_geometries())[scene]))
    _no_negative_zero_x(m)
    settings = F.witness_settings()
    n, V = len(m), len(settings)
    plain = plain_runs(capi, base, m, q, settings, F.WITNESS_VOI)
    refs, rows, n_band, exact = [], [], 0, []
    for s in settings:
        pv = base.replace(**s)
        mc, qc, rows_m, rows_q, band = F.clear_witnesses(pv, m, q, wit)
        assert len(rows_q) == len(q), "the query witnesses lie on an axis: never within a band"
        refs += reference(capi, pv, mc, qc, [{}], (scene, s))
        rows.append(rows_m)
        n_band += len(band)
        exact.append(not band)
    _report(f"witnesses {scene}", refs, n_band)
    gm = capi.Map(m)
    h = capi.Handle(base)
    h.attach_map(gm)
    for kind in ("host", "device", "packed"):
        f0 = h.fence_counts()["ambiguous_sector"]
        keep = tune(h, n, I7, [q], settings, kind, voi=F.WITNESS_VOI)
        got = keep.reshape(V, n).cpu().numpy()
        nf, nr = h.sweep_stats()
        assert h.fence_counts()["ambiguous_sector"] - f0 == sum(plain["fence"][::2]), kind      # settings come in pairs per geometry
        for v, s in enumerate(settings):
            check_call(got[v:v + 1], (nf[v:v + 1], nr[v:v + 1]), dict(keep=plain["keep"][v:v + 1], nf=plain["nf"][v:v + 1],
                       nr=plain["nr"][v:v + 1]), refs[v:v + 1], [s], (scene, kind), rows=rows[v], exact_counts=exact[v])
    h.close(); gm.close()


def test_exact_56kb_pair_takes_one_k1_launch(capi):
    """4 x 12 and 26 x 181 bins: K1 tables of 640 + 56 704 bytes, exactly 56 KB, share one launch; 26 x 182 (57 664 bytes) goes over
    and takes a launch of its own.  Masks cannot show how the geometries were packed; the launch count can."""
    base = P.preset("seq_05").replace(skip_voxelize=1)
    geos = dict(F.witness_geometries())
    m, q, _ = F.witness_frame(base.replace(**geos["26x181"]))
    n = len(m)
    pair = lambda other: [dict(geos["4x12"], scan_ratio_threshold=0.3), dict(geos[other], scan_ratio_threshold=0.3)]
    plain = {g: plain_runs(capi, base, m, q, pair(g), F.WITNESS_VOI)["keep"] for g in ("26x181", "26x182")}
    gm = capi.Map(m)
    h = capi.Handle(base)
    h.attach_map(gm)
    tune(h, n, I7, [q], pair("26x181"), voi=F.WITNESS_VOI)          # the handle's first call also launches class C
    launches = {}
    for g in ("26x181", "26x182", "26x181", "26x182"):
        l0 = h.kernel_launch_count()
        keep = tune(h, n, I7, [q], pair(g), voi=F.WITNESS_VOI)
        launches.setdefault(g, set()).add(h.kernel_launch_count() - l0)
        assert np.array_equal(keep.reshape(2, n).cpu().numpy(), plain[g]), g
    assert len(launches["26x181"]) == 1 and len(launches["26x182"]) == 1
    assert launches["26x182"].pop() - launches["26x181"].pop() == 1, "26 x 181 shares the 4 x 12 launch, 26 x 182 does not"
    h.close(); gm.close()


# ================================================================================================================================
# d. a class-C bin in one geometry only
# ================================================================================================================================
def test_class_c_bin_in_one_geometry_only(capi):
    """3600 points in one 15 m x 30 degree bin of the coarse geometry (class C), nine class-A/B bins of seq_05's geometry: both in
    one tune call, on a fresh handle and again after a call whose frame has no class-C bin."""
    p = P.preset("seq_05").replace(skip_voxelize=1)
    m, q = F.class_c_frame(p)
    _no_negative_zero_x(m)
    settings = F.CLASS_C_SETTINGS
    n, V = len(m), len(settings)
    for s in settings:                                   # the coarse geometry has one bin beyond class B, the fine one none
        pv = p.replace(**s)
        cnt = np.bincount(F.polar(pv, m)[0], minlength=pv.num_bins)
        assert (cnt.max() > 2560) == ("num_rings" in s)
    refs = reference(capi, p, m, q, settings, "class C")
    _report("class C", refs)
    assert all(r["known"].all() for r in refs)
    plain = plain_runs(capi, p, m, q, settings, 0.0)
    m_small, q_small = F.frame_of(p, [(5, 20, "flat", 300, None)], seed=44)
    h = capi.Handle(p)
    for stage in ("first call", "after a frame without class C"):
        if stage != "first call":
            gs = capi.Map(m_small)
            h.attach_map(gs)
            tune(h, len(m_small), I7, [q_small], settings, voi=0.0)
            h.attach_map(None); gs.close()
        gm = capi.Map(m)
        h.attach_map(gm)
        keep = tune(h, n, I7, [q], settings, voi=0.0)
        check_call(keep.reshape(V, n).cpu().numpy(), h.sweep_stats(), plain, refs, settings, ("class C", stage))
        h.attach_map(None); gm.close()
    h.close()
