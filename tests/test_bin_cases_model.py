"""The crafted frames of tests/bin_cases.py against the oracle (no GPU): every case lands on the intended side of the size switch it
is for, so that tests/test_gpu_capacity_edges.py compares the device's second code paths with the oracle and not the first ones
again.  Also K4b's global-scratch layout (device_types.h k4b_scratch_offset, through the host build): every flagged bin's region
is disjoint from the others, including two adjacent bins whose every map point is ground."""
import ctypes
import os

import numpy as np
import pytest

import bin_cases as C
from erasor_b200 import params as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTCHECK = os.path.join(ROOT, "erasor_b200", "_lib", "liberasor_b200_hostcheck.so")


def _oracle(oracle_mod, p, m, q):
    o = oracle_mod.Oracle(p)
    o.run(m, q)
    return o


def _spec_bins(p, specs):
    return sorted(C.bin_id(p, s.ring, s.sector) for s in specs)


def test_switches_as_read_from_the_code():
    assert C.K4_C_CAP == 8775 and C.K4B_CAP == 4549
    assert C.k2_window(14400) == 2356                   # 40 x 360: (111 KB - the slot table) / 36 bytes per slot
    assert C.k2_window(15 * 60) == 900 and C.k2_window(20 * 108) == 2160      # one window holds every bin of the KITTI grids
    assert [C.radix_passes(c) for c in (1, 256, 257, 1 << 16, (1 << 16) + 1, 1 << 24, (1 << 24) + 1, (1 << 31) - 1)] == [1, 1, 2, 2, 3, 3, 4, 4]


@pytest.mark.parametrize("version", [3, 2])
@pytest.mark.parametrize("z", C.RGPF_Z_KINDS)
def test_rgpf_frames(oracle_mod, z, version):
    p = P.preset("seq_05").replace(skip_voxelize=1, version=version)
    specs = C.rgpf_specs(z)
    m, q = C.flagged_bins(p, specs, seed=7)
    o = _oracle(oracle_mod, p, m, q)
    planes = o.planes()
    assert [x["bin"] for x in planes] == _spec_bins(p, specs), "exactly the requested bins are flagged"
    want = {C.bin_id(p, s.ring, s.sector): s.n for s in specs}
    assert all(x["n_points"] == want[x["bin"]] for x in planes)
    sizes = sorted(want.values())
    for sw in C.RGPF_SWITCHES + (C.K4_C_CAP,):
        if z in ("rough", "dup") or sw >= C.K4_C_CAP:
            assert sw in sizes and sw + 1 in sizes, f"both sides of the switch at {sw}"
    assert max(sizes) > 10 * C.K4_C_CAP


@pytest.mark.parametrize("leaf", sorted(C.K4B_FRAMES))
def test_k4b_frames(oracle_mod, leaf):
    p = P.preset("seq_05").replace(skip_voxelize=0, version=3, map_voxel_size=leaf)
    specs = C.K4B_FRAMES[leaf]
    m, q = C.flagged_bins(p, specs, seed=11)
    o = _oracle(oracle_mod, p, m, q)
    planes = {x["bin"]: x for x in o.planes()}
    assert sorted(planes) == _spec_bins(p, specs)
    bm, bq = o.bin_of_point(0), o.bin_of_point(1)
    _, _, qcnt, _ = o.bins(1)
    passes = []
    for s in specs:
        b = C.bin_id(p, s.ring, s.sector)
        x = planes[b]
        assert x["n_points"] == s.n and x["n_ground"][-1] == s.n, "a ramp bin is ground throughout"
        assert qcnt[b] == s.nq and qcnt[b] + x["n_ground"][-1] == s.n + s.nq       # K4b's n = qc + n_ground_final
        pts = np.concatenate([q[bq == b], m[bm == b]])
        cells, overflow = C.voxel_cells(pts, leaf)
        passes.append("through" if overflow else C.radix_passes(cells))
        if s.distinct_leaf is not None:
            assert len(np.unique(C.voxel_ids(pts, leaf), axis=0)) == len(pts), "one point per voxel"
    n = [s.n + s.nq for s in specs]
    expect = {0.2: [2, 2, 1, 1], 0.05: [2, 2, 3, 3], 0.01: [3, 3, 4, 3, 3, 3], 0.001: ["through"]}[leaf]
    assert passes == expect, passes
    if leaf != 0.001:
        assert n[:4] == [C.K4B_CAP, C.K4B_CAP + 1, 12000, 40000]
    else:
        assert n[0] > C.K4B_CAP


def _hostcheck():
    L = ctypes.CDLL(HOSTCHECK)
    u32p = np.ctypeslib.ndpointer(np.uint32, flags="C")
    L.erasor_hostcheck_k4b_scratch_offset.argtypes = [u32p, u32p, u32p, ctypes.c_size_t, np.ctypeslib.ndpointer(np.uint64, flags="C")]
    return L


def _k4b_offsets(dsq, dsm, bins):
    out = np.zeros(len(bins), dtype=np.uint64)
    _hostcheck().erasor_hostcheck_k4b_scratch_offset(np.ascontiguousarray(dsq, np.uint32), np.ascontiguousarray(dsm, np.uint32),
                                                     np.ascontiguousarray(bins, np.uint32), len(bins), out)
    return out.astype(np.int64)


@pytest.mark.parametrize("leaf", sorted(C.K4B_FRAMES))
def test_k4b_scratch_regions_disjoint(oracle_mod, leaf):
    """K4b's global scratch in cloud mode: bin b's region starts at k4b_scratch_offset(dsq[b], dsm[b], b), where dsq / dsm are the
    exclusive scans of the per-bin query / map counts over all bins; it spans 36 n + 4 bytes, n = qc + n_ground_final."""
    p = P.preset("seq_05").replace(skip_voxelize=0, version=3, map_voxel_size=leaf)
    specs = C.K4B_FRAMES[leaf]
    m, q = C.flagged_bins(p, specs, seed=11)
    o = _oracle(oracle_mod, p, m, q)
    _, _, cm, _ = o.bins(0)
    _, _, cq, _ = o.bins(1)
    B = p.num_bins
    assert np.array_equal(cm, np.bincount(o.bin_of_point(0)[o.bin_of_point(0) >= 0], minlength=B))
    dsm = np.concatenate([[0], np.cumsum(cm.astype(np.int64))])[:B]
    dsq = np.concatenate([[0], np.cumsum(cq.astype(np.int64))])[:B]
    planes = o.planes()
    bins = np.array([x["bin"] for x in planes], dtype=np.int64)
    n = np.array([cq[x["bin"]] + x["n_ground"][-1] for x in planes], dtype=np.int64)
    off = _k4b_offsets(dsq[bins], dsm[bins], bins)
    end = off + 36 * n + 4
    order = np.argsort(off)
    assert np.all(end[order][:-1] <= off[order][1:]), "K4b scratch regions overlap"
    size = int(_k4b_offsets([len(q)], [len(m)], [B])[0]) + 36 + 64          # d_vox_scratch's size (erasor_capi.cu)
    assert end.max() <= size
    if leaf == 0.01:
        # the adjacent all-ground pair: without the padding its first bin's footprint reaches the second bin's first point
        b0, b1 = (C.bin_id(p, r, s) for r, s in C.K4B_ADJACENT)
        assert b1 == b0 + 1 and cm[b0] > 0 and cm[b1] > 0
        i0 = int(np.flatnonzero(bins == b0)[0])
        assert n[i0] == cq[b0] + cm[b0] > C.K4B_CAP
        unpadded = 36 * (dsq + dsm)
        assert unpadded[b0] + 36 * n[i0] + 4 > unpadded[b1]


def test_k2_window_frames(oracle_mod):
    p = P.preset(C.K2_PRESET)
    B = p.num_bins
    W = C.k2_window(B)
    counts = C.k2_flag_counts(B)
    assert counts[0] < W <= counts[1] < counts[2] and counts[3] > 2 * W and counts[4] == B
    for k, nf in enumerate(counts):
        m, q, pick = C.fill_flagged(p, nf, seed=100 + k)
        o = _oracle(oracle_mod, p, m, q)
        assert [x["bin"] for x in o.planes()] == pick.tolist(), nf
