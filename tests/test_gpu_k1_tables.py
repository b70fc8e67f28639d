"""Node mode's per-bin tables (count, min z, max z) on adversarial dense rows, against the oracle's fetch_VoI + R-POD.

K1 aggregates each dense row of 32 VoI points with one shared-memory update per distinct bin of the row.  The map here is
laid out in map order so that the rows K1 forms hit the cases that scheme has to get right: 32 distinct bins in one row,
one bin for the whole row, a row of points outside the z window only (the not-binned count), equal z in many lanes, one
bin's lanes interleaved with another's, and rows cut short by points outside the VoI and by the end of a chunk."""
import numpy as np
import pytest

from erasor_b200 import params as P

pytestmark = pytest.mark.gpu


def _bin_point(p, ring, sector, rng, n):
    """n points well inside bin (ring, sector) of the polar grid around the origin (body frame == map frame here)."""
    rs, ss = p.max_range / p.num_rings, 2.0 * np.pi / p.num_sectors
    r = (ring + rng.uniform(0.2, 0.8, n)) * rs
    t = (sector + rng.uniform(0.2, 0.8, n)) * ss
    return np.stack([r * np.cos(t), r * np.sin(t)], axis=1)


def _rows(p, seed):
    rng = np.random.default_rng(seed)
    zl, zh = p.min_h, p.max_h
    R, S = p.num_rings, p.num_sectors
    rows = []
    def row(xy, z):
        rows.append(np.concatenate([xy, np.asarray(z, dtype=np.float64).reshape(-1, 1), np.full((len(xy), 1), 40.0)], axis=1))
    for k in range(8):
        # 32 distinct bins: one ring, 32 sectors (wrapping), or 32 rings / sectors mixed
        sec = (np.arange(32) + 7 * k) % S
        rg = (np.arange(32) * 3 + k) % R
        row(np.concatenate([_bin_point(p, rg[i], sec[i], rng, 1) for i in range(32)]), rng.uniform(zl + 0.01, zh - 0.01, 32))
        # all lanes in one bin, distinct z
        row(_bin_point(p, k % R, (5 * k) % S, rng, 32), rng.uniform(zl + 0.01, zh - 0.01, 32))
        # every lane outside the z window (above max_h and below min_h): counted as not binned only
        row(_bin_point(p, (k + 3) % R, (11 * k) % S, rng, 32), np.where(np.arange(32) % 2 == 0, zh + 0.5, zl - 0.5))
        # equal z in many lanes, two bins, min == max in one of them
        zz = np.full(32, zl + 0.37)
        zz[::5] = zl + 0.91
        xy = np.where((np.arange(32) < 16)[:, None], _bin_point(p, (k + 1) % R, (2 * k) % S, rng, 32),
                      _bin_point(p, (k + 2) % R, (2 * k + 1) % S, rng, 32))
        zz[16:] = zl + 0.55
        row(xy, zz)
        # two bins interleaved lane by lane, plus a third in one lane; some lanes outside the z window
        a, b, c = _bin_point(p, (k + 4) % R, (3 * k) % S, rng, 32), _bin_point(p, (k + 5) % R, (3 * k + 2) % S, rng, 32), _bin_point(p, 0, 0, rng, 32)
        xy = np.where((np.arange(32) % 2 == 0)[:, None], a, b)
        xy[17] = c[17]
        zz = rng.uniform(zl + 0.01, zh - 0.01, 32)
        zz[[3, 9, 30]] = zh + 1.0
        row(xy, zz)
        # points outside the VoI radius between rows: the next dense rows start mid-row
        n_out = int(rng.integers(1, 31))
        t = rng.uniform(0, 2 * np.pi, n_out)
        row(np.stack([1.5 * p.max_range * np.cos(t), 1.5 * p.max_range * np.sin(t)], axis=1), rng.uniform(zl, zh, n_out))
    return np.concatenate(rows)


@pytest.mark.parametrize("name", ["seq_05", "seq_00", "synthetic_40x360"])
@pytest.mark.parametrize("n_tail", [0, 7, 31])
def test_node_tables_on_adversarial_rows(oracle_mod, name, n_tail):
    from erasor_b200 import capi
    p = P.preset(name).replace(skip_voxelize=1)
    body = _rows(p, seed=5)
    # a large random part in front, so that the adversarial rows fall into several chunks and warps; n_tail points after them
    # leave the last chunk's tail shorter than a row
    rng = np.random.default_rng(17)
    n_fill = 9000
    r = p.max_range * np.sqrt(rng.uniform(0, 1.3, n_fill))
    t = rng.uniform(0, 2 * np.pi, n_fill)
    fill = np.stack([r * np.cos(t), r * np.sin(t), rng.uniform(p.min_h - 0.5, p.max_h + 0.5, n_fill), np.full(n_fill, 40.0)], axis=1)
    tail = _rows(p, seed=9)[:n_tail]
    map_world = np.concatenate([fill, body, body[::-1], tail]).astype(np.float32)
    pose = np.array([[0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]])
    q = body[:4000].astype(np.float32)
    m = capi.Map(map_world)
    h = capi.Handle(p)
    h.attach_map(m)
    h.process_nodes(pose, q, np.array([0, len(q)], dtype=np.uint64))
    voi, _ = oracle_mod.fetch_voi(map_world, pose[0], p.max_range)
    o = oracle_mod.Oracle(p)
    o.run(voi, q)
    for which in (0, 1):
        _, mn, mx, cnt = h.get_bins(which, per_point=False)
        omn, omx, ocnt, _ = o.bins(which)
        assert np.array_equal(cnt, ocnt), f"{name} cloud {which}: counts differ in {np.count_nonzero(cnt != ocnt)} bins"
        occ = ocnt > 0
        assert np.array_equal(mn[occ].astype(np.float64), omn[occ]) and np.array_equal(mx[occ].astype(np.float64), omx[occ])
        assert np.all(np.isnan(mn[~occ])) and np.all(np.isnan(mx[~occ]))
    nv, _, _ = h.node_stats()
    assert nv[0] == len(voi)                   # every VoI point counted once: binned + outside the z window
    h.close()
    m.close()
