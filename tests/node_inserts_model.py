"""Node-mode inserts built from the oracle alone (test infrastructure).

For one node (map, pose, body-frame query) the oracle's fetch_voi + ERASOR give arranged (r_pod2pc of r_pod_selected, then the
ground_viz tail), the complement and the rejected map points.  inserted_f is what the static estimate holds beyond the map points
the frame's keep mask keeps, bin by bin in r_pod2pc order:
  - a bin that ran R-GPF (the oracle's planes): bin_curr then its ground (version 3 without skip_voxelize: voxelize_preserving_labels
    of that at map_voxel_size);
  - version 2, MERGE_BINS: bin_curr (its map points are kept anyway); a bin with query points only: bin_curr;
  - every other bin: nothing (its selected points are bin_map).
frame_inserts also checks that arranged is exactly that sequence of per-bin selections and that, as multisets,
arranged + complement == map_voi[frame_keep] + inserted.  The inserts are then moved body -> origin as the updater's
body2origin does (transform by pose_to_matrix(pose))."""
import numpy as np

MERGE_BINS = 0.25


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 4).view(np.uint32)


def same_multiset(a, b) -> bool:
    a, b = _bits(a), _bits(b)
    if len(a) != len(b):
        return False
    sa = a[np.lexsort(a.T[::-1])]
    sb = b[np.lexsort(b.T[::-1])]
    return np.array_equal(sa, sb)


def frame_inserts(oracle_mod, p, map_world, pose7, q, voi_range=None):
    """-> (inserted in the map frame, frame keep mask over map_world) of one node; asserts the identity above."""
    q = np.ascontiguousarray(q, dtype=np.float32).reshape(-1, 4)
    voi, idx = oracle_mod.fetch_voi(map_world, pose7, p.max_range if voi_range is None else voi_range)
    o = oracle_mod.Oracle(p)
    o.run(voi, q)
    B = p.num_rings * p.num_sectors
    bm, bq = o.bin_of_point(0), o.bin_of_point(1)
    cq = np.bincount(bq[bq >= 0], minlength=B)
    cm = np.bincount(bm[bm >= 0], minlength=B)
    st, _ = o.status()
    flagged = {pl["bin"] for pl in o.planes()}
    arr, _ = o.cloud(o.ARRANGED)
    comp, _ = o.cloud(o.COMPLEMENT)
    gv, gsrc = o.cloud(o.GROUND_VIZ)
    _, rej = o.cloud(o.MAP_REJECTED)
    g_bin = bm[gsrc] if len(gsrc) else np.zeros(0, dtype=np.int32)
    vox = p.version == 3 and not p.skip_voxelize
    q_of = {b: q[bq == b] for b in np.unique(bq[bq >= 0])}
    m_of = {b: voi[bm == b] for b in np.unique(bm[bm >= 0])}
    empty = np.zeros((0, 4), dtype=np.float32)
    parts, pos = [], 0
    for b in range(B):
        qp, mp = q_of.get(b, empty), m_of.get(b, empty)
        ins = None
        if b in flagged:
            cur = np.concatenate([qp, gv[g_bin == b]])
            sel = ins = oracle_mod.voxelize(cur, p.map_voxel_size) if vox else cur
        elif p.version == 2 and p.minimum_num_pts >= 0 and cq[b] >= p.minimum_num_pts and cq[b] > 0 and st[b] == MERGE_BINS:
            sel, ins = np.concatenate([qp, mp]), qp
        elif p.version == 2 and p.minimum_num_pts >= 0 and cq[b] >= p.minimum_num_pts and cq[b] > 0 and cm[b] == 0:
            sel = ins = qp
        else:
            sel = mp
        assert np.array_equal(_bits(arr[pos:pos + len(sel)]), _bits(sel)), f"arranged differs from the model in bin {b}"
        pos += len(sel)
        if ins is not None and len(ins):
            parts.append(ins)
    assert np.array_equal(_bits(arr[pos:]), _bits(gv)), "arranged's tail is not ground_viz"
    inserted = np.concatenate(parts) if parts else empty
    keep_voi = np.ones(len(voi), dtype=bool)
    keep_voi[rej] = False
    assert same_multiset(np.concatenate([arr, comp]), np.concatenate([voi[keep_voi], inserted])), "arranged + complement != kept VoI + inserts"
    fk = np.ones(len(map_world), dtype=np.uint8)
    fk[idx[rej]] = 0
    return oracle_mod.transform(inserted, oracle_mod.pose_to_matrix(pose7)), fk


def node_inserts(oracle_mod, p, map_world, poses, qs, voi_range=None):
    """-> (every node's inserts concatenated in node order, uint64 offsets [F+1], frame keep masks [F][n])"""
    outs, fks = [], []
    for pose, q in zip(poses, qs):
        ins, fk = frame_inserts(oracle_mod, p, map_world, pose, q, voi_range)
        outs.append(ins)
        fks.append(fk)
    off = np.cumsum([0] + [len(x) for x in outs]).astype(np.uint64)
    return np.concatenate(outs) if outs else np.zeros((0, 4), np.float32), off, np.stack(fks)


def saved_map(oracle_mod, map_world, keep, inserts, leaf):
    """node mode's saved map with inserts: voxelize_preserving_labels(map[keep] ++ inserts of every node, in node order)"""
    kept = np.ascontiguousarray(map_world, dtype=np.float32)[np.asarray(keep) != 0]
    return oracle_mod.voxelize(np.concatenate([kept, np.ascontiguousarray(inserts, dtype=np.float32).reshape(-1, 4)]), leaf)
