"""The node-mode re-test (DESIGN.md section 8.4.1) built from the oracle alone (test infrastructure).

Pass 1 is node mode with inserts on (tests/node_inserts_model.py): keep1 over the initial map M and every node's inserts I_j.
Pass 2 runs the same nodes against the re-test map M2 = M[keep1] ++ I_0 ++ I_1 ++ ..., node j seeing the prefix
M2[:extents[j]] -- the kept map and the inserts of the nodes before it -- and keep2 is the AND over nodes of their keep masks
over that prefix (1 beyond it)."""
import numpy as np


def retest_map(map_world, keep1, inserts_per_node):
    """-> (M2, extents): M2 = map_world[keep1 != 0] ++ the inserts of node 0, node 1, ...; node j sees M2[:extents[j]]"""
    kept = np.ascontiguousarray(map_world, dtype=np.float32).reshape(-1, 4)[np.asarray(keep1) != 0]
    parts = [np.ascontiguousarray(x, dtype=np.float32).reshape(-1, 4) for x in inserts_per_node]
    sizes = np.array([len(x) for x in parts], dtype=np.uint64)
    extents = (len(kept) + np.concatenate([[0], np.cumsum(sizes)[:-1]]) if len(parts) else np.zeros(0)).astype(np.uint64)
    return np.concatenate([kept] + parts), extents


def node_keep(oracle_mod, p, map_world, pose7, q, voi_range=None):
    """one node's keep mask over map_world: the oracle's fetch_voi + ERASOR, 1 outside the VoI"""
    voi, idx = oracle_mod.fetch_voi(map_world, pose7, p.max_range if voi_range is None else voi_range)
    o = oracle_mod.Oracle(p)
    o.run(voi, np.ascontiguousarray(q, dtype=np.float32).reshape(-1, 4))
    _, rej = o.cloud(o.MAP_REJECTED)
    fk = np.ones(len(map_world), dtype=np.uint8)
    fk[idx[rej]] = 0
    return fk


def retest_keep(oracle_mod, p, M2, extents, poses, qs, voi_range=None):
    """pass 2: AND over nodes j of node j's keep mask over M2[:extents[j]] (1 beyond the prefix)"""
    keep = np.ones(len(M2), dtype=np.uint8)
    for e, pose, q in zip(extents, poses, qs):
        e = int(e)
        keep[:e] &= node_keep(oracle_mod, p, M2[:e], pose, q, voi_range)
    return keep
