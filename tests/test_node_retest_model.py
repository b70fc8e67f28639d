"""CPU checks of the node-mode re-test model (tests/node_retest_model.py: retest_map, retest_keep; DESIGN.md section 8.4.1): the
re-test map and its extents against a hand-built concatenation, the empty store, the prefix rule on the shared workload, and
the re-test rejecting dynamic points that one-pass inserts put back."""
import numpy as np
import pytest

from erasor_b200 import params as P

import node_inserts_model as NI
import node_retest_model as NR


def _nodes(small_workload, picks):
    scene = small_workload["scene"]
    poses = np.stack([scene.pose7(small_workload["frames"][i][2]) for i in picks]).astype(np.float64)
    return poses, [small_workload["frames"][i][1] for i in picks]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).reshape(-1, 4).view(np.uint32)


def _cloud(rng, n):
    return np.concatenate([rng.uniform(-30, 30, (n, 3)), rng.integers(0, 260, (n, 1))], axis=1).astype(np.float32)


@pytest.mark.parametrize("case", ["mixed", "empty store", "no nodes", "all rejected", "nodes without inserts", "all kept"])
def test_retest_map_is_the_concatenation(case):
    rng = np.random.default_rng(3)
    mw = _cloud(rng, 500)
    keep = (rng.random(500) < 0.7).astype(np.uint8)
    sizes = {"mixed": [5, 0, 17, 3], "empty store": [0, 0, 0], "no nodes": [], "all rejected": [4, 9],
             "nodes without inserts": [0, 6, 0, 0, 2, 0], "all kept": [1, 2]}[case]
    if case == "all rejected":
        keep[:] = 0
    if case == "all kept":
        keep[:] = 1
    ins = [_cloud(rng, k) for k in sizes]
    M2, ext = NR.retest_map(mw, keep, ins)
    kept = [mw[i] for i in range(len(mw)) if keep[i]]
    want = np.array(kept + [p for x in ins for p in x], dtype=np.float32).reshape(-1, 4)
    assert np.array_equal(_bits(M2), _bits(want))
    want_ext, at = [], len(kept)
    for x in ins:
        want_ext.append(at)
        at += len(x)
    assert ext.dtype == np.uint64 and ext.tolist() == want_ext
    if case == "nodes without inserts":
        assert (np.diff(ext) == 0).any()


def test_empty_store_is_the_plain_node_mask_over_the_kept_map(oracle_mod, small_workload):
    """no inserts: every node sees all of M[keep1], so the re-test is plain node mode over M[keep1]"""
    p = P.preset("seq_05").replace(skip_voxelize=1)
    mw = small_workload["map_world"]
    poses, qs = _nodes(small_workload, range(6))
    _, _, fk = NI.node_inserts(oracle_mod, p, mw, poses, qs)
    keep1 = fk.min(axis=0)
    M2, ext = NR.retest_map(mw, keep1, [np.zeros((0, 4), np.float32)] * len(qs))
    assert (ext == np.count_nonzero(keep1)).all() and len(M2) == np.count_nonzero(keep1)
    _, _, fk2 = NI.node_inserts(oracle_mod, p, M2, poses, qs)
    assert np.array_equal(NR.retest_keep(oracle_mod, p, M2, ext, poses, qs), fk2.min(axis=0))


@pytest.mark.parametrize("version,skip", [(2, 1), (3, 1), (3, 0)])
def test_no_node_sees_its_own_or_later_inserts(oracle_mod, small_workload, version, skip):
    """node j's prefix ends where its own inserts start: it holds M[keep1] and the inserts of nodes k < j only"""
    p = P.preset("seq_05").replace(version=version, skip_voxelize=skip)
    mw = small_workload["map_world"]
    poses, qs = _nodes(small_workload, range(6))
    ins, off, fk = NI.node_inserts(oracle_mod, p, mw, poses, qs)
    keep1 = fk.min(axis=0)
    per_node = [ins[int(off[j]):int(off[j + 1])] for j in range(len(qs))]
    M2, ext = NR.retest_map(mw, keep1, per_node)
    n_kept = int(np.count_nonzero(keep1))
    assert off[-1] > 0
    for j in range(len(qs)):
        assert int(ext[j]) == n_kept + int(off[j])
        assert np.array_equal(_bits(M2[:n_kept]), _bits(mw[keep1 != 0]))
        assert np.array_equal(_bits(M2[n_kept:int(ext[j])]), _bits(ins[:int(off[j])])), f"node {j} sees inserts of itself or later"
        assert np.array_equal(_bits(M2[int(ext[j]):int(ext[j]) + len(per_node[j])]), _bits(per_node[j]))


@pytest.mark.parametrize("name", ["seq_05", "seq_00"])
def test_retest_rejects_dynamic_inserts(oracle_mod, small_workload, name):
    """on the shared workload, one-pass inserts put dynamic-labelled query points (252..259) back into the map; the re-test,
    where later nodes see them, rejects at least one.  Version 2, whose MERGE_BINS and query-only bins insert far more than
    R-GPF's bins: with version 3 the six nodes (eight scans apart) reject none of their dynamic inserts."""
    p = P.preset(name).replace(version=2, skip_voxelize=1)
    mw = small_workload["map_world"]
    poses, qs = _nodes(small_workload, range(6))
    ins, off, fk = NI.node_inserts(oracle_mod, p, mw, poses, qs)
    keep1 = fk.min(axis=0)
    M2, ext = NR.retest_map(mw, keep1, [ins[int(off[j]):int(off[j + 1])] for j in range(len(qs))])
    keep2 = NR.retest_keep(oracle_mod, p, M2, ext, poses, qs)
    n_kept = int(np.count_nonzero(keep1))
    lab = M2[:, 3]
    dyn_ins = np.zeros(len(M2), dtype=bool)
    dyn_ins[n_kept:] = (lab[n_kept:] >= 252) & (lab[n_kept:] <= 259)
    assert dyn_ins.any(), "one-pass inserts keep no dynamic point on this workload"
    assert (keep2[dyn_ins] == 0).any()
    # the last node's inserts are seen by no node: the re-test cannot remove them
    assert (keep2[int(ext[-1]):] == 1).all()
