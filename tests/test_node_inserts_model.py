"""CPU checks of the node-mode insert model (tests/node_inserts_model.py) against the oracle: for every node of the shared
workload, arranged is the model's per-bin selection and arranged + complement == kept VoI + inserts, bit for bit."""
import glob
import os

import numpy as np
import pytest

from erasor_b200 import params as P

import node_inserts_model as NI

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "*.npz")))
IDENTITY = np.array([0, 0, 0, 0, 0, 0, 1], dtype=np.float64)


def golden_node(path):
    """(params, map, pose, query) of a golden frame as one node: its map VoI is the map, at the identity pose"""
    z = np.load(path, allow_pickle=True)
    p = P.preset(str(z["preset"])).replace(**{k: int(v) for k, v in z["overrides"]})
    return p, z["map_voi"], IDENTITY, z["query_voi"]


def _nodes(small_workload, picks):
    scene = small_workload["scene"]
    poses = np.stack([scene.pose7(small_workload["frames"][i][2]) for i in picks]).astype(np.float64)
    return poses, [small_workload["frames"][i][1] for i in picks]


@pytest.mark.parametrize("name", ["seq_05", "seq_00", "synthetic_40x360"])
@pytest.mark.parametrize("version,skip", [(3, 0), (3, 1), (2, 1)])
def test_identity_every_node(oracle_mod, small_workload, name, version, skip):
    p = P.preset(name).replace(version=version, skip_voxelize=skip)
    poses, qs = _nodes(small_workload, range(6))
    ins, off, fk = NI.node_inserts(oracle_mod, p, small_workload["map_world"], poses, qs)
    assert off[-1] == len(ins) and len(off) == 7
    assert off[-1] > 0, "the workload must insert something"
    assert (fk == 0).any()


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(f) for f in GOLDEN])
def test_identity_golden(oracle_mod, path):
    p, mw, pose, q = golden_node(path)
    ins, fk = NI.frame_inserts(oracle_mod, p, mw, pose, q)
    assert len(ins) > 0 and (fk == 0).any()


def test_version2_inserts_merged_and_query_only_bins(oracle_mod, small_workload):
    """version 2 inserts more than its R-GPF bins: the bins of MERGE_BINS and query-only bins add their bin_curr"""
    p = P.preset("seq_05").replace(version=2, skip_voxelize=1)
    poses, qs = _nodes(small_workload, [2])
    ins2, _ = NI.frame_inserts(oracle_mod, p, small_workload["map_world"], poses[0], qs[0])
    ins3, _ = NI.frame_inserts(oracle_mod, p.replace(version=3), small_workload["map_world"], poses[0], qs[0])
    assert len(ins2) > len(ins3)


def test_saved_map_definition(oracle_mod, small_workload):
    p = P.preset("seq_05")
    mw = small_workload["map_world"]
    poses, qs = _nodes(small_workload, range(3))
    ins, off, fk = NI.node_inserts(oracle_mod, p, mw, poses, qs)
    keep = fk.min(axis=0)
    plain = oracle_mod.voxelize(mw[keep != 0], p.map_voxel_size)
    assert np.array_equal(NI.saved_map(oracle_mod, mw, keep, np.zeros((0, 4), np.float32), p.map_voxel_size), plain)
    assert len(NI.saved_map(oracle_mod, mw, keep, ins, p.map_voxel_size)) > len(plain)
