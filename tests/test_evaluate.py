"""CPU suite: the PR/RR port (erasor_b200/evaluate.py) against the reference's own scripts/analysis_runner.py on oracle output
(the script's table for these clouds is stored in tests/golden/analysis_runner_seed41.json)."""
import json
import os

import pytest

from erasor_b200 import evaluate as E
from erasor_b200 import params as P
from erasor_b200 import synth

REF_TABLE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "analysis_runner_seed41.json")


@pytest.fixture(scope="module")
def run_pass(oracle_mod):
    sc = synth.Scene(seed=41, length=40.0, n_nodes=17, n_dynamic=6)
    kw = dict(n_beams=24, n_az=480)
    nodes = list(range(17))
    m = sc.build_map(nodes, voxel=0.2, **kw)
    ep, up = P.preset("seq_05"), P.updater_preset("seq_05")
    up.removal_interval = 2
    o = oracle_mod.OracleUpdater(up, ep, m)
    for k in nodes:
        o.callback_node(k, sc.pose7(k), sc.scan(k, seed_offset=3, **kw))
    est = o.save_static_map(0.2)
    return m, est


def test_pr_rr_moves_the_right_way(run_pass):
    gt, est = run_pass
    before = E.evaluate(gt, gt)
    after = E.evaluate(gt, est)
    assert before["PR"] == 100.0 and before["RR"] == 0.0
    assert after["RR"] > 30.0 and after["PR"] > 80.0, after      # the pass erases dynamic trails and keeps most static points


def test_matches_reference_script(tmp_path, run_pass):
    gt, est = run_pass
    gp, ep_ = str(tmp_path / "gt.pcd"), str(tmp_path / "est.pcd")
    E.write_pcd_ascii(gp, gt)
    E.write_pcd_ascii(ep_, est)
    ref = json.load(open(REF_TABLE))
    assert (len(gt), len(est)) == (ref["gt_points"], ref["est_points"]), "the pass no longer produces the clouds the table was made from"
    mine = E.evaluate(E.read_pcd_ascii(gp), E.read_pcd_ascii(ep_))
    t = ref["table"]
    assert (mine["gt_static"], mine["gt_dynamic"], mine["preserved_static"], mine["preserved_dynamic"]) == (t["gt_S"], t["gt_D"], t["kept_S"], t["kept_D"])
    # the script prints PR / RR with 3 decimals, F1 with 4
    assert abs(mine["PR"] - t["PR%"]) < 2e-3 and abs(mine["RR"] - t["RR%"]) < 2e-3, (mine, t)
    assert abs(mine["F1"] - t["F1"]) < 2e-4, (mine, t)
