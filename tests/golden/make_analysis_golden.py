"""Generates tests/golden/analysis_runner_*_stdout.txt: the reference's scripts/analysis_runner.py stdout, run unchanged on two
pairs of clouds written with erasor_b200.evaluate.write_pcd_ascii as gt.pcd / est.pcd in one directory (the script prints the
paths it is given, so it runs from that directory with the relative names):
  seed41           the clouds of tests/test_evaluate.py::run_pass (the oracle's seed-41 pass)
  seed41_jittered  the same GT; the estimate jittered by up to 0.3 m plus 300 of its points moved 1 km away
                   (tests/test_eval_overlap_model.py::jittered_estimate), so the distance percentiles are not zero
Only this script reads the reference checkout; run it by hand on a CPU machine from the repo root:
    python tests/golden/make_analysis_golden.py /path/to/reference
"""
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from erasor_b200 import evaluate as E  # noqa: E402
from oracle import oracle_py  # noqa: E402
from test_eval_grid_model import seed41_pass  # noqa: E402
from test_eval_overlap_model import GOLDEN_STDOUT, jittered_estimate  # noqa: E402


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    runner = os.path.join(ref, "scripts", "analysis_runner.py")
    oracle_py.build()
    gt, est = seed41_pass(oracle_py)
    for name, (g, e) in {"seed41": (gt, est), "seed41_jittered": (gt, jittered_estimate(est))}.items():
        with tempfile.TemporaryDirectory() as d:
            E.write_pcd_ascii(os.path.join(d, "gt.pcd"), g)
            E.write_pcd_ascii(os.path.join(d, "est.pcd"), e)
            out = subprocess.run([sys.executable, runner, "--gt", "gt.pcd", "--est", "est.pcd"], cwd=d, check=True,
                                 capture_output=True, text=True).stdout
        with open(GOLDEN_STDOUT[name], "w") as f:
            f.write(out)
        print(name, len(g), len(e))
        print(out, end="")


if __name__ == "__main__":
    main()
