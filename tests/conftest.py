"""pytest configuration: registers the `gpu` marker and shares the synthetic workloads.

`-m "not gpu"`: oracle vs its invariants / numpy restatement / golden fixtures, host logic, C-ABI symbols.
`-m gpu`     : the parity tests proper -- CUDA path through the C ABI vs the oracle.
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def small_workload():
    """One accumulated map + 6 frames, low-resolution lidar so the CPU oracle stays fast."""
    from erasor_b200 import synth
    return synth.make_frames(seed=5, n_frames=6, preset_max_range=80.0, n_map_nodes=41, n_beams=32, n_az=900)


@pytest.fixture(scope="session")
def oracle_mod():
    from oracle import oracle_py
    oracle_py.build()
    return oracle_py


def has_cuda() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False
