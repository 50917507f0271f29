import os
import sys
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


import torch
torch.set_num_threads(min(8, os.cpu_count() or 1))   # the CPU oracle oversubscribes a 128-core box


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a machine without a CUDA device skips the gpu tests instead of failing in them."""
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def rel_rms(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.sqrt(np.mean((a - b) ** 2)) / (np.sqrt(np.mean(b ** 2)) + 1e-30))


@pytest.fixture(scope="session")
def states():
    """Seeded synthetic checkpoints (same seed as tests/golden/make_golden.py)."""
    from voicefixer_b200 import synthetic
    return synthetic.make_analysis_state(0), synthetic.make_vocoder_state(1)


@pytest.fixture(scope="session")
def engine(states):
    from voicefixer_b200.engine import Engine
    return Engine(states[0], states[1], precision="fp32")
