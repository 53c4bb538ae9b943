"""pytest configuration: registers the `gpu` marker and puts the repo root on sys.path.

`-m "not gpu"` (CPU, build container): oracle vs golden vectors, host logic, C-ABI symbol
checks, world_size-2 gloo tests.   `-m gpu` (H100): CUDA path vs oracle / goldens.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def load_golden(name):
    import numpy as np

    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)
