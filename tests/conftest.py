import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


def load_golden(name):
    import torch

    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.fixture(scope="session")
def golden():
    return load_golden
