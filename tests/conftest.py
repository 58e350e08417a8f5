import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    import torch

    def load(name):
        return torch.load(os.path.join(GOLDEN, name + ".pt"), map_location="cpu", weights_only=True)

    return load
