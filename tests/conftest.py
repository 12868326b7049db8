import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (H100); run with -m gpu")


@pytest.fixture(scope="session")
def golden():
    import torch

    cache = {}

    def load(name):
        if name not in cache:
            cache[name] = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
        return cache[name]

    return load
