import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "semantic-segmentation_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def golden():
    import torch
    return torch.load(os.path.join(ROOT, "tests", "golden", "reference_outputs.pt"), map_location="cpu")
