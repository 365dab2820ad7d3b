import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) GPU; run with `-m gpu`")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")


def has_h100():
    try:
        import torch
        return torch.cuda.is_available() and torch.cuda.get_device_capability(0) == (9, 0)
    except Exception:
        return False
