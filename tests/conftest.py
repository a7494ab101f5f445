"""pytest configuration: marker registration, repo-root import path, shared helpers."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)


def rel_peak_err(a, b):
    """Per-item max|a-b| / max|b| over all non-batch dims (SURVEY.md section 8c metric)."""
    import torch

    a = torch.as_tensor(a).double()
    b = torch.as_tensor(b).double()
    bs = b.shape[0]
    num = (a - b).reshape(bs, -1).abs().amax(dim=1)
    den = b.reshape(bs, -1).abs().amax(dim=1).clamp_min(1e-30)
    return num / den


@pytest.fixture(scope="session")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
