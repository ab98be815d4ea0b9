"""pytest configuration: ``gpu`` marker = needs a real H100; everything else runs on CPU."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (sm_90a)")


@pytest.fixture(scope="session")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("gpu-marked test started without a CUDA device")
    return torch.device("cuda", 0)
