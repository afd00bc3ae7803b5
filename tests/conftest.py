import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA (sm_90, H100) device; run with `-m gpu` on an H100")


@pytest.fixture(scope="session")
def golden():
    import torch

    return torch.load(ROOT / "tests" / "golden" / "flux_step_golden.pt")
