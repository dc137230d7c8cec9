import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "stable-diffusion-xl-burn_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); select with -m gpu")


@pytest.fixture(scope="session")
def ctx():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import sdxl_b200
    c = sdxl_b200.Context(0)
    yield c
    c.close()
