import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(REPO, "tests", "golden")


@pytest.fixture(autouse=True)
def _exact_fp32_references():
    """The fp32 torch restatements the GPU tests compare against must BE fp32: torch lets cuDNN convolutions (and optionally matmuls)
    run in TF32 by default, which would put ~1e-3 of noise into the "truth"."""
    import torch
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
