import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests are skipped (not failed) on a box without a CUDA device, whatever fixtures they use."""
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def kernels():
    """The product's CUDA backend; only for -m gpu tests."""
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from torcheasyrec_b200.kernels import default_kernels

    return default_kernels()
