import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests skip (instead of erroring in a fixture) on a box without a CUDA device, so a plain `pytest tests`
    is clean on a CPU box.  On a GPU box a missing library is NOT a skip: the tests then fail loudly."""
    try:
        import torch

        have_gpu = torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def load_golden(name):
    import torch

    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.fixture(autouse=True)
def _seed_per_test(request):
    """Every test draws from its own fixed random stream: rounding-boundary statistics (fractions of bit-equal
    outputs) are then the same on every run."""
    import zlib

    import torch

    torch.manual_seed(zlib.crc32(request.node.nodeid.encode()) & 0x7FFFFFFF)
    yield
