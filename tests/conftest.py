import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

GOLDEN = os.path.join(REPO, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on a GPU machine")


def pytest_collection_modifyitems(config, items):
    """GPU tests are skipped (not failed) when no device is visible and they were not deselected."""
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(autouse=True)
def _restore_ops():
    """Every test starts and ends on the product op path."""
    from tokenflow_b200 import tokenflow_utils as tfu
    tfu._install_ops_for_testing(None)
    yield
    tfu._install_ops_for_testing(None)
