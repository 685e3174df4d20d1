import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_outputs.pt")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        # a GPU test that deadlocks (spin-wait protocols, graph capture) must fail with a stack dump, not stall the whole suite:
        # pytest-timeout's "thread" method also fires while the main thread sits inside a CUDA synchronise
        if config.pluginmanager.hasplugin("timeout"):
            for it in items:
                if "gpu" in it.keywords and it.get_closest_marker("timeout") is None:
                    it.add_marker(pytest.mark.timeout(300, method="thread"))
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def reference_outputs():
    """Outputs of the reference implementation for the differential tests' seeded inputs (scripts/make_reference_golden.py)."""
    import torch
    return torch.load(GOLDEN, weights_only=False)
