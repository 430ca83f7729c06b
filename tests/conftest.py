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
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        have_gpu = False
    # a GPU test that deadlocks (a device-side wait that never returns blocks the host in a CUDA call) must not take the whole
    # session with it for longer than this: pytest-timeout's thread method ends the process (default per-test budget, overridable)
    have_timeout = config.pluginmanager.hasplugin("timeout") and not config.getoption("timeout", None)
    for it in items:
        if have_timeout and "gpu" in it.keywords and it.get_closest_marker("timeout") is None:
            it.add_marker(pytest.mark.timeout(300, method="thread"))
        if "gpu" in it.keywords and not have_gpu:
            it.add_marker(pytest.mark.skip(reason="no CUDA device"))


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
