import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def _have_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _have_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def built():
    """Build everything once per session (a no-op when the .so files are fresh)."""
    import __graft_entry__ as g
    g.build()
    return True


@pytest.fixture(scope="session")
def cpu_oracle(built):
    from oracle import refbind
    o = refbind.CpuOracle()
    o.lib.ktoracle_set_threads(min(8, os.cpu_count() or 1))
    return o


GOLDEN = os.path.join(ROOT, "tests", "golden")
