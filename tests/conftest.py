import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")
    if os.environ.get("B200TIMG_CUSIM"):      # developer aid: replay the GPU tests on tools/cusim (no GPU needed)
        from tools import cusim
        cusim.activate()


@pytest.fixture(scope="session")
def ctx():
    """A b200timg context on cuda:0.  Fails loudly (no CPU fallback) if unavailable."""
    import timg_b200
    c = timg_b200.Context(0)
    yield c
    c.close()
