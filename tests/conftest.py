import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def built():
    """Make sure the extension and the oracle are built (no-op when fresh)."""
    import __graft_entry__ as ge
    if not os.path.exists(ge.LIB) or not os.path.exists(os.path.join(ROOT, "oracle", "liboracle.so")):
        ge.build()
    return True


@pytest.fixture(scope="session")
def encoder(built):
    import mozjpeg_b200 as mj
    enc = mj.Encoder(0)
    yield enc
    enc.close()
