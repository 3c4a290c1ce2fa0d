import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for p_ in (ROOT, HERE):
    if p_ not in sys.path:
        sys.path.insert(0, p_)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU (H100)")


@pytest.fixture(scope="session")
def ctx():
    import rawspeed_b200 as rs
    c = rs.Context(0)
    yield c
    c.close()
