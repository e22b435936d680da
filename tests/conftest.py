import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def engine():
    import grok_b200
    eng = grok_b200.Engine(0)
    yield eng
    eng.close()
