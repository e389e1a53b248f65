import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def built():
    import __graft_entry__ as g
    g.build()
    return True


@pytest.fixture(scope="session")
def oracle_mod(built):
    from oracle import oracle
    oracle.lib()
    return oracle
