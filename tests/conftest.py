import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from tests import oracle_lib
    return oracle_lib.load()


@pytest.fixture(scope="session")
def engine_cls():
    """The product engine class; building the .so here is a no-op when it is already built."""
    import __graft_entry__ as g
    g.build()
    import fgumi_b200
    return fgumi_b200.Engine


@pytest.fixture(scope="session")
def fg():
    """The product package with its library built (modules may define their own `fg` with extra set-up)."""
    import __graft_entry__ as g
    g.build()
    import fgumi_b200
    return fgumi_b200
