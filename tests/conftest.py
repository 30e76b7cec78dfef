import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "clip.cpp_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); run with `-m gpu` on a machine that has one")
    config.addinivalue_line("markers", "slow: full-size geometries")


@pytest.fixture(scope="session")
def prod():
    import __graft_entry__ as ge
    import binding as bd
    if not os.path.exists(bd.PRODUCT_LIB):
        ge.build()
    return bd.ClipLib(bd.PRODUCT_LIB)
