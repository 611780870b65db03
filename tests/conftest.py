import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def built_lib():
    """The in-tree C-ABI library (built by __graft_entry__.build() / yolosharp_b200.build())."""
    import yolosharp_b200
    path = yolosharp_b200.build()
    assert os.path.exists(path)
    return path
