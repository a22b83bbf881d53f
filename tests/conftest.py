import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def built_lib():
    """Build (if stale) and load the C-ABI library; CPU tests only check that it loads and exports."""
    import __graft_entry__ as ge
    ge.build()
    from shine_mapping_b200 import _abi
    return _abi.lib()
