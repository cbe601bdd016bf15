import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with `-m gpu`)")


@pytest.fixture(scope="session")
def built():
    """Native pieces (CUDA library, oracle, hostsim) built in-tree once per session."""
    import __graft_entry__ as g
    if not os.path.exists(os.path.join(ROOT, "rigidbodydynamics", "jl_b200", "csrc", "librbd_b200.so")):
        g.build()
    return True
