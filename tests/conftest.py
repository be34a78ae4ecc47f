"""pytest configuration: registers the `gpu` marker and makes the repo importable.

`-m "not gpu"` runs here on CPU (oracle vs the reference's own scenarios, host logic, ABI symbols);
`-m gpu` runs on an H100 and compares the CUDA path (through the C ABI) with the oracle.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
TESTS = os.path.dirname(os.path.abspath(__file__))
if TESTS not in sys.path:
    sys.path.insert(0, TESTS)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def pcdn():
    """The product package (push-cdn_b200/), loaded under the importable name push_cdn_b200."""
    import __graft_entry__ as ge

    return ge.load_package()
