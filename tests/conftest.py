import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


def find_fixture(name):
    """GGUF fixtures are the upstream project's test models; __graft_entry__.build() copies them (git-ignored) into
    oracle/_ref/testdata (oracle/fixtures.py)."""
    p = os.path.join(ROOT, "oracle", "_ref", "testdata", name)
    return p if os.path.exists(p) else None


@pytest.fixture
def fixture_path():
    def _get(name):
        p = find_fixture(name)
        if p is None:
            pytest.skip(f"fixture {name} not available (run __graft_entry__.build() with an upstream crabml checkout, see oracle/fixtures.py)")
        return p
    return _get
