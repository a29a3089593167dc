import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session", autouse=True)
def _native_libs():
    """Build the product .so and the oracle before any test (no-ops when up to date)."""
    from zstdmt_b200 import build as b
    b.build_product()
    b.build_harness()
    b.build_oracle()
