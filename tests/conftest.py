import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def lib():
    from splatt_b200 import _abi
    return _abi.load()


@pytest.fixture(scope="session")
def refmod():
    """The compiled, unmodified reference (oracle/_ref).  Skips when it was not built."""
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
    ref.load()
    return ref
