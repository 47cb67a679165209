import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(__file__))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def ref():
    """The compiled reference (oracle/_ref), built by build() where the reference tree is readable."""
    from oracle import ref as _ref
    if not _ref.available():
        pytest.skip("oracle/_ref/libmrcal_ref.so not built (needs the reference tree: make -C oracle ref)")
    return _ref
