import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_sessionstart(session):
    """A fresh checkout has no built libraries (they are git-ignored): build them once.  When they
    exist nothing is rebuilt here -- `__graft_entry__.build()` is the explicit build step."""
    needed = [os.path.join(ROOT, "scanner_b200", "lib", n) for n in
              ("libscn_kernels.so", "libscn_engine.so", "libscn_stdlib.so")] + [os.path.join(ROOT, "oracle", "liborc.so")]
    if not all(os.path.exists(p) for p in needed):
        import __graft_entry__
        __graft_entry__.build()


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
