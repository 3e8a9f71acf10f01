import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def dbx_lib():
    """libdbx must be built in-tree; the GPU tests never fall back to anything else."""
    from databend_b200 import build, lib
    build.build()
    return lib.load()


@pytest.fixture(scope="session")
def gpu(dbx_lib):
    from databend_b200 import lib
    n = lib.require_device()  # raises DbxError loudly when there is no GPU
    return n
