import os
import sys

import pytest

# the peer-history emulation tests run up to 8 emulated ranks on concurrent streams of one GPU: give every stream its own
# hardware queue (must be set before the CUDA context exists)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
# ... and load every kernel when the library is loaded: with lazy loading the FIRST launch of a kernel synchronises the
# context, which dead-locks (until the 2 s peer time-out) while another emulated rank's wait kernel is spinning
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "hybrid-rendering_b200"))
sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Make sure the oracle / product / synth libraries exist (build here when a toolchain is around)."""
    import __graft_entry__ as ge
    ge.ensure_built()
    yield
