import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

# the reference's published counterexample (TLC `dumpTrace tlc` text of VSR.tla, README constants), gzip-compressed
REF_TRACE = os.path.join(ROOT, "tests", "golden", "state_transfer_violation_trace.txt.gz")
# the reference's shipped TLC configuration, vsr-revisited/paper/VSR.cfg
REF_CFG = os.path.join(ROOT, "tests", "golden", "VSR.cfg")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def pkg():
    """The product package; builds the native library if it is missing."""
    import _pkg
    so = os.path.join(ROOT, "vsr-tlaplus_b200", "libvsr_b200.so")
    if not os.path.exists(so) or not os.path.exists(os.path.join(ROOT, "oracle", "_build", "liboracle.so")):
        import __graft_entry__
        __graft_entry__.build()
    return _pkg.load()

