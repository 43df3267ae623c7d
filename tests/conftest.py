import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the shared objects once per session (the .so files travel with the snapshot,
    so on the GPU box this is a no-op unless something is stale)."""
    import __graft_entry__ as entry

    entry.build_library()
    entry.build_hostsim()
    from oracle import oracle

    oracle.build()


def pytest_collection_modifyitems(session, config, items):
    """GPU run order: the hot path's parity tests first, then the FASTQ path, then the late additions -- with -x a
    failure in a later layer must not hide the state of the core."""
    rank = {"test_gpu_parity.py": 0, "test_gpu_fastq.py": 1, "test_gpu_z_more_goldens.py": 2}
    items.sort(key=lambda it: rank.get(os.path.basename(str(it.fspath)), -1))
