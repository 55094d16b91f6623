import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a; run with -m gpu on a machine that has one)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 GPUs (subset of gpu)")


@pytest.fixture(scope="session")
def native():
    """The product library; building is __graft_entry__.build()'s job, tests only load it."""
    from kukeon_b200 import gpupool
    if not os.path.exists(gpupool.lib_path()):
        import __graft_entry__ as g
        g.build()
    return gpupool.lib()


@pytest.fixture(scope="session")
def coracle():
    from oracle import coracle as co
    co.build()
    co.lib()
    return co


def _gpu_count():
    try:
        import torch
        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        return 0


@pytest.fixture(scope="session")
def gpu_count():
    return _gpu_count()


@pytest.fixture(scope="session")
def pool(native):
    """One single-device context for the whole GPU session (pinned-buffer allocation is slow)."""
    from kukeon_b200 import gpupool
    p = gpupool.Pool([0], n_staging_buffers=4, staging_buffer_bytes=8 << 20, n_reader_threads=2)
    yield p
    p.close()
