import os
import sys

import pytest

# The CPU oracle's OpenMP sections scale to ~32 threads; on a 128-core GPU box the runtime's default (one thread per core) makes the
# many short parallel regions slower, not faster.  Read by libgomp when the oracle library is loaded.
os.environ.setdefault("OMP_NUM_THREADS", str(min(os.cpu_count() or 1, 32)))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


@pytest.fixture(scope="session")
def oracle():
    from tests import oracle_lib
    return oracle_lib


@pytest.fixture(scope="session")
def product_lib():
    """the built CUDA library; building is part of the CPU-side check"""
    from maskfusion_b200 import build
    build.build()
    import maskfusion_b200
    return maskfusion_b200
