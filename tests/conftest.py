import os
import sys

import pytest

# tests/test_gpu_multi_local.py runs several shards of a sharded search on ONE GPU when the box has no more: kernels of different shards then
# wait for each other on the same device, which is only safe while their streams map to different hardware work queues.  The default is 8
# queues per device, assigned round-robin at stream creation; 32 (the maximum) keeps a test process that has created many streams clear of
# aliasing.  Must be set before the CUDA context exists; a deployment (one shard per GPU) does not need it.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o

    o.ensure_built()
    return o
