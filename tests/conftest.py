import os
import subprocess
import sys

import pytest

# W loopback ranks need W concurrently running streams; the default is 8 hardware queues
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs at least one CUDA device (an H100)")
    # the oracle is test infrastructure: build it on demand (gcc, < 1 s)
    if not os.path.exists(os.path.join(ROOT, "oracle", "liboracle.so")):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle")], check=True, stdout=subprocess.DEVNULL)


def pytest_collection_modifyitems(config, items):
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device on this machine")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture
def store_dir(tmp_path):
    d = tmp_path / "store"
    d.mkdir()
    return str(d)
