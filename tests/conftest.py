"""pytest configuration: `gpu` marks tests that need an H100 (`-m gpu` on a GPU machine, `-m "not gpu"` without
one)."""
import os
import sys
from pathlib import Path

import pytest

# many contexts (each with several streams) may share one device in the pool tests: give every stream its own hardware
# queue so that a flag barrier between contexts can never sit behind the kernel it waits for (read at CUDA init)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA sm_90 device (H100; run with -m gpu)")


def _cuda_available() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _cuda_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as o
    o.build()
    return o
