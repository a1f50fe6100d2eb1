import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
GOLDEN = ROOT / "tests" / "golden"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    # GPU tests must never silently pass without a device: they are selected with -m gpu on
    # the GPU box and deselected with -m "not gpu" here.  If someone runs them on a CPU box
    # they are reported as skipped, loudly.
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    from oracle.binding import Oracle
    return Oracle()


@pytest.fixture(scope="session")
def kllm_lib():
    """The product C-ABI library, built in-tree if needed (nvcc cross-compiles without a GPU)."""
    from kuiperllama_b200 import build, load_library
    build.build()
    return load_library()
