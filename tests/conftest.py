import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (run with `pytest -m gpu`)")


def _has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle_port():
    from oracle import port
    port.lib()      # builds liboracle.so on first use if needed
    return port


@pytest.fixture(scope="session")
def reference():
    """The compiled reference (oracle/_ref/libaclref.so). Tests that need it are skipped when it is absent."""
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref/libaclref.so not built (needs /root/reference)")
    ref.lib()
    return ref
