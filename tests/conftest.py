import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100)")
    config.addinivalue_line("markers", "reference: needs the reference tree under /root/reference (build container only)")


@pytest.fixture(scope="session")
def built_lib():
    """The in-tree CUDA library (built on demand; nvcc cross-compiles without a GPU)."""
    import __graft_entry__ as g

    g.build()
    from tidy3d_b200 import _cabi

    return _cabi


@pytest.fixture(scope="session")
def gpu_handle(built_lib):
    return built_lib.Handle()


def _gpu_usable():
    try:
        import torch

        return bool(torch.cuda.is_available())
    except Exception:  # noqa: BLE001
        return False


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests are skipped (not failed) on a host without a CUDA device."""
    if _gpu_usable():
        return
    skip = pytest.mark.skip(reason="no CUDA device on this host (run under gpurun)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
