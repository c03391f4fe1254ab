import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on a machine with a CUDA device)")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    import torch

    return torch.load(os.path.join(ROOT, "tests", "golden", "clip_golden.pt"), map_location="cpu", weights_only=False)


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """The C-ABI library must exist for every test session (built in-tree by __graft_entry__.build())."""
    from multimodal_b200 import _lib

    if not _lib.LIB_PATH.exists():
        _lib.build()
