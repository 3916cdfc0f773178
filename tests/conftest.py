import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    """A plain `pytest tests` on a box without a GPU (or without the built library) skips the `gpu`
    tests instead of failing at the first one; the GPU box runs them with `-m gpu`."""
    import torch
    lib = os.path.join(REPO, "neddf_b200", "libneddf_b200.so")
    reason = None
    if not torch.cuda.is_available():
        reason = "no CUDA device"
    elif not os.path.exists(lib):
        reason = "libneddf_b200.so is not built (python __graft_entry__.py)"
    if reason is None:
        return
    skip = pytest.mark.skip(reason=reason)
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def repo_root():
    return REPO
