import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3dgs-to-pc_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    # the GPU box has >100 host cores: torch-CPU oracle ops on small tensors crawl when oversubscribed
    import torch
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def lib():
    """Build (if stale) and load libg2pc.so."""
    from g2pc import build, capi
    build.build()
    return capi.load()
