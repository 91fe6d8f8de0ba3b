import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "friendly-stable-audio-tools_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with `-m gpu`)")
    config.addinivalue_line("markers", "reference: needs /root/reference (build container only)")


def pytest_collection_modifyitems(config, items):
    import torch
    has_cuda = torch.cuda.is_available()
    from oracle import ref_shims
    has_ref = ref_shims.reference_available()
    for item in items:
        if "gpu" in item.keywords and not has_cuda:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        if "reference" in item.keywords and not has_ref:
            item.add_marker(pytest.mark.skip(reason="/root/reference not available here"))


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
