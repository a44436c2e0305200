import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`gpu`-marked tests are skipped (not failed) on a box without a CUDA device.  On a GPU box a missing library is NOT a reason to
    skip: the product has no fallback and the tests must fail loudly there."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure).  Builds liboracle.so on first use."""
    from oracle import oracle as orc

    orc._lib()
    return orc


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
