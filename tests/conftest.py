import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "slow: takes more than a few seconds on CPU")


def _gpu_unavailable_reason():
    try:
        import torch
        if not torch.cuda.is_available():
            return "no CUDA device on this host (gpu-marked tests need an H100)"
    except Exception as e:          # pragma: no cover
        return "torch unavailable: %r" % (e,)
    return None                     # GPU present: nothing is skipped, a missing library fails loudly


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a host without a GPU: skip (not fail) everything marked gpu.  With a GPU present nothing is
    skipped here -- a missing / unloadable CUDA library then fails the tests loudly (no silent CPU fallback)."""
    reason = _gpu_unavailable_reason()
    if reason is None:
        return
    skip = pytest.mark.skip(reason=reason)
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
