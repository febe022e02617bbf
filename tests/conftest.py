import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN_DIR


def pytest_collection_modifyitems(config, items):
    """`-m gpu` tests need a CUDA device and the built library: on a CPU-only box they are skipped (with the reason)
    instead of erroring, so a plain `pytest` passes everywhere."""
    gpu_items = [it for it in items if it.get_closest_marker("gpu")]
    if not gpu_items:
        return
    reason = None
    try:
        import torch
        if not torch.cuda.is_available():
            reason = "no CUDA device"
        else:
            from mug_diffusion_b200 import lib as L_
            L_.load()
    except Exception as e:  # library missing / ABI mismatch: on a GPU box this must FAIL loudly, not skip
        import torch
        if torch.cuda.is_available():
            raise
        reason = f"libmugd unavailable: {e}"
    if reason:
        skip = pytest.mark.skip(reason=reason)
        for it in gpu_items:
            it.add_marker(skip)
