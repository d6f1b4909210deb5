import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))
os.environ.setdefault("MASTER_ADDR", "127.0.0.1")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # The product has no fallback when libflashy_b200.so is missing; build it (nvcc cross-compiles
    # without a GPU) so that a fresh checkout can run the suite directly.
    if not (ROOT / "flashy_b200" / "libflashy_b200.so").exists():
        import __graft_entry__ as entry
        entry.build()


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        have_gpu = torch.cuda.is_available()
    except Exception:
        have_gpu = False
    if have_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
