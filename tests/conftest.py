import os
import sys

# Gated (layer-streaming) transfers spin on device flags; a first-time lazy kernel load elsewhere in the process can wait
# for the device to idle and dead-lock against them (INTEGRATION.md §5).  Engines that use gating must load eagerly.
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices with peer access")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        ngpu = 0
    skip_gpu = pytest.mark.skip(reason="no CUDA device")
    skip_multi = pytest.mark.skip(reason="needs >= 2 CUDA devices")
    for item in items:
        if "gpu" in item.keywords and ngpu == 0:
            item.add_marker(skip_gpu)
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(skip_multi)
