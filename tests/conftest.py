import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")
    config.addinivalue_line("markers", "slow: long-running CPU test")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        ngpu = 0
    for item in items:
        if "multigpu" in item.keywords:
            item.add_marker(pytest.mark.gpu)
            if ngpu < 2:
                item.add_marker(pytest.mark.skip(reason="needs >= 2 GPUs"))
        elif "gpu" in item.keywords and ngpu < 1:
            item.add_marker(pytest.mark.skip(reason="needs a GPU"))
