import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs at least one CUDA GPU (run on the H100 box)")
    config.addinivalue_line("markers", "multigpu: test needs at least two CUDA GPUs")
    # build the native core once (incremental; a no-op when bagua_b200/_C.so is current)
    from bagua_b200 import _build

    _build.build()


def pytest_collection_modifyitems(config, items):
    import torch

    ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    for item in items:
        if "gpu" in item.keywords and ngpu == 0:
            item.add_marker(pytest.mark.skip(reason="no GPU"))
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(pytest.mark.skip(reason="needs >= 2 GPUs"))
