import importlib.util
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

# Keep the in-tree native runtime in sync with its sources *before* the package (and its _C.so)
# is imported; a no-op when everything is up to date.
_spec = importlib.util.spec_from_file_location("_pdt_build", os.path.join(ROOT, "pytorch_distributed_train_b200", "_build.py"))
_build = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_build)
_build.build()


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with `-m gpu` on an H100 box)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    import torch

    have = torch.cuda.is_available()
    n = torch.cuda.device_count() if have else 0
    for item in items:
        if "gpu" in item.keywords and not have:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        if "multigpu" in item.keywords and n < 2:
            item.add_marker(pytest.mark.skip(reason="needs >= 2 CUDA devices"))
