import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)
os.environ.setdefault("PYTHONPATH", ROOT + os.pathsep + os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


def pytest_collection_modifyitems(config, items):
    import torch
    ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    for item in items:
        if "gpu" in item.keywords and ngpu == 0:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(pytest.mark.skip(reason="needs >= 2 CUDA devices"))
