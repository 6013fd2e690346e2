import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "spark-network-traffic-classifier_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has = torch.cuda.is_available()
    except Exception:
        has = False
    if not has:
        skip = pytest.mark.skip(reason="no CUDA device")
        for it in items:
            if "gpu" in it.keywords:
                it.add_marker(skip)
