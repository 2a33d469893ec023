import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (skipped on a machine without one)")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    import torch

    def load(name):
        # a fixture may be stored in parts (every file stays under 1 MB): <stem>.<key>.pt holds entry <key> of <stem>.pt
        g = torch.load(os.path.join(GOLDEN, name), weights_only=False)
        stem = name[:-3]
        for f in sorted(os.listdir(GOLDEN)):
            if f.startswith(stem + ".") and f.endswith(".pt") and f != name:
                g[f[len(stem) + 1:-3]] = torch.load(os.path.join(GOLDEN, f), weights_only=False)
        return g

    return load
