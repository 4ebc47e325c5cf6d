import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DIAG = {}


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def diag():
    """Dict the GPU tests fill with per-case error figures; written to gpurun_out/ at session end."""
    yield DIAG
    out = os.path.join(ROOT, "gpurun_out")
    try:
        os.makedirs(out, exist_ok=True)
        path = os.path.join(out, "test_diag.json")
        old = {}
        if os.path.exists(path):
            with open(path) as fh:
                old = json.load(fh)
        old.update(DIAG)
        with open(path, "w") as fh:
            json.dump(old, fh, indent=1, sort_keys=True)
    except Exception:
        pass
