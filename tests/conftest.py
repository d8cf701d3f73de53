import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with `-m gpu`)")


def pytest_collection_modifyitems(config, items):
    """Tests marked `gpu` are skipped (not errored) on a box without a CUDA device: `pytest tests` on a CPU host then
    runs the CPU suite and reports the GPU one as skipped."""
    try:
        import torch

        have = torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def orc():
    from oracle import pyoracle

    pyoracle.lib()
    return pyoracle
