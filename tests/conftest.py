import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def ref_model_dir():
    """The reference's fresh Llama-2M test checkpoint (HF layout), vocabulary cut to its first 512 rows to stay small."""
    path = os.path.join(ROOT, "tests", "golden", "llama-2m-fresh")
    assert os.path.isfile(os.path.join(path, "model.safetensors")) and os.path.isfile(os.path.join(path, "config.json")), path
    return path
