import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def synth_state():
    from genpercept_b200 import weights as W
    return W.synth_state(1234)


@pytest.fixture(scope="session")
def text_embed():
    e = np.load(os.path.join(GOLDEN, "empty_text_embed_2x1024.npy"))
    return torch.from_numpy(e.astype(np.float32))[None]


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN
