import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = [os.path.join(ROOT, "tests", "golden", name) for name in ("clip_golden.npz", "processor_golden.npz")]


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (pytest -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    out = {}
    for path in GOLDEN:
        out.update(np.load(path, allow_pickle=False))
    return out


@pytest.fixture(scope="session")
def state_dict():
    """Seeded synthetic CLIP ViT-B/32 weights (HF names), generated once per session (~10 s)."""
    from oracle import weights
    torch.set_grad_enabled(False)
    return weights.make_state_dict(0, "rich")


@pytest.fixture(scope="session")
def engine(state_dict):
    from plip_b200.engine import Engine
    eng = Engine(state_dict, max_micro_batch=64)
    yield eng
    eng.close()
