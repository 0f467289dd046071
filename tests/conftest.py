import os
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def real_weights():
    from ai2bmd_b200.weights import load_state_dict
    return load_state_dict(os.path.join(GOLDEN, "weights_2ef43f29.npz"))


@pytest.fixture(scope="session")
def reference_outputs():
    return np.load(os.path.join(GOLDEN, "reference_outputs.npz"))


from ai2bmd_b200.fixtures import load_fragments  # noqa: E402


@pytest.fixture(scope="session")
def chig():
    return load_fragments("chig")


@pytest.fixture(scope="session")
def trpcage():
    return load_fragments("trpcage")
