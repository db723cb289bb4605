import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden():
    return {name: np.load(os.path.join(GOLDEN, f"{name}.npz")) for name in ("color_maps", "mask_builder", "attention")}


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """Build libpww_b200.so when nvcc is around (the build container); on the GPU box the prebuilt file is used."""
    from paint_with_words_sd_b200 import _native
    if not os.path.exists(_native.LIB_PATH):
        from paint_with_words_sd_b200.csrc.build import build
        build()
    yield
