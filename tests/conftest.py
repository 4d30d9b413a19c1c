import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLD = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu on a machine with one")


def pytest_collection_modifyitems(config, items):
    """Without a CUDA device (the build container) the gpu-marked tests are skipped, so a bare `pytest tests` is green there."""
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def built_library():
    """The tests exercise the in-tree libddnm_b200.so; compile it first if this checkout has not been built yet
    (nvcc cross-compiles sm_90a without a GPU)."""
    from ddnm_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import shutil
        if shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc"):
            from ddnm_b200 import build as B
            B.build()
    return _lib.LIB_PATH


def _golden(name):
    """tests/golden/<name>.npz merged with its <name>.part<i>.npz continuation files (fixtures are split to stay under 1 MB)."""
    import glob
    import numpy as np
    arrays = dict(np.load(os.path.join(GOLD, name + ".npz")))
    for part in sorted(glob.glob(os.path.join(GOLD, name + ".part*.npz"))):
        arrays.update(np.load(part))
    return arrays


@pytest.fixture(scope="session")
def gold():
    return {name: _golden(name) for name in ("unet_simple", "unet_openai", "operators", "sampler_tiny", "simplified", "general_a", "runner_io", "guided_tiny", "fullsize", "sr16", "simplified_r2", "hq")}
