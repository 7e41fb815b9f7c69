import os
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a); run with -m gpu on a GPU machine")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def ml_small():
    from lkpy_b200 import data

    return data.load_ml_small()


@pytest.fixture(scope="session")
def rng():
    return np.random.default_rng(42)


@pytest.fixture(scope="session")
def cuda_lib():
    """The built CUDA library; GPU tests must run on it, never on a fallback."""
    from lkpy_b200 import _build, _lib

    _build.build()
    return _lib.lib()


@pytest.fixture
def lk_options(cuda_lib):
    """Set diagnostic kernel switches through ``lk_set_option`` (the LK_* environment is read once, at
    load); every switch touched is restored when the test ends."""
    from lkpy_b200 import _lib

    saved: dict[str, int] = {}

    def set_(name: str, value: int) -> None:
        if name not in saved:
            saved[name] = _lib.get_option(name)
        _lib.set_option(name, value)

    yield set_
    for name, value in saved.items():
        _lib.set_option(name, value)
