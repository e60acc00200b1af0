import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


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
def golden():
    def load(name):
        return dict(np.load(os.path.join(GOLDEN, name), allow_pickle=False))
    return load


@pytest.fixture(scope="session")
def oracle_lib():
    """ctypes handle of the plain-C oracle (built on demand with gcc)."""
    import ctypes
    so = os.path.join(ROOT, "oracle", "libpsalm_oracle.so")
    src = os.path.join(ROOT, "oracle", "msda_ref.c")
    if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s"])
    return ctypes.CDLL(so)
