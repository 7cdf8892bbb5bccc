import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA (H100) device; run with -m gpu on a machine that has one")


def _has_gpu():
    try:
        import ctypes

        cuda = ctypes.CDLL("libcuda.so.1")
        n = ctypes.c_int(0)
        if cuda.cuInit(0) != 0:
            return False
        if cuda.cuDeviceGetCount(ctypes.byref(n)) != 0:
            return False
        return n.value > 0
    except OSError:
        return False


HAS_GPU = _has_gpu()


def pytest_collection_modifyitems(config, items):
    if HAS_GPU:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle_mod():
    from oracle import oracle_py

    oracle_py.build()
    return oracle_py


@pytest.fixture(scope="session")
def scene2k():
    from implicit_svsdf_planner_b200 import scenes

    return scenes.make_scene("star", 8, 2000)


@pytest.fixture(scope="session")
def scene_small_inside():
    """400 points with a narrow corridor: ~6 % of them are inside the swept volume (GSIP branch)."""
    from implicit_svsdf_planner_b200 import scenes

    return scenes.make_scene("star", 8, 400, clearance=2.35)
