import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a; select with `-m gpu`)")


@pytest.fixture(scope="session")
def backends():
    """the native `droid_backends` module (pybind layer over the C ABI); fails loudly when it was not built"""
    import droid_slam_b200
    return droid_slam_b200.install()


@pytest.fixture(scope="session")
def capi():
    from droid_slam_b200 import c_api
    return c_api.load()
