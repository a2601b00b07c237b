"""H100-native (sm_90a) dense-BA update hot path of DROID-SLAM behind the reference's `droid_backends` API.

    import droid_slam_b200
    droid_slam_b200.install()        # makes `import droid_backends` resolve to the native extension
    import droid_backends            # same nine callables as princeton-vl/DROID-SLAM src/droid.cpp:246-259

There is no CPU or PyTorch fallback: if the native extension has not been built (`python -m droid_slam_b200.build`)
`install()` / `backends()` raise ImportError.
"""
import importlib
import os
import sys

__all__ = ["install", "backends", "capi", "EXT_DIR", "LIB_PATH"]

_PKG = os.path.dirname(os.path.abspath(__file__))
EXT_DIR = os.path.join(_PKG, "_ext")
LIB_PATH = os.path.join(_PKG, "lib", "libdroid_b200.so")


def install():
    """Put the native `droid_backends` extension first on sys.path and import it (after torch)."""
    import torch  # noqa: F401  (libtorch must be loaded before the extension)
    if EXT_DIR not in sys.path:
        sys.path.insert(0, EXT_DIR)
    mod = importlib.import_module("droid_backends")
    if not getattr(mod, "_b200_native", lambda: False)():
        raise ImportError("a different `droid_backends` module shadows the native one: %r" % (mod,))
    return mod


def backends():
    return install()


def capi():
    """ctypes handle on the C ABI (include/droid_b200.h)."""
    from . import c_api
    return c_api.load()
